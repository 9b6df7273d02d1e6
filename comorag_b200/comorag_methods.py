"""Replacements for the retrieval methods of the reference's `ComoRAG` class (src/comorag/ComoRAG.py), bound onto the
class by `comorag_b200.install.install()` so an UNMODIFIED ComoRAG.py runs its probe -> retrieve -> consolidate loop
on the device shards instead of host fp32 matrices.

Each function keeps the reference method's name, signature, return type and side effects on `self`:

    prepare_retrieval_objects(self)                 ComoRAG.py:876-907
    get_query_embeddings(self, queries)             ComoRAG.py:909-935
    get_fact_scores(self, query)                    ComoRAG.py:937-948
    dense_passage_retrieval(self, query, need_cluster=False)   ComoRAG.py:950-967

`retrieve_knn` (utils/embed_utils.py:8-97, called at ComoRAG.py:678) is a module-level name and is rebound by
install() like the other imported names (comorag_b200.retrieval.retrieve_knn).

KNN_METHODS, rebound by install(knn=True) (the default), move the synonymy-edge walk onto the device:

    add_synonymy_edges(self)                        ComoRAG.py:670-712

GRAPH_METHODS, rebound only by install(graph=True), move the graph branch of tri_retrieve onto the device:

    graph_search_with_fact_entities(self, query, link_top_k, ...)    ComoRAG.py:992-1055 (+ get_top_k_weights, :972-990)
    run_ppr(self, reset_prob, damping=0.5)                           ComoRAG.py:1086-1105
"""
from __future__ import annotations

import logging
import re
from typing import Dict, List, Tuple

import numpy as np
import torch

from . import retrieval
from .coalescer import BatcherClosed
from .embedding_store import compute_mdhash_id
from .graph import DeviceGraph
from .index import rank_scores

logger = logging.getLogger(__name__)

# ComoRAG.py passes these to batch_encode (prompts/linking.py:1-11); the reference's BGE model ignores them and always
# prefixes its passage instruction (BGEEmbedding.py:150-155), ours reproduces that, so both caches hold the same rows.
_INSTRUCTION_FACT = 'Given a question, retrieve relevant triplet facts that matches this question.'
_INSTRUCTION_PASSAGE = 'Given a question, retrieve relevant documents that best answer the question.'


class ShardMatrix:
    """What `self.{entity,passage,fact,summary}_embeddings` become: the reference materialises four host fp32
    matrices with np.array(store.get_embeddings(keys)) (ComoRAG.py:897-901, 41 GB at 10M x 1024); here the rows stay
    in the store's device shard and this object only answers the questions the reference asks of those attributes
    (`.shape`, `.dtype` in its log lines) -- and still converts to the real matrix if somebody does np.asarray()."""

    def __init__(self, store):
        self._store = store

    @property
    def index(self):
        return self._store.index

    @property
    def shape(self) -> Tuple[int, int]:
        return (len(self._store.hash_ids), int(getattr(self._store, "_dim", 0) or 0))

    @property
    def dtype(self):
        return np.dtype(np.float32)

    def __len__(self) -> int:
        return self.shape[0]

    def __array__(self, dtype=None, copy=None):
        m = self._store.get_embeddings(self._store.hash_ids)
        m = np.asarray(m, dtype=np.float32).reshape(self.shape)
        return m.astype(dtype) if dtype is not None else m


def _store_has_shard(store) -> bool:
    return hasattr(store, "index") and hasattr(store, "search")


_prepare_lock = __import__("threading").RLock()


def prepare_retrieval_objects(self) -> None:
    """ComoRAG.py:876-907 with the four `np.array(store.get_embeddings(keys))` pulls replaced by views of the
    stores' device shards.  Key lists, graph index maps and `ready_to_retrieve` are set exactly as the reference does.
    The key lists are `store.get_all_ids()`, i.e. store row order, so row r of a shard is key r of its list."""
    with _prepare_lock:
        _prepare_locked(self)


def _store_signature(self):
    stores = [self.entity_embedding_store, self.ver_embedding_store, self.fact_embedding_store]
    if self.global_config.need_cluster:
        stores.append(self.sem_embedding_store)
    return tuple((id(s), len(s.hash_ids)) for s in stores) + (self.graph.vcount() if hasattr(self.graph, "vcount") else len(self.graph.vs),)


def _prepare_locked(self) -> None:
    # Up to 16 meta_control_loop threads reach `if not self.ready_to_retrieve: self.prepare_retrieval_objects()`
    # together (ComoRAG.py:436-441, :467-468).  In the reference the duplicate calls rebuild identical matrices; here
    # a late duplicate would retire the retrieval wave under the threads already using it, so a call that finds the
    # objects prepared for exactly these stores and row counts returns at once.
    sig = _store_signature(self)
    if getattr(self, "ready_to_retrieve", False) and getattr(self, "_crag_prepared_for", None) == sig:
        return
    logger.info("Preparing for fast retrieval.")
    self.query_to_embedding: Dict = {'triple': {}, 'passage': {}}

    self.entity_node_keys: List = list(self.entity_embedding_store.get_all_ids())
    self.passage_node_keys: List = list(self.ver_embedding_store.get_all_ids())
    self.fact_node_keys: List = list(self.fact_embedding_store.get_all_ids())
    if self.global_config.need_cluster:
        self.summary_node_keys: List = list(self.sem_embedding_store.get_all_ids())

    igraph_name_to_idx = {node["name"]: idx for idx, node in enumerate(self.graph.vs)}
    self.node_name_to_vertex_idx = igraph_name_to_idx
    self.entity_node_idxs = [igraph_name_to_idx[node_key] for node_key in self.entity_node_keys]
    self.passage_node_idxs = [igraph_name_to_idx[node_key] for node_key in self.passage_node_keys]

    stores = [("entity_embeddings", self.entity_embedding_store), ("passage_embeddings", self.ver_embedding_store),
              ("fact_embeddings", self.fact_embedding_store)]
    if self.global_config.need_cluster:
        stores.append(("summary_embeddings", self.sem_embedding_store))
    for attr, store in stores:
        if not _store_has_shard(store):
            raise TypeError(f"{attr}: {type(store).__module__}.{type(store).__name__} has no device shard; "
                            "install() must run before ComoRAG(...) builds its stores (there is no host fallback)")
        view = ShardMatrix(store)
        if len(store.hash_ids):
            store.index                # upload / extend the bf16 shard now, as the reference loads its matrices here
        setattr(self, attr, view)
        logger.info(f"prepare_retrieval_objects: self.{attr}.shape = {view.shape}, dtype = {view.dtype}")
    old = getattr(self, "_crag_wave", None)
    if old is not None:          # shards were rebuilt: parked results belong to the previous ones
        old.close()
        self._crag_wave = None
    self._crag_prepared_for = sig
    self.ready_to_retrieve = True


class RetrievalWave:
    """SURVEY.md section 8f item 1: one batched encode and ONE pass over each of the fact / passage / summary /
    timeline shards per wave of concurrent `tri_retrieve` calls (ComoRAG.py:436-441 answers questions from up to 16
    threads, each issuing batch-1 encodes and single-query searches, ComoRAG.py:456-554).

    `get_query_embeddings(query)` -- the first retrieval call of every tri_retrieve (ComoRAG.py:470) -- hands the
    query to a Batcher; whatever arrived within `max_wait_s` is encoded as one packed forward and scored as one query
    block per shard (a 16-query pass reads the shard once, like a 1-query pass).  The per-query results are parked and
    the four scoring entry points of that tri_retrieve (get_fact_scores, dense_passage_retrieval x2,
    get_similar_summaries) pick them up instead of launching anything."""

    def __init__(self, rag, max_queries: int = 32, max_wait_s: float = 2e-4, keep: int = 256):
        from collections import OrderedDict
        import threading
        from .coalescer import Batcher
        self.rag = rag
        self._b = Batcher(self._run, max_items=max_queries, max_wait_s=max_wait_s, name="crag-retrieval-wave")
        self._results: "OrderedDict[str, dict]" = OrderedDict()
        self._lock = threading.Lock()
        self._keep = keep

    @property
    def stats(self):
        return {"waves": self._b.batches, "queries": self._b.items}

    def close(self):
        self._b.close()

    def submit(self, query: str) -> dict:
        with self._lock:
            hit = self._results.get(query)
        if hit is not None:
            return hit
        try:
            res = self._b.call("tri_retrieve", query)
        except BatcherClosed:        # the wave was retired (shards rebuilt) between _wave() and here: answer alone
            res = self._run("tri_retrieve", [query])[0]
        with self._lock:
            self._results[query] = res
            while len(self._results) > self._keep:
                self._results.popitem(last=False)
        return res

    def lookup(self, query: str):
        with self._lock:
            return self._results.get(query)

    def _run(self, key, queries: List[str]) -> List[dict]:
        rag = self.rag
        uniq = list(dict.fromkeys(queries))
        emb = rag.embedding_model.batch_encode(uniq, instruction=_INSTRUCTION_FACT, norm=True)    # one packed forward
        n = len(uniq)
        out = [{"embedding": emb[i:i + 1]} for i in range(n)]
        fact_index = rag.fact_embeddings.index
        q_dev = fact_index.prepare_queries(emb)                  # one H2D of the wave's query block
        scores, mm = fact_index.scores_device(q_dev)             # one pass over the fact shard for the whole wave
        facts = retrieval.normalize_topk_scores(scores.cpu().numpy(), mm.cpu().numpy())
        for i in range(n):
            out[i]["fact_scores"] = facts[i]
        shards = [("passages", rag.passage_embeddings.index)]
        if rag.global_config.need_cluster:
            shards.append(("summaries", rag.summary_embeddings.index))
        for name, index in shards:
            scores, mm = index.scores_device(q_dev)              # one pass per shard
            mm_h = mm.cpu().numpy()
            for i in range(n):
                order, sorted_scores = index.rank_device(scores[i].contiguous())
                out[i][name] = (order.cpu().numpy(),
                                retrieval.normalize_topk_scores(sorted_scores.cpu().numpy()[None, :], mm_h[i:i + 1])[0])
        level_store = getattr(rag, "level_store", None)
        if level_store is not None and hasattr(level_store, "search") and len(level_store.hash_ids):
            k = min(int(getattr(rag.global_config, "qa_epi_top_k", 50)), len(level_store.hash_ids))
            ids, sc, mm = level_store.search(emb, k)             # one fused top-k pass over the timeline shard
            norm = retrieval.normalize_topk_scores(sc, mm)
            for i in range(n):
                out[i]["timeline"] = (id(level_store), k,
                                      [level_store.texts[j] for j in ids[i] if j >= 0],
                                      [float(s) for s, j in zip(norm[i], ids[i]) if j >= 0],
                                      len(level_store.hash_ids))
        by_query = dict(zip(uniq, out))
        return [by_query[q] for q in queries]


_wave_create_lock = __import__("threading").Lock()


def _wave(self):
    w = getattr(self, "_crag_wave", None)
    if w is None and getattr(self.global_config, "retrieval_wave", True) and isinstance(getattr(self, "fact_embeddings", None), ShardMatrix):
        with _wave_create_lock:      # up to 16 threads reach their first tri_retrieve together (ComoRAG.py:436-441)
            w = getattr(self, "_crag_wave", None)
            if w is None:
                w = self._crag_wave = RetrievalWave(self)
    return w


def get_query_embeddings(self, queries) -> None:
    """ComoRAG.py:909-935.  tri_retrieve passes ONE str (ComoRAG.py:470); the reference then iterates its characters,
    runs two batch encodes over single characters and fills the cache with entries nothing ever looks up.  Here a str
    is one query: it is encoded once per cache and the later lookups (get_fact_scores, dense_passage_retrieval, both
    need_cluster settings) hit.  Lists of str / QuerySolution behave as in the reference."""
    if isinstance(queries, str):
        wave = _wave(self)
        if wave is not None and len(self.fact_node_keys) and len(self.passage_node_keys):
            res = wave.submit(queries)       # encode + all four shard passes, shared with concurrent callers
            self.query_to_embedding['triple'][queries] = res["embedding"]
            self.query_to_embedding['passage'][queries] = res["embedding"]
            if "timeline" in res:
                retrieval.park_similar_summaries(queries, res["timeline"])
            return
        queries = [queries]
    cache = self.query_to_embedding
    todo: List[str] = []
    for query in queries:
        text = getattr(query, "question", query)
        if text not in cache['triple'] or text not in cache['passage']:
            if text not in todo:
                todo.append(text)
    if not todo:
        return
    model = self.embedding_model
    logger.info(f"Encoding {len(todo)} queries for query_to_fact.")
    emb_fact = model.batch_encode(todo, instruction=_INSTRUCTION_FACT, norm=True)
    if getattr(model, "instruction_is_forced", False):
        emb_passage = emb_fact     # the instruction kwarg does not reach the text (BGEEmbedding.py:150-155): same rows
    else:
        logger.info(f"Encoding {len(todo)} queries for query_to_passage.")
        emb_passage = model.batch_encode(todo, instruction=_INSTRUCTION_PASSAGE, norm=True)
    for text, e_f, e_p in zip(todo, emb_fact, emb_passage):
        cache['triple'][text] = e_f
        cache['passage'][text] = e_p


def _query_embedding(self, which: str, query: str, instruction: str) -> np.ndarray:
    emb = self.query_to_embedding[which].get(query, None)
    if emb is None:
        emb = self.embedding_model.batch_encode(query, instruction=instruction, norm=True)
    return emb


def get_fact_scores(self, query: str) -> np.ndarray:
    """ComoRAG.py:937-948: min-max-normalised score of every fact, fp32 [N_f] in fact_node_keys order."""
    wave = getattr(self, "_crag_wave", None)
    hit = wave.lookup(query) if wave is not None else None
    if hit is not None:
        return hit["fact_scores"].copy()      # callers own the array, as with the reference's fresh np result
    query_embedding = _query_embedding(self, 'triple', query, _INSTRUCTION_FACT)
    return retrieval.get_fact_scores(self.fact_embeddings.index, query_embedding)


def dense_passage_retrieval(self, query: str, need_cluster: bool = False) -> Tuple[np.ndarray, np.ndarray]:
    """ComoRAG.py:950-967: (sorted_doc_ids int64 [N], sorted min-max scores fp32 [N]) over the passage shard
    (need_cluster=False) or the summary shard (True) -- the FULL permutation, as graph_search_with_fact_entities
    consumes every rank (ComoRAG.py:1034-1042)."""
    wave = getattr(self, "_crag_wave", None)
    hit = wave.lookup(query) if wave is not None else None
    name = "summaries" if need_cluster else "passages"
    if hit is not None and name in hit:
        order, scores = hit[name]
        return order.copy(), scores.copy()
    query_embedding = _query_embedding(self, 'passage', query, _INSTRUCTION_PASSAGE)
    docs = self.summary_embeddings if need_cluster else self.passage_embeddings
    return retrieval.dense_passage_retrieval(docs.index, query_embedding)


METHODS = {
    "prepare_retrieval_objects": prepare_retrieval_objects,
    "get_query_embeddings": get_query_embeddings,
    "get_fact_scores": get_fact_scores,
    "dense_passage_retrieval": dense_passage_retrieval,
}


# ------------------------------------------------------------------------------------------------ synonymy edges
# The reference walk accepts while `num_nns > 100` is false (ComoRAG.py:699): at most 101 edges per entity.
SYNONYMY_CAP = 101


def add_synonymy_edges(self) -> None:
    """ComoRAG.py:670-712 with the k = synonymy_edge_topk kNN lists and their walk replaced by one threshold join
    (retrieval.synonymy_edges -> crag_knn_threshold): per entity only the edges the walk keeps leave the device.
    Step for step as the reference: self.entity_id_to_row is set, keys are taken in store order with embeddings from
    get_embeddings, only entities whose content keeps more than 2 alphanumerics are queries, the entity with content
    '' is never an edge target, and for each query in key order and each kept edge in rank order
    `self.node_to_node_stats[(key, nn)] = score` -- so new dict keys land, and existing ones are overwritten, in the
    reference's order.  The edges are identical to the reference walk over retrieval.retrieve_knn's lists."""
    logger.info("Expanding graph with synonymy edges")
    self.entity_id_to_row = self.entity_embedding_store.get_text_for_all_rows()
    entity_node_keys = list(self.entity_id_to_row.keys())
    logger.info(f"Performing KNN retrieval for each phrase nodes ({len(entity_node_keys)}).")
    contents = [self.entity_id_to_row[key]["content"] for key in entity_node_keys]
    queries = [r for r, text in enumerate(contents) if len(re.sub('[^A-Za-z0-9]', '', text)) > 2]
    if not queries:
        return
    entity_embs = self.entity_embedding_store.get_embeddings(entity_node_keys)
    empty = [r for r, text in enumerate(contents) if text == '']
    cfg = self.global_config
    counts, ids, scores = retrieval.synonymy_edges(entity_embs, queries, cfg.synonymy_edge_sim_threshold, SYNONYMY_CAP,
                                                   cfg.synonymy_edge_topk, exclude_rows=empty)
    stats = self.node_to_node_stats
    for i, r in enumerate(queries):
        node_key = entity_node_keys[r]
        for nn, score in zip(ids[i, :counts[i]].tolist(), scores[i, :counts[i]].tolist()):
            stats[(node_key, entity_node_keys[nn])] = score


KNN_METHODS = {
    "add_synonymy_edges": add_synonymy_edges,
}


# ------------------------------------------------------------------------------------------------ graph search
_graph_lock = __import__("threading").Lock()


def _device_graph(self) -> DeviceGraph:
    """self.graph as a DeviceGraph, built on first use and cached on the instance, keyed by (vcount, ecount): the
    reference only ever adds vertices and edges (ComoRAG.py:779-841), so a changed graph changes one of the two.
    The graph it builds coalesces the PPR of concurrent graph searches (DeviceGraph.enable_batching: one
    crag_ppr_batch pass for the questions ComoRAG.py:436-441 answers together, each result bit-identical to its own
    crag_ppr call); a rebuild closes the old graph's batcher, and calls still on their way to it run directly."""
    key = (self.graph.vcount(), self.graph.ecount())
    cached = getattr(self, "_crag_graph", None)
    if cached is None or cached[0] != key:
        with _graph_lock:               # up to 16 tri_retrieve threads reach the first graph search together
            cached = getattr(self, "_crag_graph", None)
            if cached is None or cached[0] != key:
                old = cached
                graph = DeviceGraph.from_igraph(self.graph)
                graph.enable_batching()
                cached = (key, graph)
                self._crag_graph = cached
                if old is not None:
                    old[1].disable_batching()
    return cached[1]


def _passage_vertices(self) -> np.ndarray:
    """self.passage_node_idxs as int64 (prepare_retrieval_objects assigns a new list when it rebuilds them)."""
    idxs = self.passage_node_idxs
    cached = getattr(self, "_crag_passage_vertices", None)
    if cached is None or cached[0] is not idxs or len(cached[1]) != len(idxs):
        cached = (idxs, np.asarray(idxs, dtype=np.int64).reshape(-1), {})
        self._crag_passage_vertices = cached
    return cached[1]


def _passage_vertices_on(self, graph: DeviceGraph) -> torch.Tensor:
    _passage_vertices(self)
    on_device = self._crag_passage_vertices[2]
    if graph.device not in on_device:
        on_device[graph.device] = torch.as_tensor(self._crag_passage_vertices[1], device=graph.device)
    return on_device[graph.device]


def run_ppr(self, reset_prob: np.ndarray, damping: float = 0.5) -> Tuple[np.ndarray, np.ndarray]:
    """ComoRAG.py:1086-1105: PPR over self.graph with run_ppr's reset sanitising, on the device (crag_ppr), then the
    passages ranked by score on the device (crag_rank_scores).  Returns (sorted_doc_ids int64, sorted_doc_scores
    float64) over self.passage_node_idxs; equal scores rank by ascending row."""
    if damping is None:
        damping = 0.5
    graph = _device_graph(self)
    scores = graph.personalized_pagerank(np.asarray(reset_prob, dtype=np.float64), damping,
                                         vertices=_passage_vertices_on(self, graph))
    ids, sorted_scores = rank_scores(scores)
    return ids.cpu().numpy(), sorted_scores.cpu().numpy().astype(np.float64)


def graph_search_with_fact_entities(self, query: str, link_top_k: int, query_fact_scores: np.ndarray,
                                    top_k_facts: List[Tuple], top_k_fact_indices: List[str],
                                    passage_node_weight: float = 0.05):
    """ComoRAG.py:992-1055 with get_top_k_weights (:972-990): the same node weights, bit for bit, the same
    used_phrases_with_scores and assertions, in O(facts + link_top_k) Python plus vectorised numpy:
      * phrase weights live in a dict {vertex: weight} until the end; "zero every vertex outside the top-k phrase
        keys" keeps exactly the entries whose key is among them;
      * the passage weights are one scatter of min_max_normalize(dpr scores) * passage_node_weight;
      * the per-passage linking_score_map entries (a get_row per passage) are not built: the map is local and never
        returned, so nothing observable changes."""
    linking_score_map = {}
    phrase_scores = {}
    phrase_weights = {}             # vertex -> weight: the nonzero-capable entries of the reference's dense array
    phrase_keys = {}                # vertex -> its name (phrase key)
    used_phrases_with_scores = {}
    n_vertices = self.graph.vcount()

    for rank, f in enumerate(top_k_facts):
        subject_phrase = f[0].lower()
        object_phrase = f[2].lower()
        fact_score = query_fact_scores[top_k_fact_indices[rank]] if query_fact_scores.ndim > 0 else query_fact_scores
        for phrase in [subject_phrase, object_phrase]:
            phrase_key = compute_mdhash_id(content=phrase, prefix="entity-")
            phrase_id = self.node_name_to_vertex_idx.get(phrase_key, None)
            if phrase_id is not None:
                w = np.float64(fact_score)
                if self.ent_node_to_num_chunk[phrase_key] != 0:
                    w /= self.ent_node_to_num_chunk[phrase_key]
                phrase_weights[phrase_id] = w
                phrase_keys[phrase_id] = phrase_key
                if w > 0:
                    used_phrases_with_scores[phrase] = w
            if phrase not in phrase_scores:
                phrase_scores[phrase] = []
            phrase_scores[phrase].append(fact_score)

    for phrase, scores in phrase_scores.items():
        linking_score_map[phrase] = float(np.mean(scores))
    if link_top_k:
        linking_score_map = dict(sorted(linking_score_map.items(), key=lambda x: x[1], reverse=True)[:link_top_k])
        top_k_phrases_keys = {compute_mdhash_id(content=p, prefix="entity-") for p in linking_score_map}
        phrase_weights = {v: w for v, w in phrase_weights.items() if phrase_keys[v] in top_k_phrases_keys}
        assert sum(1 for w in phrase_weights.values() if w != 0) == len(linking_score_map.keys())

    dpr_sorted_doc_ids, dpr_sorted_doc_scores = self.dense_passage_retrieval(query)
    normalized_dpr_sorted_scores = retrieval.min_max_normalize(dpr_sorted_doc_scores)
    phrase_dense = np.zeros(n_vertices)
    if phrase_weights:
        phrase_dense[np.fromiter(phrase_weights.keys(), dtype=np.int64)] = np.fromiter(phrase_weights.values(),
                                                                                   dtype=np.float64)
    passage_weights = np.zeros(n_vertices)
    passage_weights[_passage_vertices(self)[np.asarray(dpr_sorted_doc_ids, dtype=np.int64)]] = \
        normalized_dpr_sorted_scores * passage_node_weight
    node_weights = phrase_dense + passage_weights

    assert np.sum(node_weights) > 0, f'No phrases found in the graph for the given facts: {top_k_facts}'
    ppr_sorted_doc_ids, ppr_sorted_doc_scores = self.run_ppr(node_weights)
    assert len(ppr_sorted_doc_ids) == len(
        self.passage_node_idxs), f"Doc prob length {len(ppr_sorted_doc_ids)} != corpus length {len(self.passage_node_idxs)}"
    return ppr_sorted_doc_ids, ppr_sorted_doc_scores, used_phrases_with_scores


GRAPH_METHODS = {
    "graph_search_with_fact_entities": graph_search_with_fact_entities,
    "run_ppr": run_ppr,
}
