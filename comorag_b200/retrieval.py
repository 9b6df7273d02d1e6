"""Retrieval math of ComoRAG.py / utils/embed_utils.py on the fused top-k kernel.

Each function keeps the reference function's name, arguments and return convention.  Where the reference returns a
FULL ranking of all N rows (dense_passage_retrieval feeds every rank into PPR, ComoRAG.py:1034-1042) the scores come
from one score-all pass of the search kernel and the permutation from the device radix sort, at any shard size; the
truncated variants (top_k given) use the fused top-k kernel.  There is no host or library fallback.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import numpy as np

from .index import DenseIndex, MAX_K, fp32_threshold


def min_max_normalize(x: np.ndarray) -> np.ndarray:
    """misc_utils.py:141-150."""
    x = np.asarray(x)
    min_val, max_val = np.min(x), np.max(x)
    range_val = max_val - min_val
    if range_val == 0:
        return np.ones_like(x)
    return (x - min_val) / range_val


def normalize_topk_scores(scores: np.ndarray, minmax: np.ndarray) -> np.ndarray:
    """Reproduce min_max_normalize(all N scores)[top-k ids] from the k survivors and the kernel's global
    (min, max): (s - min) / (max - min), all ones if the range is 0 (misc_utils.py:141-150)."""
    mn, mx = minmax[..., 0:1], minmax[..., 1:2]
    rng = mx - mn
    out = (scores - mn) / np.where(rng == 0, 1, rng)
    return np.where(rng == 0, np.ones_like(scores), out).astype(np.float32)


def dense_topk(index: DenseIndex, query_embeddings, k: int) -> Tuple[np.ndarray, np.ndarray]:
    """Batched dense_passage_retrieval truncated to the first k ranks: (ids int64 [nq, k], min-max-normalised
    scores fp32 [nq, k]) -- what tri_retrieve consumes at ComoRAG.py:499,516 (first qa_*_top_k ids)."""
    ids, scores, minmax = index.search(query_embeddings, k)
    return ids, normalize_topk_scores(scores, minmax)


def dense_passage_retrieval(index: DenseIndex, query_embedding, top_k: Optional[int] = None) -> Tuple[np.ndarray, np.ndarray]:
    """ComoRAG.py:950-967 for one query embedding [1, D] or [D].

    top_k=None keeps the reference contract (a permutation of ALL rows + all min-max-normalised scores, consumed rank
    by rank by PPR at ComoRAG.py:1034-1042): one score-all pass of the search kernel (crag_search_scores) and the
    device radix sort (crag_rank_scores), whatever the shard size; only the int64 permutation and the fp32 scores
    come back to the host.  With top_k only the first top_k ranks are produced by the fused top-k kernel (what
    tri_retrieve consumes at ComoRAG.py:499,516).
    """
    if top_k is not None:
        ids, sc = dense_topk(index, query_embedding, top_k)
        return ids[0], sc[0]
    q = index.prepare_queries(query_embedding)
    scores, minmax = index.scores_device(q[:1])
    order, sorted_scores = index.rank_device(scores[0].contiguous())
    return order.cpu().numpy(), normalize_topk_scores(sorted_scores.cpu().numpy()[None, :], minmax.cpu().numpy())[0]


def get_fact_scores(index: DenseIndex, query_embedding) -> np.ndarray:
    """ComoRAG.py:937-948: min-max-normalised score of EVERY fact row, in row order (callers slice it with
    np.argsort(...)[-k:][::-1] and index it by fact row, ComoRAG.py:475 / :1054 / :1073).  One score-all pass of
    the search kernel; the affine rescale is the reference's own expression applied to the returned scores."""
    q = index.prepare_queries(query_embedding)
    scores, minmax = index.scores_device(q[:1])
    return normalize_topk_scores(scores.cpu().numpy(), minmax.cpu().numpy())[0]


def get_fact_scores_topk(index: DenseIndex, query_embedding, link_top_k: int) -> Tuple[np.ndarray, np.ndarray]:
    """get_fact_scores + the argsort[-k:][::-1] pick that follows it (ComoRAG.py:937-948, :475, :1073)."""
    ids, sc = dense_topk(index, query_embedding, link_top_k)
    return ids[0], sc[0]


_parked_summaries: "dict" = {}
_parked_lock = __import__("threading").Lock()


def park_similar_summaries(query: str, result) -> None:
    """A retrieval wave (comorag_methods.RetrievalWave) already ran the timeline search for `query`; keep its
    (store id, k, texts, scores, rows in the store at search time) until get_similar_summaries asks for it."""
    with _parked_lock:
        _parked_summaries[query] = result
        while len(_parked_summaries) > 512:
            _parked_summaries.pop(next(iter(_parked_summaries)))


def get_similar_summaries(query: str, level_store, embedding_model, top_k: int = 3,
                          instruction: Optional[str] = None) -> Tuple[List[str], List[float]]:
    """embed_utils.py:109-161 on an engine EmbeddingStore: no per-call matrix rebuild, fused top-k."""
    level_ids = level_store.get_all_ids()
    if not level_ids:
        return [], []
    with _parked_lock:
        parked = _parked_summaries.get(query)
    if (parked is not None and parked[0] == id(level_store) and parked[1] >= min(top_k, len(level_ids))
            and parked[4] == len(level_ids)):      # rows added since the wave ran: search again
        k = min(top_k, len(level_ids))
        return list(parked[2][:k]), list(parked[3][:k])
    query_embedding = embedding_model.batch_encode(
        query, instruction='Given a question, retrieve relevant documents that best answer the question.', norm=True)
    k = min(top_k, len(level_ids))
    ids, scores, minmax = level_store.search(query_embedding, k)
    norm = normalize_topk_scores(scores, minmax)[0]
    return [level_store.texts[i] for i in ids[0] if i >= 0], [float(s) for s, i in zip(norm, ids[0]) if i >= 0]


def knn_key_index(key_vecs, device=None) -> DenseIndex:
    """The key shard of retrieve_knn: rows L2-normalised in fp32 (embed_utils.py:8-97 normalises both sides), then
    stored as bf16 by DenseIndex.add.  synonymy_edges builds its shard here too, so both see the same words."""
    import torch
    kv = torch.nn.functional.normalize(torch.as_tensor(np.asarray(key_vecs), dtype=torch.float32), dim=1)
    index = DenseIndex(kv.shape[1], device=device, capacity=kv.shape[0])
    index.add(kv)
    return index


def synonymy_edges(key_vecs, query_rows, threshold: float, cap: int, limit: int, exclude_rows=(), device=None,
                   stream=None) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """The self-join of add_synonymy_edges as a threshold join: the keys go to a shard (knn_key_index), the queries are
    the stored rows `query_rows` of that shard (the same bf16 words retrieve_knn would send), and crag_knn_threshold
    returns, per query, the keys walk ComoRAG.py:698-710 keeps from retrieve_knn(k=limit)'s list: scores >= the
    double `threshold` in rank order, the query's own row and `exclude_rows` skipped, at most `cap`.  Returns host
    (counts int32 [nq], ids int64 [nq, w] key rows, scores fp32 [nq, w]), w = the largest count; only those columns
    leave the device."""
    import torch
    index = knn_key_index(key_vecs, device)
    rows = torch.as_tensor(np.asarray(query_rows, dtype=np.int64))
    with torch.cuda.device(index.device):
        rows_d = rows.to(index.device)
        q = index._buf[: index.n_rows].index_select(0, rows_d)
        counts, ids, scores = index.search_threshold_device(q, fp32_threshold(threshold), cap, limit, self_rows=rows_d,
                                                            exclude_rows=exclude_rows, stream=stream)
        counts_h = counts.cpu().numpy()
        w = int(counts_h.max()) if counts_h.size else 0
        return counts_h, ids[:, :w].cpu().numpy(), scores[:, :w].cpu().numpy()


def retrieve_knn(query_ids: List[str], key_ids: List[str], query_vecs, key_vecs, k: int = 2047,
                 query_batch_size: int = 1000, key_batch_size: int = 10000, device=None):
    """embed_utils.py:8-97: top-k most similar keys (cosine) for every query -> {query_id: (key ids, scores)}.

    The reference L2-normalises both sides and does blocked torch.mm + torch.topk with a two-stage merge, i.e. the
    exact top-min(k, #keys) per query, scores descending.  Here the normalised keys become a bf16 device shard and
    every group of queries goes through DenseIndex.search: for k <= 2048 and a full group (the self-join of
    add_synonymy_edges, ComoRAG.py:670-684) that is crag_knn_topk -- one wgmma GEMM per chunk of queries writing the
    fp32 score block, then a per-query radix select --, otherwise the fused scan, 128 ranks per pass chained with
    crag_search_topk_after.  The two batch size arguments are accepted for signature compatibility; blocking is the
    library's own.
    """
    import torch
    if len(key_vecs) == 0:
        return {}
    q = torch.nn.functional.normalize(torch.as_tensor(np.asarray(query_vecs), dtype=torch.float32), dim=1)
    index = knn_key_index(key_vecs, device)
    kk = min(int(k), index.n_rows)
    results = {}
    step = 1024  # queries per launch group (32 per corpus pass inside the library)
    for s0 in range(0, q.shape[0], step):
        ids, scores, _ = index.search(q[s0:s0 + step], kk)
        for i in range(ids.shape[0]):
            valid = ids[i] >= 0
            results[query_ids[s0 + i]] = ([key_ids[j] for j in ids[i][valid]], scores[i][valid].tolist())
    return results
