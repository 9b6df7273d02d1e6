"""comorag_methods.add_synonymy_edges on the CPU, with its one device call (retrieval.synonymy_edges) replaced by the
numpy walk of tests/synonymy_oracle.py over the same fp32 scores: node_to_node_stats must come out exactly as the
reference loop leaves it over retrieve_knn-shaped lists of those scores -- the same assignments, so the same dict
insertion order and the same positions for overwritten keys.  Also: the eligibility filter on the query side, the ''
entity never an edge target, entity_id_to_row set, and an empty store launching nothing."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import synonymy_oracle as so  # noqa: E402

from comorag_b200 import comorag_methods as cm  # noqa: E402
from comorag_b200 import retrieval  # noqa: E402


class _Store:
    def __init__(self, texts, emb):
        self.hash_ids = [f"entity-{i:04d}" for i in range(len(texts))]
        self.texts, self.emb = list(texts), np.asarray(emb, dtype=np.float32)

    def get_text_for_all_rows(self):
        return {h: {"hash_id": h, "content": t} for h, t in zip(self.hash_ids, self.texts)}

    def get_embeddings(self, hash_ids):
        if not hash_ids:
            return []
        return self.emb[[self.hash_ids.index(h) for h in hash_ids]]


def _scores(key_vecs):
    x = np.asarray(key_vecs, dtype=np.float64)
    x = x / np.linalg.norm(x, axis=1, keepdims=True)
    return (x @ x.T).astype(np.float32)


@pytest.fixture
def oracle_join(monkeypatch):
    calls = []

    def fake(key_vecs, query_rows, threshold, cap, limit, exclude_rows=(), device=None, stream=None):
        calls.append((list(query_rows), float(threshold), cap, limit, list(exclude_rows)))
        S = _scores(key_vecs)
        counts, ids, sc = so.walk_all(S[list(query_rows)], so.fp32_threshold(threshold), limit, cap,
                                      self_rows=list(query_rows), exclude_rows=exclude_rows)
        w = int(counts.max()) if counts.size else 0
        return counts, ids[:, :w], sc[:, :w]
    monkeypatch.setattr(retrieval, "synonymy_edges", fake)
    return calls


def _rag(texts, emb, topk=2047, threshold=0.8, stats=None):
    cfg = SimpleNamespace(synonymy_edge_topk=topk, synonymy_edge_sim_threshold=threshold,
                          synonymy_edge_query_batch_size=1000, synonymy_edge_key_batch_size=10000)
    return SimpleNamespace(entity_embedding_store=_Store(texts, emb), global_config=cfg,
                           node_to_node_stats=dict(stats or {}))


def _reference_stats(rag, stats):
    store = rag.entity_embedding_store
    rows = store.get_text_for_all_rows()
    keys = list(rows)
    S = _scores(store.get_embeddings(keys))
    k = rag.global_config.synonymy_edge_topk
    knn = {keys[q]: ([keys[r] for r in so.rank_order(S[q], k)], S[q, so.rank_order(S[q], k)].tolist())
           for q in range(len(keys))}
    out = dict(stats)
    for edge, score in so.edges_from_knn(knn, {h: r["content"] for h, r in rows.items()},
                                         rag.global_config.synonymy_edge_sim_threshold, cm.SYNONYMY_CAP):
        out[edge] = score
    return out


def _planted(n, dim, groups, seed):
    """n rows in synonym groups: rows of one group are a shared direction plus small noise."""
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((groups, dim))
    g = rng.integers(0, groups, size=n)
    return centers[g] + 0.25 * rng.standard_normal((n, dim)), g


@pytest.mark.parametrize("threshold", [0.8, 0.7])
def test_add_synonymy_edges_equals_the_reference_loop(oracle_join, threshold):
    emb, _ = _planted(300, 32, 12, 5)
    texts = [f"phrase {i}" for i in range(300)]
    texts[4], texts[9], texts[20] = "ab", "a.b", "!!?"          # fewer than 3 alphanumerics: not queries
    texts[13] = ''                                                 # never an edge target
    emb[13] = emb[14]                                              # ... even as an exact duplicate of row 14
    keys = [f"entity-{i:04d}" for i in range(300)]
    # existing entries: the pair edges of add_new_edges and one synonymy edge the walk will overwrite
    pre = {(keys[1], keys[2]): 1.0, (keys[0], keys[0]): 2.0, (keys[14], keys[13]): 7.0}
    S = _scores(emb)
    j = int(np.argsort(-S[3])[1])
    pre[(keys[3], keys[j])] = 5.0
    rag = _rag(texts, emb, threshold=threshold, stats=pre)
    want = _reference_stats(rag, pre)
    cm.add_synonymy_edges(rag)
    assert list(rag.node_to_node_stats.items()) == list(want.items())
    assert rag.node_to_node_stats[(keys[3], keys[j])] != 5.0          # overwritten in place
    assert list(rag.node_to_node_stats)[3] == (keys[3], keys[j])
    assert rag.entity_id_to_row == rag.entity_embedding_store.get_text_for_all_rows()
    new = [e for e in rag.node_to_node_stats if e not in pre]
    assert len(new) > 300
    assert not any(a in (keys[4], keys[9], keys[20]) for a, _ in new)
    assert not any(b == keys[13] for _, b in new)
    assert all(isinstance(v, float) for v in rag.node_to_node_stats.values())
    (rows, t, cap, limit, excl), = oracle_join
    assert rows == [r for r in range(300) if r not in (4, 9, 13, 20)] and excl == [13]
    assert (t, cap, limit) == (threshold, 101, 2047)


def test_the_cap_and_the_limit(oracle_join):
    emb = np.ones((400, 16)) + 1e-3 * np.random.default_rng(3).standard_normal((400, 16))   # one group of 400
    texts = [f"name {i}" for i in range(400)]
    for topk in (2047, 50):
        rag = _rag(texts, emb, topk=topk)
        cm.add_synonymy_edges(rag)
        assert list(rag.node_to_node_stats.items()) == list(_reference_stats(rag, {}).items())
        per = {}
        for a, _ in rag.node_to_node_stats:
            per[a] = per.get(a, 0) + 1
        assert set(per.values()) == {101 if topk == 2047 else 49}


def test_empty_store_and_no_eligible_query_launch_nothing(oracle_join):
    rag = _rag([], np.zeros((0, 8)))
    cm.add_synonymy_edges(rag)
    assert rag.entity_id_to_row == {} and rag.node_to_node_stats == {}
    rag = _rag(["ab", "", "x y"], np.eye(3, 8))
    cm.add_synonymy_edges(rag)
    assert len(rag.entity_id_to_row) == 3 and rag.node_to_node_stats == {}
    assert oracle_join == []


def test_add_synonymy_edges_is_bound_under_knn():
    assert cm.KNN_METHODS == {"add_synonymy_edges": cm.add_synonymy_edges}
