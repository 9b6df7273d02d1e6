"""Host side of the device PPR (no GPU): DeviceGraph.from_edges builds scipy's symmetrised, coalesced matrix and
rejects what the semantics exclude; the rebound graph_search_with_fact_entities hands run_ppr bit-identical node
weights, returns the same used_phrases_with_scores and raises the same assertions as the reference's method; and
install(graph=True) rebinds exactly its two methods."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import e2e_harness as H  # noqa: E402
from oracle import ppr_oracle as O  # noqa: E402

from comorag_b200 import comorag_methods as cm  # noqa: E402
from comorag_b200.embedding_store import compute_mdhash_id  # noqa: E402
from comorag_b200.graph import DeviceGraph, ppr_iterations  # noqa: E402

REF_ROOT = H.find_reference_root()
needs_ref = pytest.mark.skipif(REF_ROOT is None, reason="reference tree not present (build() stages it under oracle/_ref)")


# ------------------------------------------------------------------------------------------------ DeviceGraph
@pytest.mark.parametrize("seed", range(4))
def test_from_edges_builds_the_symmetrised_coalesced_csr(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(5, 80))
    a, b = rng.integers(0, n - 2, 300), rng.integers(0, n - 2, 300)        # the last two vertices stay isolated
    keep = a != b
    e = np.stack([a[keep], b[keep]], 1)
    e = np.concatenate([e, e[:40, ::-1], e[:25]])                           # both orientations, parallel edges
    w = rng.uniform(0.01, 5.0, len(e))
    g = DeviceGraph.from_edges(n, torch.as_tensor(e), torch.as_tensor(w), device="cpu")
    W = O.adjacency(n, e, w)
    A = O.transition(W)
    np.testing.assert_array_equal(g.row_ptr.numpy(), W.indptr)
    np.testing.assert_array_equal(g.col.numpy(), W.indices)
    assert g.col.dtype == torch.int32 and g.coef.dtype == torch.float32 and g.row_ptr.dtype == torch.int64
    np.testing.assert_allclose(g.coef.numpy().astype(np.float64), A.data, rtol=2.0 ** -24, atol=0)
    assert g.row_ptr[-2] == g.row_ptr[-1] == g.nnz                           # isolated vertices: empty rows


def test_from_edges_rejects_what_the_semantics_exclude():
    e = torch.tensor([[0, 1], [1, 2]])
    with pytest.raises(ValueError, match="self-loop"):
        DeviceGraph.from_edges(3, torch.tensor([[0, 1], [2, 2]]), torch.tensor([1.0, 1.0]), device="cpu")
    with pytest.raises(ValueError, match="> 0"):
        DeviceGraph.from_edges(3, e, torch.tensor([1.0, 0.0]), device="cpu")
    with pytest.raises(ValueError, match="> 0"):
        DeviceGraph.from_edges(3, e, torch.tensor([1.0, -2.0]), device="cpu")
    for bad in (float("nan"), float("inf")):
        with pytest.raises(ValueError, match="finite"):
            DeviceGraph.from_edges(3, e, torch.tensor([1.0, bad]), device="cpu")
    for bad in ([[0, 3], [1, 2]], [[-1, 1], [1, 2]]):
        with pytest.raises(ValueError, match="outside"):
            DeviceGraph.from_edges(3, torch.tensor(bad), torch.tensor([1.0, 1.0]), device="cpu")
    g = DeviceGraph.from_edges(3, e, torch.tensor([1.0, 1.0]), device="cpu")
    with pytest.raises(ValueError, match="positive"):
        g.reset_vector([0.0, -1.0, float("nan")])
    np.testing.assert_allclose(g.reset_vector([2.0, -1.0, float("nan")]).numpy(), [1.0, 0.0, 0.0])


def test_iteration_count_meets_the_tolerance():
    assert ppr_iterations(0.5) == 35
    assert ppr_iterations(0.0) == 0
    for d in (0.3, 0.5, 0.85):
        T = ppr_iterations(d, 1e-10)
        assert 2 * d ** (T + 1) / (1 - d) <= 1e-10 < 2 * d ** T / (1 - d)


# ------------------------------------------------------------------------------------------------ the rebinding
def _reference_module():
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    H.install_stand_ins()
    os.environ.setdefault("OPENAI_API_KEY", "stub")
    import src.comorag  # noqa: F401
    return sys.modules["src.comorag.ComoRAG"]


class _Rows:
    def __init__(self, texts):
        self.texts = texts

    def get_row(self, key):
        return {"content": self.texts[key]}


def _scenario(main, rng):
    """A ComoRAG instance (no __init__) with a random graph of entity and passage vertices, and a fact list."""
    phrases = [f"Phrase {i}" for i in range(25)]
    in_graph = phrases[:20]
    ent_keys = [compute_mdhash_id(p.lower(), prefix="entity-") for p in in_graph]
    n_pass = int(rng.integers(3, 15))
    pass_keys = [compute_mdhash_id(f"passage {i}", prefix="chunk-") for i in range(n_pass)]
    names = ent_keys + pass_keys
    order = rng.permutation(len(names))
    g = H._Graph()
    g.add_vertices(len(names), attributes={"name": [names[i] for i in order]})
    rag = object.__new__(main.ComoRAG)
    rag.graph = g
    rag.node_name_to_vertex_idx = {nm: i for i, nm in enumerate(g.vs["name"])}
    rag.ent_node_to_num_chunk = {k: int(rng.integers(0, 4)) for k in ent_keys}
    rag.passage_node_keys = pass_keys
    rag.passage_node_idxs = [rag.node_name_to_vertex_idx[k] for k in pass_keys]
    rag.ver_embedding_store = _Rows({k: f"text of {k}" for k in pass_keys})
    raw = rng.normal(size=n_pass).astype(np.float32)
    if rng.uniform() < 0.2:
        raw[:] = 0.25                                                         # constant: min_max_normalize gives ones
    dpr_ids = np.argsort(raw)[::-1].copy()
    dpr_scores = ((raw - raw.min()) / max(raw.max() - raw.min(), 1e-6)).astype(np.float32)[dpr_ids]
    rag.dense_passage_retrieval = lambda query, need_cluster=False: (dpr_ids.copy(), dpr_scores.copy())
    n_facts = int(rng.integers(0, 12))
    facts = [(str(rng.choice(phrases)).upper() if rng.uniform() < 0.3 else str(rng.choice(phrases)), "rel",
              str(rng.choice(phrases))) for _ in range(n_facts)]
    scores = rng.uniform(0, 1, 40).astype(np.float32)
    scores[rng.integers(0, 40, 8)] = 0.0
    idx = [int(i) for i in rng.integers(0, 40, n_facts)]
    kw = dict(query="q", link_top_k=int(rng.choice([0, 2, 5, 30])), query_fact_scores=scores, top_k_facts=facts,
              top_k_fact_indices=idx, passage_node_weight=float(rng.choice([0.0, 0.005, 0.05])))
    return rag, kw


def _call(fn, rag, kw):
    handed = {}

    def run_ppr(reset_prob, damping=0.5):
        handed["weights"] = np.array(reset_prob, copy=True)
        return np.arange(len(rag.passage_node_idxs)), np.zeros(len(rag.passage_node_idxs))
    rag.run_ppr = run_ppr
    try:
        out = fn(rag, **kw)
    except AssertionError as e:
        return {"assert": str(e).split(":")[0]}, handed
    return out, handed


@needs_ref
@pytest.mark.parametrize("seed", range(60))
def test_rebound_graph_search_hands_over_the_reference_node_weights(seed):
    main = _reference_module()
    ref_fn = main.ComoRAG.__dict__.get("_comorag_b200_originals", {}).get("graph_search_with_fact_entities") or \
        main.ComoRAG.graph_search_with_fact_entities
    if getattr(ref_fn, "__module__", "") == "comorag_b200.comorag_methods":
        pytest.skip("reference method not reachable")
    rag, kw = _scenario(main, np.random.default_rng(seed))
    want, want_w = _call(ref_fn, rag, kw)
    got, got_w = _call(cm.graph_search_with_fact_entities, rag, kw)
    if isinstance(want, dict):
        assert isinstance(got, dict) and got == want and "weights" not in got_w
        return
    assert want_w["weights"].dtype == got_w["weights"].dtype == np.float64
    np.testing.assert_array_equal(want_w["weights"].view(np.uint64), got_w["weights"].view(np.uint64))
    assert list(want[2].items()) == list(got[2].items())
    assert all(type(a) is type(b) for a, b in zip(want[2].values(), got[2].values()))


def _restore_store(main, package, ref_store):
    for name, mod in list(sys.modules.items()):
        if mod is not None and (name == package or name.startswith(package + ".")) and \
                getattr(mod, "EmbeddingStore", None) is not None and \
                getattr(mod, "EmbeddingStore").__module__ == "comorag_b200.embedding_store":
            mod.EmbeddingStore = ref_store


@needs_ref
def test_install_graph_rebinds_exactly_the_two_methods():
    import comorag_b200.install as crag
    main = _reference_module()
    cls = main.ComoRAG
    ref_store = sys.modules["src.comorag.embedding_store"].EmbeddingStore
    crag.uninstall_search("src.comorag")
    before = {k: v for k, v in cls.__dict__.items() if callable(v)}
    try:
        counts = crag.install("src.comorag", summaries=False, search=False, knn=False, encoder=False)
        assert not any(k.startswith("ComoRAG.") for k in counts)
        assert {k: v for k, v in cls.__dict__.items() if callable(v)} == before      # graph=False: nothing rebound
        counts = crag.install("src.comorag", summaries=False, search=False, knn=False, encoder=False, graph=True)
        assert sorted(k for k in counts if k.startswith("ComoRAG.")) == \
            ["ComoRAG.graph_search_with_fact_entities", "ComoRAG.run_ppr"]
        after = {k: v for k, v in cls.__dict__.items() if callable(v)}
        changed = sorted(k for k in after if after[k] is not before.get(k))
        assert changed == ["graph_search_with_fact_entities", "run_ppr"]
        assert cls.run_ppr is cm.run_ppr and cls.graph_search_with_fact_entities is cm.graph_search_with_fact_entities
        crag.uninstall_search("src.comorag")
        assert {k: v for k, v in cls.__dict__.items() if callable(v)} == before
    finally:
        crag.uninstall_search("src.comorag")
        _restore_store(main, "src.comorag", ref_store)
