"""crag_ppr on the device against the float64 oracle, held to the error bound of tests/ppr_bound.py (derived in its
docstring and in tests/test_ppr_emulated.py): hand graphs, a random ComoRAG-shaped graph, a power-law graph, a star
whose hub has 2^20 neighbours and isolated vertices carrying reset mass, at d in {0, 0.5, 0.85} and T in {0, 1,
default}.  Plus: the out_vertices gather, the passage ranking, bit-identical repeats on two streams, argument
errors."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ppr_bound  # noqa: E402

from comorag_b200 import _native  # noqa: E402
from comorag_b200.graph import DeviceGraph, ppr_iterations  # noqa: E402
from comorag_b200.index import rank_scores  # noqa: E402

pytestmark = pytest.mark.gpu
D85 = float(np.float32(0.85))       # the kernel takes d as fp32: the oracle gets the same value


def _comorag_shaped(rng, passages=3000, entities=1200, summaries=50):
    """Passages linked to 10-20 entities (both orientations), entity fact edges in both orientations, synonymy
    edges with weights in [0.8, 1], isolated summary vertices at the end."""
    links = rng.integers(10, 21, passages)
    p = np.repeat(np.arange(passages), links) + entities
    ent = rng.integers(0, entities, p.size)
    fact_a, fact_b = rng.integers(0, entities, 4000), rng.integers(0, entities, 4000)
    keep = fact_a != fact_b
    fa, fb = fact_a[keep], fact_b[keep]
    syn_a, syn_b = rng.integers(0, entities, 500), rng.integers(0, entities, 500)
    keep = syn_a != syn_b
    e = np.concatenate([np.stack([p, ent], 1), np.stack([ent, p], 1), np.stack([fa, fb], 1), np.stack([fb, fa], 1),
                        np.stack([syn_a[keep], syn_b[keep]], 1)])
    w = np.concatenate([np.ones(2 * p.size), np.ones(2 * fa.size), rng.uniform(0.8, 1.0, int(keep.sum()))])
    return entities + passages + summaries, e, w


def _power_law(rng, n=20000, m=80000):
    a = np.minimum((rng.pareto(1.2, m) * 3).astype(np.int64), n - 1)
    b = rng.integers(0, n, m)
    keep = a != b
    return n, np.stack([a[keep], b[keep]], 1), rng.uniform(0.1, 2.0, int(keep.sum()))


def _graphs():
    rng = np.random.default_rng(20251016)
    out = {}
    out["path"] = (6, np.array([[0, 1], [1, 2], [2, 3], [3, 4], [4, 5]]), np.array([1.0, 2.0, 0.5, 1.0, 3.0]))
    out["triangle + isolated"] = (5, np.array([[0, 1], [1, 2], [2, 0], [1, 0], [0, 1]]), np.array([1.0, 1.0, 2.0, 0.5, 0.25]))
    out["comorag-shaped"] = _comorag_shaped(rng)
    out["power-law"] = _power_law(rng)
    leaves = 1 << 20
    out["star 2^20"] = (leaves + 1, np.stack([np.zeros(leaves, np.int64), np.arange(1, leaves + 1)], 1),
                        rng.uniform(0.8, 1.0, leaves))
    return out


GRAPHS = _graphs()
_dev_cache = {}


def _device_graph(name):
    if name not in _dev_cache:
        n, e, w = GRAPHS[name]
        _dev_cache[name] = DeviceGraph.from_edges(n, torch.as_tensor(e, device="cuda"), torch.as_tensor(w, device="cuda"))
    return _dev_cache[name]


def _reset(name, n):
    rng = np.random.default_rng(len(name))
    r = rng.uniform(0, 1, n) * (rng.uniform(size=n) < 0.2)
    r[0] = 1.0
    r[-1] = 0.5                      # the last vertex is isolated in the triangle, comorag-shaped and power-law graphs
    return r


def _check(name, d, T):
    n, e, w = GRAPHS[name]
    g = _device_graph(name)
    reset = _reset(name, n)
    got = g.ppr_iterate(g.reset_vector(reset), d, T).cpu().numpy().astype(np.float64)
    x, bnd = ppr_bound.bound(n, e, w, reset, d, T, exact_iterate=T != ppr_iterations(d))
    err = np.abs(got - x)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(err == 0, 0.0, err / bnd)
    assert np.isfinite(got).all()
    assert ratio.max() <= 1.0, f"{name} d={d} T={T}: {ratio.max():.3f} of the bound at vertex {int(ratio.argmax())}"
    return ratio.max()


@pytest.mark.parametrize("name", list(GRAPHS))
@pytest.mark.parametrize("d", [0.0, 0.5, D85])
def test_ppr_within_the_bound_of_the_oracle(name, d):
    for T in sorted({0, 1, ppr_iterations(d)}):
        _check(name, d, T)


def test_isolated_vertices_carrying_reset_mass():
    n = 50
    e = np.array([[0, 1], [1, 2], [2, 3], [3, 0], [1, 3]])
    w = np.array([1.0, 2.0, 1.0, 0.5, 1.0])
    reset = np.zeros(n)
    reset[[0, 10, 20, 49]] = [1.0, 2.0, 0.5, 3.0]
    g = DeviceGraph.from_edges(n, torch.as_tensor(e, device="cuda"), torch.as_tensor(w, device="cuda"))
    for d in (0.5, D85):
        got = g.personalized_pagerank(reset, d).cpu().numpy().astype(np.float64)
        x, bnd = ppr_bound.bound(n, e, w, reset, d, ppr_iterations(d), exact_iterate=False)
        assert (np.abs(got - x) <= bnd).all()
        assert got[10] > 0 and got[5] == 0.0


def test_gather_equals_the_full_vector():
    g = _device_graph("comorag-shaped")
    v = g.reset_vector(_reset("comorag-shaped", g.n))
    full = g.ppr_iterate(v, 0.5, 35)
    sub = torch.as_tensor(np.random.default_rng(1).choice(g.n, 777, replace=True), device="cuda")
    part = g.ppr_iterate(v, 0.5, 35, vertices=sub)
    assert torch.equal(part.view(torch.int32), full[sub].view(torch.int32))


def test_passage_ranking_matches_the_oracle_outside_near_ties():
    name = "comorag-shaped"
    n, e, w = GRAPHS[name]
    g = _device_graph(name)
    reset = _reset(name, n)
    passages = np.arange(1200, 4200)
    scores = g.personalized_pagerank(reset, 0.5, vertices=torch.as_tensor(passages, device="cuda"))
    ids, sorted_scores = rank_scores(scores)
    ids = ids.cpu().numpy()
    x, bnd = ppr_bound.bound(n, e, w, reset, 0.5, ppr_iterations(0.5), exact_iterate=False)
    xs, tol = x[passages], 2 * bnd[passages].max()
    assert sorted(ids.tolist()) == list(range(len(passages)))
    seq = xs[ids]
    suffix_max = np.maximum.accumulate(seq[::-1])[::-1]
    # every passage outranks, in the oracle, all later ones except those within twice the bound (a near-tie set)
    assert (seq[:-1] >= suffix_max[1:] - tol).all()
    np.testing.assert_array_equal(sorted_scores.cpu().numpy(), scores.cpu().numpy()[ids])


def test_bit_identical_across_repeats_and_streams():
    g = _device_graph("power-law")
    v = g.reset_vector(_reset("power-law", g.n))
    first = g.ppr_iterate(v, 0.5, 35)
    side = torch.cuda.Stream()
    for st in (None, side, None, side):
        again = g.ppr_iterate(v, 0.5, 35, stream=st)
        torch.cuda.synchronize()
        assert torch.equal(first.view(torch.int32), again.view(torch.int32))


def test_argument_errors_return_before_any_launch():
    lib = _native.load()
    g = _device_graph("path")
    v = g.reset_vector(_reset("path", g.n))
    ws_bytes = lib.crag_ppr_workspace_bytes(g.n, g.nnz)
    ws = torch.empty(ws_bytes + 256, dtype=torch.uint8, device="cuda")
    out = torch.full((g.n,), -7.0, device="cuda")
    sub = torch.zeros(3, dtype=torch.int32, device="cuda")
    base = dict(row_ptr=g.row_ptr.data_ptr(), col=g.col.data_ptr(), coef=g.coef.data_ptr(), n=g.n, nnz=g.nnz,
                reset=v.data_ptr(), d=0.5, T=35, verts=None, n_out=g.n, out=out.data_ptr(), ws=ws.data_ptr(),
                ws_bytes=ws_bytes)

    def call(**kw):
        a = {**base, **kw}
        return lib.crag_ppr(a["row_ptr"], a["col"], a["coef"], a["n"], a["nnz"], a["reset"], a["d"], a["T"], a["verts"],
                            a["n_out"], a["out"], a["ws"], a["ws_bytes"], None)
    INVALID, WORKSPACE = -1, -3
    for kw, rc in [(dict(n=0), INVALID), (dict(nnz=-1), INVALID), (dict(d=1.0), INVALID), (dict(d=-0.1), INVALID),
                   (dict(d=float("nan")), INVALID), (dict(T=-1), INVALID), (dict(n_out=3), INVALID),
                   (dict(verts=sub.data_ptr(), n_out=-1), INVALID), (dict(row_ptr=None), INVALID), (dict(col=None), INVALID),
                   (dict(reset=None), INVALID), (dict(out=None), INVALID), (dict(ws=ws.data_ptr() + 4), INVALID),
                   (dict(ws_bytes=ws_bytes - 1), WORKSPACE)]:
        assert call(**kw) == rc, kw
        assert lib.crag_last_error().decode().startswith("crag_ppr")
    torch.cuda.synchronize()
    assert (out == -7.0).all()                   # nothing was launched
    assert lib.crag_ppr_workspace_bytes(0, 5) == 0 and lib.crag_ppr_workspace_bytes(5, -1) == 0
    assert call() == 0
    torch.cuda.synchronize()
    assert abs(out.sum().item() - 1.0) < 1e-5
