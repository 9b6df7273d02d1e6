"""crag_ivf_search (IVFIndex) on the GPU, bit for bit against scan_reference.ivf_from_scores: ids, scores and
(min, max) derived from the score-all matrix of the queries against the padded residuals, with the engine's own
probed lists (or the caller's).  Also the IVF build's assignment, bit for bit against assign_from_scores.

Covered: the shapes of test_ivf_gpu.py and 1 / 33 / 70 queries (several 32-query passes whose probes differ);
nlist not a multiple of 32; nprobe 1 and nlist; hand-made layouts with empty lists and lists of exactly 128 and 129
rows; caller probes holding -1, a repeated list and an id >= nlist; a -1 / -inf tail and a query that probes only
empty lists; ids beyond 2^33; two streams, the host entry point and ShardedIVF at world 1; and an exact tie
between two lists, which goes to the smaller stored position (the smaller list id), not the smaller original id."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import scan_reference as sr  # noqa: E402
from test_ivf_gpu import _clustered  # noqa: E402
from test_scan_exact_gpu import BIG_OFFSET, DEV, score_all  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _lib():
    assert torch.cuda.is_available()
    from comorag_b200 import _native
    _native.load()


def check(idx, qb, nprobe, k, probed=None, stream=None):
    """One search against the reference; returns the engine's (ids, scores, minmax, probed)."""
    ids, sc, mm, (p_ids, p_sc) = idx.search_device(qb, nprobe, k, stream=stream, probed=probed)
    torch.cuda.synchronize()
    S, _ = score_all(idx.residuals, qb)
    w_ids, w_sc, w_mm = sr.ivf_from_scores(S, p_ids, p_sc, idx.list_tile_start, idx.list_rows, idx.row_ids, k)
    sr.assert_bits(ids, w_ids, "ids")
    sr.assert_bits(sc, w_sc, "scores")
    sr.assert_bits(mm, w_mm, "minmax")
    return ids, sc, mm, (p_ids, p_sc)


def build(n, d, nlist, nq, seed=0, row_offset=0):
    from comorag_b200.ivf import IVFIndex
    x, q = _clustered(n, d, nq, seed)
    xd = torch.from_numpy(x).to(DEV)
    idx = IVFIndex.build(xd, nlist, iters=4, seed=seed, row_offset=row_offset)
    return idx, xd, torch.from_numpy(q).to(DEV).to(torch.bfloat16)


def hand_index(assignment, nlist, dim, residual_fn, row_offset=0, seed=0):
    """An IVFIndex over a hand-made assignment, laid out by ivf_layout; residual_fn(order) -> bf16 residuals of the
    rows in stored order (list, then original id)."""
    from comorag_b200.ivf import IVFIndex, TILE_ROWS, ivf_layout
    a = torch.as_tensor(assignment, dtype=torch.int64, device=DEV)
    order, dest, tile_start, list_rows = ivf_layout(a, nlist)
    total = max(int(tile_start[-1]), 1) * TILE_ROWS
    res = torch.zeros((total, dim), dtype=torch.bfloat16, device=DEV)
    row_ids = torch.full((total,), -1, dtype=torch.int64, device=DEV)
    res[dest] = residual_fn(order)
    row_ids[dest] = order + row_offset
    g = torch.Generator(device=DEV).manual_seed(seed)
    cent = torch.nn.functional.normalize(torch.randn(nlist, dim, generator=g, device=DEV), dim=1).bfloat16()
    return IVFIndex(cent, res, row_ids, tile_start.contiguous(), list_rows.contiguous(), a.numel())


@pytest.mark.parametrize("n,d,nlist,nprobe,k,nq", [(20000, 128, 64, 8, 10, 8), (50000, 768, 128, 16, 100, 40),
                                                   (3000, 64, 16, 16, 10, 3), (700, 64, 32, 2, 64, 5),
                                                   (20000, 128, 64, 8, 10, 1), (20000, 128, 64, 8, 10, 33),
                                                   (20000, 128, 64, 8, 10, 70), (6000, 128, 45, 1, 50, 33),
                                                   (6000, 128, 45, 45, 128, 70)])
def test_ivf_search_equals_reference(n, d, nlist, nprobe, k, nq):
    """The engine's coarse pass, plan, scan, merge and id map; and the build's row -> list map, which must be
    assign_from_scores of the score-all matrix of the bf16 centroids against the bf16 rows."""
    idx, x, qb = build(n, d, nlist, nq)
    S_cent, _ = score_all(x.to(torch.bfloat16), idx.centroids.matrix())
    w_a, _ = sr.assign_from_scores(S_cent)
    sr.assert_bits(idx.assignment, w_a.to(torch.int64), "assignment")
    ids, _, _, (p_ids, _) = check(idx, qb, nprobe, k)
    if nq > 32:                                           # the passes probe different lists
        assert len({tuple(r) for r in p_ids[:32].tolist()} ^ {tuple(r) for r in p_ids[32:].tolist()}) > 0
    h_ids, _ = idx.search(qb.float().cpu().numpy(), nprobe, k)
    assert (torch.from_numpy(h_ids) == ids.cpu()).all()


def _edge_index(seed=0):
    """nlist 37: lists of 0, 1, 128, 129 and 300 rows among random sizes; residuals of mixed magnitude; ids from
    2^33 + 7 on."""
    g = torch.Generator().manual_seed(seed)
    sizes = torch.randint(0, 60, (37,), generator=g)
    sizes[[0, 5, 36]] = 0
    sizes[[1, 6]] = torch.tensor([128, 129])
    sizes[2], sizes[7], sizes[35] = 1, 300, 129
    assignment = torch.repeat_interleave(torch.arange(37), sizes)
    assignment = assignment[torch.randperm(assignment.numel(), generator=g)]
    dim = 192

    def residuals(order):
        gd = torch.Generator(device=DEV).manual_seed(seed + 1)
        r = 0.1 * torch.randn(order.numel(), dim, generator=gd, device=DEV)
        return (r * torch.exp2((order % 9 - 4).float())[:, None]).bfloat16()
    return hand_index(assignment, 37, dim, residuals, row_offset=BIG_OFFSET, seed=seed), sizes


@pytest.mark.parametrize("nprobe,k", [(1, 10), (5, 128), (37, 64), (37, 1)])
def test_edge_layout_with_engine_probes(nprobe, k):
    idx, sizes = _edge_index()
    qb = torch.nn.functional.normalize(torch.randn(70, idx.dim, generator=torch.Generator().manual_seed(nprobe)), dim=1)
    ids, _, _, _ = check(idx, qb.to(DEV).bfloat16(), nprobe, k)
    assert bool((ids[ids >= 0] >= BIG_OFFSET).all())


def test_caller_probes_with_absent_repeated_and_empty_lists():
    """Caller probes: -1, a list twice (same coarse score), an id >= nlist, empty lists only (all -1 / -inf, minmax
    (+inf, -inf)), a lone 129-row list, fewer probed rows than k (a tail), and negative coarse scores."""
    idx, sizes = _edge_index(seed=4)
    nq, nprobe, k = 40, 6, 128
    g = torch.Generator().manual_seed(9)
    qb = torch.nn.functional.normalize(torch.randn(nq, idx.dim, generator=g), dim=1).to(DEV).bfloat16()
    p_ids = torch.randint(0, 37, (nq, nprobe), generator=g)
    p_sc = torch.randn(nq, nprobe, generator=g)
    p_ids[0] = torch.tensor([3, -1, 3, 37, 1000, 8])
    p_sc[0, 2] = p_sc[0, 0]
    p_ids[1] = torch.tensor([0, 5, 36, -1, 0, 36])                     # empty lists only
    p_sc[1, 4], p_sc[1, 5] = p_sc[1, 0], p_sc[1, 2]
    p_ids[2] = torch.tensor([6, -1, -1, -1, -1, -1])                   # one 129-row list: 128 of its rows
    p_ids[33] = torch.tensor([2, -1, 2, -1, 0, 5])                     # one real row, in the second pass
    p_sc[33, 2] = p_sc[33, 0]
    p_sc[34] = -p_sc[34].abs() - 2
    for q in range(nq):                                                # a repeated random probe repeats its score
        for j in range(nprobe):
            first = (p_ids[q, :j] == p_ids[q, j]).nonzero()
            if first.numel():
                p_sc[q, j] = p_sc[q, int(first[0])]
    probed = (p_ids.to(DEV), p_sc.to(DEV))
    ids, sc, mm, _ = check(idx, qb, nprobe, k, probed=probed)
    assert bool((ids[1] == -1).all()) and bool(torch.isneginf(sc[1]).all())
    assert mm[1, 0].item() == float("inf") and mm[1, 1].item() == float("-inf")
    assert int((ids[2] >= 0).sum()) == 128 and int((ids[33] >= 0).sum()) == 1 and bool(torch.isneginf(sc[33, 1:]).all())
    n0 = int(sizes[3] + sizes[8])
    assert int((ids[0] >= 0).sum()) == min(k, n0)


def test_cross_list_exact_tie_goes_to_the_smaller_list():
    """Lists 0 and 2 hold identical residual rows and the caller gives them equal coarse scores.  List 0's rows have
    the LARGER original ids, so a tie rule by id would put list 2's row first; the engine puts the smaller stored
    position -- list 0's row -- first, as ivf_oracle, DESIGN.md section 7 and the header say.  Dyadic residuals and
    queries make every score exact, so the ties are exact whatever the summation order."""
    dim, m = 128, 64
    g = torch.Generator(device=DEV).manual_seed(21)
    twins = (torch.randint(-3, 4, (m, dim), generator=g, device=DEV).float() / 8).bfloat16()
    other = (torch.randint(-3, 4, (50, dim), generator=g, device=DEV).float() / 8).bfloat16()
    assignment = torch.tensor([2] * m + [1] * 50 + [0] * m)             # ids 0..63 -> list 2, 114..177 -> list 0

    def residuals(order):
        r = torch.empty((order.numel(), dim), dtype=torch.bfloat16, device=DEV)
        o = order.to(DEV)
        r[o < m] = twins[o[o < m]]
        r[(o >= m) & (o < m + 50)] = other[o[(o >= m) & (o < m + 50)] - m]
        r[o >= m + 50] = twins[o[o >= m + 50] - m - 50]
        return r
    idx = hand_index(assignment, 3, dim, residuals)
    nq, k = 34, 2 * m
    qb = (torch.randint(-3, 4, (nq, dim), generator=g, device=DEV).float() / 8).bfloat16()
    p_ids = torch.tensor([[2, 0, 1], [0, 2, 1]] * (nq // 2), device=DEV)
    c = torch.full((nq, 1), 0.5, device=DEV)
    p_sc = torch.cat([c, c, c - 100.0], dim=1)
    ids, sc, _, _ = check(idx, qb, 3, k, probed=(p_ids, p_sc))
    ids, sc = ids.cpu(), sc.cpu()
    for q in range(nq):                 # each run of equal scores: list 0's rows, then their twins in list 2, in order
        for s in sc[q].unique():
            run = ids[q][sc[q] == s]
            h = run.numel() // 2
            assert run.numel() == 2 * h and bool((run[:h] >= m + 50).all()) and torch.equal(run[h:], run[:h] - m - 50)


def test_two_streams_host_entry_and_sharded_world_1():
    from comorag_b200.ivf import ShardedIVF
    idx, _, qb = build(20000, 256, 64, 37, seed=4, row_offset=BIG_OFFSET)
    want = check(idx, qb, 8, 20)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    a = idx.search_device(qb, 8, 20, stream=s1)
    b = idx.search_device(qb[:33], 8, 20, stream=s2)
    torch.cuda.synchronize()
    for g, w in zip(a[:3], want[:3]):
        sr.assert_bits(g, w)
    for g, w in zip(b[:3], want[:3]):
        sr.assert_bits(g, w[:33])
    h_ids, h_sc = idx.search(qb.float().cpu().numpy(), 8, 20)
    sr.assert_bits(torch.from_numpy(h_ids), want[0])
    sr.assert_bits(torch.from_numpy(h_sc), want[1])
    for g, w in zip(ShardedIVF(idx).search_device(qb, 8, 20), want[:3]):
        sr.assert_bits(g, w)
