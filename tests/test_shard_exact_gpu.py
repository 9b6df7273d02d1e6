"""The row-sharded search on one GPU, bit for bit: the merge kernels against shard_cases.merge_reference, and both
exchange formulations, ShardedIndex and ShardedIVF on virtual ranks (one thread and stream per rank).

  merge       crag_merge_topk and crag_merge_topk_packed at k in every selector tier (32 / 64 / 128 keys), 0 .. 64
              parts and 1 .. 100 queries, on adversarial records (ties across parts, +-0, -inf with a valid id, absent
              entries, unsorted parts), with sentinels around every output.
  all-gather  SearchSession(gather=...): scan, finalize into the packed record, a virtual all-gather, merge kernel.
  peer        SearchSession(exchange=PeerExchange.from_local_buffers(...)), eager, many epochs through one set of
              exchange buffers.  Not graph-captured: a captured session's warm-up is a collective, so all virtual
              ranks would capture at once, and torch supports one capture at a time per process.
  ShardedIndex / ShardedIVF through a test-side factory that sets what __init__ sets, without a process group.

Every rank must return the unsharded DenseIndex answer, which must equal merge_reference of the per-rank answers.
Corpora are knn_cases.int_rows with exact scores, so ties planted across shard boundaries are exact on every rank.
Real NCCL and NVLink peer memory need two GPUs or more (tools/gpu_check_dist.py)."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ivf_i8_oracle as io  # noqa: E402
import scan_reference as sr  # noqa: E402
import shard_cases as sc  # noqa: E402
from test_ivf_exact_gpu import check as ivf_check  # noqa: E402
from test_oracle_ivf_i8 import clustered  # noqa: E402
from test_scan_exact_gpu import DEV, SENTINEL  # noqa: E402

pytestmark = pytest.mark.gpu

K_TIERS = [1, 32, 33, 64, 65, 128]


@pytest.fixture(scope="module")
def lib():
    assert torch.cuda.is_available()
    from comorag_b200 import _native
    return _native.load()


def _sentinel_out(nq, k):
    """Outputs with one sentinel row before and after: (ids, scores, minmax) full buffers."""
    ids = torch.full((nq + 2, k), -7, dtype=torch.int64, device=DEV)
    s = torch.full((nq + 2, k), SENTINEL, dtype=torch.int32, device=DEV).view(torch.float32)
    mm = torch.full((nq + 2, 2), SENTINEL, dtype=torch.int32, device=DEV).view(torch.float32)
    return ids, s, mm


def _inner(bufs):
    """The outputs between the sentinels, after checking the sentinels are intact."""
    ids, s, mm = bufs
    assert bool((ids[0] == -7).all() and (ids[-1] == -7).all()), "ids sentinel overwritten"
    for t in (s, mm):
        b = t.view(torch.int32)
        assert bool((b[0] == SENTINEL).all() and (b[-1] == SENTINEL).all()), "sentinel overwritten"
    return ids[1:-1], s[1:-1], mm[1:-1]


def merge_native(lib, ids, scores, mm, k, packed):
    from comorag_b200 import _native
    from comorag_b200.index import packed_record_bytes, packed_views
    parts, nq, _ = scores.shape
    out = _sentinel_out(nq, k)
    o = [t[1:].data_ptr() for t in out]
    st = torch.cuda.current_stream().cuda_stream
    if packed:
        per = packed_record_bytes(nq, k)
        rec = torch.full((max(parts, 1) * per,), 0xA5, dtype=torch.uint8, device=DEV)   # padding bytes are noise
        for p in range(parts):
            for v, t in zip(packed_views(rec[p * per:(p + 1) * per], nq, k), (ids[p], scores[p], mm[p])):
                v.copy_(t)
        rc = lib.crag_merge_topk_packed(rec.data_ptr() if parts else 0, per, parts, nq, k, *o, st)
    else:
        ptrs = [t.data_ptr() if parts else 0 for t in (scores, ids, mm)]
        rc = lib.crag_merge_topk(*ptrs, parts, nq, k, *o, st)
    _native.check(rc, "merge")
    torch.cuda.synchronize()
    return _inner(out)


# ------------------------------------------------------------------------------------------------------ merge kernels
@pytest.mark.parametrize("k", K_TIERS)
def test_merge_kernels_equal_reference(lib, k):
    for parts in (0, 1, 2, 3, 8, 16, 64):
        for nq in (1, 5, 32, 100):
            ids, s, mm = sc.adversarial_records(parts, nq, k, seed=parts * 1000 + nq * 7 + k)
            want = sc.merge_reference(ids, s, mm, k)
            d = (ids.to(DEV), s.to(DEV), mm.to(DEV))
            for packed in (False, True):
                sc.assert_merge(merge_native(lib, *d, k, packed), want, f"parts={parts} nq={nq} packed={packed}")


def test_merge_minmax_signed_zero(lib):
    """fminf / fmaxf over the parts' (min, max) when they are +0 and -0, in both part orders and at both ends of a
    warp's shuffle tree (parts 0 / 1 and 0 / 16): the kernels order -0 below +0, as the keys do."""
    z = [(0.0, 0.0), (-0.0, -0.0)]
    for parts, a, b in [(2, 0, 1), (17, 0, 16), (33, 1, 32)]:
        for first in (0, 1):
            mm = torch.full((parts, 1, 2), 0.0)
            mm[:, 0] = torch.tensor([float("inf"), float("-inf")])
            mm[a, 0] = torch.tensor(z[first])
            mm[b, 0] = torch.tensor(z[1 - first])
            ids = torch.full((parts, 1, 1), -1, dtype=torch.int64)
            s = torch.zeros((parts, 1, 1))
            got = merge_native(lib, ids.to(DEV), s.to(DEV), mm.to(DEV), 1, packed=False)[2].cpu()
            assert got.view(torch.int32).tolist() == [[int(0x80000000) - (1 << 32), 0]], (parts, a, b, first, got)


# ------------------------------------------------------------------------------------------------- virtual ranks
def shards_of(x, offs, base):
    from comorag_b200.index import DenseIndex
    return [DenseIndex.from_tensor(x[offs[r]:offs[r + 1]], row_offset=base + offs[r]) for r in range(len(offs) - 1)]


def per_rank_reference(shards, q, k):
    parts = [s.search_device(q, k) for s in shards]
    return sc.merge_reference(*(torch.stack([p[i] for p in parts]) for i in range(3)), k)


def _case(world, k, i, n=3000):
    """(rows on the device, bounds, kind) of the i-th case of a (world, k) sweep: corpus kinds and layouts rotate."""
    kinds = ("boundary", "mixed", "all_equal")
    layouts = ("ragged", "small", "even") if world >= 3 else ("ragged", "even")
    layout = layouts[i % len(layouts)]
    kind = kinds[(i + k) % len(kinds)]
    offs = sc.edge_bounds(n, world, layout, k)
    x, _ = sc.planned_corpus(kind, n, k, offs, seed=world * 100 + k + i)
    return x.to(DEV), offs, kind


def _check_rank_outputs(outs, whole, shards, q, k, kind, what):
    want = whole.search_device(q, k)
    sc.assert_merge(want, per_rank_reference(shards, q, k), f"{what}: unsharded vs merge of the ranks")
    if kind == "all_equal":
        assert torch.equal(want[0][0].cpu(), sc.BIG_BASE + torch.arange(k)), what
    for r, o in enumerate(outs):
        sc.assert_merge(o, want, f"{what} rank {r}")


@pytest.mark.parametrize("world", [2, 3, 5, 8, 16])
def test_all_gather_formulation(world):
    """scan + finalize into the packed record + virtual all-gather + crag_merge_topk_packed on every rank: the
    unsharded answer, for every k tier and nq in {1, 7, 32}, over three consecutive runs with new queries."""
    from comorag_b200.index import DenseIndex, SearchSession
    i = 0
    for k in K_TIERS:
        for nq in (1, 7, 32):
            x, offs, kind = _case(world, k, i)
            i += 1
            whole = DenseIndex.from_tensor(x, row_offset=sc.BIG_BASE)
            shards = shards_of(x, offs, sc.BIG_BASE)
            group = sc.VirtualGroup(world)
            sessions = [SearchSession(shards[r], nq, k, gather=group.rank(r).gather, world=world, use_graph=False)
                        for r in range(world)]
            for run in range(3):
                q = sc.exact_queries(nq, seed=1000 * run + i).to(DEV)
                outs = sc.run_ranks(world, lambda r: tuple(t.clone() for t in sessions[r].run(q)), DEV)
                _check_rank_outputs(outs, whole, shards, q, k, kind, f"k={k} nq={nq} {kind} {offs} run {run}")


PEER_CASES = [(1, 1), (32, 7), (33, 7), (40, 1), (48, 32), (64, 7), (65, 32), (128, 7), (128, 32)]


@pytest.mark.parametrize("world", [2, 4, 8])
def test_peer_formulation(world):
    """finalize_exchange_kernel through SearchSession on `world` virtual ranks, one set of exchange buffers for all
    cases (epochs 1 .. 30+ per query slot, both parities, sessions of different nq and k), an empty rank wherever the
    layout has one; the exchange status is checked after every run.  Sessions run eagerly: a captured session's
    warm-up is a collective, so every virtual rank would capture at once, and torch supports one capture at a time
    per process (concurrent builds were invalidated on H100).  Each run is enqueued from one thread in rank order,
    as test_fused_finalize_exchange_merge_virtual_ranks does.  8 ranks run the cases of fewer than 32 queries: with
    32 queries on each of 8 ranks (256 exchange CTAs spinning at once on one GPU) the exchange timed out on H100,
    eager and captured, while every case below 32 queries passes.  The likely cause is that the spinning CTAs hold
    the SM resources a later rank's scan needs; a real rank's exchange shares its GPU with no other rank."""
    from comorag_b200 import _native
    from comorag_b200.dist import PeerExchange
    from comorag_b200.index import DenseIndex, SearchSession
    lib = _native.load()
    nbytes = int(lib.crag_exchange_buffer_bytes(world))
    bufs = [torch.zeros(nbytes, dtype=torch.uint8, device=DEV) for _ in range(world)]
    peers = [PeerExchange.from_local_buffers(bufs, r) for r in range(world)]
    streams = [torch.cuda.Stream(DEV) for _ in range(world)]
    for i, (k, nq) in enumerate(PEER_CASES):
        if world == 8 and nq == 32:
            continue
        x, offs, kind = _case(world, k, i)
        whole = DenseIndex.from_tensor(x, row_offset=sc.BIG_BASE)
        shards = shards_of(x, offs, sc.BIG_BASE)

        sessions = [SearchSession(shards[r], nq, k, exchange=peers[r], world=world, use_graph=False)
                    for r in range(world)]
        for p in peers:
            p.check()
        for run in range(4):
            q = sc.exact_queries(nq, seed=500 * run + i).to(DEV)
            torch.cuda.synchronize()
            outs = []
            for r in range(world):       # every rank's step in flight at once, enqueued from this thread in rank order
                with torch.cuda.stream(streams[r]):
                    outs.append(sessions[r].run(q))
            torch.cuda.synchronize()
            outs = [tuple(t.clone() for t in o) for o in outs]
            for p in peers:
                p.check()
            _check_rank_outputs(outs, whole, shards, q, k, kind, f"k={k} nq={nq} {kind} {offs} run {run}")


# ------------------------------------------------------------------------------------------------------ ShardedIndex
def _sharded_index_case(mode):
    """4 virtual ranks with a ragged split, a tie run cut across a boundary, rows from 2^33 on: (whole, shards, the
    ranks' ShardedIndex, their PeerExchange objects or Nones)."""
    from comorag_b200 import _native
    from comorag_b200.dist import PeerExchange
    from comorag_b200.index import DenseIndex
    world, n, k = 4, 5000, 128
    offs = sc.edge_bounds(n, world, "ragged", k)
    x, _ = sc.planned_corpus("boundary", n, k, offs, seed=77)
    x = x.to(DEV)
    whole = DenseIndex.from_tensor(x, row_offset=sc.BIG_BASE)
    shards = shards_of(x, offs, sc.BIG_BASE)
    group = sc.VirtualGroup(world)
    peers = [None] * world
    if mode == "peer":
        nbytes = int(_native.load().crag_exchange_buffer_bytes(world))
        bufs = [torch.zeros(nbytes, dtype=torch.uint8, device=DEV) for _ in range(world)]
        peers = [PeerExchange.from_local_buffers(bufs, r) for r in range(world)]
    return whole, shards, [sc.virtual_sharded_index(shards[r], group.rank(r), peers[r]) for r in range(world)], peers


def test_sharded_index_all_gather_blocks_and_host_entry(monkeypatch):
    """ShardedIndex in the all-gather formulation: search_device at nq = 70 (blocks of 32 + 32 + 6, each block's
    answer copied out before the next) and k = 128 on every rank at once, k = 129 refused, and the host search()
    entry."""
    import torch.distributed as dist
    monkeypatch.setattr(dist, "all_gather_into_tensor", sc.virtual_all_gather)
    whole, shards, idx, _ = _sharded_index_case("nccl")
    world, k, nq = len(idx), 128, 70
    q = sc.exact_queries(nq, seed=78).to(DEV)
    want = whole.search_device(q, k)
    sc.assert_merge(want, per_rank_reference(shards, q, k), "unsharded vs merge of the ranks")
    for use_graph in (True, False):          # the all-gather formulation is never captured: both run eagerly
        outs = sc.run_ranks(world, lambda r: idx[r].search_device(q, k, use_graph=use_graph), DEV)
        for r, o in enumerate(outs):
            sc.assert_merge(o, want, f"use_graph={use_graph} rank {r}")
    assert sorted(idx[0]._sessions) == [(6, k, False), (6, k, True), (32, k, False), (32, k, True)]
    with pytest.raises(ValueError):
        idx[0].search_device(q, 129)
    host = sc.run_ranks(world, lambda r: idx[r].search(q.float().cpu().numpy(), k), DEV)
    for r, (h_ids, h_s, h_mm) in enumerate(host):
        sc.assert_merge((torch.from_numpy(h_ids), torch.from_numpy(h_s), torch.from_numpy(h_mm)), want, f"host rank {r}")


def test_sharded_index_peer_blocks():
    """ShardedIndex in the peer formulation: search_device for the two block shapes of a 70-query batch (32 and 6
    queries) at k = 128, twice each, and k = 129 refused; eager sessions, as in test_peer_formulation.

    Each call is enqueued from one thread in rank order and nothing is enqueued behind a rank's exchange until every
    rank's exchange is in flight.  Virtual ranks share one GPU's hardware work queues: work a rank enqueues after its
    exchange kernel (the next block of a 70-query call, the copy of its answer, the host entry's device-to-host copy)
    waits for that kernel to finish, which waits for every other rank's record; in a queue that another rank's stream
    also feeds, it holds back that rank's scan, and the exchange times out.  So one call per block here; the block
    loop and the host entry run in the all-gather formulation above, whose collective does not spin on the device."""
    whole, shards, idx, peers = _sharded_index_case("peer")
    world, k = len(idx), 128
    q = sc.exact_queries(70, seed=79).to(DEV)
    blocks = (q[:32], q[64:70])
    streams = [torch.cuda.Stream(DEV) for _ in range(world)]
    for rep in range(2):
        for b in blocks:
            want = whole.search_device(b, k)
            sc.assert_merge(want, per_rank_reference(shards, b, k), "unsharded vs merge of the ranks")
            torch.cuda.synchronize()
            outs = []
            for r in range(world):
                with torch.cuda.stream(streams[r]):
                    outs.append(idx[r].search_device(b, k, use_graph=False))
            torch.cuda.synchronize()
            for p in peers:
                p.check()
            for r, o in enumerate(outs):
                sc.assert_merge(o, want, f"nq={b.shape[0]} rep {rep} rank {r}")
    assert sorted(idx[0]._sessions) == [(6, k, False), (32, k, False)]
    with pytest.raises(ValueError):
        idx[0].search_device(q, 129)


# -------------------------------------------------------------------------------------------------------- ShardedIVF
def _ivf_shards(xd, offs, nlist, base):
    from comorag_b200.ivf import IVFIndex
    whole = IVFIndex.build(xd, nlist, iters=4, seed=0, row_offset=base)
    c = whole.centroids.matrix().contiguous()
    ranks = [IVFIndex.build(xd[offs[r]:offs[r + 1]], nlist, centroids=c, row_offset=base + offs[r])
             for r in range(len(offs) - 1)]
    return whole, ranks


def _sharded_ivf(ranks, monkeypatch, qb, nprobe, k):
    import torch.distributed as dist
    monkeypatch.setattr(dist, "all_gather_into_tensor", sc.virtual_all_gather)
    group = sc.VirtualGroup(len(ranks))
    return sc.run_ranks(len(ranks), lambda r: sc.virtual_sharded_ivf(ranks[r], group.rank(r)).search_device(qb, nprobe, k), DEV)


@pytest.mark.parametrize("world,nprobe,k", [(2, 8, 10), (3, 16, 64), (5, 4, 127)])
def test_sharded_ivf_bf16(monkeypatch, world, nprobe, k):
    """Each rank's IVFIndex over its contiguous rows (same centroids, row_offset = its first global row) is pinned by
    ivf_from_scores; ShardedIVF equals merge_reference of those answers on every rank, and the unsharded IVFIndex
    wherever no exact tie reaches the (k+1)-th score."""
    n, d, nq, nlist = 6000, 128, 40, 32
    x, q = clustered(n, d, nq, seed=world)
    xd = torch.from_numpy(x).to(DEV)
    qb = torch.from_numpy(q).to(DEV).to(torch.bfloat16)
    offs = sc.edge_bounds(n, world, "ragged")
    whole, ranks = _ivf_shards(xd, offs, nlist, sc.BIG_BASE)
    per = [ivf_check(ix, qb, nprobe, k)[:3] for ix in ranks]
    want = sc.merge_reference(*(torch.stack([p[i] for p in per]) for i in range(3)), k)
    for r, o in enumerate(_sharded_ivf(ranks, monkeypatch, qb, nprobe, k)):
        sc.assert_merge(o, want, f"rank {r}")
    w_ids, w_sc, w_mm = ivf_check(whole, qb, nprobe, k + 1)[:3]
    sr.assert_bits(want[2], w_mm, "minmax vs unsharded")
    valid = w_ids >= 0
    strict = ((w_sc[:, :-1] > w_sc[:, 1:]) | ~valid[:, 1:]).all(dim=1)
    assert int(strict.sum()) >= nq // 2, "too few tie-free queries to compare with the unsharded index"
    sr.assert_bits(want[0][strict], w_ids[strict, :k], "ids vs unsharded")
    sr.assert_bits(want[1][strict], w_sc[strict, :k], "scores vs unsharded")


def _hand_ivf(assignment, dim, residual_of, centroids, row_offset):
    """An IVFIndex over a hand-made assignment of rows with global ids row_offset + i; residual_of(global ids)."""
    from comorag_b200.ivf import IVFIndex, TILE_ROWS, ivf_layout
    a = torch.as_tensor(assignment, dtype=torch.int64, device=DEV)
    order, dest, tile_start, list_rows = ivf_layout(a, centroids.shape[0])
    total = max(int(tile_start[-1]), 1) * TILE_ROWS
    res = torch.zeros((total, dim), dtype=torch.bfloat16, device=DEV)
    row_ids = torch.full((total,), -1, dtype=torch.int64, device=DEV)
    res[dest] = residual_of(order + row_offset)
    row_ids[dest] = order + row_offset
    return IVFIndex(centroids, res, row_ids, tile_start.contiguous(), list_rows.contiguous(), a.numel())


def test_sharded_ivf_cross_rank_tie_departs_from_ivf_index(monkeypatch):
    """Lists 0 and 2 have identical centroids and hold identical residual rows; global rows 0..63 are in list 2 on
    rank 0, rows 114..177 in list 0 on rank 1.  IVFIndex over all rows puts list 0's row (the larger id) first in each
    tie; ShardedIVF merges by (score, rank, position) and puts rank 0's row (list 2, the smaller id) first.  Both
    answers hold the same scores; the sharded one is merge_reference of the per-rank answers."""
    dim, m = 128, 64
    g = torch.Generator(device=DEV).manual_seed(21)
    twins = (torch.randint(-3, 4, (m, dim), generator=g, device=DEV).float() / 8).bfloat16()
    other = (torch.randint(-3, 4, (50, dim), generator=g, device=DEV).float() / 8).bfloat16()

    def residual_of(ids):
        r = torch.empty((ids.numel(), dim), dtype=torch.bfloat16, device=DEV)
        lo, mid, hi = ids < m, (ids >= m) & (ids < m + 50), ids >= m + 50
        r[lo], r[mid], r[hi] = twins[ids[lo]], other[ids[mid] - m], twins[ids[hi] - m - 50]
        return r
    e0 = torch.zeros(dim, device=DEV)
    e0[0] = 1.0
    cent = torch.stack([e0, -e0, e0]).bfloat16()                 # coarse: q0, -q0, q0; every query has q0 = 3/8
    whole = _hand_ivf([2] * m + [1] * 50 + [0] * m, dim, residual_of, cent, 0)
    ranks = [_hand_ivf([2] * m + [1] * 50, dim, residual_of, cent, 0), _hand_ivf([0] * m, dim, residual_of, cent, m + 50)]
    nq, nprobe, k = 34, 2, 2 * m
    qb = (torch.randint(-3, 4, (nq, dim), generator=g, device=DEV).float() / 8)
    qb[:, 0] = 0.375
    qb = qb.bfloat16()
    per = [ivf_check(ix, qb, nprobe, k)[:3] for ix in ranks]
    want = sc.merge_reference(*(torch.stack([p[i] for p in per]) for i in range(3)), k)
    outs = _sharded_ivf(ranks, monkeypatch, qb, nprobe, k)
    for r, o in enumerate(outs):
        sc.assert_merge(o, want, f"rank {r}")
    w_ids, w_sc, w_mm = ivf_check(whole, qb, nprobe, k)[:3]
    sr.assert_bits(want[1], w_sc, "scores vs unsharded")
    sr.assert_bits(want[2], w_mm, "minmax vs unsharded")
    ids, s, u_ids = want[0].cpu(), want[1].cpu(), w_ids.cpu()
    for q in range(nq):
        for v in s[q].unique():
            run, u_run = ids[q][s[q] == v], u_ids[q][s[q] == v]
            h = run.numel() // 2
            assert run.numel() == 2 * h and bool((run[:h] < m).all()) and torch.equal(run[h:], run[:h] + m + 50)
            assert torch.equal(u_run, torch.cat([run[h:], run[:h]]))         # IVFIndex: list 0 (rank 1's rows) first
    assert not torch.equal(ids, u_ids)


def test_sharded_quantized_ivf_rescores_the_union(monkeypatch, record_property):
    """ShardedIVF over QuantizedIVF: every rank keeps its own top n_cand by S1 and rescores them, so the result is
    merge_reference of the per-rank ivf_i8_oracle answers, and its S2 at every position is >= the unsharded
    QuantizedIVF's (the global top n_cand by S1 lies inside the union of the ranks')."""
    from comorag_b200.ivf import QuantizedIVF
    world, n, d, nq, nlist, nprobe, k = 3, 6000, 128, 12, 32, 8, 16
    x, q = clustered(n, d, nq, seed=9)
    xd = torch.from_numpy(x).to(DEV)
    qb = torch.from_numpy(q).to(DEV).to(torch.bfloat16)
    offs = sc.edge_bounds(n, world, "ragged")
    whole, ranks = _ivf_shards(xd, offs, nlist, sc.BIG_BASE)
    qranks = [QuantizedIVF.from_ivf(ix) for ix in ranks]
    n_cand = min(128, 4 * k)
    per = []
    for ix, qi in zip(ranks, qranks):
        ids, s, mm, probed = qi.search_device(qb, nprobe, k)
        o_ids, o_s, o_mm, _ = io.search_i8(ix.residuals.float().cpu().numpy(), ix.row_ids.cpu().numpy(),
                                           ix.list_tile_start.cpu().numpy(), ix.list_rows.cpu().numpy(),
                                           qb.float().cpu().numpy(), (probed[0].cpu().numpy(), probed[1].cpu().numpy()),
                                           k, n_cand)
        o = (torch.from_numpy(o_ids), torch.from_numpy(o_s), torch.from_numpy(o_mm.astype(np.float32)))
        sc.assert_merge((ids, s, mm), o, "rank vs ivf_i8_oracle")
        per.append(o)
    want = sc.merge_reference(*(torch.stack([p[i] for p in per]) for i in range(3)), k)
    for r, o in enumerate(_sharded_ivf(qranks, monkeypatch, qb, nprobe, k)):
        sc.assert_merge(o, want, f"rank {r}")
    u_ids, u_s, u_mm, _ = QuantizedIVF.from_ivf(whole).search_device(qb, nprobe, k)
    u_s = u_s.cpu()
    assert bool((want[1] >= u_s).all()), "a sharded S2 below the unsharded one"
    sr.assert_bits(want[2], u_mm, "S1 minmax vs unsharded")
    record_property("positions_above_unsharded", int((want[1] > u_s).sum()))
