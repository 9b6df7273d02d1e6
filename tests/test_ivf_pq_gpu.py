"""crag_ivf_search_pq / crag_pq_encode / PQIVF on the GPU, bit for bit against tests/ivf_pq_oracle.py.

The hand-made layout (dim 192, so m = 8, 96 and 192 all divide it) has lists of 0, 1, 127, 128 and 129 rows among
random ones.  Over m in {8, 96, 192} the cases cover k in {1, 10, 100, 128} with candidates in {k, 128}, nprobe in
{1, 32, nlist} and nq in {1, 31, 32, 33, 100}, each with the residuals on the device and in page-locked host memory,
which must agree.  Caller-supplied probes hold -1, out-of-range ids, duplicates and two lists with equal coarse terms
that share an identical row.  Lossless codebooks make PQIVF equal IVFIndex.search_device bit for bit, two streams and
repeated runs agree, ShardedIVF over PQIVF on 2 to 8 virtual ranks is the merge of the per-rank oracle answers, and
every argument error names its argument."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ivf_pq_oracle as po  # noqa: E402
import scan_reference as sr  # noqa: E402
import shard_cases as sc  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
DIM, NLIST = 192, 64
FIXED_ROWS = [0, 1, 127, 128, 129, 0]


@pytest.fixture(scope="module", autouse=True)
def _lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from comorag_b200 import _native
    _native.load()


def _hand_ivf(list_rows, dim, residuals_f32, centroids, row_offset=0):
    """IVFIndex over a given padded layout (lists back to back in whole tiles)."""
    from comorag_b200.ivf import IVFIndex
    tiles = [(r + 127) // 128 for r in list_rows]
    starts = np.concatenate([[0], np.cumsum(tiles)]).astype(np.int32)
    n = int(starts[-1]) * 128
    row_ids = np.full(n, -1, np.int64)
    nid = 0
    for l, r in enumerate(list_rows):
        row_ids[starts[l] * 128 + np.arange(r)] = row_offset + nid + np.arange(r)
        nid += r
    res = torch.from_numpy(residuals_f32).to(DEV).to(torch.bfloat16).contiguous()
    return IVFIndex(torch.from_numpy(centroids).to(DEV).to(torch.bfloat16), res, torch.from_numpy(row_ids).to(DEV),
                    torch.from_numpy(starts).to(DEV), torch.from_numpy(np.array(list_rows, np.int32)).to(DEV), nid)


def _random_index(seed=0):
    rng = np.random.default_rng(seed)
    rows = FIXED_ROWS + list(rng.integers(0, 300, NLIST - len(FIXED_ROWS)))
    n = sum((r + 127) // 128 for r in rows) * 128
    res = np.zeros((n, DIM), np.float32)
    tiles = np.concatenate([[0], np.cumsum([(r + 127) // 128 for r in rows])])
    for l, r in enumerate(rows):
        res[tiles[l] * 128 + np.arange(r)] = rng.standard_normal((r, DIM)).astype(np.float32) * 0.05
    c = rng.standard_normal((NLIST, DIM)).astype(np.float32)
    c /= np.linalg.norm(c, axis=1, keepdims=True)
    return _hand_ivf(rows, DIM, res, c)


@pytest.fixture(scope="module")
def base():
    return _random_index()


@pytest.fixture(scope="module")
def pq_pairs(base):
    """m -> (PQIVF with device residuals, the same codes with host residuals)."""
    from comorag_b200.pq import PQIVF
    out = {}
    for m in (8, 96, 192):
        dev = PQIVF.from_ivf(base, m, iters=3, seed=m)
        host = PQIVF.from_ivf(base, m, codebooks=dev.codebooks, residuals="host")
        assert torch.equal(dev.codes, host.codes)
        out[m] = (dev, host)
    return out


def _np(t):
    return t.cpu().numpy()


def _oracle(pq, qb, probed, k, n_cand):
    return po.search_pq(_np(pq._rows.float()), _np(pq.codes), _np(pq.codebooks), _np(pq.row_ids),
                        _np(pq.list_tile_start), _np(pq.list_rows), _np(qb.float()),
                        (_np(probed[0]), _np(probed[1])), k, n_cand)


def _assert_oracle(got, want, what):
    ids, s, mm = (_np(t) for t in got[:3])
    assert np.array_equal(ids, want[0]), f"{what}: ids {np.argwhere(ids != want[0])[:5]}"
    assert np.array_equal(s.view(np.uint32), want[1].view(np.uint32)), f"{what}: scores"
    assert np.array_equal(mm.view(np.uint32), want[2].view(np.uint32)), f"{what}: minmax"


def test_codes_match_oracle(base, pq_pairs):
    res = _np(base.residuals.float())
    real = _np(base.row_ids) >= 0
    for m, (pq, _) in pq_pairs.items():
        codes = _np(pq.codes)
        want = po.encode(res[real], _np(pq.codebooks))
        assert np.array_equal(codes[real, :m], want), f"m={m}"
        assert not codes[~real].any() and not codes[:, m:].any()


def _grid():
    cases, i = [], 0
    for m in (8, 96, 192):
        for k in (1, 10, 100, 128):
            for cand in sorted({k, 128}):
                cases.append((m, k, cand, (1, 32, NLIST)[i % 3], (1, 31, 32, 33, 100)[i % 5]))
                i += 1
    return cases


@pytest.mark.parametrize("m,k,cand,nprobe,nq", _grid())
def test_search_matches_oracle_on_device_and_host_residuals(base, pq_pairs, m, k, cand, nprobe, nq):
    g = torch.Generator(device="cpu").manual_seed(m * 1000 + k * 10 + nq)
    qb = torch.nn.functional.normalize(torch.randn(nq, DIM, generator=g), dim=1).to(DEV).to(torch.bfloat16)
    dev, host = pq_pairs[m]
    got = dev.search_device(qb, nprobe, k, candidates=cand)
    assert dev.residuals_on_device and not host.residuals_on_device
    got_h = host.search_device(qb, nprobe, k, candidates=cand, probed=got[3])
    for a, b in zip(got[:3], got_h[:3]):
        assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                           b.view(torch.int32) if b.dtype == torch.float32 else b), "host vs device residuals"
    _assert_oracle(got, _oracle(dev, qb, got[3], k, cand), f"m={m} k={k} cand={cand} nprobe={nprobe} nq={nq}")


def test_caller_probes_with_absent_out_of_range_duplicate_and_tied_lists(base, pq_pairs):
    """Lists 3 and 4 (128 and 129 rows) get the same coarse term and share a row: the tie goes to list 3's copy."""
    from comorag_b200.pq import PQIVF
    ivf = _random_index(seed=1)
    res = ivf.residuals.clone()
    a = int(ivf.list_tile_start[3]) * 128 + 7
    b = int(ivf.list_tile_start[4]) * 128 + 128
    res[b] = res[a]
    ivf.residuals = res
    pq = PQIVF.from_ivf(ivf, 96, codebooks=pq_pairs[96][0].codebooks)
    nq = 33
    g = torch.Generator(device="cpu").manual_seed(5)
    qb = torch.randn(nq, DIM, generator=g)
    qb[:, :] = qb + 40 * res[a].float().cpu()                   # every query wants the shared row
    qb = torch.nn.functional.normalize(qb, dim=1).to(DEV).to(torch.bfloat16)
    ids = torch.tensor([[3, -1, 4, NLIST + 5, 3, 0, 5, 1]] * nq, dtype=torch.int64)
    sc_ = torch.full((nq, 8), 0.25)
    sc_[:, 6:] = torch.randn(nq, 2, generator=g)
    probed = (ids.to(DEV), sc_.to(DEV))
    for k, cand in ((10, 128), (128, 128), (1, 1)):
        got = pq.search_device(qb, 8, k, candidates=cand, probed=probed)
        want = _oracle(pq, qb, probed, k, cand)
        _assert_oracle(got, want, f"k={k}")
        if k > 1:
            row_a, row_b = int(ivf.row_ids[a]), int(ivf.row_ids[b])
            got_ids = _np(got[0])
            for q in range(nq):
                lst = list(got_ids[q])
                if row_a in lst and row_b in lst:
                    assert lst.index(row_a) < lst.index(row_b)


def _lossless_ivf(m, seed=0):
    """IVFIndex whose residual sub-vectors take at most 200 values per subspace, all exact in bf16, plus codebooks
    holding them: PQ is lossless and every product and sum below is exact in fp32."""
    rng = np.random.default_rng(seed)
    dsub = DIM // m
    rows = FIXED_ROWS + list(rng.integers(0, 200, 10))
    n = sum((r + 127) // 128 for r in rows) * 128
    cb = np.empty((m, 256, dsub), np.float32)
    for j in range(m):
        v = rng.integers(-8, 9, (200, dsub)).astype(np.float32) / 8
        cb[j, :200], cb[j, 200:] = v, v[-1]
    res = np.zeros((n, DIM), np.float32)
    tiles = np.concatenate([[0], np.cumsum([(r + 127) // 128 for r in rows])])
    for l, r in enumerate(rows):
        p = tiles[l] * 128 + np.arange(r)
        for j in range(m):
            res[p, j * dsub:(j + 1) * dsub] = cb[j, rng.integers(0, 200, r)]
    c = rng.integers(-4, 5, (len(rows), DIM)).astype(np.float32) / 16
    return _hand_ivf(rows, DIM, res, c), torch.from_numpy(cb)


@pytest.mark.parametrize("m", [8, 96, 192])
def test_lossless_codebooks_equal_ivf_index(m):
    from comorag_b200.pq import PQIVF
    ivf, cb = _lossless_ivf(m, seed=m)
    pq = PQIVF.from_ivf(ivf, m, codebooks=cb)
    g = torch.Generator(device="cpu").manual_seed(m)
    qb = (torch.randint(-16, 17, (40, DIM), generator=g).float() / 16).to(DEV).to(torch.bfloat16)
    for nprobe, k in ((ivf.nlist, 10), (3, 128), (1, 1)):
        want = ivf.search_device(qb, nprobe, k)
        for cand in sorted({k, 128}):
            got = pq.search_device(qb, nprobe, k, candidates=cand)
            sr.assert_bits(got[0], want[0], f"ids m={m} nprobe={nprobe} k={k} cand={cand}")
            sr.assert_bits(got[1], want[1], "scores")
            sr.assert_bits(got[2], want[2], "minmax")


def test_two_streams_and_repeats_agree(pq_pairs):
    pq = pq_pairs[96][1]
    g = torch.Generator(device="cpu").manual_seed(7)
    qb = torch.nn.functional.normalize(torch.randn(70, DIM, generator=g), dim=1).to(DEV).to(torch.bfloat16)
    s1, s2 = torch.cuda.Stream(DEV), torch.cuda.Stream(DEV)
    torch.cuda.synchronize()
    a = pq.search_device(qb, 16, 100, stream=s1)
    b = pq.search_device(qb, 16, 100, stream=s2)
    c = pq.search_device(qb, 16, 100)
    torch.cuda.synchronize()
    for x, y in ((a, b), (a, c)):
        for u, v in zip(x[:3], y[:3]):
            sr.assert_bits(u, v, "streams / repeats")


@pytest.mark.parametrize("world", [2, 5, 8])
def test_sharded_pq_ivf_merges_the_rank_answers(monkeypatch, pq_pairs, world):
    """Each rank's PQIVF (same centroids and codebooks, its own rows) keeps its own top candidates by S1 and rescores
    them: ShardedIVF is merge_reference of the per-rank oracle answers, and its S2 at every position is >= the
    unsharded PQIVF's (the global top candidates by S1 lie inside the union of the ranks')."""
    import torch.distributed as dist
    from comorag_b200.ivf import IVFIndex
    from comorag_b200.pq import PQIVF
    from test_oracle_ivf_i8 import clustered
    n, nq, nlist, nprobe, k = 6000, 12, 32, 8, 16
    x, q = clustered(n, DIM, nq, seed=world)
    xd = torch.from_numpy(x).to(DEV)
    qb = torch.from_numpy(q).to(DEV).to(torch.bfloat16)
    offs = sc.edge_bounds(n, world, "ragged")
    whole = IVFIndex.build(xd, nlist, iters=4, seed=0, row_offset=sc.BIG_BASE)
    c = whole.centroids.matrix().contiguous()
    ranks = [IVFIndex.build(xd[offs[r]:offs[r + 1]], nlist, centroids=c, row_offset=sc.BIG_BASE + offs[r])
             for r in range(world)]
    cb = PQIVF.from_ivf(whole, 48, iters=3).codebooks
    pranks = [PQIVF.from_ivf(ix, 48, codebooks=cb) for ix in ranks]
    per = []
    for pq in pranks:
        got = pq.search_device(qb, nprobe, k)
        want = _oracle(pq, qb, got[3], k, min(128, 4 * k))
        _assert_oracle(got, want, "rank vs oracle")
        per.append(tuple(torch.from_numpy(np.ascontiguousarray(w)) for w in want[:3]))
    want = sc.merge_reference(*(torch.stack([p[i] for p in per]) for i in range(3)), k)
    monkeypatch.setattr(dist, "all_gather_into_tensor", sc.virtual_all_gather)
    group = sc.VirtualGroup(world)
    outs = sc.run_ranks(world, lambda r: sc.virtual_sharded_ivf(pranks[r], group.rank(r)).search_device(qb, nprobe, k), DEV)
    for r, o in enumerate(outs):
        sc.assert_merge(o, want, f"rank {r}")
    u = PQIVF.from_ivf(whole, 48, codebooks=cb).search_device(qb, nprobe, k)
    assert bool((want[1] >= u[1].cpu()).all()), "a sharded S2 below the unsharded one"
    sr.assert_bits(want[2], u[2], "S1 minmax vs unsharded")


def _raw(pq, qb, over=None):
    """crag_ivf_search_pq at k = 4, n_cand = 8 with the arguments in `over` replaced (nothing launches when one is
    bad, so the outputs are sized for k = 128)."""
    k, n_cand = 4, 8
    from comorag_b200 import _native
    lib = _native.load()
    nq = qb.shape[0]
    pid = torch.zeros((nq, 1), dtype=torch.int64, device=DEV)
    psc = torch.zeros((nq, 1), dtype=torch.float32, device=DEV)
    ids = torch.empty((nq, 128), dtype=torch.int64, device=DEV)
    sc_ = torch.empty((nq, 128), dtype=torch.float32, device=DEV)
    mm = torch.empty((nq, 2), dtype=torch.float32, device=DEV)
    wsb = lib.crag_ivf_pq_workspace_bytes(pq.nlist, pq.total_tiles, n_cand, pq.m)
    ws = torch.empty(wsb + 256, dtype=torch.uint8, device=DEV)
    a = dict(codes=pq.codes.data_ptr(), m=pq.m, code_stride=pq.codes.stride(0), codebooks=pq.codebooks.data_ptr(),
             rows=pq._rows.data_ptr(), dim=pq.dim, row_stride=pq._rows.stride(0), n_rows=pq._rows.shape[0],
             starts=pq.list_tile_start.data_ptr(), lrows=pq.list_rows.data_ptr(), nlist=pq.nlist,
             total_tiles=pq.total_tiles, row_ids=pq.row_ids.data_ptr(), queries=qb.data_ptr(), nq=nq,
             pid=pid.data_ptr(), psc=psc.data_ptr(), nprobe=1, n_cand=n_cand, k=k, ids=ids.data_ptr(),
             scores=sc_.data_ptr(), minmax=mm.data_ptr(), ws=ws.data_ptr(), wsb=wsb, stream=None)
    a.update(over or {})
    rc = lib.crag_ivf_search_pq(*a.values())
    return rc, lib.crag_last_error().decode()


def test_argument_errors_name_the_argument(pq_pairs):
    from comorag_b200 import _native
    from comorag_b200.pq import PQIVF
    lib = _native.load()
    pq = pq_pairs[8][0]
    qb = torch.zeros((2, DIM), dtype=torch.bfloat16, device=DEV)
    pageable = torch.empty(16)
    assert _raw(pq, qb)[0] == 0
    for over, word in [(dict(k=0), "k"), (dict(k=9), "n_cand"), (dict(n_cand=129, k=4), "n_cand"), (dict(nq=0), "nq"),
                       (dict(m=7), "m"), (dict(m=193), "m"), (dict(code_stride=8), "code_stride"),
                       (dict(codes=None), "codes"), (dict(codebooks=None), "codebooks"),
                       (dict(codes=pq.codes.data_ptr() + 4), "aligned"), (dict(dim=100), "dim"),
                       (dict(row_stride=8), "stride"), (dict(nprobe=0), "nprobe"), (dict(nlist=0), "nlist"),
                       (dict(n_rows=100), "n_rows_padded"), (dict(queries=None), "queries_bf16"),
                       (dict(ws=None), "workspace"), (dict(wsb=16), "workspace"), (dict(ids=None), "null"),
                       (dict(rows=pageable.data_ptr()), "pageable")]:
        rc, msg = _raw(pq, qb, over)
        assert rc != 0 and word in msg, (over, rc, msg)
    assert lib.crag_ivf_pq_workspace_bytes(pq.nlist, pq.total_tiles, 129, 8) == 0
    assert lib.crag_ivf_pq_workspace_bytes(pq.nlist, pq.total_tiles, 8, 193) == 0
    rows = pq._rows[:10]
    codes = torch.zeros((10, 16), dtype=torch.uint8, device=DEV)
    enc = lambda **o: lib.crag_pq_encode(*dict(dict(rows=rows.data_ptr(), n=10, dim=DIM, stride=DIM,
                                                    cb=pq.codebooks.data_ptr(), m=8, codes=codes.data_ptr(), cs=16,
                                                    st=None), **o).values())
    assert enc() == 0
    for over, word in [(dict(m=5), "m"), (dict(dim=96), "dim"), (dict(n=-1), "n_rows"), (dict(stride=8), "row_stride"),
                       (dict(cs=4), "code_stride"), (dict(codes=None), "codes"), (dict(cb=None), "codebooks")]:
        assert enc(**over) != 0 and word in lib.crag_last_error().decode(), over
    with pytest.raises(ValueError, match="m must divide"):
        PQIVF.from_ivf(_random_index(), 7)
    with pytest.raises(ValueError, match="candidates"):
        pq.search_device(qb, 1, 10, candidates=8)
    with pytest.raises(ValueError, match="residuals"):
        PQIVF.from_ivf(_random_index(), 8, residuals="disk")
