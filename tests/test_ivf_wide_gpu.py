"""crag_ivf_search_i8_wide / crag_ivf_search_pq_wide and QuantizedIVF / PQIVF.search_device_wide on the GPU, bit for
bit against the narrow entries and tests/ivf_i8_oracle.py / tests/ivf_pq_oracle.py (DESIGN.md section 7).

The hand-made layout of tests/test_ivf_pq_gpu.py (lists of 0, 1, 127, 128, 129 rows among random ones) gets duplicate
residual rows inside and across lists, and caller probes give two lists equal coarse terms, so S1 and S2 tie across
the candidate cut-off.  Cases: the wide C entries forced to n_cand <= 128 equal the narrow entries in ids, scores,
minmax and candidates for nq in {1, 31, 32, 33, 100}; n_cand in {129, 512, 2048} equal the oracles, candidates
included; a max_probe_rows below most queries' probed rows keeps their first slots, and a query without probed rows
gives -1 / -inf and minmax (+inf, -inf); S2 never drops at any rank as candidates grow from 128 to 2048; host and
device residuals agree; two streams and a repeated call agree; argument errors are refused before any launch."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ivf_i8_oracle as io  # noqa: E402
import ivf_pq_oracle as po  # noqa: E402
import ivf_wide_oracle as wo  # noqa: E402
import scan_reference as sr  # noqa: E402
from oracle import quant_oracle as qo  # noqa: E402
from test_ivf_pq_gpu import DIM, NLIST, _hand_ivf  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
FIXED_ROWS = [0, 1, 127, 128, 129, 0, 700, 1500]
NQ, ALIGN = 32, 256


@pytest.fixture(scope="module", autouse=True)
def _lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from comorag_b200 import _native
    _native.load()


def _np(t):
    return t.cpu().numpy()


@pytest.fixture(scope="module")
def base():
    rng = np.random.default_rng(3)
    rows = FIXED_ROWS + list(rng.integers(0, 400, NLIST - len(FIXED_ROWS)))
    tiles = np.concatenate([[0], np.cumsum([(r + 127) // 128 for r in rows])])
    res = np.zeros((int(tiles[-1]) * 128, DIM), np.float32)
    for l, r in enumerate(rows):
        res[tiles[l] * 128 + np.arange(r)] = rng.standard_normal((r, DIM)).astype(np.float32) * 0.05
    src = tiles[6] * 128 + 5
    for dst in (tiles[6] * 128 + 600, tiles[7] * 128 + 9, tiles[3] * 128 + 127, tiles[4] * 128 + 128):
        res[dst] = res[src]                                   # duplicates inside list 6 and in lists 7, 3 and 4
    c = rng.standard_normal((NLIST, DIM)).astype(np.float32)
    c /= np.linalg.norm(c, axis=1, keepdims=True)
    return _hand_ivf(rows, DIM, res, c)


@pytest.fixture(scope="module")
def snaps(base):
    """name -> (device-residual snapshot, host-residual snapshot)."""
    from comorag_b200.ivf import QuantizedIVF
    from comorag_b200.pq import PQIVF
    out = {"i8": (QuantizedIVF.from_ivf(base), QuantizedIVF.from_ivf(base, "host"))}
    for m in (8, 96):
        d = PQIVF.from_ivf(base, m, iters=3, seed=m)
        out[f"pq{m}"] = (d, PQIVF.from_ivf(base, m, codebooks=d.codebooks, residuals="host"))
    return out


def _queries(nq, seed, base=None):
    g = torch.Generator(device="cpu").manual_seed(seed)
    q = torch.randn(nq, DIM, generator=g)
    if base is not None:                                      # pull the queries towards the duplicated row
        q = q + 30 * base._rows[int(base.list_tile_start[6]) * 128 + 5].float().cpu()
    return torch.nn.functional.normalize(q, dim=1).to(DEV).to(torch.bfloat16)


def _tied_probes(nq, nprobe, seed):
    """Probes of lists 3, 4, 6 and 7 with one shared coarse term, plus -1, out-of-range and repeated probes."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    ids = torch.stack([torch.randperm(NLIST, generator=g)[:nprobe] for _ in range(nq)])
    ids[:, :4] = torch.tensor([6, 3, 7, 4])
    ids[:, 4], ids[:, 5], ids[:, 6] = -1, NLIST + 2, 6
    sc = torch.randn(nq, nprobe, generator=g) * 0.1
    sc[torch.isin(ids, torch.tensor([3, 4, 6, 7]))] = 0.125   # a list probed twice has one coarse term
    return ids.to(DEV), sc.float().to(DEV)


def _raw(snap, qb, probed, nprobe, n_cand, k, max_probe_rows, wide=True, over=None):
    """One call of the C entry on a fresh workspace: (rc, ids, scores, minmax, candidate positions, candidate S1) with
    the candidates of the last 32-query pass read from the workspace."""
    from comorag_b200 import _native
    from comorag_b200.quantized import quantize_rows
    lib = _native.load()
    pq = hasattr(snap, "codes")
    nq = qb.shape[0]
    ids = torch.empty((nq, k), dtype=torch.int64, device=DEV)
    sc = torch.empty((nq, k), dtype=torch.float32, device=DEV)
    mm = torch.empty((nq, 2), dtype=torch.float32, device=DEV)
    if wide:
        wsb = (lib.crag_ivf_pq_wide_workspace_bytes(snap.nlist, snap.total_tiles, n_cand, max_probe_rows, snap.m) if pq
               else lib.crag_ivf_i8_wide_workspace_bytes(snap.nlist, snap.total_tiles, n_cand, max_probe_rows))
    else:
        wsb = (lib.crag_ivf_pq_workspace_bytes(snap.nlist, snap.total_tiles, n_cand, snap.m) if pq
               else lib.crag_ivf_i8_workspace_bytes(snap.nlist, snap.total_tiles, n_cand))
    ws = torch.zeros(wsb, dtype=torch.uint8, device=DEV)
    common = dict(rows=snap._rows.data_ptr(), dim=snap.dim, row_stride=snap._rows.stride(0), n_rows=snap._rows.shape[0],
                  starts=snap.list_tile_start.data_ptr(), lrows=snap.list_rows.data_ptr(), nlist=snap.nlist,
                  total_tiles=snap.total_tiles, row_ids=snap.row_ids.data_ptr())
    if pq:
        a = dict(codes=snap.codes.data_ptr(), m=snap.m, code_stride=snap.codes.stride(0),
                 codebooks=snap.codebooks.data_ptr(), **common, queries=qb.data_ptr(), nq=nq)
    else:
        q8, qs = quantize_rows(qb, snap.dim8)
        a = dict(codes=snap._i8.data_ptr(), scales=snap._scales.data_ptr(), dim8=snap.dim8, stride8=snap._i8.stride(0),
                 **common, q8=q8.data_ptr(), qs=qs.data_ptr(), queries=qb.data_ptr(), nq=nq)
    a.update(pid=probed[0].data_ptr(), psc=probed[1].data_ptr(), nprobe=nprobe, n_cand=n_cand, k=k)
    if wide:
        a["max_probe_rows"] = max_probe_rows
    a.update(ids=ids.data_ptr(), scores=sc.data_ptr(), minmax=mm.data_ptr(), ws=ws.data_ptr(), wsb=wsb, stream=None)
    a.update(over or {})
    fn = ("crag_ivf_search_pq" if pq else "crag_ivf_search_i8") + ("_wide" if wide else "")
    rc = getattr(lib, fn)(*a.values())
    torch.cuda.synchronize()
    if rc != 0:
        return (rc,)
    # the candidate buffers sit at the end of the layout (before the PQ tables): [32][n_cand] int64, then fp32
    lut = ((NQ * snap.m * 256 * 4 + ALIGN - 1) // ALIGN * ALIGN) if pq else 0
    c_sc_bytes = (NQ * n_cand * 4 + ALIGN - 1) // ALIGN * ALIGN
    c_id_bytes = (NQ * n_cand * 8 + ALIGN - 1) // ALIGN * ALIGN
    end = wsb - lut
    c_ids = ws[end - c_sc_bytes - c_id_bytes:end - c_sc_bytes - c_id_bytes + NQ * n_cand * 8].view(torch.int64)
    c_s1 = ws[end - c_sc_bytes:end - c_sc_bytes + NQ * n_cand * 4].view(torch.float32)
    last = (nq - 1) // NQ * NQ
    n_last = nq - last
    return rc, ids, sc, mm, c_ids.reshape(NQ, n_cand)[:n_last], c_s1.reshape(NQ, n_cand)[:n_last], last


def _oracle(snap, qb, probed, k, n_cand):
    res = _np(snap._rows.float())
    args = (_np(snap.row_ids), _np(snap.list_tile_start), _np(snap.list_rows), _np(qb.float()),
            (_np(probed[0]), _np(probed[1])), k, n_cand)
    if hasattr(snap, "codes"):
        return po.search_pq(res, _np(snap.codes), _np(snap.codebooks), *args)
    return io.search_i8(res, *args)


@pytest.mark.parametrize("name", ["i8", "pq8", "pq96"])
@pytest.mark.parametrize("nq", [1, 31, 32, 33, 100])
def test_wide_entry_at_128_or_fewer_equals_the_narrow_entry(snaps, name, nq):
    snap = snaps[name][0]
    nprobe = 8
    qb = _queries(nq, nq, snap)
    probed = _tied_probes(nq, nprobe, nq)
    bound = snap.probe_rows_bound(nprobe)
    for n_cand, k in ((128, 100), (40, 40), (1, 1)):
        a = _raw(snap, qb, probed, nprobe, n_cand, k, bound, wide=False)
        b = _raw(snap, qb, probed, nprobe, n_cand, k, bound, wide=True)
        assert a[0] == 0 and b[0] == 0
        for x, y, what in zip(a[1:6], b[1:6], ("ids", "scores", "minmax", "candidates", "candidate S1")):
            sr.assert_bits(x, y, f"{name} nq={nq} n_cand={n_cand} {what}")


@pytest.mark.parametrize("name", ["i8", "pq8", "pq96"])
@pytest.mark.parametrize("n_cand", [129, 512, 2048])
def test_wide_entry_matches_the_oracle(snaps, name, n_cand):
    snap = snaps[name][0]
    nq, nprobe, k = 33, 12, min(n_cand, 300)
    qb = _queries(nq, n_cand, snap)
    probed = _tied_probes(nq, nprobe, n_cand)
    rc, ids, sc, mm, c_ids, c_s1, last = _raw(snap, qb, probed, nprobe, n_cand, k, snap.probe_rows_bound(nprobe))
    assert rc == 0
    want = _oracle(snap, qb, probed, k, n_cand)
    assert np.array_equal(_np(ids), want[0]), np.argwhere(_np(ids) != want[0])[:5]
    assert np.array_equal(_np(sc).view(np.uint32), want[1].view(np.uint32))
    assert np.array_equal(_np(mm).view(np.uint32), want[2].view(np.uint32))
    assert np.array_equal(_np(c_ids), want[3][0][last:])
    assert np.array_equal(_np(c_s1).view(np.uint32), want[3][1][last:].view(np.uint32))


@pytest.mark.parametrize("name", ["i8", "pq96"])
def test_s2_never_drops_as_candidates_grow_and_host_equals_device(snaps, name):
    dev, host = snaps[name]
    nq, nprobe, k = 40, 16, 128
    qb = _queries(nq, 9)
    prev = None
    for cand in (128, 256, 512, 1024, 2048):
        got = dev.search_device_wide(qb, nprobe, k, cand)
        got_h = host.search_device_wide(qb, nprobe, k, cand, probed=got[3])
        for a, b in zip(got[:3], got_h[:3]):
            sr.assert_bits(a, b, f"host vs device residuals, candidates {cand}")
        if prev is not None:
            assert bool((got[1] >= prev).all()), f"an S2 dropped going to {cand} candidates"
        prev = got[1]
    ids, _ = dev.search_wide(_np(qb.float()), nprobe, 10, 600)
    sr.assert_bits(torch.from_numpy(ids), dev.search_device_wide(qb, nprobe, 10, 600)[0].cpu(), "search_wide")


@pytest.mark.parametrize("name", ["i8", "pq96"])
def test_undersized_max_probe_rows_and_a_query_without_rows(snaps, name):
    """max_probe_rows below most queries' probed rows keeps each query's first slots (ivf_wide_oracle.slot_positions);
    the last query probes only -1, out-of-range and empty lists, so n_q = 0: -1 / -inf and minmax (+inf, -inf)."""
    snap = snaps[name][0]
    nq, nprobe, n_cand, k, cap = 33, 12, 300, 50, 1000
    qb = _queries(nq, 5, snap)
    p_ids, p_sc = _tied_probes(nq, nprobe, 5)
    p_ids[nq - 1] = torch.tensor([0, 5, -1, NLIST + 1] + [0] * (nprobe - 4), device=DEV)   # lists 0 and 5 are empty
    probed = (p_ids, p_sc)
    rc, ids, sc, mm, c_ids, c_s1, last = _raw(snap, qb, probed, nprobe, n_cand, k, cap)
    assert rc == 0
    ids_np, starts, lrows = _np(p_ids), _np(snap.list_tile_start), _np(snap.list_rows)
    res, qf = _np(snap._rows.float()), _np(qb.float())
    per_q = io._probed_of((ids_np, _np(p_sc)), nq, snap.nlist)
    if hasattr(snap, "codes"):
        lut, codes = po.table(qf, _np(snap.codebooks)), _np(snap.codes)[:, :snap.m]
        s1_of = lambda i, p: po.pq_sums(lut[i], codes[p])
    else:
        r8, rs = qo.quantize(res, snap.dim8)
        q8, qs = qo.quantize(qf, snap.dim8)
        s1_of = lambda i, p: qo.s1_scores(r8[p], rs[p], q8[i:i + 1], qs[i:i + 1])[0]
    cand = np.full((nq, n_cand), -1, np.int64)
    clamped = 0
    for i in range(nq):
        p = wo.slot_positions(ids_np[i], starts, lrows, snap.nlist, cap)
        clamped += p.size == cap
        lists = io.list_of_positions(starts, p)
        s1 = (s1_of(i, p) + np.array([per_q[i][int(l)] for l in lists], np.float32)).astype(np.float32) if p.size \
            else np.zeros(0, np.float32)
        _, pos, s, want_mm = wo.stage1(s1, p, n_cand)
        cand[i] = pos
        assert np.array_equal(_np(mm)[i].view(np.uint32), want_mm.view(np.uint32)), f"query {i}: minmax"
        if i >= last:
            assert np.array_equal(_np(c_ids)[i - last], pos), f"query {i}: candidates"
            assert np.array_equal(_np(c_s1)[i - last].view(np.uint32), s.view(np.uint32)), f"query {i}: candidate S1"
    assert clamped > nq // 2, "the cap should cut most queries' probed rows"
    want_pos, want_s2 = io.rescore(res, starts, lambda j, l: per_q[j][int(l)], qf, cand, k)
    want_ids = np.where(want_pos >= 0, _np(snap.row_ids)[np.maximum(want_pos, 0)], -1)
    assert np.array_equal(_np(ids), want_ids)
    assert np.array_equal(_np(sc).view(np.uint32), want_s2.view(np.uint32))
    assert (_np(ids)[nq - 1] == -1).all() and np.isneginf(_np(sc)[nq - 1]).all()
    assert _np(mm)[nq - 1][0] == np.inf and _np(mm)[nq - 1][1] == -np.inf


def test_two_streams_and_repeats_agree(snaps):
    pq = snaps["pq96"][1]
    qb = _queries(70, 7)
    s1, s2 = torch.cuda.Stream(DEV), torch.cuda.Stream(DEV)
    torch.cuda.synchronize()
    a = pq.search_device_wide(qb, 16, 100, 1000, stream=s1)
    b = pq.search_device_wide(qb, 16, 100, 1000, stream=s2)
    c = pq.search_device_wide(qb, 16, 100, 1000)
    torch.cuda.synchronize()
    for x, y in ((a, b), (a, c)):
        for u, v in zip(x[:3], y[:3]):
            sr.assert_bits(u, v, "streams / repeats")


@pytest.mark.parametrize("name", ["i8", "pq8"])
def test_argument_errors(snaps, name):
    from comorag_b200 import _native
    lib = _native.load()
    snap = snaps[name][0]
    qb = _queries(2, 1)
    probed = _tied_probes(2, 8, 1)
    bound = snap.probe_rows_bound(8)
    assert _raw(snap, qb, probed, 8, 200, 10, bound)[0] == 0
    for over, word in [(dict(k=0), "k"), (dict(k=201), "n_cand"), (dict(n_cand=2049, k=4), "n_cand"),
                       (dict(max_probe_rows=0), "max_probe_rows"), (dict(max_probe_rows=-5), "max_probe_rows"),
                       (dict(nq=0), "nq"), (dict(ws=None), "workspace"), (dict(wsb=1024), "workspace"), (dict(ids=None), "null")]:
        rc = _raw(snap, qb, probed, 8, 200, 10, bound, over=over)[0]
        assert rc != 0 and word in lib.crag_last_error().decode(), (over, rc, lib.crag_last_error().decode())
    for k, cand in ((0, 10), (11, 10), (10, 2049)):
        with pytest.raises(ValueError, match="candidates"):
            snap.search_device_wide(qb, 8, k, cand)
