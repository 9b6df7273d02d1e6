"""Up to 2048 rescored candidates for int8 and one-bit shards on the GPU, bit for bit against oracle/quant_oracle.py and
tests/binary_oracle.py: the S1 block of the score-all passes over the codes, crag_knn_topk_i8 / _b1 against the top-k
scans at k <= 128 and against the oracle's top k by (S1 desc, row asc) up to 2048 with ties across the cut-off, the
final answers of search_device_wide with rows on the device and in page-locked host memory, its equality with
search_device at <= 128 candidates and across the two codes when every row is a candidate, the monotone S2 per rank,
two streams and a repeated call, and argument errors with nothing launched."""
import numpy as np
import pytest
import torch

import binary_oracle as bo
from comorag_b200 import _native
from comorag_b200.binary import BinaryIndex, binarize_rows
from comorag_b200.index import DenseIndex
from comorag_b200.quantized import QuantizedIndex, quantize_rows
from oracle import quant_oracle as qo

pytestmark = pytest.mark.gpu
DEV = "cuda"
ALIGN, NQ = 256, 32
INVALID, WORKSPACE = -1, -3
CODES = ["i8", "b1"]


def _bf16(x):
    """numpy float32 -> (device bf16 tensor, its values as numpy float32)."""
    t = torch.from_numpy(np.ascontiguousarray(x, np.float32)).bfloat16()
    return t.to(DEV), t.float().numpy()


def _assert_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape
    bad = a.view(np.uint32) != b.view(np.uint32) if a.dtype == np.float32 else a != b
    assert not bad.any(), f"{bad.sum()} of {bad.size} differ, first at {np.argwhere(bad)[:4].tolist()}"


def _corpus(n, dim, rng, distinct=None):
    """Unit rows; with `distinct`, only that many different rows (ties at every cut-off), plus duplicates and zeros."""
    x = rng.standard_normal((n if distinct is None else distinct, dim), dtype=np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    if distinct is not None:
        x = x[rng.integers(0, distinct, n)]
    if n >= 40:
        x[10:14] = x[3]
        x[31:33] = 0.0
    return x


def _queries(nq, dim, rng, corpus=None):
    q = rng.standard_normal((nq, dim), dtype=np.float32)
    if nq > 2:
        q[nq - 1] = 0.0                                   # every S1 ties at 0
    if corpus is not None and nq > 3 and corpus.shape[0] > 3:
        q[1] = corpus[3]
    return q


def _encode(code, xd, n, dim8):
    """(codes, scales, row_stride) of device bf16 rows."""
    if code == "i8":
        if n == 0:
            return torch.zeros((0, dim8), dtype=torch.int8, device=DEV), torch.zeros(0, device=DEV), dim8
        c, s = quantize_rows(xd, dim8)
        return c, s, dim8
    if n == 0:
        return torch.zeros((0, dim8 // 8), dtype=torch.uint8, device=DEV), torch.zeros(0, device=DEV), dim8 // 8
    c, s = binarize_rows(xd)
    return c, s, dim8 // 8


def _oracle_s1(code, codes, scales, q8, qs):
    c, s, q, x = codes.cpu().numpy(), scales.cpu().numpy(), q8.cpu().numpy(), qs.cpu().numpy()
    return qo.s1_scores(c, s, q, x) if code == "i8" else bo.s1_scores(c, s, q, x)


def _oracle_topk(code, codes, scales, q8, qs, k, row_offset=0):
    c, s, q, x = codes.cpu().numpy(), scales.cpu().numpy(), q8.cpu().numpy(), qs.cpu().numpy()
    return qo.search_i8(c, s, q, x, k, row_offset) if code == "i8" else bo.search_b1(c, s, q, x, k, row_offset)


def _knn(code, codes, scales, n, dim8, stride, q8, qs, k, row_offset=0, ws_queries=None, stream=None, ws=None):
    """crag_knn_topk_<code>; ws_queries caps the workspace at that many score rows.  Returns device (ids, S1, minmax,
    workspace)."""
    lib = _native.load()
    nq = q8.shape[0]
    ids = torch.full((nq, k), -7, dtype=torch.int64, device=DEV)
    sc = torch.full((nq, k), -7.0, device=DEV)
    mm = torch.full((nq, 2), -7.0, device=DEV)
    if ws is None:
        ws = torch.empty(lib.crag_knn_code_workspace_bytes(n, ws_queries or nq), dtype=torch.uint8, device=DEV)
    st = stream.cuda_stream if stream is not None else torch.cuda.current_stream().cuda_stream
    rc = getattr(lib, f"crag_knn_topk_{code}")(codes.data_ptr() if n else 0, scales.data_ptr() if n else 0, n, dim8,
                                                 stride, row_offset, q8.data_ptr(), qs.data_ptr(), nq, k, ids.data_ptr(),
                                                 sc.data_ptr(), mm.data_ptr(), ws.data_ptr(), ws.numel(), st)
    _native.check(rc, f"crag_knn_topk_{code}")
    return ids, sc, mm, ws


def _setup(code, n, dim, nq, seed, distinct=None):
    rng = np.random.default_rng(seed)
    dim8 = qo.dim8_of(dim)
    x = _corpus(n, dim, rng, distinct)
    xd, xv = _bf16(x)
    qd, _ = _bf16(_queries(nq, dim, rng, xv))
    codes, scales, stride = _encode(code, xd, n, dim8)
    q8, qs = quantize_rows(qd, dim8)
    return codes, scales, stride, dim8, q8, qs


# ------------------------------------------------------------------------------------------------ 1. the S1 block
@pytest.mark.parametrize("code", CODES)
@pytest.mark.parametrize("n", [1, 127, 128, 129, 1000, 5000])
def test_s1_block_bit_identical(code, n):
    """The score block left in the workspace (one chunk holding every query) is the oracle's S1, row for row; with a
    workspace of 7 score rows the chunked call still returns the oracle's top k."""
    lib = _native.load()
    grid = lib.crag_sm_count()
    parts = (grid * NQ * 2 * 4 + ALIGN - 1) // ALIGN * ALIGN
    ld = (n + 3) // 4 * 4
    for dim, nq in ((64, 1), (320, 33), (768, 100), (1024, 32)):
        codes, scales, stride, dim8, q8, qs = _setup(code, n, dim, nq, seed=n * 7 + dim)
        _, _, _, ws = _knn(code, codes, scales, n, dim8, stride, q8, qs, 1)
        torch.cuda.synchronize()
        block = ws[parts:parts + nq * ld * 4].view(torch.float32).reshape(nq, ld)[:, :n].cpu().numpy()
        _assert_bits(block, _oracle_s1(code, codes, scales, q8, qs))
        k = min(n, 300)
        ids, sc, mm, _ = _knn(code, codes, scales, n, dim8, stride, q8, qs, k, row_offset=1 << 33, ws_queries=7)
        for g, w in zip((ids, sc, mm), _oracle_topk(code, codes, scales, q8, qs, k, 1 << 33)):
            _assert_bits(g.cpu().numpy(), w)


# ------------------------------------------------------------------------------------------------ 2. against the scans
@pytest.mark.parametrize("code", CODES)
def test_equals_topk_scan_up_to_128(code):
    lib = _native.load()
    n, nq = 20_000, 40
    codes, scales, stride, dim8, q8, qs = _setup(code, n, 768, nq, seed=5)
    for k in (1, 10, 64, 65, 128):
        ids, sc, mm, _ = _knn(code, codes, scales, n, dim8, stride, q8, qs, k, row_offset=3)
        s_ids = torch.full((nq, k), -7, dtype=torch.int64, device=DEV)
        s_sc = torch.full((nq, k), -7.0, device=DEV)
        s_mm = torch.full((nq, 2), -7.0, device=DEV)
        ws = torch.empty(lib.crag_search_workspace_bytes(nq, k), dtype=torch.uint8, device=DEV)
        rc = getattr(lib, f"crag_search_topk_{code}")(codes.data_ptr(), scales.data_ptr(), n, dim8, stride, 3,
                                                      q8.data_ptr(), qs.data_ptr(), nq, k, s_ids.data_ptr(),
                                                      s_sc.data_ptr(), s_mm.data_ptr(), ws.data_ptr(), ws.numel(), None)
        _native.check(rc, "scan")
        assert torch.equal(ids, s_ids), k
        assert torch.equal(sc.view(torch.int32), s_sc.view(torch.int32)), k
        assert torch.equal(mm, s_mm), k


# ------------------------------------------------------------------------------------------------ 3. beyond 128
@pytest.mark.parametrize("code", CODES)
@pytest.mark.parametrize("k", [129, 700, 2047, 2048])
def test_candidates_beyond_128_with_ties(code, k):
    """300 distinct rows among 5000 (plus duplicates and zero rows): S1 ties straddle every cut-off."""
    codes, scales, stride, dim8, q8, qs = _setup(code, 5000, 320, 35, seed=k, distinct=300)
    ids, sc, mm, _ = _knn(code, codes, scales, 5000, dim8, stride, q8, qs, k, ws_queries=16)
    for g, w in zip((ids, sc, mm), _oracle_topk(code, codes, scales, q8, qs, k)):
        _assert_bits(g.cpu().numpy(), w)


@pytest.mark.parametrize("code", CODES)
def test_empty_shard(code):
    codes, scales, stride, dim8, q8, qs = _setup(code, 0, 256, 3, seed=1)
    ids, sc, mm, _ = _knn(code, codes, scales, 0, dim8, stride, q8, qs, 200)
    assert (ids.cpu() == -1).all() and torch.isneginf(sc.cpu()).all()
    assert torch.isposinf(mm[:, 0].cpu()).all() and torch.isneginf(mm[:, 1].cpu()).all()


# ------------------------------------------------------------------------------------------------ 4. final answers
def _index(n, dim, rng, row_offset=0, planted=False):
    x = _corpus(n, dim, rng)
    ix = DenseIndex(dim, device=torch.device(DEV, 0), row_offset=row_offset)
    ix.add(x)
    pad = ix.dim_pad - dim
    xv = np.pad(torch.from_numpy(x).bfloat16().float().numpy(), ((0, 0), (0, pad)))
    return ix, x, xv, pad


def _cls(code):
    return QuantizedIndex if code == "i8" else BinaryIndex


def _pipeline(code, xv, qv, k, c, row_offset):
    f = qo.quantized_search if code == "i8" else bo.binary_search
    return f(xv, qv, k, c, row_offset=row_offset)[:2]


@pytest.mark.parametrize("code", CODES)
@pytest.mark.parametrize("rows", ["device", "host"])
def test_search_wide_bit_identical(code, rows):
    rng = np.random.default_rng(21)
    n, dim = 20_000, 1000
    ix, x, xv, pad = _index(n, dim, rng, row_offset=1 << 33)
    wix = _cls(code).from_dense(ix, rows=rows)
    q = _queries(40, dim, rng, x)
    qv = np.pad(torch.from_numpy(q).bfloat16().float().numpy(), ((0, 0), (0, pad)))
    for k, c in ((10, 129), (100, 1000), (1, 2048), (2048, 2048)):
        ids, sc = wix.search_wide(q, k, c)
        w_ids, w_sc = _pipeline(code, xv, qv, k, c, 1 << 33)
        _assert_bits(ids, w_ids)
        _assert_bits(sc, w_sc)


@pytest.mark.parametrize("code", CODES)
def test_wide_at_most_128_is_search_device(code):
    rng = np.random.default_rng(3)
    ix, x, _, _ = _index(5000, 384, rng)
    wix = _cls(code).from_dense(ix)
    qd, _ = _bf16(_queries(33, 384, rng, x))
    for k, c in ((1, 1), (10, 40), (128, 128)):
        a, b = wix.search_device_wide(qd, k, c), wix.search_device(qd, k, c)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))


def test_every_row_a_candidate_codes_agree():
    """With candidates >= n_rows both stage 1s keep every row, so the rescored answers are bit-identical."""
    rng = np.random.default_rng(9)
    ix, x, _, _ = _index(1000, 320, rng)
    q = _queries(35, 320, rng, x)
    bix, qix = BinaryIndex.from_dense(ix), QuantizedIndex.from_dense(ix)
    for k, c in ((1, 1000), (10, 1500), (1000, 2048)):
        bi, bs = bix.search_wide(q, k, c)
        qi, qs_ = qix.search_wide(q, k, c)
        _assert_bits(bi, qi)
        _assert_bits(bs, qs_)


# ------------------------------------------------------------------------------------------------ 5. monotone S2
@pytest.mark.parametrize("code", CODES)
def test_more_candidates_never_lower_s2(code):
    """The 2048-candidate set contains the 128-candidate set (both are top-k lists of one S1 order), so the S2 at
    every rank can only rise."""
    rng = np.random.default_rng(17)
    n, dim = 50_000, 1024
    base = rng.standard_normal((n, dim), dtype=np.float32)
    q = rng.standard_normal((32, dim), dtype=np.float32)
    for j in range(32):                                   # planted neighbours: 20 rows near each query
        base[j * 20:(j + 1) * 20] = q[j] + rng.standard_normal((20, dim), dtype=np.float32) * np.float32(0.6)
    ix = DenseIndex(dim, device=torch.device(DEV, 0))
    ix.add(base)
    wix = _cls(code).from_dense(ix)
    qd, _ = _bf16(q)
    _, s128 = wix.search_device(qd, 100, 128)
    _, s2048 = wix.search_device_wide(qd, 100, 2048)
    s128, s2048 = s128.cpu().numpy(), s2048.cpu().numpy()
    assert (s2048 >= s128).all()
    if code == "b1":   # int8 codes already find these answers among 128 candidates; one-bit codes do not
        assert (s2048 > s128).any()


# ------------------------------------------------------------------------------------------------ 6. streams, repeats
def test_two_streams_and_repeat_identical():
    rng = np.random.default_rng(8)
    ix, x, _, _ = _index(30_000, 768, rng)
    a, b = BinaryIndex.from_dense(ix, "device"), BinaryIndex.from_dense(ix, "host")
    qd, _ = _bf16(_queries(45, 768, rng, x))
    ref = a.search_device_wide(qd, 50, 1500)
    again = a.search_device_wide(qd, 50, 1500)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    s1.wait_stream(torch.cuda.current_stream())
    s2.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s1):
        r1 = a.search_device_wide(qd, 50, 1500, stream=s1)
    with torch.cuda.stream(s2):
        r2 = b.search_device_wide(qd, 50, 1500, stream=s2)
    torch.cuda.synchronize()
    for r in (again, r1, r2):
        assert torch.equal(r[0], ref[0]) and torch.equal(r[1].view(torch.int32), ref[1].view(torch.int32))


# ------------------------------------------------------------------------------------------------ 7. errors
@pytest.mark.parametrize("code", CODES)
def test_errors_launch_nothing(code):
    lib = _native.load()
    rng = np.random.default_rng(1)
    ix, x, _, _ = _index(500, 256, rng)
    wix = _cls(code).from_dense(ix)
    qd, _ = _bf16(x[:4])
    for k, c in ((20, 10), (10, 2049), (0, 5), (1, 0)):
        with pytest.raises(ValueError):
            wix.search_device_wide(qd, k, c)
        with pytest.raises(ValueError):
            wix.search_wide(x[:4], k, c)
    codes, scales, stride, dim8, q8, qs = _setup(code, 500, 256, 4, seed=2)
    out_i = torch.full((4 * 2048 + 8,), -7, dtype=torch.int64, device=DEV)
    out_s = torch.full((4 * 2048 + 8,), -7.0, device=DEV)
    ws = torch.empty(lib.crag_knn_code_workspace_bytes(500, 4), dtype=torch.uint8, device=DEV)
    parts = lib.crag_knn_code_workspace_bytes(500, 4) - (4 * 500 * 4 + ALIGN - 1) // ALIGN * ALIGN
    fn = getattr(lib, f"crag_knn_topk_{code}")

    def call(k=100, d8=dim8, st=stride, cp=codes.data_ptr(), ws_bytes=ws.numel()):
        return fn(cp, scales.data_ptr(), 500, d8, st, 0, q8.data_ptr(), qs.data_ptr(), 4, k, out_i.data_ptr(),
                  out_s.data_ptr(), 0, ws.data_ptr(), ws_bytes, None)
    assert call(k=2049) == INVALID and "k=" in lib.crag_last_error().decode()
    assert call(k=0) == INVALID
    assert call(d8=192) == INVALID and "dim8" in lib.crag_last_error().decode()
    assert call(st=stride + 8) == INVALID and "row_stride" in lib.crag_last_error().decode()
    assert call(cp=0) == INVALID and "null" in lib.crag_last_error().decode()
    assert call(ws_bytes=parts + 500 * 4 - 1) == WORKSPACE and "score row" in lib.crag_last_error().decode()
    cand = torch.zeros((4, 2049), dtype=torch.int64, device=DEV)
    rc = lib.crag_rescore_topk(ix._snapshot()[0].data_ptr(), 500, ix.dim_pad, ix.dim_pad, 0, qd.data_ptr(), 4,
                               cand.data_ptr(), 2049, 10, out_i.data_ptr(), out_s.data_ptr(), None)
    assert rc == INVALID and "n_cand" in lib.crag_last_error().decode()
    torch.cuda.synchronize()
    assert (out_i.cpu() == -7).all() and (out_s.cpu() == -7.0).all()
