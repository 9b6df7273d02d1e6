"""One-bit shards on the GPU: crag_binarize_rows, crag_search_topk_b1 and BinaryIndex against tests/binary_oracle.py bit
for bit -- codes and alpha, stage-1 ids, S1 and (min, max) over shard edges, dims, query blocks and k, the final ids and
scores with rows on the device and in page-locked host memory, ties, zero rows, two streams, the equality with
QuantizedIndex when every row is a candidate, and argument errors with nothing launched."""
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


def _bf16(x):
    """numpy float32 -> (device bf16 tensor, its values as numpy float32)."""
    t = torch.from_numpy(np.ascontiguousarray(x, np.float32)).bfloat16()
    return t.to(DEV), t.float().numpy()


def _corpus(n, dim, rng):
    x = rng.standard_normal((n, dim), dtype=np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True) + 1e-30
    if n >= 40:
        x[10:14] = x[3]               # duplicate rows: tied S1 and S2
        x[20:30] = x[20]              # a block of equal rows
        x[31:33] = 0.0                # zero rows: alpha = 0, S1 = 0
    return x


def _queries(nq, dim, rng, corpus_vals=None):
    q = rng.standard_normal((nq, dim), dtype=np.float32)
    if nq > 2:
        q[nq - 1] = 0.0               # an all-zero query: every S1 is 0
    if corpus_vals is not None and nq > 3 and corpus_vals.shape[0] > 0:
        q[1] = corpus_vals[min(3, corpus_vals.shape[0] - 1)]
    return q


def _assert_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape
    if a.dtype == np.float32:
        bad = a.view(np.uint32) != b.view(np.uint32)
    else:
        bad = a != b
    assert not bad.any(), f"{bad.sum()} of {bad.size} differ, first at {np.argwhere(bad)[:4].tolist()}"


@pytest.mark.parametrize("n,dim", [(1, 64), (1000, 64), (777, 320), (1000, 768), (2000, 1024)])
def test_codes_and_alpha_bit_identical(n, dim):
    rng = np.random.default_rng(n + dim)
    xd, xv = _bf16(_corpus(n, dim, rng))
    bits, alpha = binarize_rows(xd)
    want_c, want_a = bo.binarize(xv)
    _assert_bits(bits.cpu().numpy(), want_c)
    _assert_bits(alpha.cpu().numpy(), want_a)


def _stage1(codes, alpha, n, dim8, q8, qs, k, row_offset=0):
    lib = _native.load()
    nq = q8.shape[0]
    ids = torch.full((nq, k), -7, dtype=torch.int64, device=DEV)
    sc = torch.full((nq, k), -7.0, device=DEV)
    mm = torch.full((nq, 2), -7.0, device=DEV)
    ws_bytes = lib.crag_search_workspace_bytes(nq, k)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
    rc = lib.crag_search_topk_b1(codes.data_ptr() if n else 0, alpha.data_ptr() if n else 0, n, dim8, dim8 // 8,
                                 row_offset, q8.data_ptr(), qs.data_ptr(), nq, k, ids.data_ptr(), sc.data_ptr(),
                                 mm.data_ptr(), ws.data_ptr(), ws_bytes, None)
    _native.check(rc, "crag_search_topk_b1")
    return ids.cpu().numpy(), sc.cpu().numpy(), mm.cpu().numpy()


def _check_stage1(n, dim, nq, k, seed, row_offset=0):
    rng = np.random.default_rng(seed)
    xd, xv = _bf16(_corpus(n, dim, rng))
    qd, qv = _bf16(_queries(nq, dim, rng, xv))
    dim8 = bo.dim8_of(dim)
    codes, alpha = binarize_rows(xd) if n else (torch.zeros((0, dim8 // 8), dtype=torch.uint8, device=DEV),
                                                torch.zeros(0, device=DEV))
    q8, qs = quantize_rows(qd, dim8)
    got = _stage1(codes, alpha, n, dim8, q8, qs, k, row_offset)
    want = bo.search_b1(codes.cpu().numpy(), alpha.cpu().numpy(), q8.cpu().numpy(), qs.cpu().numpy(), k, row_offset)
    w_codes, w_alpha = bo.binarize(xv, dim8)
    _assert_bits(codes.cpu().numpy(), w_codes)
    _assert_bits(alpha.cpu().numpy(), w_alpha)
    for g, w in zip(got, want):
        _assert_bits(g, w)
    return got


@pytest.mark.parametrize("n", [0, 1, 127, 128, 129])
@pytest.mark.parametrize("dim,nq,k", [(64, 1, 1), (320, 31, 10), (768, 33, 65), (1024, 100, 128)])
def test_stage1_bit_identical_shard_edges(n, dim, nq, k):
    ids, _, mm = _check_stage1(n, dim, nq, k, seed=n * 7 + dim)
    if n == 0:
        assert (ids == -1).all() and np.isposinf(mm[:, 0]).all() and np.isneginf(mm[:, 1]).all()


@pytest.mark.parametrize("nq", [1, 31, 32, 33, 100])
@pytest.mark.parametrize("k", [1, 10, 64, 65, 128])
def test_stage1_bit_identical_query_blocks_and_k(nq, k):
    _check_stage1(5000, 320, nq, k, seed=nq * 131 + k)


@pytest.mark.parametrize("dim,k", [(1024, 10), (768, 128), (64, 64)])
def test_stage1_bit_identical_large_shard_pooled_floor(dim, k):
    _check_stage1(300_000, dim, 32, k, seed=dim + k, row_offset=1 << 33)


def test_stage1_all_zero_rows_and_ties():
    """Zero rows score 0 and tie in ascending row order; duplicate rows tie likewise."""
    rng = np.random.default_rng(4)
    x = np.zeros((600, 1024), np.float32)
    x[100:200] = rng.standard_normal((100, 1024))
    x[300:340] = x[100]
    xd, xv = _bf16(x)
    qd, _ = _bf16(_queries(3, 1024, rng))
    codes, alpha = binarize_rows(xd)
    q8, qs = quantize_rows(qd, 1024)
    got = _stage1(codes, alpha, 600, 1024, q8, qs, 128)
    want = bo.search_b1(codes.cpu().numpy(), alpha.cpu().numpy(), q8.cpu().numpy(), qs.cpu().numpy(), 128)
    for g, w in zip(got, want):
        _assert_bits(g, w)


def _index(n, dim, rng, row_offset=0):
    x = _corpus(n, dim, rng)
    ix = DenseIndex(dim, device=torch.device(DEV, 0), row_offset=row_offset)
    ix.add(x)
    pad = ix.dim_pad - dim
    xv = np.pad(torch.from_numpy(x).bfloat16().float().numpy(), ((0, 0), (0, pad)))
    return ix, x, xv, pad


@pytest.mark.parametrize("rows", ["device", "host"])
def test_binary_index_bit_identical(rows):
    rng = np.random.default_rng(21)
    n, dim = 20_000, 1000                                          # dim_pad 1024, dim8 1024
    ix, x, xv, pad = _index(n, dim, rng, row_offset=1 << 33)
    bix = BinaryIndex.from_dense(ix, rows=rows)
    assert bix.rows_on_device == (rows == "device") and bix.n_rows == n
    q = _queries(40, dim, rng, x)
    qv = np.pad(torch.from_numpy(q).bfloat16().float().numpy(), ((0, 0), (0, pad)))
    for k, c in ((10, None), (1, 1), (64, 65), (100, 128)):
        ids, sc = bix.search(q, k, c)
        w_ids, w_sc, _ = bo.binary_search(xv, qv, k, c or min(128, 4 * k), row_offset=1 << 33)
        _assert_bits(ids, w_ids)
        _assert_bits(sc, w_sc)
    assert bix.device_bytes == n * (128 + 4) + (n * 1024 * 2 if rows == "device" else 0)


def test_device_and_pinned_rows_and_two_streams_identical():
    rng = np.random.default_rng(8)
    ix, x, _, _ = _index(50_000, 768, rng)
    a, b = BinaryIndex.from_dense(ix, "device"), BinaryIndex.from_dense(ix, "host")
    qd, _ = _bf16(_queries(45, 768, rng, x))
    ref = a.search_device(qd, 10)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    s1.wait_stream(torch.cuda.current_stream())
    s2.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s1):
        r1 = a.search_device(qd, 10, stream=s1)
    with torch.cuda.stream(s2):
        r2 = b.search_device(qd, 10, stream=s2)
    torch.cuda.synchronize()
    for r in (r1, r2):
        assert torch.equal(r[0], ref[0]) and torch.equal(r[1].view(torch.int32), ref[1].view(torch.int32))


@pytest.mark.parametrize("n,dim", [(1, 64), (100, 320), (128, 1024)])
def test_all_candidates_equal_quantized_index(n, dim):
    """With candidates >= n_rows both stage 1s keep every row, so the rescored answers are bit-identical."""
    rng = np.random.default_rng(n)
    ix, x, _, _ = _index(n, dim, rng)
    q = _queries(35, dim, rng, x)
    bix, qix = BinaryIndex.from_dense(ix), QuantizedIndex.from_dense(ix)
    for k in (1, min(n, 10), n):
        bi, bs = bix.search(q, k, 128)
        qi, qs = qix.search(q, k, 128)
        _assert_bits(bi, qi)
        _assert_bits(bs, qs)


def test_errors_launch_nothing():
    lib = _native.load()
    n = 500
    rng = np.random.default_rng(1)
    ix, x, _, _ = _index(n, 256, rng)
    bix = BinaryIndex.from_dense(ix)
    qd, _ = _bf16(x[:4])
    with pytest.raises(ValueError):
        bix.search_device(qd, 20, candidates=10)
    with pytest.raises(ValueError):
        bix.search_device(qd, 10, candidates=129)
    with pytest.raises(ValueError):
        bix.search_device(qd[:, :128], 10)
    with pytest.raises(ValueError):
        binarize_rows(qd.float())
    bits = torch.zeros((n, 32), dtype=torch.uint8, device=DEV)
    alpha = torch.zeros(n, device=DEV)
    q8 = torch.zeros((1, 256), dtype=torch.int8, device=DEV)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
    out = torch.full((130,), -7, dtype=torch.int64, device=DEV)
    for dim8, stride, k, word in ((192, 32, 5, "dim8"), (256, 24, 5, "row_stride"), (256, 16, 5, "row_stride"),
                                  (256, 32, 129, "k")):
        rc = lib.crag_search_topk_b1(bits.data_ptr(), alpha.data_ptr(), n, dim8, stride, 0, q8.data_ptr(),
                                     alpha.data_ptr(), 1, k, out.data_ptr(), out.data_ptr(), 0, ws.data_ptr(),
                                     ws.numel(), None)
        assert rc == -1 and word in lib.crag_last_error().decode()
    rc = lib.crag_binarize_rows(qd.data_ptr(), 4, 256, 256, bits.data_ptr(), 16, alpha.data_ptr(), None)
    assert rc == -1 and "out_stride" in lib.crag_last_error().decode()
    torch.cuda.synchronize()
    assert (out.cpu() == -7).all() and not bits.cpu().any()
