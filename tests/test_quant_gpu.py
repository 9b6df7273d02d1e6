"""Int8 shards on the GPU: crag_quantize_rows_i8, crag_search_topk_i8, crag_rescore_topk and QuantizedIndex against
oracle/quant_oracle.py bit for bit, plus argument errors, pinned host rows, streams and recall."""
import ctypes as C

import numpy as np
import pytest
import torch

from comorag_b200 import _native
from comorag_b200.index import DenseIndex
from comorag_b200.quantized import QuantizedIndex, quantize_rows
from oracle import quant_oracle as qo

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _bf16(x):
    """numpy float32 -> (device bf16 tensor, its values as numpy float32)."""
    t = torch.from_numpy(np.ascontiguousarray(x, np.float32)).bfloat16()
    return t.to(DEV), t.float().numpy()


def _corpus(n, dim, rng, specials=True):
    x = rng.standard_normal((n, dim), dtype=np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True) + 1e-30
    if specials and n >= 40:
        x[10:14] = x[3]               # duplicate rows
        x[20:30] = x[20]              # a block of equal rows
        x[31:33] = 0.0                # zero rows
    return x


def _queries(nq, dim, rng, corpus_vals=None):
    q = rng.standard_normal((nq, dim), dtype=np.float32)
    if nq > 2:
        q[nq - 1] = 0.0               # an all-zero query: every S1 is 0
    if corpus_vals is not None and nq > 3 and corpus_vals.shape[0] > 0:
        q[1] = corpus_vals[min(3, corpus_vals.shape[0] - 1)]   # a query on a (duplicated) row
    return q


def _assert_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape
    if a.dtype == np.float32:
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), np.argwhere(a.view(np.uint32) != b.view(np.uint32))[:5]
    else:
        assert np.array_equal(a, b), np.argwhere(a != b)[:5]


# ------------------------------------------------------------------------------------------------ quantiser
@pytest.mark.parametrize("n", [1, 127, 128, 129, 100_003])
@pytest.mark.parametrize("dim", [64, 384, 768, 1024])
def test_quantiser_bit_identical(n, dim):
    rng = np.random.default_rng(n * 7 + dim)
    x = _corpus(n, dim, rng) * rng.uniform(1e-3, 4.0, (n, 1)).astype(np.float32)
    if n > 5:
        x[5, :2] = [1e-39, -3.0]
        x[6] = rng.integers(-127, 128, dim) * np.float32(2.0 ** -133)
    full = np.zeros((n, dim + 40), np.float32)    # strided input: rows dim + 40 apart, garbage past dim
    full[:, :dim] = x
    full[:, dim:] = 1e30
    dev, vals = _bf16(full)
    q8, s = quantize_rows(dev[:, :dim], qo.dim8_of(dim))
    want_q, want_s = qo.quantize(vals[:, :dim])
    _assert_bits(s.cpu().numpy(), want_s)
    _assert_bits(q8.cpu().numpy(), want_q)


# ------------------------------------------------------------------------------------------------ int8 scan
def _search_i8(r8, rs, q8, qs, k, row_offset=0, stream=None):
    lib = _native.load()
    n, nq = r8.shape[0], q8.shape[0]
    ids = torch.full((nq, k), -7, dtype=torch.int64, device=DEV)
    sc = torch.full((nq, k), -7.0, device=DEV)
    mm = torch.full((nq, 2), -7.0, device=DEV)
    ws_bytes = lib.crag_search_workspace_bytes(nq, k)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
    st = stream or torch.cuda.current_stream()
    rc = lib.crag_search_topk_i8(r8.data_ptr() if n else 0, rs.data_ptr() if n else 0, n, r8.shape[1], r8.shape[1],
                                 row_offset, q8.data_ptr(), qs.data_ptr(), nq, k, ids.data_ptr(), sc.data_ptr(),
                                 mm.data_ptr(), ws.data_ptr(), ws_bytes, st.cuda_stream)
    _native.check(rc, "crag_search_topk_i8")
    return ids, sc, mm


def _check_scan(n, dim, nq, ks, row_offset=0, seed=0, specials=True):
    rng = np.random.default_rng(seed)
    xd, xv = _bf16(_corpus(n, dim, rng, specials))
    qd, qv = _bf16(_queries(nq, dim, rng, xv))
    dim8 = qo.dim8_of(dim)
    r8, rs = quantize_rows(xd, dim8)
    q8, qs = quantize_rows(qd, dim8)
    o_r8, o_rs = qo.quantize(xv, dim8)
    o_q8, o_qs = qo.quantize(qv, dim8)
    _assert_bits(r8.cpu().numpy(), o_r8)
    _assert_bits(qs.cpu().numpy(), o_qs)
    for k in ks:
        ids, sc, mm = _search_i8(r8, rs, q8, qs, k, row_offset)
        w_ids, w_sc, w_mm = qo.search_i8(o_r8, o_rs, o_q8, o_qs, k, row_offset)
        _assert_bits(ids.cpu().numpy(), w_ids)
        _assert_bits(sc.cpu().numpy(), w_sc)
        _assert_bits(mm.cpu().numpy(), w_mm)


@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, 5000])
def test_scan_bit_identical_small_shards(n):
    _check_scan(n, 384, 33, [1, 10, 64, 65, 128], seed=n)


@pytest.mark.parametrize("nq", [1, 31, 32, 33, 70])
def test_scan_bit_identical_query_blocks(nq):
    _check_scan(3000, 1024, nq, [10, 65], seed=nq)


def test_scan_bit_identical_row_offset_2_33():
    _check_scan(2000, 768, 5, [1, 128], row_offset=1 << 33, seed=3)


def test_scan_bit_identical_1m_rows_pooled_floor():
    """1M rows: ~7800 tiles, many per CTA, so the pooled admission floor is in play."""
    _check_scan(1_000_000, 128, 33, [10, 128], seed=11)


def test_scan_all_zero_rows_and_queries():
    n, dim = 300, 256
    r8 = torch.zeros((n, 256), dtype=torch.int8, device=DEV)
    rs = torch.zeros(n, device=DEV)
    q8 = torch.zeros((3, 256), dtype=torch.int8, device=DEV)
    qs = torch.zeros(3, device=DEV)
    ids, sc, mm = _search_i8(r8, rs, q8, qs, 7)
    assert (ids.cpu() == torch.arange(7)).all() and (sc.cpu() == 0).all() and (mm.cpu() == 0).all()


# ------------------------------------------------------------------------------------------------ rescore / index
def _rescore(rows, n, row_offset, qd, cand, k):
    lib = _native.load()
    nq = qd.shape[0]
    ids = torch.full((nq, k), -7, dtype=torch.int64, device=DEV)
    sc = torch.full((nq, k), -7.0, device=DEV)
    rc = lib.crag_rescore_topk(rows.data_ptr() if n else 0, n, rows.shape[1], rows.stride(0), row_offset,
                               qd.data_ptr(), nq, cand.data_ptr(), cand.shape[1], k, ids.data_ptr(), sc.data_ptr(),
                               torch.cuda.current_stream().cuda_stream)
    return rc, ids, sc


def test_rescore_bit_identical_and_skips_out_of_range_ids():
    rng = np.random.default_rng(5)
    n, dim, nq, nc, off = 4000, 1024, 9, 100, 12345
    xd, xv = _bf16(_corpus(n, dim, rng))
    qd, qv = _bf16(_queries(nq, dim, rng, xv))
    cand = np.stack([rng.permutation(n)[:nc] for _ in range(nq)]).astype(np.int64) + off
    cand[0, :4] = [3 + off, 12 + off, 11 + off, 10 + off]        # duplicates of row 3: tied S2
    cand[:, -1] = -1
    cand[:, -2] = off - 1
    cand[:, -3] = off + n
    cand[2] = -1                                                  # a query without candidates
    for k in (1, 10, nc):
        rc, ids, sc = _rescore(xd, n, off, qd, torch.from_numpy(cand).to(DEV), k)
        assert rc == 0
        w_ids, w_sc = qo.rescore(xv, n, off, qv, cand, k)
        _assert_bits(ids.cpu().numpy(), w_ids)
        _assert_bits(sc.cpu().numpy(), w_sc)
    assert (ids[2].cpu() == -1).all() and (ids[0].cpu().numpy()[-3:] == -1).all()


@pytest.mark.parametrize("rows", ["device", "host"])
def test_quantized_index_bit_identical(rows):
    rng = np.random.default_rng(21)
    n, dim = 20_000, 1000                                          # dim_pad 1024, dim8 1024
    x = _corpus(n, dim, rng)
    ix = DenseIndex(dim, device=torch.device(DEV, 0), row_offset=1 << 33)
    ix.add(x)
    qix = QuantizedIndex.from_dense(ix, rows=rows)
    assert qix.rows_on_device == (rows == "device")
    xv = torch.from_numpy(x).bfloat16().float().numpy()
    xv = np.pad(xv, ((0, 0), (0, 24)))
    q = _queries(40, dim, rng, x)
    qv = np.pad(torch.from_numpy(q).bfloat16().float().numpy(), ((0, 0), (0, 24)))
    for k, c in ((10, None), (1, 1), (100, 128)):
        ids, sc = qix.search(q, k, c)
        w_ids, w_sc, _ = qo.quantized_search(xv, qv, k, c or min(128, 4 * k), row_offset=1 << 33)
        _assert_bits(ids, w_ids)
        _assert_bits(sc, w_sc)
    i8_bytes = n * 1024 + 4 * n
    assert qix.device_bytes == i8_bytes + (n * 1024 * 2 if rows == "device" else 0)


def test_device_and_pinned_rows_and_two_streams_identical():
    rng = np.random.default_rng(8)
    x = _corpus(50_000, 768, rng)
    ix = DenseIndex(768, device=torch.device(DEV, 0))
    ix.add(x)
    a, b = QuantizedIndex.from_dense(ix, "device"), QuantizedIndex.from_dense(ix, "host")
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


def test_errors_launch_nothing():
    lib = _native.load()
    rng = np.random.default_rng(1)
    n, dim = 500, 256
    x = torch.from_numpy(rng.standard_normal((n, dim), dtype=np.float32)).bfloat16()
    pageable = x.clone()                                          # ordinary host memory
    qd = x[:4].to(DEV)
    cand = torch.arange(40, dtype=torch.int64, device=DEV).repeat(4, 1)
    rc, ids, sc = _rescore(pageable, n, 0, qd, cand, 10)
    assert rc == -1 and "pageable" in lib.crag_last_error().decode()
    rc, ids2, _ = _rescore(x.to(DEV), n, 0, qd, cand[:, :8], 10)  # k > candidates
    assert rc == -1
    torch.cuda.synchronize()
    assert (ids.cpu() == -7).all() and (sc.cpu() == -7).all() and (ids2.cpu() == -7).all()
    assert lib.crag_quantize_rows_i8(0, 5, 1025, 1025, 0, 1152, 0, None) == -1
    assert lib.crag_quantize_rows_i8(0, 5, 100, 100, 0, 120, 0, None) == -1      # out_stride < dim8
    ix = DenseIndex(dim, device=torch.device(DEV, 0))
    ix.add(x)
    qix = QuantizedIndex.from_dense(ix)
    with pytest.raises(ValueError):
        qix.search_device(qd, 20, candidates=10)
    with pytest.raises(ValueError):
        qix.search_device(qd, 10, candidates=129)
    r8 = torch.zeros((n, 256), dtype=torch.int8, device=DEV)
    rs = torch.zeros(n, device=DEV)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
    out = torch.empty(64, dtype=torch.int64, device=DEV)
    for dim8, stride, k in ((192, 192, 5), (256, 200, 5), (256, 256, 129)):
        rc = lib.crag_search_topk_i8(r8.data_ptr(), rs.data_ptr(), n, dim8, stride, 0, r8.data_ptr(), rs.data_ptr(), 1,
                                     k, out.data_ptr(), out.data_ptr(), 0, ws.data_ptr(), ws.numel(), None)
        assert rc == -1


def test_recall_vs_dense_index_1m_1024():
    """1M x 1024 random unit rows, 32 queries: recall@10 and @100 of the default candidates against the bf16 scan."""
    g = torch.Generator(device=DEV).manual_seed(99)
    n, dim = 1_000_000, 1024
    rows = torch.empty((n, dim), dtype=torch.bfloat16, device=DEV)
    for r0 in range(0, n, 100_000):
        c = torch.randn((100_000, dim), generator=g, device=DEV)
        rows[r0:r0 + 100_000] = torch.nn.functional.normalize(c, dim=1).bfloat16()
    ix = DenseIndex.from_tensor(rows)
    qix = QuantizedIndex.from_dense(ix)
    q = torch.nn.functional.normalize(torch.randn((32, dim), generator=g, device=DEV), dim=1).bfloat16()
    for k in (10, 100):
        want = ix.search_device(q, k)[0].cpu().numpy()
        got = qix.search_device(q, k)[0].cpu().numpy()
        recall = np.mean([len(set(got[j]) & set(want[j])) / k for j in range(32)])
        print(f"recall@{k} (candidates {min(128, 4 * k)}) at 1M x 1024: {recall:.4f}")
        assert recall >= 0.99, recall
