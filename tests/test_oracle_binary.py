"""tests/binary_oracle.py against plain scalar loops, and the properties the one-bit search is built on: with
candidates >= n_rows the answer is the exact rescore of every row, and rows whose entries share one magnitude lose
nothing to the code but the query's rounding.  Also the C ABI of the two new entry points without a device: both are
declared, exported and bound, the workspace is crag_search_workspace_bytes', and every malformed argument is refused
before any launch with a message naming it."""
import ctypes as C

import numpy as np
import pytest

import binary_oracle as bo
from oracle import quant_oracle as qo

F32 = np.float32


def _bf16_values(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, F32)).bfloat16().float().numpy()


def test_binarize_matches_scalar_loops():
    rng = np.random.default_rng(0)
    for dim in (64, 320, 1024):
        x = _bf16_values(rng.standard_normal((9, dim)) * 0.1)
        x[0] = 0.0
        x[1, :5] = -0.0
        codes, alpha = bo.binarize(x)
        dim8 = bo.dim8_of(dim)
        for r in range(x.shape[0]):
            for c in range(dim8):
                bit = (int(codes[r, c // 8]) >> (c % 8)) & 1
                assert bit == (1 if c < dim and x[r, c] > 0 else 0)
            lanes = [F32(0)] * 32
            for ch in range((dim + 7) // 8):
                for e in range(8):
                    if 8 * ch + e < dim:
                        lanes[ch % 32] = F32(lanes[ch % 32] + F32(abs(x[r, 8 * ch + e])))
            for o in (16, 8, 4, 2, 1):
                lanes = [F32(lanes[lane] + lanes[lane ^ o]) for lane in range(32)]
            assert alpha[r] == F32(lanes[0] / F32(dim))
        assert alpha[0] == 0 and not codes[0].any()


def test_s1_matches_scalar_loops():
    rng = np.random.default_rng(1)
    dim = 320
    x = _bf16_values(rng.standard_normal((50, dim)))
    q = _bf16_values(rng.standard_normal((3, dim)))
    codes, alpha = bo.binarize(x)
    q8, qs = qo.quantize(q, bo.dim8_of(dim))
    s1 = bo.s1_scores(codes, alpha, q8, qs, block=7)
    for j in range(3):
        for r in range(50):
            acc = 0
            for c in range(bo.dim8_of(dim)):
                acc += int(q8[j, c]) * (1 if (int(codes[r, c // 8]) >> (c % 8)) & 1 else -1)
            assert abs(acc) <= 127 * 1024
            assert s1[j, r] == F32(F32(acc) * F32(qs[j] * alpha[r]))


@pytest.mark.parametrize("n", [1, 60, 128])
def test_all_candidates_give_the_exact_rescore(n):
    rng = np.random.default_rng(n)
    dim = 320
    x = _bf16_values(rng.standard_normal((n, dim)))
    q = _bf16_values(rng.standard_normal((5, dim)))
    k = min(n, 10)
    ids, sc, (c_ids, _, _) = bo.binary_search(x, q, k, 128, row_offset=7)
    assert (np.sort(c_ids[:, :n], axis=1) == np.arange(n) + 7).all()   # every row is a candidate
    want_ids, want_sc = qo.rescore(x, n, 7, q, np.tile(np.arange(n) + 7, (5, 1)), k)
    assert np.array_equal(ids, want_ids)
    assert np.array_equal(sc.view(np.uint32), want_sc.view(np.uint32))


def test_one_magnitude_rows_lose_only_query_rounding():
    """x_i = +-c_r: alpha = c_r exactly, so S1 = float(s_q * c_r * (q^ . sign x)) up to two float32 roundings, the
    dequantised query's dot with the row itself."""
    rng = np.random.default_rng(3)
    n, dim = 400, 768
    c = _bf16_values(rng.uniform(0.01, 2.0, n))
    x = np.where(rng.random((n, dim)) < 0.5, -1.0, 1.0).astype(F32) * c[:, None]
    q = _bf16_values(rng.standard_normal((4, dim)))
    codes, alpha = bo.binarize(x)
    assert np.array_equal(alpha, c)
    q8, qs = qo.quantize(q, dim)
    s1 = bo.s1_scores(codes, alpha, q8, qs)
    exact = (q8.astype(np.float64) * qs[:, None].astype(np.float64)) @ x.astype(np.float64).T
    assert np.all(np.abs(s1 - exact) <= 2.0 ** -22 * np.abs(exact) + 1e-30)


# ------------------------------------------------------------------------------------------------ C ABI, no device
INVALID, WORKSPACE = -1, -3


@pytest.fixture(scope="module")
def lib():
    from comorag_b200 import _native
    return _native.load()


@pytest.fixture(scope="module")
def p():
    buf = (C.c_char * 8192)()
    p.keepalive = buf
    return (C.addressof(buf) + 255) & ~255


def test_new_symbols_are_declared_exported_and_bound(lib):
    import os
    import re
    from comorag_b200 import _native
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, "include", "comorag_b200.h")).read()
    for name in ("crag_binarize_rows", "crag_search_topk_b1"):
        assert re.search(r"CRAG_API\s+int\s+" + name + r"\s*\(", header)
        assert name in _native.SIGNATURES
        assert getattr(lib, name).argtypes == _native.SIGNATURES[name][1]


def _expect(lib, rc, code, word):
    msg = lib.crag_last_error().decode()
    assert rc == code, (rc, msg)
    assert word in msg, msg


def _b1(lib, p, **kw):
    a = dict(bits=p, alpha=p, n_rows=1000, dim8=1024, stride=128, row_offset=0, q=p, qs=p, nq=4, k=10, ids=p, sc=p,
             mm=p, ws=p, ws_bytes=1 << 24, stream=None)
    a.update(kw)
    return lib.crag_search_topk_b1(*a.values())


def test_search_b1_argument_errors(lib, p):
    for kw, code, word in [
            (dict(nq=0), INVALID, "nq"), (dict(k=0), INVALID, "k"), (dict(k=129), INVALID, "k"),
            (dict(dim8=1000), INVALID, "dim8"), (dict(dim8=0), INVALID, "dim8"), (dict(dim8=2048, stride=256), INVALID, "dim8"),
            (dict(n_rows=-1), INVALID, "n_rows"), (dict(n_rows=1 << 31), INVALID, "n_rows"),
            (dict(stride=112), INVALID, "row_stride"), (dict(stride=136), INVALID, "row_stride"),
            (dict(bits=None), INVALID, "bits"), (dict(bits=p + 8), INVALID, "bits"), (dict(alpha=None), INVALID, "alpha"),
            (dict(q=None), INVALID, "queries_i8"), (dict(q=p + 4), INVALID, "queries_i8"),
            (dict(qs=None), INVALID, "query_scales"), (dict(ids=None), INVALID, "output"), (dict(sc=None), INVALID, "output"),
            (dict(ws=None), INVALID, "workspace"), (dict(ws=p + 16), INVALID, "workspace"),
            (dict(ws_bytes=1024), WORKSPACE, "workspace")]:
        _expect(lib, _b1(lib, p, **kw), code, word)


def test_search_b1_workspace_is_the_scan_workspace(lib, p):
    """The one-bit scan sizes its workspace as the other flat scans do: crag_search_workspace_bytes(nq, k), whose
    per-CTA partials a short workspace cannot hold.  (A full-size call would launch: tests/test_binary_gpu.py.)"""
    for nq, k in ((1, 1), (33, 65), (100, 128)):
        need = lib.crag_search_workspace_bytes(nq, k)
        assert need > 0
        _expect(lib, _b1(lib, p, nq=nq, k=k, ws_bytes=256), WORKSPACE, "workspace")


def _bin(lib, p, **kw):
    a = dict(rows=p, n_rows=100, dim=1000, stride=1000, out=p, out_stride=128, alpha=p, stream=None)
    a.update(kw)
    return lib.crag_binarize_rows(*a.values())


def test_binarize_argument_errors(lib, p):
    for kw, word in [(dict(dim=0), "dim"), (dict(dim=1025), "dim"), (dict(n_rows=-1), "n_rows"),
                     (dict(stride=999), "row_stride"), (dict(out_stride=112), "out_stride"),
                     (dict(out_stride=136), "out_stride"), (dict(rows=None), "rows"), (dict(out=None), "out_bits"),
                     (dict(alpha=None), "out_alpha"), (dict(rows=p + 1), "rows"), (dict(out=p + 4), "out_bits")]:
        _expect(lib, _bin(lib, p, **kw), INVALID, word)
    assert _bin(lib, p, n_rows=0, rows=None, out=None, alpha=None) == 0   # nothing to do, nothing read
