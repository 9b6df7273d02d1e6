"""Argument validation of every C entry point of the shard scan, without a device: the flat bf16 and int8 top-k scans,
the one-bit scan, the one-pass scan, the score-all pass, the IVF assignment, the bf16, int8 and PQ IVF searches, the PQ
encode, the exact large-k top-k and the threshold join.  Each case breaks exactly one argument of an otherwise valid
call and must be refused before any launch with INVALID (or WORKSPACE for a short workspace) and a crag_last_error()
naming that argument.  The host buffer passed as every pointer is never dereferenced.  Pageable-memory refusals need a
device and are tested in test_ivf_i8_gpu.py and test_ivf_pq_gpu.py."""
import ctypes as C

import pytest

from comorag_b200 import _native

INVALID, WORKSPACE = -1, -3


@pytest.fixture(scope="module")
def lib():
    return _native.load()


@pytest.fixture(scope="module")
def p():
    buf = (C.c_char * 8192)()
    p.keepalive = buf
    return (C.addressof(buf) + 255) & ~255


def caller(lib, fn, defaults):
    """fn(**overrides) with the arguments of `defaults` (an ordered list of (name, value)) in order."""
    names = [n for n, _ in defaults]

    def call(**kw):
        assert set(kw) <= set(names), kw
        return getattr(lib, fn)(*[kw.get(n, d) for n, d in defaults])
    return call


def expect(lib, rc, code, word):
    assert rc == code, (rc, lib.crag_last_error().decode())
    msg = lib.crag_last_error().decode()
    assert word in msg, msg


def flat_topk_args(p, after):
    a = [("corpus", p), ("n_rows", 1000), ("dim", 1024), ("stride", 1024), ("row_offset", 0), ("queries", p),
         ("nq", 4), ("k", 10)]
    if after:
        a.append(("after", None))
    a += [("ids", p), ("scores", p), ("minmax", p)]
    if after:
        a.append(("last", None))
    return a + [("ws", p), ("ws_bytes", 1 << 24), ("stream", None)]


BF16_CASES = [   # (overrides, return code, word of the message), common to every bf16 flat entry point
    (dict(nq=0), INVALID, "nq"),
    (dict(dim=1000), INVALID, "dim"),
    (dict(dim=0), INVALID, "dim"),
    (dict(dim=2048, stride=2048), INVALID, "dim"),
    (dict(stride=512), INVALID, "stride"),
    (dict(stride=1028), INVALID, "stride"),
    (dict(n_rows=-1), INVALID, "n_rows"),
    (dict(n_rows=1 << 31), INVALID, "n_rows"),
    (dict(corpus=None), INVALID, "null"),
    (dict(queries=None), INVALID, "null"),
    (dict(ws=None), INVALID, "null"),
    (dict(corpus=8), INVALID, "aligned"),
    (dict(queries=8), INVALID, "aligned"),
    (dict(ws=64), INVALID, "workspace"),
    (dict(ws_bytes=16), WORKSPACE, "workspace"),
]


def rebase(p, case):
    """pointer overrides given as small ints are offsets from the aligned buffer"""
    kw, code, word = case
    ptrs = {"corpus", "queries", "ws", "rows", "centroids"}
    return {n: (p + v if n in ptrs and isinstance(v, int) else v) for n, v in kw.items()}, code, word


@pytest.mark.parametrize("fn", ["crag_search_topk", "crag_search_topk_after"])
def test_flat_topk(lib, p, fn):
    call = caller(lib, fn, flat_topk_args(p, fn.endswith("_after")))
    for case in BF16_CASES:
        kw, code, word = rebase(p, case)
        expect(lib, call(**kw), code, word)
    expect(lib, call(k=0), INVALID, "k=")
    expect(lib, call(k=129), INVALID, "k=")
    expect(lib, call(ids=None), INVALID, "null")
    expect(lib, call(scores=None), INVALID, "null")


def test_search_scan(lib, p):
    call = caller(lib, "crag_search_scan", [("corpus", p), ("n_rows", 1000), ("dim", 1024), ("stride", 1024),
                                            ("queries", p), ("nq", 4), ("k", 10), ("ws", p), ("ws_bytes", 1 << 24),
                                            ("stream", None)])
    for case in BF16_CASES:
        kw, code, word = rebase(p, case)
        expect(lib, call(**kw), code, word)
    expect(lib, call(k=129), INVALID, "k=")
    expect(lib, call(nq=33), INVALID, "nq")


def test_search_scores(lib, p):
    call = caller(lib, "crag_search_scores", [("corpus", p), ("n_rows", 1000), ("dim", 1024), ("stride", 1024),
                                              ("queries", p), ("nq", 4), ("out", p), ("ld", 1000), ("minmax", p),
                                              ("ws", p), ("ws_bytes", 1 << 24), ("stream", None)])
    for case in BF16_CASES:
        kw, code, word = rebase(p, case)
        expect(lib, call(**kw), code, word)
    expect(lib, call(out=None), INVALID, "out_ld")
    expect(lib, call(ld=999), INVALID, "out_ld")


def test_ivf_assign(lib, p):
    call = caller(lib, "crag_ivf_assign", [("rows", p), ("n_rows", 1000), ("dim", 1024), ("stride", 1024),
                                           ("centroids", p), ("nq", 64), ("best_score", p), ("best_id", p),
                                           ("ws", p), ("ws_bytes", 1 << 24), ("stream", None)])
    rename = {"corpus": "rows", "queries": "centroids"}
    for case in BF16_CASES:
        kw, code, word = rebase(p, ({rename.get(n, n): v for n, v in case[0].items()},) + case[1:])
        expect(lib, call(**kw), code, word)
    expect(lib, call(best_score=None), INVALID, "null")
    expect(lib, call(best_id=None), INVALID, "null")


def test_knn_topk(lib, p):
    call = caller(lib, "crag_knn_topk", flat_topk_args(p, False))
    for case in BF16_CASES:
        kw, code, word = rebase(p, case)
        expect(lib, call(**kw), code, word)
    expect(lib, call(k=0), INVALID, "k=")
    expect(lib, call(k=2049), INVALID, "k=")
    expect(lib, call(ids=None), INVALID, "null")


def test_topk_i8(lib, p):
    call = caller(lib, "crag_search_topk_i8", [
        ("corpus", p), ("row_scales", p), ("n_rows", 1000), ("dim8", 1024), ("stride", 1024), ("row_offset", 0),
        ("queries", p), ("query_scales", p), ("nq", 4), ("k", 10), ("ids", p), ("scores", p), ("minmax", p),
        ("ws", p), ("ws_bytes", 1 << 24), ("stream", None)])
    expect(lib, call(nq=0), INVALID, "nq")
    expect(lib, call(k=0), INVALID, "k=")
    expect(lib, call(k=129), INVALID, "k=")
    expect(lib, call(dim8=1000), INVALID, "dim")
    expect(lib, call(dim8=64, stride=64), INVALID, "dim")
    expect(lib, call(dim8=2048, stride=2048), INVALID, "dim")
    expect(lib, call(stride=512), INVALID, "stride")
    expect(lib, call(stride=1032), INVALID, "stride")
    expect(lib, call(n_rows=-1), INVALID, "n_rows")
    expect(lib, call(n_rows=1 << 31), INVALID, "n_rows")
    for name in ("corpus", "row_scales", "queries", "query_scales", "ids", "scores", "ws"):
        expect(lib, call(**{name: None}), INVALID, "null")
    expect(lib, call(corpus=p + 8), INVALID, "aligned")
    expect(lib, call(queries=p + 8), INVALID, "aligned")
    expect(lib, call(ws=p + 64), INVALID, "workspace")
    expect(lib, call(ws_bytes=16), WORKSPACE, "workspace")


def test_ivf_search(lib, p):
    call = caller(lib, "crag_ivf_search", [
        ("residuals", p), ("n_rows_padded", 1024), ("dim", 1024), ("stride", 1024), ("list_tile_start", p),
        ("list_rows", p), ("nlist", 8), ("total_tiles", 8), ("row_ids", p), ("queries", p), ("nq", 4),
        ("probed_ids", p), ("probed_scores", p), ("nprobe", 2), ("k", 10), ("ids", p), ("scores", p), ("minmax", p),
        ("ws", p), ("ws_bytes", 1 << 24), ("stream", None)])
    expect(lib, call(nq=0), INVALID, "nq")
    expect(lib, call(k=0), INVALID, "k=")
    expect(lib, call(k=129), INVALID, "k=")
    expect(lib, call(nprobe=0), INVALID, "nprobe")
    expect(lib, call(nprobe=9), INVALID, "nprobe")
    expect(lib, call(nlist=0), INVALID, "nprobe")
    expect(lib, call(nlist=(1 << 20) + 1, nprobe=2), INVALID, "nprobe")
    expect(lib, call(total_tiles=7), INVALID, "total_tiles")
    expect(lib, call(total_tiles=-1), INVALID, "total_tiles")
    expect(lib, call(total_tiles=0, n_rows_padded=0), INVALID, "empty")
    expect(lib, call(total_tiles=1 << 24, n_rows_padded=1 << 31), INVALID, "n_rows")
    expect(lib, call(dim=1000), INVALID, "dim")
    expect(lib, call(dim=2048, stride=2048), INVALID, "dim")
    expect(lib, call(stride=512), INVALID, "stride")
    expect(lib, call(stride=1028), INVALID, "stride")
    for name in ("residuals", "list_tile_start", "list_rows", "row_ids", "queries", "probed_ids", "probed_scores",
                 "ids", "scores", "ws"):
        expect(lib, call(**{name: None}), INVALID, "null")
    expect(lib, call(residuals=p + 8), INVALID, "aligned")
    expect(lib, call(queries=p + 8), INVALID, "aligned")
    expect(lib, call(ws=p + 64), INVALID, "workspace")
    expect(lib, call(ws_bytes=16), WORKSPACE, "workspace")
    short = lib.crag_ivf_workspace_bytes(8, 8, 10) - 256
    expect(lib, call(ws_bytes=short), WORKSPACE, "workspace")


def test_ivf_search_i8(lib, p):
    call = caller(lib, "crag_ivf_search_i8", [
        ("res_i8", p), ("row_scales", p), ("dim8", 768), ("stride_i8", 768), ("res_bf16", p), ("dim", 704),
        ("stride", 704), ("n_rows_padded", 1024), ("list_tile_start", p), ("list_rows", p), ("nlist", 8),
        ("total_tiles", 8), ("row_ids", p), ("queries_i8", p), ("query_scales", p), ("queries_bf16", p), ("nq", 4),
        ("probed_ids", p), ("probed_scores", p), ("nprobe", 2), ("n_cand", 40), ("k", 10), ("ids", p),
        ("scores", p), ("minmax", p), ("ws", p), ("ws_bytes", 1 << 24), ("stream", None)])
    expect(lib, call(nq=0), INVALID, "nq")
    expect(lib, call(k=0), INVALID, "n_cand")
    expect(lib, call(k=41), INVALID, "n_cand")
    expect(lib, call(n_cand=129), INVALID, "n_cand")
    expect(lib, call(nprobe=0), INVALID, "nprobe")
    expect(lib, call(nprobe=9), INVALID, "nprobe")
    expect(lib, call(nlist=0), INVALID, "nprobe")
    expect(lib, call(total_tiles=7), INVALID, "total_tiles")
    expect(lib, call(total_tiles=0, n_rows_padded=0), INVALID, "empty")
    expect(lib, call(total_tiles=1 << 24, n_rows_padded=1 << 31), INVALID, "n_rows")
    expect(lib, call(dim=700), INVALID, "dim")
    expect(lib, call(dim=0, dim8=0), INVALID, "dim")
    expect(lib, call(dim=2048, dim8=2048, stride=2048, stride_i8=2048), INVALID, "dim")
    expect(lib, call(dim8=896), INVALID, "dim8")
    expect(lib, call(stride_i8=640), INVALID, "stride")
    expect(lib, call(stride_i8=776), INVALID, "stride")
    expect(lib, call(stride=640), INVALID, "stride")
    expect(lib, call(stride=708), INVALID, "stride")
    for name in ("res_i8", "row_scales", "res_bf16", "list_tile_start", "list_rows", "row_ids", "queries_i8",
                 "query_scales", "queries_bf16", "probed_ids", "probed_scores", "ids", "scores", "ws"):
        expect(lib, call(**{name: None}), INVALID, "null")
    for name in ("res_i8", "res_bf16", "queries_i8", "queries_bf16"):
        expect(lib, call(**{name: p + 8}), INVALID, "aligned")
    expect(lib, call(ws=p + 64), INVALID, "workspace")
    expect(lib, call(ws_bytes=16), WORKSPACE, "workspace")
    short = lib.crag_ivf_i8_workspace_bytes(8, 8, 40) - 256
    expect(lib, call(ws_bytes=short), WORKSPACE, "workspace")


def test_topk_b1(lib, p):
    call = caller(lib, "crag_search_topk_b1", [
        ("bits", p), ("alpha", p), ("n_rows", 1000), ("dim8", 1024), ("stride", 128), ("row_offset", 0),
        ("queries", p), ("query_scales", p), ("nq", 4), ("k", 10), ("ids", p), ("scores", p), ("minmax", p),
        ("ws", p), ("ws_bytes", 1 << 24), ("stream", None)])
    expect(lib, call(nq=0), INVALID, "nq")
    expect(lib, call(k=0), INVALID, "k=")
    expect(lib, call(k=129), INVALID, "k=")
    for dim8 in (0, 192, 1000, 2048):
        expect(lib, call(dim8=dim8), INVALID, "dim8")
    expect(lib, call(stride=120), INVALID, "row_stride")
    expect(lib, call(stride=136), INVALID, "row_stride")
    expect(lib, call(n_rows=-1), INVALID, "n_rows")
    expect(lib, call(n_rows=1 << 31), INVALID, "n_rows")
    expect(lib, call(bits=None), INVALID, "bits")
    expect(lib, call(alpha=None), INVALID, "alpha")
    for name in ("bits", "alpha", "queries", "query_scales", "ids", "scores", "ws"):
        expect(lib, call(**{name: None}), INVALID, "null")
    expect(lib, call(bits=p + 8), INVALID, "aligned")
    expect(lib, call(queries=p + 8), INVALID, "aligned")
    expect(lib, call(ws=p + 64), INVALID, "workspace")
    expect(lib, call(ws_bytes=16), WORKSPACE, "workspace")


def test_ivf_search_pq(lib, p):
    call = caller(lib, "crag_ivf_search_pq", [
        ("codes", p), ("m", 8), ("code_stride", 16), ("codebooks", p), ("res_bf16", p), ("dim", 768), ("stride", 768),
        ("n_rows_padded", 1024), ("list_tile_start", p), ("list_rows", p), ("nlist", 8), ("total_tiles", 8),
        ("row_ids", p), ("queries_bf16", p), ("nq", 4), ("probed_ids", p), ("probed_scores", p), ("nprobe", 2),
        ("n_cand", 40), ("k", 10), ("ids", p), ("scores", p), ("minmax", p), ("ws", p), ("ws_bytes", 1 << 24),
        ("stream", None)])
    expect(lib, call(nq=0), INVALID, "nq")
    expect(lib, call(k=0), INVALID, "n_cand")
    expect(lib, call(k=41), INVALID, "n_cand")
    expect(lib, call(n_cand=129), INVALID, "n_cand")
    expect(lib, call(nprobe=0), INVALID, "nprobe")
    expect(lib, call(nprobe=9), INVALID, "nprobe")
    expect(lib, call(nlist=0), INVALID, "nlist")
    expect(lib, call(total_tiles=7), INVALID, "total_tiles")
    expect(lib, call(n_rows_padded=100), INVALID, "n_rows_padded")
    expect(lib, call(total_tiles=0, n_rows_padded=0), INVALID, "empty")
    for m in (0, 7, 193):
        expect(lib, call(m=m), INVALID, "m must divide")
    expect(lib, call(m=192), INVALID, "code_stride")
    expect(lib, call(dim=100), INVALID, "dim")
    expect(lib, call(dim=2048, stride=2048), INVALID, "dim")
    expect(lib, call(code_stride=8), INVALID, "code_stride")
    expect(lib, call(code_stride=24), INVALID, "code_stride")
    expect(lib, call(codes=None), INVALID, "codes")
    expect(lib, call(codebooks=None), INVALID, "codebooks")
    for name in ("codes", "codebooks", "list_tile_start", "list_rows", "row_ids", "probed_ids", "probed_scores", "ids",
                 "scores", "ws"):
        expect(lib, call(**{name: None}), INVALID, "null")
    for name in ("codes", "codebooks"):
        expect(lib, call(**{name: p + 4}), INVALID, "aligned")
    expect(lib, call(ws=p + 64), INVALID, "workspace")
    expect(lib, call(ws_bytes=16), WORKSPACE, "workspace")
    short = lib.crag_ivf_pq_workspace_bytes(8, 8, 40, 8) - 256
    expect(lib, call(ws_bytes=short), WORKSPACE, "workspace")


def test_pq_encode(lib, p):
    call = caller(lib, "crag_pq_encode", [("rows", p), ("n_rows", 10), ("dim", 768), ("stride", 768),
                                          ("codebooks", p), ("m", 8), ("codes", p), ("code_stride", 16),
                                          ("stream", None)])
    for m in (0, 5, 193):
        expect(lib, call(m=m), INVALID, "m must divide")
    expect(lib, call(dim=96), INVALID, "dim")
    expect(lib, call(dim=2048, stride=2048), INVALID, "dim")
    expect(lib, call(n_rows=-1), INVALID, "n_rows")
    expect(lib, call(n_rows=1 << 31), INVALID, "n_rows")
    expect(lib, call(stride=512), INVALID, "row_stride")
    expect(lib, call(code_stride=4), INVALID, "code_stride")
    for name in ("rows", "codebooks", "codes"):
        expect(lib, call(**{name: None}), INVALID, name)
    expect(lib, call(rows=p + 1), INVALID, "aligned")
    expect(lib, call(codebooks=p + 2), INVALID, "aligned")


def test_knn_threshold(lib, p):
    call = caller(lib, "crag_knn_threshold", [
        ("corpus", p), ("n_rows", 1000), ("dim", 1024), ("stride", 1024), ("queries", p), ("nq", 4),
        ("threshold", 0.5), ("limit", 10), ("cap", 5), ("self_rows", None), ("exclude", p), ("n_exclude", 0),
        ("counts", p), ("ids", p), ("scores", p), ("ws", p), ("ws_bytes", 1 << 24), ("stream", None)])
    for case in BF16_CASES:
        kw, code, word = rebase(p, case)
        expect(lib, call(**kw), code, word)
    for t in (float("nan"), float("inf"), float("-inf")):
        expect(lib, call(threshold=t), INVALID, "threshold")
    expect(lib, call(limit=0), INVALID, "k=")
    expect(lib, call(cap=0), INVALID, "cap")
    expect(lib, call(cap=2048), INVALID, "cap")
    expect(lib, call(n_exclude=-1), INVALID, "n_exclude")
    expect(lib, call(n_exclude=65), INVALID, "n_exclude")
    expect(lib, call(cap=2048 - 64, n_exclude=64), INVALID, "cap")
    expect(lib, call(n_exclude=3, exclude=None), INVALID, "null")
    for name in ("counts", "ids", "scores"):
        expect(lib, call(**{name: None}), INVALID, "null")
    expect(lib, call(ws_bytes=1000 * 4 - 1), WORKSPACE, "workspace")
