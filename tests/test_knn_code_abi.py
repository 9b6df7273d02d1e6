"""The C ABI of the exact top-k over int8 and one-bit codes (crag_knn_topk_i8, crag_knn_topk_b1,
crag_knn_code_workspace_bytes), without a device: the prototypes in the header and a plain C99 call site against them,
the workspace size against its layout restated here (the score-all pass's per-CTA (min, max), then the score block,
each region on a 256-byte boundary), and argument errors refused before any launch with the scans' rules and k up to
2048.  The host buffer passed as every pointer is never dereferenced."""
import ctypes as C
import itertools
import os
import re
import shutil
import subprocess

import pytest

from comorag_b200 import _native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "comorag_b200.h")
INVALID, WORKSPACE = -1, -3
ALIGN, NQ = 256, 32

TOPK_PARAMS = ["int64_t n_rows", "int dim8", "int64_t row_stride", "int64_t row_offset", "const void* queries_i8",
               "const float* query_scales", "int nq", "int k", "int64_t* out_ids", "float* out_scores",
               "float* out_minmax", "void* workspace", "size_t workspace_bytes", "crag_stream_t stream"]
PROTOTYPES = {
    "crag_knn_code_workspace_bytes": ("size_t", ["int64_t n_rows", "int q_chunk"]),
    "crag_knn_topk_i8": ("int", ["const void* codes", "const float* row_scales"] + TOPK_PARAMS),
    "crag_knn_topk_b1": ("int", ["const void* bits", "const float* alpha"] + TOPK_PARAMS),
}


def total(regions):
    return sum((r + ALIGN - 1) // ALIGN * ALIGN for r in regions)


@pytest.fixture(scope="module")
def lib():
    return _native.load()


@pytest.fixture(scope="module")
def grid(lib):
    g = lib.crag_sm_count()
    return g if g > 0 else 132


@pytest.mark.parametrize("name", list(PROTOTYPES))
def test_header_prototype(name):
    src = open(HEADER).read()
    m = re.search(r"CRAG_API\s+(\w+)\s+" + name + r"\(([^)]*)\);", src)
    assert m, name
    ret, params = PROTOTYPES[name]
    assert m.group(1) == ret
    assert [" ".join(p.split()) for p in m.group(2).split(",")] == params


def test_c99_call_site(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("gcc not installed")
    (tmp_path / "call.c").write_text(r'''
#include "comorag_b200.h"
int call(const void* codes, const void* bits, const float* scales, const void* q, const float* qs, int64_t* ids,
         float* sc, float* mm, void* ws) {
  size_t bytes = crag_knn_code_workspace_bytes((int64_t)1000, 7);
  int rc = crag_knn_topk_i8(codes, scales, (int64_t)1000, 1024, (int64_t)1024, (int64_t)0, q, qs, 7, 2048, ids, sc,
                            mm, ws, bytes, (crag_stream_t)0);
  return rc | crag_knn_topk_b1(bits, scales, (int64_t)1000, 1024, (int64_t)128, (int64_t)0, q, qs, 7, 2048, ids, sc,
                               mm, ws, bytes, (crag_stream_t)0);
}
''')
    r = subprocess.run(["gcc", "-std=c99", "-pedantic", "-Wall", "-Werror", "-I", os.path.dirname(HEADER), "-c",
                        str(tmp_path / "call.c"), "-o", str(tmp_path / "call.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_workspace_layout(lib, grid):
    for n, q_chunk in itertools.product([0, 1, 2, 3, 4, 5, 63, 64, 65, 1000, 1 << 20, 10_000_000], [1, 2, 7, 26, 32, 1024]):
        ld = (max(n, 1) + 3) // 4 * 4
        want = total([grid * NQ * 2 * 4, q_chunk * ld * 4])
        assert lib.crag_knn_code_workspace_bytes(n, q_chunk) == want, (n, q_chunk)
    assert lib.crag_knn_code_workspace_bytes(-1, 1) == 0
    assert lib.crag_knn_code_workspace_bytes(10, 0) == 0


@pytest.fixture(scope="module")
def p():
    buf = (C.c_char * 8192)()
    p.keepalive = buf
    return (C.addressof(buf) + 255) & ~255


def _caller(lib, fn, p, ws_bytes):
    b1 = fn.endswith("_b1")
    defaults = [("codes", p), ("scales", p), ("n_rows", 1000), ("dim8", 1024), ("stride", 128 if b1 else 1024),
                ("row_offset", 0), ("queries", p), ("qscales", p), ("nq", 4), ("k", 2048), ("ids", p), ("scores", p),
                ("minmax", p), ("ws", p), ("ws_bytes", ws_bytes), ("stream", None)]
    names = [n for n, _ in defaults]

    def call(**kw):
        assert set(kw) <= set(names), kw
        return getattr(lib, fn)(*[kw.get(n, d) for n, d in defaults])
    return call


def _expect(lib, rc, code, word):
    assert rc == code, (rc, lib.crag_last_error().decode())
    msg = lib.crag_last_error().decode()
    assert word in msg, msg


@pytest.mark.parametrize("fn", ["crag_knn_topk_i8", "crag_knn_topk_b1"])
def test_argument_errors(lib, p, grid, fn):
    parts = total([grid * NQ * 2 * 4])
    call = _caller(lib, fn, p, 1 << 30)
    b1 = fn.endswith("_b1")
    _expect(lib, call(k=0), INVALID, "k=")
    _expect(lib, call(k=2049), INVALID, "k=")
    _expect(lib, call(nq=0), INVALID, "nq")
    _expect(lib, call(dim8=192), INVALID, "dim8")
    _expect(lib, call(dim8=2048, stride=2048), INVALID, "dim8")
    _expect(lib, call(stride=120 if b1 else 1000), INVALID, "row_stride")
    _expect(lib, call(stride=136 if b1 else 1032), INVALID, "row_stride")
    _expect(lib, call(n_rows=-1), INVALID, "n_rows")
    _expect(lib, call(codes=None), INVALID, "null")
    _expect(lib, call(queries=None), INVALID, "null")
    _expect(lib, call(codes=p + 8), INVALID, "aligned")
    _expect(lib, call(scales=None), INVALID, "null")
    _expect(lib, call(qscales=None), INVALID, "null")
    _expect(lib, call(ids=None), INVALID, "null")
    _expect(lib, call(scores=None), INVALID, "null")
    _expect(lib, call(ws=None), INVALID, "null")
    _expect(lib, call(ws=p + 64), INVALID, "workspace")
    _expect(lib, call(ws_bytes=parts - 1), WORKSPACE, "workspace")
    # the partials fit, one query's score row (4 * 1000 bytes) does not
    _expect(lib, call(ws_bytes=parts + 3999), WORKSPACE, "score row")
