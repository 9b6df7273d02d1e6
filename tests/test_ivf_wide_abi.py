"""The C ABI of the wide IVF searches (crag_ivf_search_i8_wide, crag_ivf_search_pq_wide and their workspace functions),
without a device: the prototypes in the header and a plain C99 call site against them, the workspace size against its
layout restated here (the IVF plan of a 1-key scan, the wide plan, the S1 block, the candidates, then the PQ tables,
each region on a 256-byte boundary), and argument errors refused before any launch.  The host buffer passed as every
pointer is never dereferenced."""
import ctypes as C
import itertools
import os
import re
import shutil
import subprocess

import pytest

from comorag_b200 import _native
from test_workspace_layout import NQ, ivf_regions, total

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "comorag_b200.h")
INVALID, WORKSPACE = -1, -3
MAX_PROBE = 128

TAIL = ["const int64_t* probed_ids", "const float* probed_scores", "int nprobe", "int n_cand", "int k",
        "int64_t max_probe_rows", "int64_t* out_ids", "float* out_scores", "float* out_minmax", "void* workspace",
        "size_t workspace_bytes", "crag_stream_t stream"]
LISTS = ["const int32_t* list_tile_start", "const int32_t* list_rows", "int nlist", "int64_t total_tiles",
         "const int64_t* row_ids"]
BF16 = ["const void* residuals_bf16", "int dim", "int64_t row_stride", "int64_t n_rows_padded"]
PROTOTYPES = {
    "crag_ivf_i8_wide_workspace_bytes": ("size_t", ["int nlist", "int64_t total_tiles", "int n_cand",
                                                    "int64_t max_probe_rows"]),
    "crag_ivf_pq_wide_workspace_bytes": ("size_t", ["int nlist", "int64_t total_tiles", "int n_cand",
                                                    "int64_t max_probe_rows", "int m"]),
    "crag_ivf_search_i8_wide": ("int", ["const void* residuals_i8", "const float* row_scales", "int dim8",
                                        "int64_t row_stride_i8"] + BF16 + LISTS +
                                ["const void* queries_i8", "const float* query_scales", "const void* queries_bf16",
                                 "int nq"] + TAIL),
    "crag_ivf_search_pq_wide": ("int", ["const void* codes", "int m", "int64_t code_stride", "const float* codebooks"] +
                                BF16 + LISTS + ["const void* queries_bf16", "int nq"] + TAIL),
}


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
int call(const void* p, const float* f, const int32_t* i32, const int64_t* i64, int64_t* ids, float* sc, void* ws) {
  size_t a = crag_ivf_i8_wide_workspace_bytes(64, (int64_t)10, 2048, (int64_t)5000);
  size_t b = crag_ivf_pq_wide_workspace_bytes(64, (int64_t)10, 2048, (int64_t)5000, 96);
  int rc = crag_ivf_search_i8_wide(p, f, 768, (int64_t)768, p, 768, (int64_t)768, (int64_t)1280, i32, i32, 64,
                                   (int64_t)10, i64, p, f, p, 7, i64, f, 32, 2048, 100, (int64_t)5000, ids, sc, sc, ws,
                                   a, (crag_stream_t)0);
  return rc | crag_ivf_search_pq_wide(p, 96, (int64_t)96, f, p, 768, (int64_t)768, (int64_t)1280, i32, i32, 64,
                                      (int64_t)10, i64, p, 7, i64, f, 32, 2048, 100, (int64_t)5000, ids, sc, sc, ws, b,
                                      (crag_stream_t)0);
}
''')
    r = subprocess.run(["gcc", "-std=c99", "-pedantic", "-Wall", "-Werror", "-I", os.path.dirname(HEADER), "-c",
                        str(tmp_path / "call.c"), "-o", str(tmp_path / "call.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def wide_regions(grid, nlist, tiles, n_cand, max_probe_rows, m=0):
    ld = (max_probe_rows + 3) // 4 * 4
    return ivf_regions(grid, 1, nlist, tiles) + [nlist * NQ * 4, NQ * MAX_PROBE * 4, NQ * MAX_PROBE * 4, NQ * 4, NQ * 4,
                                                 NQ * ld * 4, NQ * n_cand * 8, NQ * n_cand * 4, NQ * m * 256 * 4]


def test_workspace_layout(lib, grid):
    for nlist, tiles, n_cand, rows in itertools.product([1, 65, 4096], [0, 3, 1000], [1, 128, 129, 2048],
                                                        [1, 2, 5, 300_001, (1 << 31) - 128]):
        assert lib.crag_ivf_i8_wide_workspace_bytes(nlist, tiles, n_cand, rows) == \
            total(wide_regions(grid, nlist, tiles, n_cand, rows)), (nlist, tiles, n_cand, rows)
        for m in (1, 96, 192):
            assert lib.crag_ivf_pq_wide_workspace_bytes(nlist, tiles, n_cand, rows, m) == \
                total(wide_regions(grid, nlist, tiles, n_cand, rows, m)), (nlist, tiles, n_cand, rows, m)
    for bad in [(0, 1, 1, 1), (1, -1, 1, 1), (1, 1, 0, 1), (1, 1, 2049, 1), (1, 1, 1, 0), (1, 1, 1, (1 << 31) - 127)]:
        assert lib.crag_ivf_i8_wide_workspace_bytes(*bad) == 0, bad
        assert lib.crag_ivf_pq_wide_workspace_bytes(*bad, 8) == 0, bad
    assert lib.crag_ivf_pq_wide_workspace_bytes(1, 1, 1, 1, 0) == 0
    assert lib.crag_ivf_pq_wide_workspace_bytes(1, 1, 1, 1, 193) == 0


@pytest.fixture(scope="module")
def p():
    buf = (C.c_char * 8192)()
    p.keepalive = buf
    return (C.addressof(buf) + 255) & ~255


def _caller(lib, fn, p):
    pq = "_pq_" in fn
    lead = ([("codes", p), ("m", 96), ("code_stride", 96), ("codebooks", p)] if pq else
            [("codes", p), ("scales", p), ("dim8", 768), ("stride8", 768)])
    bf = [("rows", p), ("dim", 768), ("row_stride", 768), ("n_rows", 1280), ("starts", p), ("lrows", p), ("nlist", 64),
          ("tiles", 10), ("row_ids", p)]
    qs = [("queries", p), ("nq", 4)] if pq else [("q8", p), ("qs", p), ("queries", p), ("nq", 4)]
    tail = [("pid", p), ("psc", p), ("nprobe", 8), ("n_cand", 2048), ("k", 100), ("max_probe_rows", 5000), ("ids", p),
            ("scores", p), ("minmax", p), ("ws", p), ("ws_bytes", 1 << 40), ("stream", None)]
    defaults = lead + bf + qs + tail
    names = [n for n, _ in defaults]

    def call(**kw):
        assert set(kw) <= set(names), kw
        return getattr(lib, fn)(*[kw.get(n, d) for n, d in defaults])
    return call


def _expect(lib, rc, code, word):
    assert rc == code, (rc, lib.crag_last_error().decode())
    msg = lib.crag_last_error().decode()
    assert word in msg, msg


@pytest.mark.parametrize("fn", ["crag_ivf_search_i8_wide", "crag_ivf_search_pq_wide"])
def test_argument_errors(lib, p, fn):
    call = _caller(lib, fn, p)
    _expect(lib, call(k=2049), INVALID, "n_cand")
    _expect(lib, call(n_cand=99), INVALID, "n_cand")          # k > n_cand
    _expect(lib, call(n_cand=2049), INVALID, "n_cand <= 2048")
    _expect(lib, call(k=0), INVALID, "k=")
    _expect(lib, call(nq=0), INVALID, "nq")
    _expect(lib, call(max_probe_rows=0), INVALID, "max_probe_rows")
    _expect(lib, call(max_probe_rows=-1), INVALID, "max_probe_rows")
    _expect(lib, call(max_probe_rows=1 << 31), INVALID, "max_probe_rows")
    _expect(lib, call(nprobe=129, nlist=200), INVALID, "nprobe")
    _expect(lib, call(nprobe=0), INVALID, "nprobe")
    _expect(lib, call(n_rows=1000), INVALID, "n_rows_padded")
    _expect(lib, call(ids=None), INVALID, "null")
    _expect(lib, call(dim=100), INVALID, "dim")
    _expect(lib, call(ws=None), INVALID, "null")
    _expect(lib, call(ws=p + 64), INVALID, "workspace")
    need = (lib.crag_ivf_pq_wide_workspace_bytes(64, 10, 2048, 5000, 96) if "_pq_" in fn
            else lib.crag_ivf_i8_wide_workspace_bytes(64, 10, 2048, 5000))
    _expect(lib, call(ws_bytes=need - 1), WORKSPACE, "workspace")
    if "_pq_" in fn:
        _expect(lib, call(m=7), INVALID, "m must divide")
        _expect(lib, call(code_stride=8), INVALID, "code_stride")
        _expect(lib, call(codes=None), INVALID, "codes")
    else:
        _expect(lib, call(dim8=640, stride8=640), INVALID, "dim8")
        _expect(lib, call(scales=None), INVALID, "null")
