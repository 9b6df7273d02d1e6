"""The select kernel of crag_knn_threshold (csrc/knn_threshold.cuh) on the CPU: the header holds no wgmma / TMA /
mbarrier code, so tests/warp_emu/knn_threshold_emu_test.cpp compiles the very header search.cu includes, runs
knn_threshold_kernel on emulated 512-thread blocks and compares counts, ids and scores bit for bit with a C++ model
of the walk (sort every key, walk the first min(limit, n_rows), stop below the threshold, skip self and excluded rows,
accept up to cap).  Regimes: no row above the threshold, fewer than cap, up to 2 048, more than 2 048 (the radix-select
path, with the cut decided by each of its three digits and by a tie), more than `limit`, every row excluded, and
row counts that are not a multiple of 4 with NaN in the padding columns.  Four mutants of the header must fail it."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "warp_emu")
CSRC = os.path.join(ROOT, "comorag_b200", "csrc")


def _build(csrc_dir, exe):
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unknown-pragmas", "-Wno-unused-function", "-pthread",
                        "-I", os.path.join(EMU, "stub"), "-I", str(csrc_dir), os.path.join(EMU, "knn_threshold_emu_test.cpp"),
                        "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def _mutant(tmp_path, replacements):
    mutated = tmp_path / "csrc"
    mutated.mkdir()
    for h in os.listdir(CSRC):
        if h.endswith(".cuh"):
            shutil.copy(os.path.join(CSRC, h), mutated / h)
    src = (mutated / "knn_threshold.cuh").read_text()
    for needle, repl in replacements:
        assert src.count(needle) == 1, needle
        src = src.replace(needle, repl)
    (mutated / "knn_threshold.cuh").write_text(src)
    return _build(mutated, tmp_path / "mutant")


def _fails(exe):
    r = subprocess.run([str(exe), "quick"], capture_output=True, text=True, timeout=1800)
    return r.returncode != 0 and "FAILED" in r.stderr


@pytest.fixture(autouse=True)
def _need_gxx():
    if shutil.which("g++") is None:
        pytest.skip("g++ not installed")


def test_the_emulated_threshold_select_is_the_header_search_cu_includes():
    assert '#include "knn_threshold.cuh"' in open(os.path.join(CSRC, "search.cu")).read()
    assert '#include "knn_threshold.cuh"' in open(os.path.join(EMU, "knn_threshold_emu_test.cpp")).read()
    src = open(os.path.join(CSRC, "knn_threshold.cuh")).read()
    for arch_only in ("wgmma_", "mbar_", "tma_load", "asm("):
        assert arch_only not in src, arch_only


def test_knn_threshold_kernel_on_emulated_blocks(tmp_path):
    exe = _build(CSRC, tmp_path / "knn_threshold_emu_test")
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.strip().endswith("ALL OK")
    for group in ("n_rows = 4097, c in", "ties at the threshold and the limit", "c > 2048 (overflow), cut by radix digits",
                  "every row excluded, n_rows % 4 != 0", "70001 rows"):
        assert f"ok  knn_threshold_kernel: {group}" in r.stdout, group


def test_emulation_catches_a_strict_threshold(tmp_path):
    """`>` where `>=` is needed drops the rows scoring exactly the threshold, which the walk accepts."""
    assert _fails(_mutant(tmp_path, [("hit[j] = live && e[j] >= threshold", "hit[j] = live && e[j] > threshold")]))


def test_emulation_catches_an_ignored_limit(tmp_path):
    """Walking every row above the threshold instead of the first `limit` of the list."""
    assert _fails(_mutant(tmp_path, [("int k_sel = limit < c ? limit : c;", "int k_sel = c;")]))


def test_emulation_catches_excluded_rows_counted_toward_the_cap(tmp_path):
    """Skipped rows that still take a place (and a slot of the cap) in the compaction."""
    assert _fails(_mutant(tmp_path, [("n_take += take[j] ? 1 : 0;", "n_take += 4 * tid + j < k_sel ? 1 : 0;"),
                                     ("    if (take[j]) {\n      if (r < cap) {",
                                      "    if (4 * tid + j < k_sel) {\n      if (r < cap && take[j]) {")]))


def test_emulation_catches_reading_the_padding_columns(tmp_path):
    """A pass that takes the whole last float4 as rows reads the NaN padding of rows whose count is not a multiple of 4."""
    assert _fails(_mutant(tmp_path, [("const bool live = i < n4 && 4 * i + j < n_rows;", "const bool live = i < n4;")]))
