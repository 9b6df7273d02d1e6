"""The select kernel of crag_knn_topk (csrc/knn_select.cuh) on the CPU: the header holds no wgmma / TMA / mbarrier code,
so tests/warp_emu/knn_emu_test.cpp compiles the very header search.cu includes, runs knn_select_kernel on emulated
512-thread blocks and compares ids, scores and (min, max) bit for bit with std::sort over the packed keys.  Two
mutants of the header must fail it: a tie gather that keeps the LAST equal rows, and a digit search that counts `>`
where `>=` is needed."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "warp_emu")
CSRC = os.path.join(ROOT, "comorag_b200", "csrc")


def _build(csrc_dir, exe):
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unknown-pragmas", "-pthread", "-I", os.path.join(EMU, "stub"),
                        "-I", str(csrc_dir), os.path.join(EMU, "knn_emu_test.cpp"), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def _mutant(tmp_path, replacements):
    mutated = tmp_path / "csrc"
    mutated.mkdir()
    for h in os.listdir(CSRC):
        if h.endswith(".cuh"):
            shutil.copy(os.path.join(CSRC, h), mutated / h)
    src = (mutated / "knn_select.cuh").read_text()
    for needle, repl in replacements:
        assert src.count(needle) == 1, needle
        src = src.replace(needle, repl)
    (mutated / "knn_select.cuh").write_text(src)
    return _build(mutated, tmp_path / "mutant")


@pytest.fixture(autouse=True)
def _need_gxx():
    if shutil.which("g++") is None:
        pytest.skip("g++ not installed")


def test_the_emulated_select_is_the_header_search_cu_includes():
    assert '#include "knn_select.cuh"' in open(os.path.join(CSRC, "search.cu")).read()
    assert '#include "knn_select.cuh"' in open(os.path.join(EMU, "knn_emu_test.cpp")).read()
    src = open(os.path.join(CSRC, "knn_select.cuh")).read()
    for arch_only in ("wgmma_", "mbar_", "tma_load", "asm("):
        assert arch_only not in src, arch_only


def test_knn_select_kernel_on_emulated_blocks(tmp_path):
    """Random rows, all-equal rows, three score levels, scores ascending with the row id, +-0 / +-inf / denormals;
    k in {1, 2, 127, 128, 129, 2047, 2048} against n_rows in {1, k-1, k, k+1, 5000, 70001}; row offsets beyond 2^32
    and the empty shard."""
    exe = _build(CSRC, tmp_path / "knn_emu_test")
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.strip().endswith("ALL OK")
    for group in ("k = 1, n_rows", "k = 129, n_rows", "k = 2048, n_rows", "all rows equal, k = 2047 of 70001",
                  "three score levels, k = 2047", "ascending with the row id, k = 2047", "+-0, +-inf and denormals, k = 2047",
                  "empty shard"):
        assert f"ok  knn_select_kernel: {group}" in r.stdout, group


def test_emulation_catches_a_gather_that_keeps_the_last_ties(tmp_path):
    """Mutation check: keeping the LAST quota rows equal to the threshold (instead of the first, in row order) breaks
    the ascending-row tie rule -- the all-equal and three-level rows must expose it."""
    exe = _mutant(tmp_path, [("if (r < quota) s_keys[c_above + r]", "if (r >= n_eq - quota) s_keys[c_above + r - (n_eq - quota)]"),
                             ("if (ordered_ties && taken_ties < quota)", "if (ordered_ties)")])
    r = subprocess.run([str(exe), "ties"], capture_output=True, text=True, timeout=1800)
    assert r.returncode != 0 and "FAILED" in r.stderr


def test_emulation_catches_a_digit_search_that_counts_strictly(tmp_path):
    """Mutation check: a digit search that picks the bin where the rows above it plus the bin EXCEED the rank (`>`
    instead of `>=`) selects the wrong threshold whenever the k-th row is the last of its bin."""
    exe = _mutant(tmp_path, [("above + h[c] >= quota", "above + h[c] > quota")])
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=1800)
    assert r.returncode != 0 and "FAILED" in r.stderr
