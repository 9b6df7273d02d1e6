"""The SIMT parts of the kernels on the CPU.  csrc/topk.cuh, pool_floor.cuh, merge_kernels.cuh, rank_kernels.cuh and
encoder_simt.cuh hold no wgmma / TMA / mbarrier code, so the SAME headers the library compiles are compiled for the
host with CUDA threads as fibers (tests/warp_emu: warp collectives, __syncthreads, shared memory, one OS thread per
rank with real atomics for the cross-rank exchange) and checked against plain C++ models:
  selector_emu_test.cpp  bitonic sort, flush / insert list maintenance, select_stream, and the pooled admission
                         floors -- above all the property exactness rests on: >= k published keys reach the floor
  select_emu_test.cpp    the SELECT WARPS of the headline kernel (csrc/select_warps.inc.cuh, the text search_topk_kernel
                         #includes): admission, warp-ballot compaction, flushes, pooled-floor refreshes across CTAs,
                         drain, rank continuation, score-all and IVF variants -- fed a score matrix in place of
                         the score-tile read, merged by the emulated merge kernel, compared bit for bit with the exact top-k
  encoder_emu_test.cpp   embedding + LayerNorm, LayerNorm, masked mean pool + L2 normalise (K3) and the classifier
                         head (csrc/encoder_simt.cuh) against double-precision models
  kernel_emu_test.cpp    the IVF plan / id-map kernels, the radix-rank kernels (full permutation == stable descending
                         sort), merge_topk_kernel in
                         both layouts, and finalize_exchange_kernel on 2 / 3 / 4 / 8 ranks, calls back to back with
                         a deliberately slow reader (the slot-parity protocol)."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "warp_emu")
CSRC = os.path.join(ROOT, "comorag_b200", "csrc")


@pytest.fixture(scope="module")
def emu_binary(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not installed")
    exe = tmp_path_factory.mktemp("warp_emu") / "selector_emu_test"
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Wno-unknown-pragmas", "-pthread", "-I", os.path.join(EMU, "stub"), "-I", CSRC,
                        os.path.join(EMU, "selector_emu_test.cpp"), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def _build_kernel_test(csrc_dir, exe):
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Wno-unknown-pragmas", "-pthread", "-I", os.path.join(EMU, "stub"), "-I", str(csrc_dir),
                        os.path.join(EMU, "kernel_emu_test.cpp"), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


@pytest.fixture(scope="module")
def kernel_binary(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not installed")
    return _build_kernel_test(CSRC, tmp_path_factory.mktemp("warp_emu_k") / "kernel_emu_test")


def test_selector_primitives_match_their_models_on_emulated_lanes(emu_binary):
    r = subprocess.run([str(emu_binary), "3"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.strip().endswith("ALL OK")
    for group in ("warp_sort_desc<8>", "flush_query<128, 128>", "first-tile flush_query<128, 0>", "insert_few<128, 128>",
                  "select_stream<128, 128>", "lane_kth_of_pool<4>", "pooled_floor_batch8", "pooled_kth_key / pooled_max_kth"):
        assert f"ok  {group}" in r.stdout, group


def test_the_emulated_headers_are_the_ones_the_kernel_includes():
    """No copy of the selector lives under tests/: the emulation includes csrc/topk.cuh and csrc/pool_floor.cuh, and
    search.cu includes the same two files."""
    test_src = open(os.path.join(EMU, "selector_emu_test.cpp")).read()
    assert '#include "topk.cuh"' in test_src and '#include "pool_floor.cuh"' in test_src
    kernel_src = open(os.path.join(CSRC, "search.cu")).read()
    assert '#include "topk.cuh"' in kernel_src and '#include "pool_floor.cuh"' in kernel_src
    ktest_src = open(os.path.join(EMU, "kernel_emu_test.cpp")).read()
    assert '#include "merge_kernels.cuh"' in ktest_src and '#include "rank_kernels.cuh"' in ktest_src
    assert '#include "merge_kernels.cuh"' in kernel_src
    assert '#include "rank_kernels.cuh"' in open(os.path.join(CSRC, "rank_all.cu")).read()
    for name in os.listdir(EMU):
        assert not name.endswith(".cuh"), f"{name}: kernel headers must not be duplicated under tests/"


def test_emulation_catches_a_broken_floor(emu_binary, tmp_path):
    """Mutation check: a floor bisection that counts `>` instead of `>=` (a floor one key too high -- it would drop a
    true top-k row) must fail the property test."""
    mutated = tmp_path / "csrc"
    mutated.mkdir()
    for h in ("topk.cuh", "pool_floor.cuh"):
        shutil.copy(os.path.join(CSRC, h), mutated / h)
    src = (mutated / "pool_floor.cuh").read_text()
    needle = "for (int i = 0; i < NC; ++i) c += (hi[j][i] >= cand) ? 1 : 0;"
    assert src.count(needle) == 1
    (mutated / "pool_floor.cuh").write_text(src.replace(needle, needle.replace(">= cand", "> cand")))
    exe = tmp_path / "mutant"
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wno-unknown-pragmas", "-I", os.path.join(EMU, "stub"), "-I", str(mutated),
                        os.path.join(EMU, "selector_emu_test.cpp"), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe), "1"], capture_output=True, text=True, timeout=600)
    assert r.returncode != 0 and "FAILED" in r.stderr


def test_rank_merge_and_exchange_kernels_on_emulated_blocks(kernel_binary):
    r = subprocess.run([str(kernel_binary), "1"], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.strip().endswith("ALL OK")
    for group in ("ivf_plan_kernel + ivf_map_ids_kernel: nlist = 4096", "rank kernels: n = 6000", "merge_topk_kernel<128, 128, keys>", "merge_topk_kernel<64, 64, packed records>",
                  "finalize_exchange_kernel<64, 64>: world = 3", "finalize_exchange_kernel<128, 128>: world = 8"):
        assert f"ok  {group}" in r.stdout, group


def test_emulation_catches_a_broken_exchange_protocol(tmp_path):
    """Mutation check of the cross-rank protocol: with ONE slot parity a rank that ran a call ahead overwrites the record
    a slow peer is still reading -- the emulated ranks (one OS thread each, the last one a slow reader) must see it."""
    if shutil.which("g++") is None:
        pytest.skip("g++ not installed")
    mutated = tmp_path / "csrc"
    mutated.mkdir()
    for h in os.listdir(CSRC):
        if h.endswith(".cuh"):
            shutil.copy(os.path.join(CSRC, h), mutated / h)
    src = (mutated / "merge_kernels.cuh").read_text()
    needle = "const int parity = int(epoch & 1);"
    assert src.count(needle) == 1
    (mutated / "merge_kernels.cuh").write_text(src.replace(needle, "const int parity = 0;"))
    exe = _build_kernel_test(mutated, tmp_path / "mutant")
    # whether the overwrite lands inside the slow reader's window depends on thread scheduling: 24 calls per run give
    # it 24 chances, and a loaded box gets three runs
    for _ in range(3):
        r = subprocess.run([str(exe), "1"], capture_output=True, text=True, timeout=900)
        if r.returncode != 0:
            break
    assert r.returncode != 0 and "FAILED" in r.stderr and "exchange" in r.stderr


def test_encoder_simt_kernels_on_emulated_blocks(tmp_path):
    """embed_layernorm / layernorm / pool_normalize (BGEEmbedding.py:15-28, :127) / cls_head from csrc/encoder_simt.cuh,
    the file encoder_kernels.cu includes, against double-precision models (bf16 outputs within one bf16 step, fp32
    outputs within 2e-6)."""
    if shutil.which("g++") is None:
        pytest.skip("g++ not installed")
    assert '#include "encoder_simt.cuh"' in open(os.path.join(CSRC, "encoder_kernels.cu")).read()
    exe = tmp_path / "encoder_emu_test"
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Wno-unknown-pragmas", "-pthread", "-I", os.path.join(EMU, "stub"), "-I", CSRC,
                        os.path.join(EMU, "encoder_emu_test.cpp"), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.strip().endswith("ALL OK")
    for group in ("layernorm_kernel<4>: H = 1024", "embed_layernorm_kernel<4>: H = 1024, position offset 2",
                  "pool_normalize_kernel: H = 1024", "cls_head_kernel: H = 1024"):
        assert f"ok  {group}" in r.stdout, group


def _build_select_test(csrc_dir, exe):
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wno-unknown-pragmas", "-pthread", "-I", os.path.join(EMU, "stub"), "-I", str(csrc_dir),
                        os.path.join(EMU, "select_emu_test.cpp"), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def test_select_warps_of_the_scan_kernel_on_emulated_blocks(tmp_path):
    """search_topk_kernel's select warps -- the text the kernel itself #includes -- on adversarial score matrices
    (ascending with the row id, all rows equal, three score levels, planted neighbours in the tail, random), k from 1
    to 128, 1 to 148 CTAs sharing the pooled floor -- run one after the other and all resident together in random
    interleavings --, with and without the tile permutation; rank continuation over
    several pages; the score-all and IVF variants.  Ids, scores and (min, max) must equal the exact answer."""
    if shutil.which("g++") is None:
        pytest.skip("g++ not installed")
    kernel_src = open(os.path.join(CSRC, "search.cu")).read()
    assert kernel_src.count('#include "select_warps.inc.cuh"') == 3      # the kernel is built from the very same text
    exe = _build_select_test(CSRC, tmp_path / "select_emu_test")
    r = subprocess.run([str(exe), "1"], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.strip().endswith("ALL OK")
    for group in ("select warps <64, 64>: all rows equal", "select warps <128, 128>: planted neighbours in the last rows, 75699 rows on 148 CTAs",
                  "select warps <128, 128>: all rows equal, 75699 rows on 148 CTAs (4 tiles each), nq = 32, k = 100, pool on, permutation on, CTAs interleaved",
                  "rank continuation <128, 128>: random", "IVF variant <128, 128>: 64 lists", "score-all variant: 4475 rows"):
        assert f"ok  {group}" in r.stdout, group


def test_emulation_catches_a_selector_that_drops_a_tie(tmp_path):
    """Mutation check: an admission test that compares scores only (strictly) loses rows that tie the k-th score with a
    smaller row id -- the all-equal / few-levels corpora and the continuation pages must expose it."""
    if shutil.which("g++") is None:
        pytest.skip("g++ not installed")
    mutated = tmp_path / "csrc"
    mutated.mkdir()
    for h in os.listdir(CSRC):
        if h.endswith(".cuh"):
            shutil.copy(os.path.join(CSRC, h), mutated / h)
    src = (mutated / "select_warps.inc.cuh").read_text()
    needle = "if (s >= thr_f[q] && s <= bnd_f[q] && make_key(s, uint32_t(row)) > thr_key[q]) pending |= 1u << q;"
    assert src.count(needle) == 2          # flat and IVF admission
    (mutated / "select_warps.inc.cuh").write_text(src.replace(needle, "if (s > thr_f[q] && s <= bnd_f[q]) pending |= 1u << q;"))
    exe = _build_select_test(mutated, tmp_path / "mutant")
    r = subprocess.run([str(exe), "ties"], capture_output=True, text=True, timeout=1800)
    assert r.returncode != 0 and "FAILED" in r.stderr
