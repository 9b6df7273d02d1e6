"""The kernels of crag_ppr_batch (csrc/ppr_batch_kernels.cuh) against those of crag_ppr (csrc/ppr_kernels.cuh) on
the CPU.  tests/warp_emu/ppr_batch_emu_test.cpp runs both headers on emulated blocks, in ppr.cu's launch order:
every reset alone through the single-source kernels, then the batch through the batched kernels, block after block
and in random block interleavings.  Column b of every batched run must equal the single run of reset b bit for bit.

Graphs as in test_ppr_emulated.py: a path, a star whose hub row spans about a hundred segments, isolated vertices
with reset mass, empty rows next to every segment edge, and n = 1.  Columns differ: mass on a dangling vertex,
uniform, mass on the hub, and random sparse resets.  B in {1, 2, 3, 8, 31, 32} (widths 2 to 32), T in {0, 1, 35},
with and without out_vertices.

Both kernels are compiled with -ffp-contract=off: the batched kernels' ppr_mul / ppr_row_value are the single
kernels' plain expressions here, so the emulator checks the batched structure (chunks, open-row partials, carries,
columns, sums) and the GPU test (test_ppr_batch_gpu.py) pins the device's rounding.  Four mutants of the batched
header must fail: a gather off by one column, a row spanning chunks that loses its earlier partial, a fix-up that
drops a row's last carry, and every column normalised by column 0's total.  The star runs two batch sizes and one
random interleaving only: at 50 000 leaves it is the slowest case to emulate."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from comorag_b200.graph import DeviceGraph, ppr_iterations

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EMU = os.path.join(ROOT, "tests", "warp_emu")
CSRC = os.path.join(ROOT, "comorag_b200", "csrc")
BATCHES = "1,2,3,8,31,32"


def _build(csrc_dir, exe):
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-pthread",
                        "-I", os.path.join(EMU, "stub"), "-I", str(csrc_dir), os.path.join(EMU, "ppr_batch_emu_test.cpp"),
                        "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


@pytest.fixture(autouse=True)
def _need_gxx():
    if shutil.which("g++") is None:
        pytest.skip("g++ not installed")


@pytest.fixture(scope="module")
def emulator(tmp_path_factory):
    return _build(CSRC, tmp_path_factory.mktemp("ppr_batch_emu") / "ppr_batch_emu_test")


# ------------------------------------------------------------------------------------------------ graphs
def _path(n, rng):
    e = np.stack([np.arange(n - 1), np.arange(1, n)], 1)
    return n, e, rng.uniform(0.5, 2.0, n - 1)


def _star(leaves, rng):
    e = np.stack([np.zeros(leaves, np.int64), np.arange(1, leaves + 1)], 1)
    return leaves + 1, e, rng.uniform(0.8, 1.0, leaves)


def _isolated(rng):
    """120 vertices, the first 70 in a random graph with parallel edges and both orientations, 50 isolated."""
    a = rng.integers(0, 70, 400)
    b = rng.integers(0, 70, 400)
    keep = a != b
    e = np.stack([a[keep], b[keep]], 1)
    e = np.concatenate([e, e[:50, ::-1], e[:30]])
    return 120, e, rng.uniform(0.1, 3.0, len(e))


def _ladder(rng):
    """Pairs joined by one edge, an isolated vertex after every pair: an empty row next to every segment edge."""
    n = 3000
    trip = np.arange(0, n, 3)
    e = np.stack([trip, trip + 1], 1)
    return n, e, rng.uniform(0.5, 1.5, len(e))


def _resets(n, e, rng, hub=0, count=32):
    """count distinct resets: mass on a dangling vertex (or vertex n - 1), uniform, on the hub, then random sparse
    ones, some with mass on every dangling vertex."""
    deg = np.bincount(np.asarray(e, np.int64).reshape(-1), minlength=n)
    dangling = np.flatnonzero(deg == 0)
    out = np.zeros((count, n))
    out[0, dangling[0] if dangling.size else n - 1] = 1.0
    out[1] = 1.0
    out[2, hub] = 1.0
    for b in range(3, count):
        r = rng.uniform(0.0, 1.0, n) * (rng.uniform(size=n) < 0.3)
        r[rng.integers(0, n)] = 1.0
        if b % 4 == 0 and dangling.size:
            r[dangling] = 0.7
        out[b] = r
    return out


def _write_case(path, n, edges, weights, resets, damping, iterations, out_vertices=None):
    g = DeviceGraph.from_edges(n, torch.as_tensor(np.asarray(edges, np.int64).reshape(-1, 2)), torch.as_tensor(weights),
                               device="cpu")
    v = g.reset_vector(resets).numpy()
    with open(path, "wb") as f:
        np.array([n, g.nnz, -1 if out_vertices is None else len(out_vertices), iterations, len(v)], np.int64).tofile(f)
        np.array([damping], np.float32).tofile(f)
        g.row_ptr.numpy().astype(np.int64).tofile(f)
        g.col.numpy().astype(np.int32).tofile(f)
        g.coef.numpy().astype(np.float32).tofile(f)
        v.astype(np.float32).tofile(f)
        if out_vertices is not None:
            np.asarray(out_vertices, np.int32).tofile(f)


def _cases():
    rng = np.random.default_rng(20251017)
    T = ppr_iterations(0.5)
    d85 = float(np.float32(0.85))
    out = []
    n, e, w = _path(700, rng)
    r = _resets(n, e, rng, hub=350)
    for t in (0, 1, T):
        out.append(("path", n, e, w, r, 0.5, t, None))
    out.append(("path gathered", n, e, w, r, 0.5, T, rng.choice(n, 100, replace=False)))
    out.append(("path d=0.85", n, e, w, r, d85, ppr_iterations(d85), None))
    n, e, w = _star(50_000, rng)            # the hub's row spans ~100 segments of 512 items
    r = _resets(n, e, rng)
    r[3:, -1500:] = 5.0                      # heavy leaves at the end of the hub's row: its last carries matter
    out.append(("star", n, e, w, r, 0.5, 1, None))
    out.append(("star gathered", n, e, w, r, 0.5, 3, rng.choice(n, 300, replace=False)))
    n, e, w = _isolated(rng)
    r = _resets(n, e, rng, hub=int(np.bincount(e.reshape(-1)).argmax()))
    for t in (0, 1, T):
        out.append(("isolated", n, e, w, r, 0.5, t, None))
    out.append(("isolated gathered", n, e, w, r, 0.5, T, rng.choice(n, 40, replace=False)))
    n, e, w = _ladder(rng)
    r = _resets(n, e, rng)
    for t in (1, T):
        out.append(("ladder", n, e, w, r, 0.5, t, None))
    for t in (0, 1, T):
        out.append(("n = 1", 1, np.zeros((0, 2), np.int64), np.zeros(0), np.ones((32, 1)), 0.5, t, None))
    return out


CASES = _cases()


def _run(exe, tmp_path, names, batches=BATCHES, interleavings=2):
    files = []
    for i, (name, n, e, w, r, d, T, sub) in enumerate(CASES):
        if name in names:
            path = tmp_path / f"case{i}.bin"
            _write_case(path, n, e, w, r, d, T, sub)
            files.append(str(path))
    assert files, names
    return subprocess.run([str(exe), batches, str(interleavings), *files], capture_output=True, text=True, timeout=3000)


def test_the_emulated_kernels_are_the_headers_ppr_cu_includes():
    ppr_cu = open(os.path.join(CSRC, "ppr.cu")).read()
    assert '#include "ppr_batch_kernels.cuh"' in ppr_cu
    assert '#include "ppr_batch_kernels.cuh"' in open(os.path.join(EMU, "ppr_batch_emu_test.cpp")).read()
    src = open(os.path.join(CSRC, "ppr_batch_kernels.cuh")).read()
    assert '#include "ppr_kernels.cuh"' in src
    for arch_only in ("wgmma_", "mbar_", "tma_load", "asm(", "atomicAdd", "atomicCAS"):
        assert arch_only not in src, arch_only


@pytest.mark.parametrize("names, batches, interleavings", [
    (("path", "path gathered", "path d=0.85"), BATCHES, 2),
    (("star", "star gathered"), "3,32", 1),                  # the largest graph: one width below and the widest
    (("isolated", "isolated gathered"), BATCHES, 2),
    (("ladder",), BATCHES, 2),
    (("n = 1",), BATCHES, 2),
], ids=["path", "star", "isolated", "ladder", "n=1"])
def test_batched_columns_equal_single_source_runs_bit_for_bit(emulator, tmp_path, names, batches, interleavings):
    proc = _run(emulator, tmp_path, set(names), batches, interleavings)
    assert proc.returncode == 0, proc.stdout + proc.stderr
    assert proc.stdout.strip().endswith("ALL OK")


@pytest.mark.parametrize("mutant, needle, repl, names, batches", [
    ("gather off by one column", "y[vtx * W + b]", "y[vtx * W + (b + 1) % W]", ("path gathered",), "3"),
    ("a row spanning chunks loses its earlier partial", "(continued ? s_open[b] : 0.f) + x[b]", "0.f + x[b]",
     ("path",), "2,8"),
    ("fix-up drops a row's last carry", "k < s; ++k", "k < s - 1; ++k", ("star",), "3"),
    ("every column normalised by column 0's total", "b] / totals[b];", "b] / totals[0];", ("isolated",), "3,8"),
])
def test_emulation_catches_mutant(tmp_path, mutant, needle, repl, names, batches):
    mutated = tmp_path / "csrc"
    mutated.mkdir()
    for h in os.listdir(CSRC):
        if h.endswith(".cuh"):
            shutil.copy(os.path.join(CSRC, h), mutated / h)
    src = (mutated / "ppr_batch_kernels.cuh").read_text()
    assert src.count(needle) == 1, needle
    (mutated / "ppr_batch_kernels.cuh").write_text(src.replace(needle, repl))
    exe = _build(mutated, tmp_path / "mutant")
    proc = _run(exe, tmp_path, set(names), batches=batches, interleavings=0)
    assert proc.returncode != 0 and "FAILED" in proc.stderr, f"{mutant}: {proc.stdout}"
