"""The kernels of crag_ppr (csrc/ppr_kernels.cuh) on the CPU.  The header holds no wgmma / TMA / mbarrier code, so
tests/warp_emu/ppr_emu_test.cpp compiles the very header ppr.cu includes and runs plan, init, step, fix-up, sum and
gather on emulated blocks, once block after block and twice with all blocks resident in random interleavings; the
three outputs must be bit-identical.  The output is then held to the error bound of tests/ppr_bound.py against the
float64 oracle:

    |x_hat_p - x_p| <= num_p / s_lo + u (x_p + num_p / s_lo),  num_p = b_p + trunc + x_p (E + gamma_D (S + E)),
    b = (I - d A)^-1 (gamma_{deg + 3} (.) y*),  E = sum(b) + trunc,  s_lo = (S - E)(1 - gamma_D),

where gamma_{deg_i + 3} bounds the relative rounding of row i's deg_i + 1 nonnegative terms (each a product of
fp32-rounded factors), b carries it through the contraction, trunc = d^(T+1) is the truncation (0 against the exact
T-step iterate) and gamma_D the fixed-shape tree of the normalising sum (ppr_bound.py derives each term).

Calibration: the emulated fp32 arithmetic stays under half of the bound on every graph, and three mutants of the
header exceed it: a fix-up that drops a row's last carry, a step that skips empty rows, and a finalize that
normalises by the sum of the gathered outputs instead of all vertices."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import ppr_bound  # noqa: E402

from comorag_b200.graph import DeviceGraph, ppr_iterations  # noqa: E402

EMU = os.path.join(ROOT, "tests", "warp_emu")
CSRC = os.path.join(ROOT, "comorag_b200", "csrc")


def _build(csrc_dir, exe):
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unknown-pragmas", "-pthread", "-I", os.path.join(EMU, "stub"),
                        "-I", str(csrc_dir), os.path.join(EMU, "ppr_emu_test.cpp"), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def _mutant(tmp_path, needle, repl):
    mutated = tmp_path / "csrc"
    mutated.mkdir()
    for h in os.listdir(CSRC):
        if h.endswith(".cuh"):
            shutil.copy(os.path.join(CSRC, h), mutated / h)
    src = (mutated / "ppr_kernels.cuh").read_text()
    assert src.count(needle) == 1, needle
    (mutated / "ppr_kernels.cuh").write_text(src.replace(needle, repl))
    return _build(mutated, tmp_path / "mutant")


@pytest.fixture(autouse=True)
def _need_gxx():
    if shutil.which("g++") is None:
        pytest.skip("g++ not installed")


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
    """Pairs joined by one edge, an isolated vertex after every pair: rows of 2, 2 and 1 merge-path items, so over the
    segments of 512 items an empty row lands on every position next to a segment edge."""
    n = 3000
    trip = np.arange(0, n, 3)
    e = np.stack([trip, trip + 1], 1)
    return n, e, rng.uniform(0.5, 1.5, len(e))


def _reset(n, rng, isolated=None):
    r = rng.uniform(0.0, 1.0, n) * (rng.uniform(size=n) < 0.3)
    r[rng.integers(0, n)] = 1.0
    if isolated is not None:
        r[isolated] = 0.7            # reset mass on isolated vertices
    return r


def _write_case(path, n, edges, weights, reset, damping, iterations, out_vertices=None):
    g = DeviceGraph.from_edges(n, torch.as_tensor(np.asarray(edges, np.int64).reshape(-1, 2)), torch.as_tensor(weights),
                               device="cpu")
    v = g.reset_vector(reset).numpy()
    with open(path, "wb") as f:
        np.array([n, g.nnz, -1 if out_vertices is None else len(out_vertices), iterations], np.int64).tofile(f)
        np.array([damping], np.float32).tofile(f)
        g.row_ptr.numpy().astype(np.int64).tofile(f)
        g.col.numpy().astype(np.int32).tofile(f)
        g.coef.numpy().astype(np.float32).tofile(f)
        v.astype(np.float32).tofile(f)
        if out_vertices is not None:
            np.asarray(out_vertices, np.int32).tofile(f)


def _cases():
    rng = np.random.default_rng(20251016)
    out = []
    d_half = 0.5
    T_def = ppr_iterations(d_half)
    n, e, w = _path(700, rng)
    r = _reset(n, rng)
    sub = rng.choice(n, 100, replace=False)
    for T in (0, 1, T_def):
        out.append(("path", n, e, w, r, d_half, T, None))
    out.append(("path gathered", n, e, w, r, d_half, T_def, sub))
    d85 = float(np.float32(0.85))
    out.append(("path d=0.85", n, e, w, r, d85, ppr_iterations(d85), None))
    n, e, w = _star(120_000, rng)
    r = _reset(n, rng)
    r[-1500:] = 5.0          # heavy leaves at the end of the hub's row: its last carries hold most of its sum
    for T in (1, T_def):
        out.append(("star", n, e, w, r, d_half, T, None))
    n, e, w = _isolated(rng)
    r = _reset(n, rng, isolated=np.arange(70, 120, 7))
    for T in (0, 1, T_def):
        out.append(("isolated", n, e, w, r, d_half, T, None))
    out.append(("isolated gathered", n, e, w, r, d_half, T_def, rng.choice(n, 40, replace=False)))
    n, e, w = _ladder(rng)
    r = _reset(n, rng, isolated=np.arange(2, n, 3)[::5])
    for T in (1, T_def):
        out.append(("ladder", n, e, w, r, d_half, T, None))
    for T in (0, 1, T_def):
        out.append(("n = 1", 1, np.zeros((0, 2), np.int64), np.zeros(0), np.ones(1), d_half, T, None))
    return out


CASES = _cases()


def _run_cases(exe, tmp_path, names=None):
    """Run the emulator over the cases; returns {index: (out, x_ref, bound)}, or the failed process."""
    args, sel = [], []
    for i, (name, n, e, w, r, d, T, sub) in enumerate(CASES):
        if names is not None and name not in names:
            continue
        case, out = tmp_path / f"case{i}.bin", tmp_path / f"out{i}.bin"
        _write_case(case, n, e, w, r, d, T, sub)
        args += [str(case), str(out)]
        sel.append(i)
    proc = subprocess.run([str(exe), *args], capture_output=True, text=True, timeout=3000)
    if proc.returncode != 0:
        return proc
    res = {}
    for i in sel:
        name, n, e, w, r, d, T, sub = CASES[i]
        got = np.fromfile(tmp_path / f"out{i}.bin", dtype=np.float32).astype(np.float64)
        x, bnd = ppr_bound.bound(n, e, w, r, d, T, exact_iterate=T != ppr_iterations(d))
        if sub is not None:
            x, bnd = x[sub], bnd[sub]
        res[i] = (got, x, bnd)
    return res


def _ratio(got, x, bnd):
    """|got - x| / bound per entry (0 where both are exactly equal, e.g. unreachable vertices; inf for NaN)."""
    err = np.abs(got - x)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(err == 0, 0.0, err / bnd)


def _worst(res):
    """max over every case and entry of |got - x| / bound (inf for NaN)."""
    worst = 0.0
    for got, x, bnd in res.values():
        ratio = _ratio(got, x, bnd)
        worst = max(worst, float(np.nanmax(np.where(np.isfinite(ratio), ratio, np.inf))))
    return worst


def test_the_emulated_kernels_are_the_header_ppr_cu_includes():
    assert '#include "ppr_kernels.cuh"' in open(os.path.join(CSRC, "ppr.cu")).read()
    assert '#include "ppr_kernels.cuh"' in open(os.path.join(EMU, "ppr_emu_test.cpp")).read()
    src = open(os.path.join(CSRC, "ppr_kernels.cuh")).read()
    for arch_only in ("wgmma_", "mbar_", "tma_load", "asm(", "atomicAdd", "atomicCAS"):
        assert arch_only not in src, arch_only


def test_ppr_kernels_on_emulated_blocks_within_half_the_bound(tmp_path):
    """Path (T in {0, 1, default}, d = 0.5 and 0.85, a gathered subset), a star whose hub spans ~235 segments,
    isolated vertices with reset mass, empty rows at every position next to a segment edge, and n = 1."""
    exe = _build(CSRC, tmp_path / "ppr_emu_test")
    res = _run_cases(exe, tmp_path)
    assert not isinstance(res, subprocess.CompletedProcess), res.stdout + res.stderr
    for i, (got, x, bnd) in res.items():
        name, T = CASES[i][0], CASES[i][6]
        ratio = _ratio(got, x, bnd)
        assert np.isfinite(got).all(), name
        assert ratio.max() <= 0.5, f"{name} T={T}: error {ratio.max():.3f} of the bound"
        if CASES[i][7] is None:
            assert abs(got.sum() - 1.0) < 1e-5, name


@pytest.mark.parametrize("mutant, needle, repl, cases", [
    ("fix-up drops a row's last carry", "k < s; ++k", "k < s - 1; ++k", ["star"]),
    ("step skips empty rows", "    else y_out[x0 + i] =", "    else if (row_ptr[x0 + i + 1] > row_ptr[x0 + i]) y_out[x0 + i] =",
     ["isolated", "ladder"]),
    ("finalize normalises by the gathered outputs", "const float total = ppr_block_sum(acc, s_red);",
     "const float total = ppr_block_sum(p < n_out ? y[out_vertices ? out_vertices[p] : p] : 0.f, s_red);",
     ["path gathered", "isolated gathered"]),
])
def test_emulation_catches_mutant(tmp_path, mutant, needle, repl, cases):
    exe = _mutant(tmp_path, needle, repl)
    res = _run_cases(exe, tmp_path, names=set(cases))
    if isinstance(res, subprocess.CompletedProcess):
        assert "FAILED" in res.stderr, res.stdout + res.stderr
        return
    assert _worst(res) > 1.0, mutant
