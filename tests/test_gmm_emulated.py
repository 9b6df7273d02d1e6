"""The kernels of crag_gmm_sweep (csrc/gmm_kernels.cuh) on the CPU.  The header holds no wgmma / TMA / mbarrier code,
so tests/warp_emu/gmm_emu_test.cpp compiles the very header gmm.cu includes and runs the whole sweep -- moments,
k-means++ seeding, Lloyd, EM, BIC and the winner's memberships -- on emulated blocks, once block after block and once
with every launch's blocks resident in a random interleaving; the two outputs must be bit-identical.  The output is
then checked against the float64 oracle (oracle/gmm_oracle.py, pinned to scikit-learn by tests/test_oracle_gmm.py):
k-means++ rows, k-means labels and iteration counts, EM iteration counts and the chosen n exactly, weights, means and memberships to
1e-9 relative and BIC to 1e-9 relative plus the rounding a near-singular covariance amplifies
(oracle.gmm_oracle.bic_tolerance).  That covers, through their outputs, the warp Cholesky and triangular inverse (means, BIC), the
Mahalanobis term and logsumexp (memberships), the chunk-order statistic reduction (bit-identity) and the k-means++
candidate pick (seeds).

The Lloyd loop also runs alone from given centres, some beyond every row, so that its first pass relocates empty
clusters (--lloyd), against the oracle's Lloyd.

Three mutants of the header must fail: a Lloyd loop that treats every stop as strict convergence (and so skips the
final assignment after a stop on the centre shift), an M-step without reg_covar (the duplicate rows make a
covariance singular), and a statistics reduction in which every chunk writes chunk 0's slot."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
from oracle import gmm_oracle as G  # noqa: E402

EMU = os.path.join(ROOT, "tests", "warp_emu")
CSRC = os.path.join(ROOT, "comorag_b200", "csrc")


def _build(csrc_dir, exe):
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unknown-pragmas", "-pthread", "-I",
                        os.path.join(EMU, "stub"), "-I", str(csrc_dir), os.path.join(EMU, "gmm_emu_test.cpp"), "-o",
                        str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def _mutant(tmp_path, needle, repl):
    mutated = tmp_path / "csrc"
    mutated.mkdir()
    for h in os.listdir(CSRC):
        if h.endswith(".cuh"):
            shutil.copy(os.path.join(CSRC, h), mutated / h)
    src = (mutated / "gmm_kernels.cuh").read_text()
    assert src.count(needle) == 1, needle
    (mutated / "gmm_kernels.cuh").write_text(src.replace(needle, repl))
    return _build(mutated, tmp_path / "mutant")


@pytest.fixture(autouse=True)
def _need_gxx():
    if shutil.which("g++") is None:
        pytest.skip("g++ not installed")


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return _build(CSRC, tmp_path_factory.mktemp("gmm_emu") / "gmm_emu_test")


def _write_case(path, X, M):
    X = np.ascontiguousarray(X, dtype=np.float64)
    first, draws = G.draws(len(X), M)
    with open(path, "wb") as f:
        np.asarray([len(X)], np.int64).tofile(f)
        np.asarray([X.shape[1], M], np.int32).tofile(f)
        X.tofile(f)
        first.astype(np.int64).tofile(f)
        np.asarray([draws.size], np.int64).tofile(f)
        draws.tofile(f)


def _read_out(path, n, d, M):
    raw = open(path, "rb").read()
    o, pos = {}, 0

    def take(name, dtype, count):
        nonlocal pos
        a = np.frombuffer(raw, dtype=dtype, count=count, offset=pos)
        pos += a.nbytes
        o[name] = a
    take("bic", np.float64, M)
    take("iters", np.int32, M)
    take("conv", np.int32, M)
    take("best", np.int32, 1)
    take("weights", np.float64, M)
    take("means", np.float64, M * d)
    k = int(o["best"][0])
    take("memb", np.float64, n * k)
    take("seeds", np.int32, M * (M + 1) // 2)
    take("labels", np.int32, M * n)
    take("lloyd_iters", np.int32, M)
    o["means"] = o["means"].reshape(M, d)
    o["memb"] = o["memb"].reshape(n, k)
    o["labels"] = o["labels"].reshape(M, n)
    return o


def _cases():
    rng = np.random.default_rng(0)
    c = rng.normal(0, 4, size=(3, 2))
    blobs = c[rng.integers(0, 3, 40)] + rng.normal(0, 0.5, size=(40, 2))
    dup = np.concatenate([blobs[:10]] * 3)                                  # duplicates: singular but for reg_covar
    shift_stop = np.random.default_rng(0).normal(size=(300, 2))           # m = 2 stops on the centre shift
    flat = np.concatenate([blobs, blobs]) @ np.array([[1.0, 0.0, 2.0], [0.0, 1.0, -1.0]])   # duplicates, rank 2 in 3-d
    line = rng.normal(size=(12, 1))
    return {"blobs": (blobs, 8), "duplicates": (dup, 12), "shift_stop": (shift_stop, 3), "rank_deficient": (flat, 6), "d1": (line, 5)}


def _run(exe, tmp_path, cases):
    args, outs = [], {}
    for name, (X, M) in cases.items():
        cp, op = tmp_path / f"{name}.bin", tmp_path / f"{name}.out"
        _write_case(cp, X, M)
        args += [str(cp), str(op)]
        outs[name] = op
    r = subprocess.run([str(exe)] + args, capture_output=True, text=True, timeout=1800)
    return r, outs


def _compare(X, M, o):
    """Decisions are compared where the oracle takes them with a relative margin above 1e-9 (a model seeded through
    an exact tie between two points is not),
    and the chosen n where every model is."""
    sw = G.sweep(X, M)
    decided = [mo.seed_margin > 1e-9 for mo in sw.models]
    for m, mo in enumerate(sw.models, start=1):
        if not decided[m - 1]:
            continue
        seeds = o["seeds"][m * (m - 1) // 2: m * (m + 1) // 2]       # as points: duplicate rows are the same seed
        np.testing.assert_array_equal(X[seeds], X[mo.seeds], err_msg=f"m={m}")
        np.testing.assert_array_equal(o["labels"][m - 1], mo.labels, err_msg=f"m={m}")
        assert int(o["lloyd_iters"][m - 1]) == mo.kmeans_iters, (m, o["lloyd_iters"][m - 1], mo.kmeans_iters)
        assert int(o["iters"][m - 1]) == mo.iters, (m, o["iters"][m - 1], mo.iters)
        assert bool(o["conv"][m - 1]) == mo.converged
        tol = G.bic_tolerance(mo, len(X), X.shape[1], 1e-9)
        assert abs(o["bic"][m - 1] - mo.bic) <= tol, (m, o["bic"][m - 1], mo.bic, tol)
    if not all(decided):
        return
    assert int(o["best"][0]) == sw.best
    k = sw.best
    mo = sw.models[k - 1]
    np.testing.assert_allclose(o["weights"][:k], mo.weights, rtol=1e-9)
    np.testing.assert_allclose(o["means"][:k], mo.means, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(o["memb"], sw.memberships, rtol=0, atol=1e-9)


def test_sweep_on_emulated_blocks_matches_the_oracle(emu, tmp_path):
    cases = _cases()
    r, outs = _run(emu, tmp_path, cases)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr
    for name, (X, M) in cases.items():
        _compare(X, M, _read_out(outs[name], len(X), X.shape[1], M))


def _fails(exe, tmp_path, cases):
    r, outs = _run(exe, tmp_path, cases)
    if r.returncode != 0:
        return True
    try:
        for name, (X, M) in cases.items():
            _compare(X, M, _read_out(outs[name], len(X), X.shape[1], M))
    except AssertionError:
        return True
    return False


def test_mutant_lloyd_without_strict_convergence_fails(tmp_path):
    # every stop counts as strict convergence, so a loop that ends on the centre shift skips its final assignment
    exe = _mutant(tmp_path, "if (changed == 0) st->lloyd_strict = 1;", "st->lloyd_strict = 1;")
    assert _fails(exe, tmp_path, {"shift_stop": _cases()["shift_stop"]})


def _lloyd(exe, tmp_path, X, centres):
    cp, op = tmp_path / "lloyd.bin", tmp_path / "lloyd.out"
    with open(cp, "wb") as f:
        np.asarray([len(X)], np.int64).tofile(f)
        np.asarray([X.shape[1], len(centres)], np.int32).tofile(f)
        np.ascontiguousarray(X, np.float64).tofile(f)
        np.ascontiguousarray(centres, np.float64).tofile(f)
    r = subprocess.run([str(exe), "--lloyd", str(cp), str(op)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = np.fromfile(op, dtype=np.uint8)
    n, m, d = len(X), len(centres), X.shape[1]
    labels = raw[:4 * n].view(np.int32)
    iters = int(raw[4 * n:4 * n + 4].view(np.int32)[0])
    return labels, iters, raw[4 * n + 4:].view(np.float64).reshape(m, d)


@pytest.mark.parametrize("far", [1, 2])
def test_lloyd_relocates_empty_clusters(emu, tmp_path, far):
    """Lloyd from given centres, `far` of them beyond every row: the first pass leaves them empty with every row off
    its centre, so each takes one of the farthest rows (_relocate_empty_clusters_dense).  Labels, iteration count
    and centres as the oracle's lloyd (scikit-learn's, tests/test_oracle_gmm.py)."""
    rng = np.random.default_rng(far)
    X = rng.normal(size=(60, 2)) * np.array([3.0, 1.0])
    Xc = X - X.mean(0)
    centres = np.concatenate([Xc[[3, 17, 40]], 50.0 + 10.0 * np.arange(far)[:, None] * np.ones((1, 2))])
    tol = np.var(X, axis=0).mean() * G.KMEANS_TOL
    labels, iters, got = _lloyd(emu, tmp_path, X, centres)
    want_labels, want_centres, want_iters, _ = G.lloyd(Xc, centres, tol)
    np.testing.assert_array_equal(labels, want_labels)
    assert iters == want_iters
    np.testing.assert_allclose(got, want_centres, rtol=1e-12, atol=1e-12)


def test_mutant_without_reg_covar_fails(tmp_path):
    exe = _mutant(tmp_path, "if (j == lane) v += kGmmRegCovar;", "")
    assert _fails(exe, tmp_path, {"duplicates": _cases()["duplicates"]})


def test_mutant_reduction_in_arrival_order_fails(tmp_path):
    # every chunk adds its statistics into chunk 0's slot as it finishes, instead of writing its own
    exe = _mutant(tmp_path, "double* part = esum + (int64_t(r) * comps + off) * S;",
                  "double* part = esum + (int64_t(0) * comps + off) * S;")
    X = np.random.default_rng(4).normal(size=(1500, 2))      # 6 row chunks
    assert _fails(exe, tmp_path, {"chunks": (X, 3)})
