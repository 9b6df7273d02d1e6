"""The kernels of crag_umap_* (csrc/umap_kernels.cuh) on the CPU.  The header holds no wgmma / TMA code, so
tests/warp_emu/umap_emu_test.cpp compiles the very header umap.cu includes and runs each stage -- the fuzzy graph,
the spectral start, layout epochs -- on emulated blocks, once block after block and once in a random interleaving;
the two outputs must be bit-identical.  Then against the float64 oracle (tests/umap_oracle.py):

* fuzzy graph: lists and distances exactly, rho exactly, sigma within 1e-5 relative (the bisection's sums run in
  another order), memberships within 2e-6;
* spectral start: Ritz values within 1e-9, the span of the Ritz vectors within 1e-6 rad, the start layout within
  2e-5 of the oracle's post-processing of the emulated vectors;
* epochs: per epoch, each vertex within 2^-14 per update step (two attractions per due edge plus its negative
  samples) + 1e-4, a calibrated bound (the worst vertex seen uses under a third of it), except vertices with a snapshot point within d^2 < 1e-2, where the fp32 / fp64 difference of d^2
  is amplified by the repulsion's 1 / (0.001 + d^2) and only the clip bounds a step.

Three mutants of the header must fail: the epoch kernel reading the buffer it writes (interleaving-dependent), a
negative sample that hits i itself not being skipped, and rho taken from the search's self entry."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import umap_oracle as U  # noqa: E402

EMU = os.path.join(ROOT, "tests", "warp_emu")
CSRC = os.path.join(ROOT, "comorag_b200", "csrc")
SEED = 224


def _build(csrc_dir, exe):
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wno-unknown-pragmas", "-pthread", "-I",
                        os.path.join(EMU, "stub"), "-I", str(csrc_dir), os.path.join(EMU, "umap_emu_test.cpp"), "-o",
                        str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def _mutant(tmp_path, needle, repl):
    mutated = tmp_path / "csrc"
    mutated.mkdir()
    for h in os.listdir(CSRC):
        if h.endswith(".cuh"):
            shutil.copy(os.path.join(CSRC, h), mutated / h)
    src = (mutated / "umap_kernels.cuh").read_text()
    assert src.count(needle) == 1, needle
    (mutated / "umap_kernels.cuh").write_text(src.replace(needle, repl))
    return _build(mutated, tmp_path / "mutant")


@pytest.fixture(autouse=True)
def _need_gxx():
    if shutil.which("g++") is None:
        pytest.skip("g++ not installed")


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return _build(CSRC, tmp_path_factory.mktemp("umap_emu") / "umap_emu_test")


def _run(exe, mode, case, out):
    return subprocess.run([str(exe), mode, str(case), str(out)], capture_output=True, text=True, timeout=600)


def _lists(n, dim, k, seed, dup=0):
    X, labels = U.planted(n, dim, 4, seed=seed, spread=0.6)
    if dup:
        X[n - dup:] = X[:dup]
    Xb = U.bf16_rows(X)
    S = (Xb @ Xb.T).astype(np.float32)
    return U.topk_lists(S, k)


# ------------------------------------------------------------------------------------------------- fuzzy graph
def _fuzzy(exe, tmp_path, ids, sc):
    n, k = ids.shape
    case, out = tmp_path / "fuzzy.bin", tmp_path / "fuzzy.out"
    with open(case, "wb") as f:
        np.asarray([n], np.int64).tofile(f)
        np.asarray([k], np.int32).tofile(f)
        ids.astype(np.int64).tofile(f)
        sc.astype(np.float32).tofile(f)
    r = _run(exe, "--fuzzy", case, out)
    assert r.returncode == 0, r.stdout + r.stderr
    raw = open(out, "rb").read()
    pos = 0

    def take(dtype, count):
        nonlocal pos
        a = np.frombuffer(raw, dtype=dtype, count=count, offset=pos)
        pos += a.nbytes
        return a
    nbr = take(np.int32, n * k).reshape(n, k)
    dist = take(np.float32, n * k).reshape(n, k)
    rho, sigma = take(np.float32, n), take(np.float32, n)
    return nbr, dist, rho, sigma, take(np.float32, n * k).reshape(n, k)


def _check_fuzzy(got, ids, sc):
    nbr, dist, rho, sigma, memb = got
    want_nbr, want_dist = U.knn_lists(ids, sc)
    np.testing.assert_array_equal(nbr, want_nbr)
    np.testing.assert_array_equal(dist, want_dist)
    o_rho, o_sigma, _ = U.smooth_knn(dist)
    np.testing.assert_array_equal(rho, o_rho)
    np.testing.assert_allclose(sigma, o_sigma, rtol=1e-5, atol=0)
    np.testing.assert_allclose(memb, U.memberships(nbr, dist, rho, sigma.astype(np.float64)), rtol=0, atol=2e-6)


@pytest.mark.parametrize("n,k,dup", [(150, 15, 10), (70, 40, 0), (40, 39, 3)])
def test_fuzzy_graph(emu, tmp_path, n, k, dup):
    ids, sc = _lists(n, 64, k, seed=n, dup=dup)
    # a list in which the search did not return the row itself: the last entry is dropped
    ids[5] = np.concatenate([ids[5][ids[5] != 5], [ids[5][-1]]])[:k] if 5 in ids[5] else ids[5]
    ids[5][ids[5] == 5] = (ids[5].max() + 1) % n
    _check_fuzzy(_fuzzy(emu, tmp_path, ids, sc), ids, sc)


def test_mutant_rho_from_the_self_entry_fails(tmp_path):
    exe = _mutant(tmp_path, "if (q < k) self_d = 0.0f;", "if (q < k) self_d = fmaxf(0.0f, 1.0f - sc[q]);")
    ids, sc = _lists(150, 64, 15, seed=1)
    assert (sc[ids == np.arange(150)[:, None]] < 1).any()
    with pytest.raises(AssertionError):
        _check_fuzzy(_fuzzy(exe, tmp_path, ids, sc), ids, sc)


# ---------------------------------------------------------------------------------------------- spectral start
def _graph(n, k, seed, clusters=4, spread=1.2):
    X, _ = U.planted(n, 64, clusters, seed=seed, spread=spread)
    Xb = U.bf16_rows(X)
    ids, sc = U.topk_lists((Xb @ Xb.T).astype(np.float32), k)
    nbr, dist = U.knn_lists(ids, sc)
    rho, sigma, _ = U.smooth_knn(dist)
    return U.fuzzy_union(nbr, U.memberships(nbr, dist, rho, sigma), 500)


@pytest.mark.parametrize("n,d,iters", [(400, 3, 60), (2500, 10, 20), (12, 10, 5), (17, 15, 4)])
def test_spectral_start(emu, tmp_path, n, d, iters):
    ip, ix, w, eps = _graph(n, min(15, n - 1), seed=1)
    case, out = tmp_path / "spec.bin", tmp_path / "spec.out"
    with open(case, "wb") as f:
        np.asarray([n, len(ix)], np.int64).tofile(f)
        np.asarray([d, iters], np.int32).tofile(f)
        np.asarray([SEED], np.uint64).tofile(f)
        ip.tofile(f)
        ix.tofile(f)
        w.tofile(f)
    r = _run(emu, "--spectral", case, out)
    assert r.returncode == 0, r.stdout + r.stderr
    p = U.n_columns(n, d)
    raw = open(out, "rb").read()
    y = np.frombuffer(raw, np.float32, n * d).reshape(n, d)
    vec = np.frombuffer(raw, np.float64, n * d, offset=4 * n * d).reshape(n, d)
    vals = np.frombuffer(raw, np.float64, p, offset=12 * n * d)
    want, wvals = U.spectral_subspace(ip, ix, w, d, iters, SEED)
    np.testing.assert_allclose(vals, wvals, rtol=0, atol=1e-9)
    # near-degenerate Ritz values leave the individual vectors free to rotate: compare the subspace
    assert U.principal_angle(vec, want) <= 1e-6
    np.testing.assert_allclose(y, U.post(vec, SEED), rtol=0, atol=2e-5)
    assert y.min() == 0 and np.isclose(y.max(axis=0), 10, atol=1e-5).all()


# ------------------------------------------------------------------------------------------------------ epochs
def _epoch_case(path, ip, ix, eps, ns, nn, y, n_epochs, e0, e1, a, b):
    n, d = y.shape
    with open(path, "wb") as f:
        np.asarray([n, len(ix)], np.int64).tofile(f)
        np.asarray([d, n_epochs, e0, e1], np.int32).tofile(f)
        np.asarray([SEED], np.uint64).tofile(f)
        np.asarray([a, b], np.float32).tofile(f)
        ip.tofile(f)
        ix.tofile(f)
        eps.tofile(f)
        ns.tofile(f)
        nn.tofile(f)
        y.astype(np.float32).tofile(f)


def _epochs(exe, tmp_path, n=120, epochs=(0, 1, 6)):
    """Per epoch e: (device y, oracle y, per-vertex bound, near-coincident mask) from the oracle's state at e."""
    ip, ix, w, eps = _graph(n, 10, seed=7, clusters=3, spread=1.0)
    a, b = U.find_ab_params()
    Yr, _ = U.spectral_subspace(ip, ix, w, 3, 40, SEED)
    y = U.post(Yr, SEED)
    ns, nn = U.schedule(eps)
    results = []
    n_epochs = 200
    for e in range(max(epochs) + 1):
        if e in epochs:
            case, out = tmp_path / f"ep{e}.bin", tmp_path / f"ep{e}.out"
            snap = y.astype(np.float32)
            _epoch_case(case, ip, ix, eps, ns, nn, snap, n_epochs, e, e + 1, a, b)
            r = _run(exe, "--epochs", case, out)
            assert r.returncode == 0, r.stdout + r.stderr
            got = np.frombuffer(open(out, "rb").read(), np.float32, n * 3).reshape(n, 3)
            due = ns <= e
            n_neg = np.where(due, np.floor((e - nn) / (eps / 5.0)), 0)
            steps = np.zeros(n)
            np.add.at(steps, np.repeat(np.arange(n), np.diff(ip)), np.where(due, 2 + n_neg, 0))
            diff = snap[:, None, :].astype(np.float64) - snap[None, :, :]
            d2 = (diff ** 2).sum(-1) + np.eye(n) * 1e9
            close = (d2 < 1e-2).any(axis=1)
            ns_o, nn_o = ns.copy(), nn.copy()
            want = U.epoch(ip, ix, eps, snap, ns_o, nn_o, e, n_epochs, a, b, SEED)
            results.append((got, want, steps * 2.0 ** -14 + 1e-4, close))
        y = U.epoch(ip, ix, eps, y.astype(np.float32), ns, nn, e, n_epochs, a, b, SEED)
    return results


def _check_epochs(results):
    for got, want, bound, close in results:
        err = np.abs(got.astype(np.float64) - want).max(axis=1)
        assert not ((err > bound) & ~close).any(), (err / bound).max()


def test_epochs(emu, tmp_path):
    _check_epochs(_epochs(emu, tmp_path))


def test_mutant_epoch_reads_the_buffer_it_writes_fails(tmp_path):
    exe = _mutant(tmp_path, "const float* snap = prev;", "const float* snap = next;")
    with pytest.raises(AssertionError, match="interleavings"):
        _epochs(exe, tmp_path)


def test_mutant_negative_sample_hitting_i_fails(tmp_path):
    exe = _mutant(tmp_path, "if (kk == i) continue;", "")
    with pytest.raises(AssertionError):
        _check_epochs(_epochs(exe, tmp_path, n=40, epochs=(0, 1)))
