"""crag_gmm_sweep on the device against the float64 oracle (oracle/gmm_oracle.py, itself pinned to scikit-learn by
tests/test_oracle_gmm.py), fed the same host-made draws.

Decisions -- the k-means++ rows, the final k-means labels, the EM iteration counts and the chosen n -- must be
identical wherever the oracle decides with a margin above the bound below; continuous outputs (BIC, weights, means,
memberships) are held to a relative tolerance.

Bound.  Device and oracle run the same float64 algorithm and differ only in the order of their sums and in how a
distance or a log-density is expanded (x.c expansion and X P - mu P in the oracle, direct differences on the
device).  Each such sum of n terms carries a relative error of at most gamma_n = n u / (1 - n u) (u = 2^-53), so a
quantity built from a few of them differs by a few gamma_n between the two, far below 1e-9 for n <= 5e4 (gamma_5e4
~ 5.6e-12).  EM amplifies that difference by at most its contraction per step; on the cases below the measured
spread between the two is ~1e-12 relative (a calibration run printed it), so a margin of 1e-6 -- relative to the
quantity compared -- leaves six orders of magnitude.  Margins:
  * chosen n: the BIC gap between the best and the second-best model, relative to |BIC_best|;
  * EM iterations: min over the iterations checked of ||lower bound change| - 1e-3|, relative to 1e-3 (per model);
  * k-means++ rows: the smallest distance of a scaled draw from a running-sum value, and of the chosen candidate's
    potential from another row's, relative to the potential (oracle.gmm_oracle.kmeans_plusplus(margin=True));
  * k-means labels: the smallest gap between a row's nearest and second-nearest final centre, relative to the
    mean squared distance (per model).
A model whose seeding or label margin falls below the bound is not compared (nor, then, the chosen n); one whose
lower-bound margin does is compared on everything but its iteration count.
"""
import os
import sys

import numpy as np
import pytest
import torch
from scipy.special import logsumexp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from comorag_b200 import _native  # noqa: E402
from comorag_b200.cluster import gmm_sweep, seed_draws  # noqa: E402
from oracle import gmm_oracle as G  # noqa: E402

pytestmark = pytest.mark.gpu
MARGIN = 1e-6
CONT_TOL = 1e-8


def _mixture(rng, n, d, k, spread, scale=1.0):
    centres = rng.normal(0, spread, size=(k, d))
    lab = rng.integers(0, k, n)
    return centres[lab] + rng.normal(0, scale, size=(n, d))


def _lb_margin(X, mo_m):
    """Smallest distance of |lower bound change| from the tolerance over the EM loop of the oracle's model."""
    X = np.asarray(X, np.float64)
    n = len(X)
    resp = np.zeros((n, mo_m.weights.size))
    resp[np.arange(n), mo_m.labels] = 1.0
    nk, means, prec = G._m_step(X, resp)
    weights = nk / n
    lb, worst = -np.inf, np.inf
    for _ in range(mo_m.iters):
        wlp = G.weighted_log_prob(X, weights, means, prec)
        lpn = logsumexp(wlp, axis=1)
        nk, means, prec = G._m_step(X, np.exp(wlp - lpn[:, None]))
        weights = nk / nk.sum()
        new = lpn.mean()
        if np.isfinite(lb):
            worst = min(worst, abs(abs(new - lb) - G.EM_TOL) / G.EM_TOL)
        lb = new
    return worst


def _label_margin(X, labels):
    Xc = X - X.mean(0)
    m = labels.max() + 1
    c = np.stack([Xc[labels == k].mean(0) if (labels == k).any() else np.full(X.shape[1], np.inf) for k in range(m)])
    if m == 1:
        return np.inf
    d2 = ((Xc[:, None, :] - c[None]) ** 2).sum(-1)
    s = np.sort(d2, axis=1)
    return float((s[:, 1] - s[:, 0]).min() / max(d2[np.isfinite(d2)].mean(), 1e-300))


def _check(X, M, models=None, expect_n=None):
    X = np.asarray(X)
    Xd = X.astype(np.float64)
    r = gmm_sweep(X, M, keep_kmeans=True)
    first, seed = G.draws(len(X), M)
    offs = np.concatenate([[0], np.cumsum([(m - 1) * G.trials(m) for m in range(1, M + 1)])])
    ms = range(1, M + 1) if models is None else sorted(set(models) | {r.n_components})
    fitted, decided = {}, {}
    for m in ms:
        mo = G.fit(Xd, m, first[m - 1], seed[offs[m - 1]:offs[m]])
        fitted[m] = mo
        tag = f"m={m}"
        decided[m] = mo.seed_margin > MARGIN and (_label_margin(Xd, mo.labels) > MARGIN or m == 1)
        if decided[m]:
            seeds = r.seeds[m * (m - 1) // 2: m * (m + 1) // 2]     # as points: duplicate rows are the same seed
            np.testing.assert_array_equal(Xd[seeds], Xd[mo.seeds], err_msg=tag)
            np.testing.assert_array_equal(r.labels[m - 1], mo.labels, err_msg=tag)
            if _lb_margin(Xd, mo) > MARGIN:
                assert int(r.iterations[m - 1]) == mo.iters, (tag, r.iterations[m - 1], mo.iters)
                assert bool(r.converged[m - 1]) == mo.converged, tag
            tol = G.bic_tolerance(mo, len(X), X.shape[1], CONT_TOL)
            assert abs(r.bic[m - 1] - mo.bic) <= tol, (tag, r.bic[m - 1], mo.bic, tol)
    if models is None:
        bics = np.array([fitted[m].bic for m in ms])
        order = np.argsort(bics, kind="stable")
        gap = (bics[order[1]] - bics[order[0]]) / abs(bics[order[0]]) if M > 1 else np.inf
        if gap > MARGIN and all(decided.values()):
            assert r.n_components == int(order[0]) + 1, (r.n_components, int(order[0]) + 1)
    if expect_n is not None:
        assert r.n_components == expect_n
    k = r.n_components
    mo = fitted[k]
    np.testing.assert_allclose(r.weights, mo.weights, rtol=CONT_TOL, atol=1e-12)
    np.testing.assert_allclose(r.means, mo.means, rtol=CONT_TOL, atol=CONT_TOL * np.abs(mo.means).max())
    np.testing.assert_allclose(r.memberships, G.memberships(Xd, mo), rtol=0, atol=1e-8)
    return r


@pytest.mark.parametrize("n,d,M", [(3, 1, 2), (12, 2, 11), (13, 2, 12), (13, 16, 12), (200, 10, 50), (200, 1, 50),
                                   (200, 16, 64), (64, 2, 1)])
def test_sweep_matches_oracle_small(n, d, M):
    rng = np.random.default_rng(n * 100 + d)
    _check(_mixture(rng, n, d, 4, 3.0), M)


@pytest.mark.parametrize("n,d,M,k", [(5000, 10, 50, 5), (5000, 16, 64, 3), (50000, 10, 50, 6), (50000, 2, 2, 2)])
def test_well_separated_mixture_finds_its_n(n, d, M, k):
    rng = np.random.default_rng(n + d)
    X = _mixture(rng, n, d, k, 30.0)
    _check(X, M, models=[1, 2, k, M], expect_n=k)


def test_overlapping_mixture():
    rng = np.random.default_rng(7)
    _check(_mixture(rng, 2000, 2, 6, 1.5), 50, models=[1, 2, 3, 7, 20, 50])


def test_duplicates_and_rank_deficient_rows():
    """Rows on a 3-d subspace of R^10, each row twice: every covariance is singular but for reg_covar."""
    rng = np.random.default_rng(11)
    base = _mixture(rng, 150, 3, 3, 4.0) @ rng.normal(size=(3, 10))
    X = np.concatenate([base, base])
    _check(X, 20)


def test_more_components_than_distinct_points():
    """19 rows on 5 points: the 6-component model has an empty cluster, which scikit-learn relocates
    (oracle.gmm_oracle.relocation_layout).  Its sixth seed is rounding noise (margin 0), so that model and the chosen
    n are not compared; the relocation itself is pinned on emulated blocks (tests/test_gmm_emulated.py)."""
    X, m = _relocation_layout()
    _check(X, m)


def _relocation_layout():
    return G.relocation_layout(), 6


def test_float32_input():
    rng = np.random.default_rng(5)
    X = _mixture(rng, 500, 10, 4, 5.0).astype(np.float32)
    r = _check(X, 30)
    assert r.memberships.dtype == np.float64


def test_bit_identical_on_two_streams():
    rng = np.random.default_rng(3)
    X = _mixture(rng, 3000, 10, 5, 2.0)
    a = gmm_sweep(X, 50, keep_kmeans=True)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        b = gmm_sweep(X, 50, keep_kmeans=True, stream=s)
    for f in ("bic", "iterations", "converged", "weights", "means", "memberships", "seeds", "labels"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f
    assert a.bic.tobytes() == b.bic.tobytes() and a.memberships.tobytes() == b.memberships.tobytes()


def test_argument_errors():
    lib = _native.load()
    dev = torch.device("cuda")
    n, d, M = 100, 4, 10
    x = torch.zeros(n, d, dtype=torch.float64, device=dev)
    first = torch.zeros(M, dtype=torch.int64, device=dev)
    draws = torch.zeros(1000, dtype=torch.float64, device=dev)
    f = torch.zeros(n * M, dtype=torch.float64, device=dev)
    i = torch.zeros(M, dtype=torch.int32, device=dev)
    wsb = lib.crag_gmm_sweep_workspace_bytes(n, d, M)
    assert wsb > 0
    ws = torch.zeros(wsb + 512, dtype=torch.uint8, device=dev)
    base = ws.data_ptr() + (-ws.data_ptr()) % 256

    def call(n=n, d=d, M=M, x=x.data_ptr(), first=first.data_ptr(), draws=draws.data_ptr(), out=f.data_ptr(),
             ws=base, wsb=wsb):
        return lib.crag_gmm_sweep(x, n, d, M, first, draws, out, i.data_ptr(), i.data_ptr(), i.data_ptr(), out, out, out,
                                  None, None, ws, wsb, None)

    for kw, word in [(dict(n=1), "n out of range"), (dict(d=0), "d must be"), (dict(d=17), "d must be"),
                     (dict(M=0), "max_components"), (dict(M=65), "max_components"), (dict(n=5, M=5), "max_components"),
                     (dict(x=None), "null pointer"), (dict(first=None), "null pointer"), (dict(draws=None), "null pointer"),
                     (dict(out=None), "null pointer"), (dict(ws=None), "null pointer"),
                     (dict(ws=base + 8), "256-byte aligned"), (dict(wsb=wsb - 1), "workspace")]:
        rc = call(**kw)
        assert rc != 0, kw
        assert word in lib.crag_last_error().decode(), (kw, lib.crag_last_error())
    torch.cuda.synchronize()
    for bad in [(1, 4, 1), (10, 0, 2), (10, 17, 2), (10, 4, 10), (100, 4, 65)]:
        assert lib.crag_gmm_sweep_workspace_bytes(*bad) == 0
    with pytest.raises(ValueError, match="d = 17"):
        gmm_sweep(np.zeros((20, 17)), 3)
    with pytest.raises(ValueError, match="max_components"):
        gmm_sweep(np.zeros((20, 3)), 20)


def test_seed_draws_match_the_oracle():
    a, b = seed_draws(500, 64)
    c, e = G.draws(500, 64)
    assert np.array_equal(a, c) and np.array_equal(b, e)
