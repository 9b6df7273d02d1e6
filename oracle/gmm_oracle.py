"""Float64 numpy restatement of the BIC sweep behind ComoRAG's soft clustering (cluster_utils.py:175-189, 252-260):
for m = 1..M, scikit-learn's GaussianMixture(n_components=m, covariance_type="full", random_state=224) -- KMeans
(k-means++ seeding, Lloyd) then EM -- and its BIC.  It is fed the host-made random draws (`draws`) that the device
sweep takes, and follows scikit-learn's own arithmetic where that decides a discrete choice (the seeding's
distance expansion and running sum, Lloyd's ||c||^2 - 2 x.c, the empty-cluster relocation and placement), so that
tests/test_oracle_gmm.py can pin it to the installed scikit-learn.  DESIGN.md section 2b."""
from __future__ import annotations

from dataclasses import dataclass
from typing import List

import numpy as np
from scipy import linalg
from scipy.special import logsumexp

REG_COVAR = 1e-6
EM_TOL = 1e-3
EM_MAX_ITER = 100
KMEANS_TOL = 1e-4
KMEANS_MAX_ITER = 300

def relocation_layout() -> np.ndarray:
    """19 rows, copies of 5 points in the plane, on which scikit-learn's Lloyd relocates an empty cluster in the
    6-component model.  With k-means++ seeds an empty cluster needs more seeds than distinct points, and then the
    sixth seed is picked by the rounding noise of the expanded distances (kmeans_plusplus's margin is 0), so the
    device need not pick the same one; the layout pins the oracle's relocation to scikit-learn's."""
    rng = np.random.default_rng(1)
    k, d = int(rng.integers(3, 9)), int(rng.integers(1, 3))
    base = rng.normal(0, 1, size=(k, d)) * rng.choice([0.1, 1, 10], size=(k, 1))
    return np.concatenate([base, base[rng.integers(0, k, int(rng.integers(k + 2, 16)))]])


def trials(m: int) -> int:
    return 2 + int(np.log(m))


def draws(n: int, max_components: int, random_state: int = 224):
    """(first_centre int64 [M], seed_draws fp64 [sum_m (m - 1) trials(m)]): what a fresh RandomState(random_state)
    yields, model by model, to _kmeans_plusplus with unit sample weights."""
    first, rest = [], []
    w = np.ones(n, dtype=np.float64)
    for m in range(1, max_components + 1):
        rs = np.random.RandomState(random_state)
        first.append(rs.choice(n, p=w / w.sum()))
        for _ in range(1, m):
            rest.append(rs.uniform(size=trials(m)))
    seed = np.concatenate(rest) if rest else np.zeros(0)
    return np.asarray(first, dtype=np.int64), seed.astype(np.float64)


def _sq_dist(A, X, x_sq):
    d = -2.0 * (A @ X.T)
    d += np.einsum("ij,ij->i", A, A)[:, None]
    d += x_sq[None, :]
    return np.maximum(d, 0.0)


def kmeans_plusplus(Xc: np.ndarray, m: int, first: int, u: np.ndarray, margin: bool = False):
    """Row indices of the m seeds; u = the model's (m - 1) x trials(m) draws.  With margin=True also the smallest
    relative distance of a decision from flipping: of a scaled draw from a running-sum value, and of the chosen
    candidate's potential from a different point's (a tie between two points is decided by rounding alone); 0 once
    the potential has fallen to rounding noise, as when every distinct point is already a seed."""
    n = Xc.shape[0]
    x_sq = np.einsum("ij,ij->i", Xc, Xc)
    idx = [int(first)]
    closest = _sq_dist(Xc[[first]], Xc, x_sq)[0]
    pot = closest.sum()
    u = np.asarray(u).reshape(max(m - 1, 0), trials(m))
    worst, pot0 = np.inf, pot
    for c in range(1, m):
        cs = np.cumsum(closest)
        v = u[c - 1] * pot
        cand = np.searchsorted(cs, v)
        np.clip(cand, None, n - 1, out=cand)
        dc = np.minimum(closest, _sq_dist(Xc[cand], Xc, x_sq))
        pots = dc.sum(axis=1)
        b = int(np.argmin(pots))
        if margin and pot <= 1e-9 * pot0:
            worst = 0.0     # every row (nearly) on a seed: the potential and the draw's row are rounding noise
        elif margin:
            worst = min(worst, float(np.abs(cs[None, :] - v[:, None]).min() / pot))
            other = pots[(Xc[cand] != Xc[cand[b]]).any(axis=1)]     # a duplicate of the chosen row is the same seed
            if other.size:
                worst = min(worst, float((other.min() - pots[b]) / pot))
        pot, closest = pots[b], dc[b]
        idx.append(int(cand[b]))
    idx = np.asarray(idx, dtype=np.int64)
    return (idx, worst) if margin else idx


def lloyd(Xc: np.ndarray, centres: np.ndarray, tol: float):
    """scikit-learn's _kmeans_single_lloyd (unit weights): (labels, centres, iterations, strict)."""
    n, d = Xc.shape
    m = centres.shape[0]
    centres = centres.copy()
    labels_old = np.full(n, -1, dtype=np.int64)
    strict = False

    def assign(c):
        dd = (c * c).sum(axis=1)[None, :] - 2.0 * (Xc @ c.T)
        return np.argmin(dd, axis=1)

    for it in range(KMEANS_MAX_ITER):
        labels = assign(centres)
        sums = np.zeros((m, d))
        np.add.at(sums, labels, Xc)
        w = np.bincount(labels, minlength=m).astype(np.float64)
        empty = np.where(w == 0)[0]
        if len(empty):
            dist = ((Xc - centres[labels]) ** 2).sum(axis=1)
            far = np.argpartition(dist, -len(empty))[:-len(empty) - 1:-1]
            if dist.max() > 0:                # every row on its centre (duplicates): no relocation
                for e, i in zip(empty, far):
                    old = labels[i]
                    sums[old] -= Xc[i]
                    sums[e] = Xc[i]
                    w[e] = 1.0
                    w[old] -= 1.0
        new = sums.copy()
        big = int(np.argmax(w))
        for k in range(m):                    # in order: an empty cluster before `big` takes big's unscaled sum
            new[k] = new[k] * (1.0 / w[k]) if w[k] > 0 else new[big]
        shift = (np.sqrt(((new - centres) ** 2).sum(axis=1)) ** 2).sum()
        centres = new
        if np.array_equal(labels, labels_old):
            strict = True
            break
        if shift <= tol:
            break
        labels_old = labels
    if not strict:
        labels = assign(centres)
    return labels, centres, it + 1, strict


def _chol_prec(cov):
    out = np.empty_like(cov)
    for k, c in enumerate(cov):
        L = linalg.cholesky(c, lower=True)
        out[k] = linalg.solve_triangular(L, np.eye(c.shape[0]), lower=True).T
    return out


def _m_step(X, resp):
    nk = resp.sum(axis=0) + 10 * np.finfo(np.float64).eps
    means = resp.T @ X / nk[:, None]
    cov = np.empty((len(nk), X.shape[1], X.shape[1]))
    for k in range(len(nk)):
        diff = X - means[k]
        cov[k] = (resp[:, k] * diff.T) @ diff / nk[k]
        cov[k].flat[:: X.shape[1] + 1] += REG_COVAR
    return nk, means, _chol_prec(cov)


def weighted_log_prob(X, weights, means, prec_chol):
    d = X.shape[1]
    log_det = np.log(np.stack([np.diag(p) for p in prec_chol])).sum(axis=1)
    lp = np.empty((X.shape[0], len(weights)))
    for k, (mu, p) in enumerate(zip(means, prec_chol)):
        y = X @ p - mu @ p
        lp[:, k] = (y * y).sum(axis=1)
    return -0.5 * (d * np.log(2 * np.pi) + lp) + log_det + np.log(weights)


@dataclass
class Model:
    seeds: np.ndarray
    labels: np.ndarray
    kmeans_iters: int
    weights: np.ndarray
    means: np.ndarray
    prec_chol: np.ndarray
    iters: int
    converged: bool
    bic: float
    seed_margin: float = np.inf   # kmeans_plusplus(margin=True)


def fit(X: np.ndarray, m: int, first: int, u: np.ndarray) -> Model:
    X = np.asarray(X, dtype=np.float64)
    n, d = X.shape
    tol = np.var(X, axis=0).mean() * KMEANS_TOL
    Xc = X - X.mean(axis=0)
    seeds, seed_margin = kmeans_plusplus(Xc, m, first, u, margin=True)
    labels, _, k_it, _ = lloyd(Xc, Xc[seeds], tol)
    resp = np.zeros((n, m))
    resp[np.arange(n), labels] = 1.0
    nk, means, prec = _m_step(X, resp)
    weights = nk / n
    lb, converged = -np.inf, False
    for it in range(1, EM_MAX_ITER + 1):
        prev = lb
        wlp = weighted_log_prob(X, weights, means, prec)
        lpn = logsumexp(wlp, axis=1)
        resp = np.exp(wlp - lpn[:, None])
        nk, means, prec = _m_step(X, resp)
        weights = nk / nk.sum()
        lb = lpn.mean()
        if abs(lb - prev) < EM_TOL:
            converged = True
            break
    score = logsumexp(weighted_log_prob(X, weights, means, prec), axis=1).mean()
    p = m * d * (d + 1) / 2.0 + m * d + m - 1
    return Model(seeds, labels, k_it, weights, means, prec, it, converged, -2 * score * n + int(p) * np.log(n),
                 seed_margin)


def bic_tolerance(model: Model, n: int, d: int, rel: float) -> float:
    """How far a BIC summed in another order may lie from this one: rel |BIC| plus 4 n d u kappa, kappa the largest
    condition number of the model's covariances -- the relative rounding of the smallest eigenvalue, which reg_covar
    keeps at >= 1e-6 when rows are duplicated or rank-deficient, enters the log-density of each of the n rows."""
    kappa = max(np.linalg.cond(p) ** 2 for p in model.prec_chol)
    return rel * abs(model.bic) + 4 * n * d * np.finfo(np.float64).eps / 2 * kappa


def memberships(X: np.ndarray, model: Model) -> np.ndarray:
    wlp = weighted_log_prob(np.asarray(X, np.float64), model.weights, model.means, model.prec_chol)
    return np.exp(wlp - logsumexp(wlp, axis=1)[:, None])


@dataclass
class Sweep:
    best: int
    models: List[Model]
    memberships: np.ndarray

    @property
    def bic(self):
        return np.array([mo.bic for mo in self.models])


def sweep(X: np.ndarray, max_components: int, random_state: int = 224) -> Sweep:
    first, seed = draws(X.shape[0], max_components, random_state)
    models, off = [], 0
    for m in range(1, max_components + 1):
        cnt = (m - 1) * trials(m)
        models.append(fit(X, m, first[m - 1], seed[off:off + cnt]))
        off += cnt
    best = int(np.argmin([mo.bic for mo in models])) + 1
    return Sweep(best, models, memberships(X, models[best - 1]))
