"""UMAP as the device computes it (DESIGN.md section 2c), restated in numpy / scipy float64: the self rule on the
k-NN lists, smooth kNN, memberships, the fuzzy union, a and b, the spectral start (the device's subspace iteration,
and scipy's eigsh for comparison), the post-processing and the snapshot layout epochs.  The counter hash is
restated in integer arithmetic, so every random choice is the device's.  The epochs are vectorised over vertices (each
vertex reads only the snapshot and its own position), which keeps full runs at a few hundred rows affordable."""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
from scipy.optimize import curve_fit
from scipy.sparse.linalg import eigsh

MIN_DIST, SPREAD, NEG_RATE, GAMMA = 0.1, 1.0, 5.0, 1.0
STREAM_BASIS = 0xFFFFFFFF00000001
STREAM_NOISE = 0xFFFFFFFF00000002
_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


# ------------------------------------------------------------------------------------------------------- hash
def _mix(z):
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = z + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def counter_hash(seed, stream, a, b):
    """splitmix64's finaliser chained over (seed, stream, a, b), as umap_hash; arrays broadcast."""
    u = np.uint64
    return _mix(_mix(_mix(_mix(u(seed)) ^ u(stream)) ^ np.asarray(a, dtype=np.uint64)) ^ np.asarray(b, dtype=np.uint64))


def unit(h):
    return ((np.asarray(h, dtype=np.uint64) >> np.uint64(11)).astype(np.float64) + 1.0) * (1.0 / 9007199254740992.0)


# ----------------------------------------------------------------------------------------------- parameters
def find_ab_params(spread: float = SPREAD, min_dist: float = MIN_DIST):
    """umap-learn's find_ab_params: fit 1 / (1 + a x^2b) to the offset exponential on 300 points of [0, 3 spread]."""
    def curve(x, a, b):
        return 1.0 / (1.0 + a * x ** (2 * b))
    xv = np.linspace(0, spread * 3, 300)
    yv = np.zeros(xv.shape)
    yv[xv < min_dist] = 1.0
    yv[xv >= min_dist] = np.exp(-(xv[xv >= min_dist] - min_dist) / spread)
    params, _ = curve_fit(curve, xv, yv)
    return float(params[0]), float(params[1])


def default_epochs(n: int) -> int:
    return 500 if n <= 10000 else 200


# ------------------------------------------------------------------------------------------------- neighbours
def bf16_rows(X):
    """Rows normalised in fp32 (a zero row stays zero), rounded to bf16 (round to nearest even), as float64."""
    X = np.asarray(X, dtype=np.float32)
    nrm = np.sqrt((X * X).sum(axis=1, dtype=np.float32))
    Xn = np.where(nrm[:, None] > 0, X / np.where(nrm > 0, nrm, 1)[:, None], 0).astype(np.float32)
    u = Xn.view(np.uint32).astype(np.uint64)
    r = ((u + np.uint64(0x7FFF) + ((u >> np.uint64(16)) & np.uint64(1))) >> np.uint64(16)) << np.uint64(16)
    return r.astype(np.uint32).view(np.float32).astype(np.float64)


def topk_lists(S, k):
    """(ids, scores) of each row's k best columns by (score desc, column asc), from a score matrix."""
    n = S.shape[0]
    order = np.lexsort((np.broadcast_to(np.arange(S.shape[1]), S.shape), -S), axis=1)[:, :k]
    return order.astype(np.int64), np.take_along_axis(S, order, axis=1).astype(np.float32)


def knn_lists(ids, scores):
    """The self rule: i first at distance 0, then the k - 1 best other rows (i's entry removed, else the last
    dropped); distance max(0, 1 - score) in fp32."""
    ids = np.asarray(ids)
    scores = np.asarray(scores, dtype=np.float32)
    n, k = ids.shape
    nbr = np.empty((n, k), np.int32)
    dist = np.empty((n, k), np.float32)
    for i in range(n):
        hit = np.where(ids[i] == i)[0]
        keep = np.delete(np.arange(k), hit[0]) if hit.size else np.arange(k - 1)
        nbr[i, 0], dist[i, 0] = i, 0.0
        nbr[i, 1:] = ids[i, keep]
        dist[i, 1:] = np.maximum(np.float32(0), np.float32(1) - scores[i, keep])
    return nbr, dist


def smooth_knn(dist, n_iter=64, tol=1e-5):
    """(rho fp32, sigma float64, stopped_early bool) per row, as umap-learn's smooth_knn_dist with
    local_connectivity 1 and bandwidth 1."""
    dist = np.asarray(dist, dtype=np.float32)
    n, k = dist.shape
    target = np.log2(k)
    mean_all = dist.astype(np.float64).mean()
    rho = np.zeros(n, np.float32)
    sigma = np.zeros(n)
    early = np.zeros(n, bool)
    for i in range(n):
        di = dist[i].astype(np.float64)
        nz = di[di > 0]
        rho[i] = nz[0] if nz.size else 0.0
        lo, hi, mid = 0.0, np.inf, 1.0
        x = di[1:] - float(rho[i])
        for _ in range(n_iter):
            psum = float(np.where(x > 0, np.exp(-(np.maximum(x, 0) / mid)), 1.0).sum())
            if abs(psum - target) < tol:
                early[i] = True
                break
            if psum > target:
                hi = mid
                mid = (lo + hi) / 2.0
            else:
                lo = mid
                mid = mid * 2 if hi == np.inf else (lo + hi) / 2.0
        floor = 1e-3 * (di.mean() if rho[i] > 0 else mean_all)
        sigma[i] = max(mid, floor)
    return rho, sigma, early


def memberships(nbr, dist, rho, sigma):
    n, k = nbr.shape
    x = dist.astype(np.float64) - rho.astype(np.float64)[:, None]
    mu = np.where((x <= 0) | (sigma[:, None] == 0), 1.0, np.exp(-(np.maximum(x, 0) / sigma[:, None])))
    mu[nbr == np.arange(n)[:, None]] = 0.0
    return mu.astype(np.float32)


def fuzzy_union(nbr, memb, n_epochs):
    """G = P + P^T - P o P^T in fp32, zeros dropped, entries below max(G) / n_epochs dropped; CSR with ascending
    columns: (indptr int64, indices int32, weights fp32, epochs_per_sample float64)."""
    n, k = nbr.shape
    rows = np.repeat(np.arange(n), k)
    P = sp.csr_matrix((memb.ravel().astype(np.float32), (rows, nbr.ravel())), shape=(n, n))
    P.eliminate_zeros()
    G = (P + P.T - P.multiply(P.T)).tocsr().astype(np.float32)
    G.eliminate_zeros()
    G.data[G.data < G.data.max() / np.float32(n_epochs)] = 0
    G.eliminate_zeros()
    G.sort_indices()
    eps = float(G.data.max()) / G.data.astype(np.float64)
    return G.indptr.astype(np.int64), G.indices.astype(np.int32), G.data.astype(np.float32), eps


# ------------------------------------------------------------------------------------------------ spectral
def _operator(indptr, indices, w):
    n = len(indptr) - 1
    G = sp.csr_matrix((w.astype(np.float64), indices, indptr), shape=(n, n))
    deg = np.asarray(G.sum(axis=1)).ravel()
    dis = np.where(deg > 0, 1.0 / np.sqrt(np.where(deg > 0, deg, 1)), 0.0)
    return G, deg, dis


def n_columns(n, d):
    return min(max(16, d + 1), n)


def _signed(Y):
    Y = Y.copy()
    for c in range(Y.shape[1]):
        if Y[np.argmax(np.abs(Y[:, c])), c] < 0:
            Y[:, c] = -Y[:, c]
    return Y


def spectral_subspace(indptr, indices, w, d, iters, seed):
    """The device's start: block subspace iteration with CholQR after every step, then Rayleigh-Ritz.  Returns
    (signed Ritz vectors 2..d+1 [n][d], Ritz values [p] descending)."""
    G, deg, dis = _operator(indptr, indices, w)
    n = G.shape[0]
    p = n_columns(n, d)
    if n <= 16:
        V = np.eye(n)
        iters = 0
    else:
        i, c = np.meshgrid(np.arange(n), np.arange(p), indexing="ij")
        V = 2.0 * unit(counter_hash(seed, STREAM_BASIS, i, c)) - 1.0
        V[:, 0] = np.sqrt(deg)

    def apply(V):
        return 0.5 * (V + dis[:, None] * (G @ (dis[:, None] * V)))
    for _ in range(iters):
        W = apply(V)
        L = np.linalg.cholesky(W.T @ W)
        V = np.linalg.solve(L, W.T).T
    H = V.T @ apply(V)
    vals, Q = np.linalg.eigh(0.5 * (H + H.T))
    order = np.argsort(-vals, kind="stable")
    return _signed(V @ Q[:, order[1:d + 1]]), vals[order]


def spectral_eigsh(indptr, indices, w, d):
    """The reference subspace: the d eigenvectors of S' after the top one, from ARPACK at full precision."""
    G, deg, dis = _operator(indptr, indices, w)
    n = G.shape[0]
    S = 0.5 * (sp.identity(n) + sp.diags(dis) @ G @ sp.diags(dis))
    vals, vecs = eigsh(S, k=d + 1, which="LA", v0=np.ones(n))
    order = np.argsort(-vals, kind="stable")
    return _signed(vecs[:, order[1:d + 1]]), vals[order]


def principal_angle(A, B):
    """Largest principal angle (radians) between the column spans of A and B."""
    qa, _ = np.linalg.qr(A)
    qb, _ = np.linalg.qr(B)
    s = np.linalg.svd(qa.T @ qb, compute_uv=False)
    return float(np.arccos(np.clip(s.min(), -1.0, 1.0)))


def post(Y, seed):
    """umap-learn's post-processing of the start: x 10 / max|Y| in fp32, + 1e-4 N(0, 1) noise (Box-Muller on the
    counter hash), per-column min-max rescale to [0, 10] in fp32."""
    n, d = Y.shape
    i, c = np.meshgrid(np.arange(n), np.arange(d), indexing="ij")
    u1 = unit(counter_hash(seed, STREAM_NOISE, i, 2 * c))
    u2 = unit(counter_hash(seed, STREAM_NOISE, i, 2 * c + 1))
    g = np.sqrt(-2.0 * np.log(u1)) * np.cos(6.283185307179586 * u2)
    E = (Y * (10.0 / np.abs(Y).max())).astype(np.float32) + (1e-4 * g).astype(np.float32)
    mn, mx = E.min(axis=0), E.max(axis=0)
    return (np.float32(10.0) * (E - mn) / (mx - mn)).astype(np.float32)


# -------------------------------------------------------------------------------------------------- layout
def schedule(eps):
    """Schedule counters before epoch 0: (next_sample, next_neg)."""
    return eps.copy(), eps / NEG_RATE


def epoch(indptr, indices, eps, Y, next_sample, next_neg, e, n_epochs, a, b, seed, skip_self=True):
    """Layout epoch e in float64: every vertex moves from its own position against the snapshot Y.  Returns the new
    layout; next_sample / next_neg advance in place."""
    snap = np.asarray(Y, dtype=np.float64)
    y = snap.copy()
    n = snap.shape[0]
    alpha = 1.0 - max(e - 1, 0) / n_epochs
    deg = np.diff(indptr)
    clip = lambda v: np.clip(v, -4.0, 4.0)  # noqa: E731
    for t in range(int(deg.max()) if n else 0):
        v = np.where(deg > t)[0]
        p = indptr[v] + t
        due = next_sample[p] <= e
        v, p = v[due], p[due]
        o = snap[indices[p]]
        for _ in range(2):
            diff = y[v] - o
            d2 = (diff * diff).sum(axis=1)
            pos = d2 > 0
            g = np.zeros_like(d2)
            g[pos] = -2.0 * a * b * d2[pos] ** (b - 1.0) / (a * d2[pos] ** b + 1.0)
            y[v] += clip(g[:, None] * diff) * alpha
        epn = eps[p] / NEG_RATE
        next_sample[p] += eps[p]
        n_neg = ((e - next_neg[p]) / epn).astype(np.int64)
        for s in range(int(n_neg.max()) if n_neg.size else 0):
            m = n_neg > s
            vs, ps = v[m], p[m]
            kk = (counter_hash(seed, e, ps, s) % np.uint64(n)).astype(np.int64)
            diff = y[vs] - snap[kk]
            d2 = (diff * diff).sum(axis=1)
            ok = d2 > 0
            if skip_self:
                ok &= kk != vs
            g = np.zeros_like(d2)
            g[ok] = 2.0 * GAMMA * b / ((0.001 + d2[ok]) * (a * d2[ok] ** b + 1.0))
            y[vs] += np.where(ok[:, None], clip(g[:, None] * diff), 0.0) * alpha
        next_neg[p] += n_neg * epn
    return y


# ------------------------------------------------------------------------------------------------ whole run
def umap(X, n_neighbors, d, seed=224, n_epochs=None, iters=None, start="subspace", epochs_run=None):
    """The whole reduction on the CPU: dict with every stage's output."""
    Xb = bf16_rows(X)
    n = len(Xb)
    k = n_neighbors if n > n_neighbors else n - 1
    ids, sc = topk_lists((Xb @ Xb.T).astype(np.float32), k)
    nbr, dist = knn_lists(ids, sc)
    rho, sigma, early = smooth_knn(dist)
    mu = memberships(nbr, dist, rho, sigma)
    n_epochs = n_epochs or default_epochs(n)
    indptr, indices, w, eps = fuzzy_union(nbr, mu, n_epochs)
    a, b = find_ab_params()
    if start == "eigsh":
        Yr, vals = spectral_eigsh(indptr, indices, w, d)
    else:
        Yr, vals = spectral_subspace(indptr, indices, w, d, iters, seed)
    Y = post(Yr, seed)
    y0 = Y.copy()
    ns, nn = schedule(eps)
    for e in range(n_epochs if epochs_run is None else epochs_run):
        Y = epoch(indptr, indices, eps, Y, ns, nn, e, n_epochs, a, b, seed)
    return dict(nbr=nbr, dist=dist, rho=rho, sigma=sigma, early=early, memb=mu, indptr=indptr, indices=indices,
                weights=w, eps=eps, a=a, b=b, start_vectors=Yr, eigenvalues=vals, y0=y0, y=Y, k=k, n_epochs=n_epochs)


def planted(n, dim, clusters, seed=0, spread=0.35):
    """Rows around `clusters` random directions, with labels."""
    rs = np.random.RandomState(seed)
    centres = rs.normal(size=(clusters, dim))
    labels = np.arange(n) % clusters
    X = centres[labels] + spread * rs.normal(size=(n, dim)) * np.sqrt(1.0 / 1.0)
    return X.astype(np.float32), labels
