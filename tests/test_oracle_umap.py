"""The UMAP oracle (tests/umap_oracle.py) on its own, on the CPU: a and b are umap-learn's, the bisection reaches its
target, the fuzzy union is a symmetric graph in [0, 1], the subspace-iteration start spans eigsh's subspace on a
connected graph, and a whole run lays out planted clusters well.

Calibration of the whole-run bars (N = 400, 64 columns, 6 planted clusters, n_neighbors 15, d = 10, n_epochs 200, the
default 300-step start): trustworthiness 0.969 (15 neighbours, cosine; the start alone scores 0.953) and a
GaussianMixture(6) on the layout recovers the labels with ARI 1.0.  The bars are 0.95 and 0.95."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import umap_oracle as U  # noqa: E402

ITERS = 300          # comorag_b200.umap_layout.SPECTRAL_ITERS (importing the package would load torch)


def _graph(n, dim, clusters, spread, k=15, seed=1, n_epochs=500):
    X, labels = U.planted(n, dim, clusters, seed=seed, spread=spread)
    Xb = U.bf16_rows(X)
    ids, sc = U.topk_lists((Xb @ Xb.T).astype(np.float32), k)
    nbr, dist = U.knn_lists(ids, sc)
    rho, sigma, early = U.smooth_knn(dist)
    mu = U.memberships(nbr, dist, rho, sigma)
    return X, labels, nbr, dist, rho, sigma, early, mu, U.fuzzy_union(nbr, mu, n_epochs)


def test_ab_params():
    a, b = U.find_ab_params()
    assert abs(a - 1.576943) <= 1e-5 and abs(b - 0.895061) <= 1e-5


def test_self_rule():
    ids = np.array([[0, 1, 2], [0, 2, 1], [0, 1, 2]])
    sc = np.array([[0.99, 0.5, 0.4], [0.9, 0.8, 0.7], [0.6, 0.5, 0.4]], np.float32)
    nbr, dist = U.knn_lists(ids, sc)
    np.testing.assert_array_equal(nbr, [[0, 1, 2], [1, 0, 2], [2, 0, 1]])
    np.testing.assert_array_equal(dist[:, 0], 0)
    assert dist[1, 1] == np.float32(1) - np.float32(0.9)
    assert dist[2, 2] == np.float32(1) - np.float32(0.5)


def test_bisection_reaches_target_and_graph_is_symmetric():
    X, labels, nbr, dist, rho, sigma, early, mu, (ip, ix, w, eps) = _graph(300, 64, 5, 0.35)
    k = nbr.shape[1]
    assert early.mean() > 0.9
    for i in np.where(early)[0]:
        x = dist[i, 1:].astype(np.float64) - float(rho[i])
        psum = np.where(x > 0, np.exp(-np.maximum(x, 0) / sigma[i]), 1.0).sum()
        if sigma[i] > 1e-3 * dist[i].mean():          # not floored
            assert abs(psum - np.log2(k)) < 1e-5
    assert (rho == np.array([d[d > 0][0] if (d > 0).any() else 0 for d in dist], np.float32)).all()
    import scipy.sparse as sp
    G = sp.csr_matrix((w, ix, ip), shape=(300, 300))
    assert (abs(G - G.T) > 0).nnz == 0
    assert w.min() > 0 and w.max() <= 1
    assert (G.diagonal() == 0).all()
    assert np.all(np.diff(ix[ip[0]:ip[1]]) > 0)
    np.testing.assert_array_equal(eps, w.max() / w.astype(np.float64))


def test_rho_ignores_the_self_entry():
    # a duplicate row sits at distance 0 beside i itself: rho is the first nonzero distance after both
    X, _ = U.planted(50, 32, 2, seed=3)
    X[1] = X[0]
    Xb = U.bf16_rows(X)
    ids, sc = U.topk_lists((Xb @ Xb.T).astype(np.float32), 10)
    nbr, dist = U.knn_lists(ids, sc)
    rho, _, _ = U.smooth_knn(dist)
    assert dist[0, 0] == 0 and rho[0] > 0


@pytest.mark.parametrize("n,dim,d,spread", [(400, 64, 3, 1.2), (400, 64, 3, 1.6)])
def test_subspace_start_matches_eigsh(n, dim, d, spread):
    import scipy.sparse as sp
    import scipy.sparse.csgraph as cg
    X, labels, *_, (ip, ix, w, eps) = _graph(n, dim, d + 1, spread)
    assert cg.connected_components(sp.csr_matrix((w, ix, ip), shape=(n, n)))[0] == 1
    ref, vals = U.spectral_eigsh(ip, ix, w, d)
    mine, mvals = U.spectral_subspace(ip, ix, w, d, ITERS, 224)
    assert U.principal_angle(mine, ref) <= 1e-2
    np.testing.assert_allclose(mvals[:d + 1], vals, atol=1e-8)


def test_hash_is_the_documented_splitmix_chain():
    def mix(z):
        z = (z + 0x9E3779B97F4A7C15) & (2**64 - 1)
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & (2**64 - 1)
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & (2**64 - 1)
        return z ^ (z >> 31)
    for seed, s, a, b in [(224, 0, 0, 0), (224, 499, 123456, 4), (7, U.STREAM_NOISE, 3, 5)]:
        assert int(U.counter_hash(seed, s, a, b)) == mix(mix(mix(mix(seed) ^ s) ^ a) ^ b)


def test_whole_run_on_planted_clusters():
    from sklearn.manifold import trustworthiness
    from sklearn.metrics import adjusted_rand_score
    from sklearn.mixture import GaussianMixture
    X, labels = U.planted(400, 64, 6, seed=2)
    r = U.umap(X, 15, 10, seed=224, n_epochs=200, iters=ITERS)
    Y = r["y"]
    assert np.isfinite(Y).all()
    assert trustworthiness(X, Y, n_neighbors=15, metric="cosine") >= 0.95
    pred = GaussianMixture(6, random_state=224).fit(Y).predict(Y)
    assert adjusted_rand_score(labels, pred) >= 0.95
