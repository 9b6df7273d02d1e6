"""UMAP on the device (comorag_b200/umap_layout.py, csrc/umap.cu) against its float64 restatement
(tests/umap_oracle.py), stage by stage:

* neighbour lists equal the self rule applied to the exact top-k (tests/scan_reference.py) of the crag_search_scores
  matrix of the same bf16 rows, bit for bit, including duplicate rows, zero rows and n_neighbors > N - 1;
* rho equals the oracle's exactly on the device's own lists; sigma within 1e-5 relative (the two sum the bisection's
  terms in different orders, so a step can stop one iteration apart, which moves sigma by less than that near the
  root); memberships within 2e-6; the symmetric CSR graph identical except entries within 1e-6 of the max / n_epochs
  cut, which are named;
* the spectral start's subspace is within 1e-2 (principal angle) of eigsh's on a connected planted-cluster graph;
* one layout epoch from a given device state matches the oracle's epoch (schedule counters exactly) within a
  per-vertex bound of 2^-14 per update step + 1e-4, calibrated on the emulated kernel.  Exempt are the vertices
  that met a near-coincident point (d^2 < 1e-2), where the fp32 / fp64 difference of d^2 is amplified by the
  repulsion's 1 / (0.001 + d^2) and only the clip bounds the step, and at most 0.5% of the others: a vertex's walk
  over its edges is a sequential map whose steps can expand a rounding difference in a dense region (one vertex in
  2 000 exceeded the bound six-fold at epoch 3 on an H100);
* a whole run is bit-identical twice and on a second stream;
* on planted clusters (N = 2000, 1024 columns) the layout is finite, its trustworthiness clears the oracle-calibrated
  bar and the device GMM sweep recovers the labels (ARI >= 0.95);
* small N follows _reduce_dimensions' control flow, including the fallback at N = 2."""
import logging
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import scan_reference as SR  # noqa: E402
import umap_oracle as U  # noqa: E402

pytestmark = pytest.mark.gpu

logger = logging.getLogger(__name__)
TRUST_BAR = 0.95


@pytest.fixture(scope="module")
def ul():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from comorag_b200 import umap_layout
    return umap_layout


def _rows(n, dim, seed, dup=0, zero=0, spread=0.35, clusters=6):
    X, labels = U.planted(n, dim, clusters, seed=seed, spread=spread)
    if dup:
        X[n - dup:] = X[:dup]
    if zero:
        X[1:1 + zero] = 0
    return X, labels


@pytest.mark.parametrize("n,dim,k,dup,zero", [(300, 64, 15, 20, 3), (200, 1024, 30, 0, 0), (40, 100, 64, 5, 2),
                                              (17, 64, 17, 0, 1), (3, 64, 5, 1, 0)])
def test_neighbour_lists_equal_the_self_rule_on_score_all(ul, n, dim, k, dup, zero):
    from comorag_b200.index import DenseIndex
    X, _ = _rows(n, dim, seed=n + dim, dup=dup, zero=zero)
    kk = k if n > k else n - 1
    ids, scores = ul.knn_self_join(X, kk)
    nbr, dist, rho, sigma, memb = ul.fuzzy_graph(ids, scores)
    x = torch.as_tensor(X).cuda()
    nrm = torch.linalg.vector_norm(x, dim=1, keepdim=True)
    xn = torch.where(nrm > 0, x / torch.where(nrm > 0, nrm, torch.ones_like(nrm)), torch.zeros_like(x))
    index = DenseIndex(dim)
    index.add(xn)
    S, _ = index.scores_device(index.prepare_queries(xn))
    rid, rsc, _, _ = SR.topk_from_scores(S, kk)
    assert torch.equal(ids, rid) and torch.equal(scores, rsc)
    want_nbr, want_dist = U.knn_lists(rid.cpu().numpy(), rsc.cpu().numpy())
    np.testing.assert_array_equal(nbr.cpu().numpy(), want_nbr)
    np.testing.assert_array_equal(dist.cpu().numpy(), want_dist)
    assert (nbr[:, 0].cpu().numpy() == np.arange(n)).all()


@pytest.mark.parametrize("n,dim,k", [(600, 128, 15), (2000, 1024, 30)])
def test_fuzzy_graph_matches_the_oracle(ul, n, dim, k):
    X, _ = _rows(n, dim, seed=3, dup=10, zero=2)
    ids, scores = ul.knn_self_join(X, k)
    nbr, dist, rho, sigma, memb = ul.fuzzy_graph(ids, scores)
    nbr_h, dist_h = nbr.cpu().numpy(), dist.cpu().numpy()
    o_rho, o_sigma, early = U.smooth_knn(dist_h)
    np.testing.assert_array_equal(rho.cpu().numpy(), o_rho)
    np.testing.assert_allclose(sigma.cpu().numpy(), o_sigma, rtol=1e-5, atol=0)
    o_mu = U.memberships(nbr_h, dist_h, rho.cpu().numpy(), sigma.cpu().numpy().astype(np.float64))
    np.testing.assert_allclose(memb.cpu().numpy(), o_mu, rtol=0, atol=2e-6)
    n_epochs = U.default_epochs(n)
    indptr, indices, w, eps = ul.symmetric_graph(nbr, memb, n_epochs)
    ip, ix, ow, oeps = U.fuzzy_union(nbr_h, memb.cpu().numpy(), n_epochs)
    got = set(zip(np.repeat(np.arange(n), np.diff(indptr.cpu().numpy())), indices.cpu().numpy()))
    want = set(zip(np.repeat(np.arange(n), np.diff(ip)), ix))
    cut = float(ow.max()) / n_epochs
    gw = dict(zip(got, w.cpu().numpy()))
    for e in got ^ want:                  # named: an entry within rounding of the max / n_epochs cut
        val = gw.get(e)
        assert val is not None and abs(float(val) - cut) <= 1e-6, e
    if got == want:
        np.testing.assert_array_equal(w.cpu().numpy(), ow)
        np.testing.assert_array_equal(eps.cpu().numpy(), oeps)
    # exactly symmetric
    G = torch.sparse_csr_tensor(indptr, indices.long(), w, (n, n)).to_dense()
    assert torch.equal(G, G.T)


def _connected_graph(ul, n, dim, d, spread, seed=1):
    X, _ = U.planted(n, dim, d + 1, seed=seed, spread=spread)
    ids, scores = ul.knn_self_join(X, 15)
    nbr, dist, rho, sigma, memb = ul.fuzzy_graph(ids, scores)
    return ul.symmetric_graph(nbr, memb, 500)


@pytest.mark.parametrize("n,dim,d,spread", [(400, 64, 3, 1.2), (2000, 1024, 4, 6.0), (2000, 1024, 4, 8.0)])
def test_spectral_start_spans_eigsh_subspace(ul, n, dim, d, spread):
    import scipy.sparse as sp
    import scipy.sparse.csgraph as cg
    indptr, indices, w, eps = _connected_graph(ul, n, dim, d, spread)
    ip, ix, ww = indptr.cpu().numpy(), indices.cpu().numpy(), w.cpu().numpy()
    assert cg.connected_components(sp.csr_matrix((ww, ix, ip), shape=(n, n)))[0] == 1
    y0, vec, vals = ul.spectral_init(indptr, indices, w, d, vectors=True)
    ref, ref_vals = U.spectral_eigsh(ip, ix, ww, d)
    angle = U.principal_angle(vec.cpu().numpy(), ref)
    assert angle <= 1e-2, angle
    # the start is the oracle's post-processing of the device's own vectors
    want = U.post(vec.cpu().numpy(), 224)
    np.testing.assert_allclose(y0.cpu().numpy(), want, rtol=0, atol=2e-5)
    mine, mine_vals = U.spectral_subspace(ip, ix, ww, d, ul.SPECTRAL_ITERS, 224)
    np.testing.assert_allclose(vals.cpu().numpy(), mine_vals, rtol=0, atol=1e-9)


@pytest.mark.parametrize("n", [3, 12, 16])
def test_spectral_start_is_exact_for_small_n(ul, n):
    X, _ = U.planted(n, 64, 2, seed=n, spread=1.0)
    ids, scores = ul.knn_self_join(X, n - 1)
    nbr, dist, rho, sigma, memb = ul.fuzzy_graph(ids, scores)
    indptr, indices, w, eps = ul.symmetric_graph(nbr, memb, 500)
    d = n - 2
    y0, vec, vals = ul.spectral_init(indptr, indices, w, d, vectors=True)
    G, deg, dis = U._operator(indptr.cpu().numpy(), indices.cpu().numpy(), w.cpu().numpy())
    S = 0.5 * (np.eye(n) + dis[:, None] * G.toarray() * dis[None, :])
    ev = np.sort(np.linalg.eigvalsh(S))[::-1]
    np.testing.assert_allclose(vals.cpu().numpy(), ev, atol=1e-12)
    assert np.isfinite(y0.cpu().numpy()).all()


def test_one_epoch_matches_the_oracle(ul):
    n, dim, k = 2000, 1024, 30
    X, _ = U.planted(n, dim, 8, seed=5)
    _, st = ul.umap_reduce(X, k, 10, n_epochs=500, return_stages=True)
    a, b = st.a, st.b
    for e0 in (0, 3, 250):
        sched = (st.eps.clone(), st.eps / 5.0)
        y = ul.optimize(st.indptr, st.indices, st.eps, st.y0, a, b, 500, 0, e0, schedule=sched)
        ns, nn = sched[0].cpu().numpy(), sched[1].cpu().numpy()
        y_dev = ul.optimize(st.indptr, st.indices, st.eps, y, a, b, 500, e0, e0 + 1, schedule=sched)
        ns_o, nn_o = ns.copy(), nn.copy()
        y_o = U.epoch(st.indptr.cpu().numpy(), st.indices.cpu().numpy(), st.eps.cpu().numpy(), y.cpu().numpy(),
                      ns_o, nn_o, e0, 500, a, b, 224)
        np.testing.assert_array_equal(sched[0].cpu().numpy(), ns_o)
        np.testing.assert_array_equal(sched[1].cpu().numpy(), nn_o)
        # update steps per vertex this epoch: two attractions per due edge plus its negative samples
        ip = st.indptr.cpu().numpy()
        steps = np.zeros(n)
        due = ns <= e0
        epn = st.eps.cpu().numpy() / 5.0
        n_neg = np.where(due, np.floor((e0 - nn) / epn), 0)
        per_edge = np.where(due, 2 + n_neg, 0)
        row = np.repeat(np.arange(n), np.diff(ip))
        np.add.at(steps, row, per_edge)
        err = np.abs(y_dev.cpu().numpy().astype(np.float64) - y_o).max(axis=1)
        bound = steps * 2.0 ** -14 + 1e-4
        yh = y.cpu().numpy().astype(np.float64)
        # vertices whose snapshot has a point within d^2 < 1e-2 (the amplified case)
        from scipy.spatial import cKDTree
        close = np.array([len(x) > 1 for x in cKDTree(yh).query_ball_point(yh, 0.1)])
        bad = (err > bound) & ~close
        assert bad.mean() <= 0.005, (e0, np.where(bad)[0][:10], err[bad][:10], bound[bad][:10])
        assert (err[close] <= 8.0 + 1e-3).all()
        assert (err <= bound).mean() >= 0.95, (e0, (err <= bound).mean())


def test_whole_run_is_bit_identical_across_runs_and_streams(ul):
    X, _ = U.planted(1500, 256, 6, seed=7)
    y1 = ul.umap_reduce(X, 15, 10)
    y2 = ul.umap_reduce(X, 15, 10)
    side = torch.cuda.Stream()
    y3 = ul.umap_reduce(X, 15, 10, stream=side)
    assert np.isfinite(y1).all()
    np.testing.assert_array_equal(y1, y2)
    np.testing.assert_array_equal(y1, y3)


def test_planted_clusters_layout_and_gmm_recover_labels(ul):
    from sklearn.manifold import trustworthiness
    from sklearn.metrics import adjusted_rand_score
    from comorag_b200.cluster import gmm_sweep
    X, labels = U.planted(2000, 1024, 8, seed=11)
    Y = ul.umap_reduce(X, 30, 10)
    assert Y.shape == (2000, 10) and Y.dtype == np.float32 and np.isfinite(Y).all()
    sub = np.random.RandomState(0).choice(2000, 1000, replace=False)
    tw = trustworthiness(X[sub], Y[sub], n_neighbors=15, metric="cosine")
    assert tw >= TRUST_BAR, tw
    r = gmm_sweep(Y, 12)
    ari = adjusted_rand_score(labels, r.memberships.argmax(axis=1))
    assert ari >= 0.95, (r.n_components, ari)


class _Clustering:
    reduction_dimension = 10
    verbose = True


@pytest.mark.parametrize("n", [2, 3, 6, 12, 17])
def test_small_n_follows_reduce_dimensions(ul, n, caplog):
    X, _ = U.planted(n, 1024, 2, seed=n, spread=1.0)
    with caplog.at_level(logging.INFO):
        out = ul.reduce_dimensions(_Clustering(), X)
    dim = min(10, n - 2)
    if n == 2:
        assert out is X                       # n_components = 0 raises, as in umap-learn: the original rows
        assert "n_components must be greater than 0" in caplog.text
    else:
        assert out.shape == (n, dim) and out.dtype == np.float32 and np.isfinite(out).all()
        assert f"Reduced dimensions from 1024 to {dim}" in caplog.text


def test_argument_errors(ul):
    X = np.ones((10, 8), np.float32)
    with pytest.raises(ValueError, match="n_components must be greater than 0"):
        ul.umap_reduce(X, 5, 0)
    with pytest.raises(ValueError):
        ul.umap_reduce(X, 5, 17)
    with pytest.raises(ValueError):
        ul.umap_reduce(X, 300, 2)
    with pytest.raises(ValueError):
        ul.umap_reduce(X, 1, 2)
    with pytest.raises(ValueError):
        ul.umap_reduce(np.ones((4, 2000), np.float32), 3, 2)
