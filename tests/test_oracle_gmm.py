"""oracle/gmm_oracle.py pinned to the installed scikit-learn on float64 input: the same k-means++ rows
(sklearn.cluster.kmeans_plusplus), k-means labels (KMeans(n_init=1)), EM iteration counts, converged flags and chosen
n as GaussianMixture(m, random_state=224); weights, means, BIC and memberships within 1e-9 relative.  The
relocation layout is checked to empty a cluster.  Then the whole of cluster.perform_clustering, with the oracle's
arithmetic in place of the device sweep, against the reference's ChunkSoftClustering.perform_clustering on the same
store and the harness's UMAP stand-in: the same clusters, centroids and memberships.  CPU only."""
import os
import sys
import types
import warnings

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from oracle import gmm_oracle as G  # noqa: E402

sklearn = pytest.importorskip("sklearn")
from sklearn.cluster import KMeans, kmeans_plusplus  # noqa: E402
from sklearn.mixture import GaussianMixture  # noqa: E402

REL = 1e-9


def _mixture(rng, n, d, k, spread):
    c = rng.normal(0, spread, size=(k, d))
    return c[rng.integers(0, k, n)] + rng.normal(0, 1.0, size=(n, d))


CASES = {
    "blobs_d10": lambda rng: (_mixture(rng, 300, 10, 4, 4.0), 25),
    "overlap_d2": lambda rng: (_mixture(rng, 400, 2, 6, 1.5), 30),
    "tiny_d1": lambda rng: (rng.normal(size=(13, 1)), 12),
    "d16": lambda rng: (_mixture(rng, 120, 16, 3, 3.0), 20),
    "duplicates": lambda rng: (np.concatenate([_mixture(rng, 80, 3, 3, 4.0)] * 2) @ rng.normal(size=(3, 10)), 15),
    "relocate": lambda rng: (G.relocation_layout(), 6),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_sklearn(name):
    X, M = CASES[name](np.random.default_rng(sorted(CASES).index(name)))
    sw = G.sweep(X, M)
    Xc = X - X.mean(0)
    bics = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for m in range(1, M + 1):
            mo = sw.models[m - 1]
            _, idx = kmeans_plusplus(Xc, m, random_state=np.random.RandomState(224), x_squared_norms=(Xc ** 2).sum(1))
            np.testing.assert_array_equal(idx, mo.seeds, err_msg=f"m={m}")
            km = KMeans(m, n_init=1, random_state=np.random.RandomState(224)).fit(X)
            np.testing.assert_array_equal(km.labels_, mo.labels, err_msg=f"m={m}")
            gm = GaussianMixture(m, random_state=224).fit(X)
            assert gm.n_iter_ == mo.iters and gm.converged_ == mo.converged, (m, gm.n_iter_, mo.iters)
            np.testing.assert_allclose(mo.weights, gm.weights_, rtol=REL)
            np.testing.assert_allclose(mo.means, gm.means_, rtol=REL, atol=REL * np.abs(gm.means_).max())
            bic = gm.bic(X)
            assert abs(mo.bic - bic) <= REL * abs(bic), (m, mo.bic, bic)
            bics.append(bic)
        best = int(np.argmin(bics)) + 1
        assert sw.best == best
        proba = GaussianMixture(best, random_state=224, covariance_type="full").fit(X).predict_proba(X)
    np.testing.assert_allclose(sw.memberships, proba, rtol=0, atol=REL)


def test_relocation_layout_relocates(monkeypatch):
    """Lloyd on relocation_layout() meets an empty cluster while some row is off its centre, so it relocates."""
    X, M = CASES["relocate"](None)
    seen = []

    class _Numpy(types.ModuleType):
        def __getattr__(self, name):
            return getattr(np, name)

        @staticmethod
        def argpartition(a, k, *rest, **kw):
            seen.append(bool(np.max(a) > 0))
            return np.argpartition(a, k, *rest, **kw)
    monkeypatch.setattr(G, "np", _Numpy("numpy"))
    G.sweep(X, M)
    assert any(seen)


def test_draws_follow_sklearn_consumption():
    """The host-made draws reproduce kmeans_plusplus's rows when fed to the oracle's seeding."""
    rng = np.random.default_rng(9)
    X = rng.normal(size=(3000, 4))
    Xc = X - X.mean(0)
    first, draws = G.draws(len(X), 50)
    off = 0
    for m in range(1, 51):
        cnt = (m - 1) * G.trials(m)
        if m in (1, 2, 7, 20, 50):
            _, idx = kmeans_plusplus(Xc, m, random_state=np.random.RandomState(224), x_squared_norms=(Xc ** 2).sum(1))
            np.testing.assert_array_equal(G.kmeans_plusplus(Xc, m, first[m - 1], draws[off:off + cnt]), idx)
        off += cnt


# ------------------------------------------------------------------------------------------------ perform_clustering
class _Store:
    def __init__(self, emb):
        self.ids = [f"chunk-{i:04d}" for i in range(len(emb))]
        self.emb = dict(zip(self.ids, emb))

    def get_all_ids(self):
        return list(self.ids)

    def get_embeddings(self, ids):
        return [self.emb[i] for i in ids]


def _reference_cluster_module():
    import e2e_harness as H
    root = H.find_reference_root()
    if root is None:
        pytest.skip("reference tree not present (build() stages it under oracle/_ref)")
    if root not in sys.path:
        sys.path.insert(0, root)
    H.install_stand_ins()
    from src.comorag.utils import cluster_utils
    return cluster_utils


def _oracle_fit_best(X, max_components, random_state=224):
    X = np.asarray(X, dtype=np.float64)
    if max_components == 1:
        return 1, (X.sum(0) / (len(X) + 10 * np.finfo(np.float64).eps))[None], np.ones((len(X), 1))
    sw = G.sweep(X, max_components, random_state)
    return sw.best, sw.models[sw.best - 1].means, sw.memberships


def _summary(clustering):
    out = []
    for c in clustering.clusters:
        cen = None if c.centroid is None else np.asarray(c.centroid, np.float64)
        out.append((c.id, cen, dict(c.members)))
    return out, {h: dict(v) for h, v in clustering.hash_id_to_cluster_memberships.items()}


@pytest.mark.parametrize("n", [2, 9, 140])
def test_perform_clustering_matches_the_reference_method(n, monkeypatch):
    cu = _reference_cluster_module()
    from comorag_b200 import cluster as cl
    monkeypatch.setattr(cl, "fit_best", _oracle_fit_best)
    rng = np.random.default_rng(n)
    centres = rng.normal(size=(5, 64))
    emb = centres[rng.integers(0, 5, n)] + 0.3 * rng.normal(size=(n, 64))
    emb /= np.linalg.norm(emb, axis=1, keepdims=True)

    def make():
        obj = object.__new__(cu.ChunkSoftClustering)
        obj.embedding_store, obj.reduction_dimension, obj.threshold = _Store(emb.astype(np.float32)), 10, 0.1
        obj.max_clusters, obj.verbose, obj.clusters, obj.hash_id_to_cluster_memberships = 50, False, [], {}
        obj.db_filename = None
        return obj

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref = make()
        cu.ChunkSoftClustering.perform_clustering(ref)
        got = make()
        cl.perform_clustering(got)
    (rc, rm), (gc, gm) = _summary(ref), _summary(got)
    assert [c[0] for c in rc] == [c[0] for c in gc]
    assert all(type(c) is cu.SoftCluster for c in got.clusters)
    for (i, rcen, rmem), (_, gcen, gmem) in zip(rc, gc):
        assert (rcen is None) == (gcen is None)
        if rcen is not None:
            np.testing.assert_allclose(gcen, rcen, rtol=REL, atol=REL * max(1.0, np.abs(rcen).max()))
        assert rmem.keys() == gmem.keys(), i
        for h in rmem:
            assert abs(gmem[h] - rmem[h]) <= REL, (i, h)
    assert rm.keys() == gm.keys()
    for h in rm:
        assert rm[h].keys() == gm[h].keys()
