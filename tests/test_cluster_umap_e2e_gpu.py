"""End to end with UMAP and the soft clustering on the device: the reference's unmodified ComoRAG.py on its cinderella
sample (tests/e2e_harness.py) with install("src.comorag", encoder=False, cluster=True, umap=True).  The harness's
UMAP stand-in is never constructed: every reduction is comorag_b200.umap_layout.reduce_dimensions.  Each
perform_clustering call's clusters, centroids and memberships equal what the reference's own method returns on a twin
whose _reduce_dimensions returns the device's recorded reductions.  The committed reference trace is not compared: it
was made with the stand-in's PCA layout."""
import copy
import os
import sys
import tempfile

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import e2e_harness as H  # noqa: E402
from test_e2e_cinderella import REF_ROOT, needs_ref  # noqa: E402


@needs_ref
@pytest.mark.gpu
def test_umap_and_clustering_on_the_device_match_the_reference_method(monkeypatch):
    from comorag_b200 import cluster as cl
    from comorag_b200 import umap_layout as ul
    import comorag_b200.install as crag

    def no_stand_in(*a, **kw):
        raise AssertionError("the harness's UMAP stand-in was constructed")
    monkeypatch.setattr(H._UMAP, "__init__", no_stand_in)
    reductions = []
    real_reduce = ul.reduce_dimensions

    def recording_reduce(self, embeddings):
        out = real_reduce(self, embeddings)
        reductions.append((np.asarray(embeddings).shape, out))
        return out
    monkeypatch.setattr(ul, "reduce_dimensions", recording_reduce)
    calls = []
    real_perform = cl.perform_clustering

    def recording_perform(self, hash_ids=None):
        before = len(reductions)
        twin = copy.copy(self)
        out = real_perform(self, hash_ids)
        recorded = [r for _, r in reductions[before:]]
        replay = iter(recorded)
        twin._reduce_dimensions = lambda embeddings: next(replay)
        self._comorag_b200_originals["perform_clustering"](twin, hash_ids)
        calls.append((self.clusters, self.hash_id_to_cluster_memberships, twin.clusters,
                      twin.hash_id_to_cluster_memberships, recorded))
        return out
    monkeypatch.setattr(cl, "perform_clustering", recording_perform)
    real_install = crag.install
    monkeypatch.setattr(crag, "install",
                        lambda pkg, **kw: real_install(pkg, **{**kw, "cluster": True, "umap": True}))
    try:
        with tempfile.TemporaryDirectory() as tmp:
            H.run_cinderella("shim_search", tmp, REF_ROOT)
    finally:
        crag.uninstall_search("src.comorag")
        crag.uninstall_cluster("src.comorag")
    assert calls, "perform_clustering never ran"
    n_device = 0
    for clusters, memb, ref_clusters, ref_memb, recorded in calls:
        for r in recorded:
            if r.ndim == 2 and r.shape[1] <= 16:
                n_device += 1
                assert r.dtype == np.float32 and np.isfinite(r).all()
        assert [c.id for c in clusters] == [c.id for c in ref_clusters]
        for c, r in zip(clusters, ref_clusters):
            assert type(c) is type(r)
            assert (c.centroid is None) == (r.centroid is None)
            if r.centroid is not None:
                np.testing.assert_allclose(c.centroid, r.centroid, rtol=1e-6, atol=1e-6)
            assert c.members.keys() == r.members.keys()
            for h in r.members:
                assert abs(c.members[h] - r.members[h]) <= 1e-6, (c.id, h)
        assert memb.keys() == ref_memb.keys()
        for h in ref_memb:
            assert memb[h].keys() == ref_memb[h].keys()
    assert n_device >= 1
