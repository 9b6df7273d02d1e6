"""End to end with the soft clustering on the device: the reference's unmodified ComoRAG.py on its cinderella sample
(tests/e2e_harness.py) with install("src.comorag", encoder=False, cluster=True) -- the reference's fp32 encoder, the
engine's stores and device search, and ChunkSoftClustering.perform_clustering rebound onto crag_gmm_sweep.  Both arms
reduce with the harness's UMAP stand-in.  Checks: the trace matches the reference arm's (compare_traces, raw_tol
4e-3); every perform_clustering call ran its sweeps on the device; and each call's clusters, centroids and
memberships equal what the reference's own method returns on the same instance (the same reduced embeddings)."""
import copy
import os
import sys
import tempfile

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import e2e_harness as H  # noqa: E402
from test_e2e_cinderella import REF_ROOT, needs_ref, reference_arm  # noqa: E402


@needs_ref
@pytest.mark.gpu
def test_clustering_on_the_device_matches_the_reference(monkeypatch):
    from comorag_b200 import cluster as cl
    import comorag_b200.install as crag

    ref = reference_arm()
    sweeps = []
    real_sweep = cl.gmm_sweep

    def recording_sweep(X, max_components, *a, **kw):
        out = real_sweep(X, max_components, *a, **kw)
        sweeps.append((np.asarray(X).shape, max_components))
        return out
    monkeypatch.setattr(cl, "gmm_sweep", recording_sweep)
    calls = []
    real_perform = cl.perform_clustering

    def recording_perform(self, hash_ids=None):
        before = len(sweeps)
        twin = copy.copy(self)
        out = real_perform(self, hash_ids)
        reference = self._comorag_b200_originals["perform_clustering"]
        reference(twin, hash_ids)
        calls.append((self.clusters, self.hash_id_to_cluster_memberships, twin.clusters,
                      twin.hash_id_to_cluster_memberships, sweeps[before:]))
        return out
    monkeypatch.setattr(cl, "perform_clustering", recording_perform)
    real_install = crag.install
    monkeypatch.setattr(crag, "install", lambda pkg, **kw: real_install(pkg, **{**kw, "cluster": True}))
    try:
        with tempfile.TemporaryDirectory() as tmp:
            got = H.run_cinderella("shim_search", tmp, REF_ROOT)
    finally:
        crag.uninstall_search("src.comorag")
        crag.uninstall_cluster("src.comorag")
    summary = H.compare_traces(ref, got, raw_tol=4e-3)
    assert not summary["problems"], summary["problems"]
    assert calls, "perform_clustering never ran"
    device_sweeps = 0
    for clusters, memb, ref_clusters, ref_memb, ran in calls:
        device_sweeps += len(ran)
        # every sweep with more than one candidate model ran on the device
        assert len(ran) == sum(1 for c in ran if c[1] > 1)
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
    assert device_sweeps >= 1
