"""End to end with the synonymy edges on the device: the reference's unmodified ComoRAG.py on its cinderella sample
(tests/e2e_harness.py) with install("src.comorag", encoder=False), which binds add_synonymy_edges to the threshold
join (crag_knn_threshold).  On the same instance, at the moment the index phase calls it, the reference's own method
(_comorag_b200_originals) runs over our retrieve_knn on a copy of node_to_node_stats, then the device method on the
real one: the two must hold the same items in the same order, with at least one synonymy edge.  crag_knn_threshold
ran and crag_knn_topk at k = 2047 did not, and the trace matches the reference arm's (compare_traces)."""
import os
import sys
import tempfile

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import e2e_harness as H  # noqa: E402
from test_e2e_cinderella import REF_ROOT, needs_ref, reference_arm  # noqa: E402


@needs_ref
@pytest.mark.gpu
def test_synonymy_edges_on_the_device_match_the_reference_method(monkeypatch):
    import comorag_b200.install as crag
    from comorag_b200 import index as crag_index

    ref = reference_arm()
    seen = {"threshold": 0, "topk_2047": 0, "checked": 0, "edges": 0}
    real_thr = crag_index.DenseIndex.search_threshold_device
    real_knn = crag_index.DenseIndex._search_device_knn

    def counting_thr(self, *a, **kw):
        seen["threshold"] += 1
        return real_thr(self, *a, **kw)

    def counting_knn(self, queries, k, *a, **kw):
        if k == 2047 and not seen.get("in_reference"):
            seen["topk_2047"] += 1
        return real_knn(self, queries, k, *a, **kw)
    monkeypatch.setattr(crag_index.DenseIndex, "search_threshold_device", counting_thr)
    monkeypatch.setattr(crag_index.DenseIndex, "_search_device_knn", counting_knn)

    real_install = crag.install

    def install_and_wrap(pkg, **kw):
        counts = real_install(pkg, **kw)
        cls = sys.modules[pkg + ".ComoRAG"].ComoRAG
        device_method = cls.add_synonymy_edges
        reference_method = cls._comorag_b200_originals["add_synonymy_edges"]
        assert device_method.__module__ == "comorag_b200.comorag_methods"

        def both(self):
            before = dict(self.node_to_node_stats)
            real_stats = self.node_to_node_stats
            self.node_to_node_stats = dict(before)
            seen["in_reference"] = True
            try:
                reference_method(self)
            finally:
                seen["in_reference"] = False
            want = list(self.node_to_node_stats.items())
            self.node_to_node_stats = real_stats
            device_method(self)
            assert list(self.node_to_node_stats.items()) == want
            seen["checked"] += 1
            seen["edges"] += sum(1 for k in dict(want) if k not in before or before[k] != dict(want)[k])
        cls.add_synonymy_edges = both           # uninstall_search puts the reference method back
        return counts
    monkeypatch.setattr(crag, "install", install_and_wrap)
    try:
        with tempfile.TemporaryDirectory() as tmp:
            got = H.run_cinderella("shim_search", tmp, REF_ROOT)
    finally:
        crag.uninstall_search("src.comorag")
    assert seen["checked"] >= 1 and seen["edges"] >= 1, seen
    assert seen["threshold"] >= seen["checked"] and seen["topk_2047"] == 0, seen
    summary = H.compare_traces(ref, got, raw_tol=4e-3)
    assert not summary["problems"], summary["problems"]
