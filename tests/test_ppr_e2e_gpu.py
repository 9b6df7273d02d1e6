"""End to end with the graph search on the device: the reference's unmodified ComoRAG.py on its cinderella sample
(tests/e2e_harness.py) with install("src.comorag", encoder=False, graph=True) -- the reference's fp32 encoder, the
engine's stores and device search, and graph_search_with_fact_entities / run_ppr rebound onto crag_ppr.  The
harness's igraph stand-in gets the two edge accessors DeviceGraph.from_igraph reads (get_edgelist, es["weight"])
here, for this test only.  Checks: the trace matches the reference arm's (compare_traces, raw_tol 4e-3), every
"ppr" entry went through crag_ppr, and every device PPR vector is within the error bound of tests/ppr_bound.py
against the float64 oracle on the same graph and reset."""
import os
import sys
import tempfile

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import e2e_harness as H  # noqa: E402
import ppr_bound  # noqa: E402
from test_e2e_cinderella import REF_ROOT, needs_ref, reference_arm  # noqa: E402


@needs_ref
@pytest.mark.gpu
def test_graph_search_on_the_device_matches_the_reference_trace(monkeypatch):
    from comorag_b200 import graph as crag_graph
    from comorag_b200.graph import ppr_iterations
    import comorag_b200.install as crag

    ref = reference_arm()
    monkeypatch.setattr(H._Graph, "get_edgelist", lambda self: list(self._edges), raising=False)
    monkeypatch.setattr(H._EdgeSeq, "__getitem__", lambda self, k: list(self._g._weights) if k == "weight" else {}[k],
                        raising=False)
    built = {}
    real_from_igraph = crag_graph.DeviceGraph.from_igraph.__func__

    def recording_build(cls, g, device=None):
        dg = real_from_igraph(cls, g, device)
        built[id(dg)] = (np.asarray(g.get_edgelist(), dtype=np.int64).reshape(-1, 2), np.asarray(g.es["weight"]))
        return dg
    monkeypatch.setattr(crag_graph.DeviceGraph, "from_igraph", classmethod(recording_build))
    calls = []
    real = crag_graph.DeviceGraph.personalized_pagerank

    def recording(self, reset, damping=0.5, tol=1e-10, vertices=None, stream=None):
        out = real(self, reset, damping, tol, vertices, stream)
        calls.append((self, np.asarray(reset, dtype=np.float64).copy(), float(damping), vertices.cpu().numpy(),
                      out.cpu().numpy()))
        return out
    monkeypatch.setattr(crag_graph.DeviceGraph, "personalized_pagerank", recording)
    real_install = crag.install
    monkeypatch.setattr(crag, "install", lambda pkg, **kw: real_install(pkg, **{**kw, "graph": True}))
    try:
        with tempfile.TemporaryDirectory() as tmp:
            got = H.run_cinderella("shim_search", tmp, REF_ROOT)
    finally:
        crag.uninstall_search("src.comorag")
    summary = H.compare_traces(ref, got, raw_tol=4e-3)
    assert not summary["problems"], summary["problems"]
    ppr_entries = [q for q, t in got["trace"].items() if "ppr" in t]
    assert len(ppr_entries) == len([q for q, t in ref["trace"].items() if "ppr" in t]) >= 9
    # every graph search ran PPR on the device: one crag_ppr call per graph search, at least one per traced query
    assert len(calls) >= len(ppr_entries)
    worst = 0.0
    for g, reset, d, verts, out in calls:
        edges, weights = built[id(g)]
        x, bnd = ppr_bound.bound(g.n, edges, weights, reset, d, ppr_iterations(d), exact_iterate=False)
        err = np.abs(out.astype(np.float64) - x[verts])
        worst = max(worst, float(np.where(err == 0, 0.0, err / bnd[verts]).max()))
    assert worst <= 1.0, worst
