"""crag_ppr_batch on the device: column b of every batched call is bit-identical to crag_ppr on reset b alone --
hand graphs, a ComoRAG-shaped graph, a power-law graph and a star whose hub has 2^20 neighbours, at d in {0, 0.5,
0.85}, B in {1, 2, 3, 5, 12, 32, 33} (every width; 33: two calls through DeviceGraph's chunking), with and without out_vertices.  Plus:
bit-identical repeats on two streams, argument errors before any launch, reset_vector's row errors, and coalescing:
16 threads calling personalized_pagerank at once through the graph's Batcher get exactly their lone results, also
through the rebound run_ppr."""
import os
import sys
import threading

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

from comorag_b200 import _native  # noqa: E402
from comorag_b200 import comorag_methods as cm  # noqa: E402
from comorag_b200.graph import DeviceGraph, ppr_iterations  # noqa: E402
from test_ppr_gpu import GRAPHS, D85  # noqa: E402

pytestmark = pytest.mark.gpu
_dev_cache = {}


def _device_graph(name):
    if name not in _dev_cache:
        n, e, w = GRAPHS[name]
        _dev_cache[name] = DeviceGraph.from_edges(n, torch.as_tensor(e, device="cuda"), torch.as_tensor(w, device="cuda"))
    return _dev_cache[name]


def _resets(n, count, seed):
    """count distinct resets: uniform, mass on the last vertex (isolated in most graphs), on vertex 0, then random
    sparse ones."""
    rng = np.random.default_rng(seed)
    r = rng.uniform(0, 1, (count, n)) * (rng.uniform(size=(count, n)) < 0.2)
    r[:, 0] += 1.0
    r[0] = 1.0
    if count > 1:
        r[1] = 0.0
        r[1, -1] = 1.0
    if count > 2:
        r[2] = 0.0
        r[2, 0] = 1.0
    return r


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("name", list(GRAPHS))
@pytest.mark.parametrize("d", [0.0, 0.5, D85])
def test_batched_columns_are_bit_identical_to_crag_ppr(name, d):
    g = _device_graph(name)
    T = ppr_iterations(d)
    v = g.reset_vector(_resets(g.n, 33, len(name)))
    sub = torch.as_tensor(np.random.default_rng(3).choice(g.n, min(g.n, 500), replace=False), device="cuda")
    for verts in (None, sub):
        single = torch.stack([g.ppr_iterate(v[b], d, T, verts) for b in range(33)])
        for B in (1, 2, 3, 5, 12, 32, 33):          # every width: 2, 4, 8, 16, 32 (and 32 + 1)
            got = g.ppr_iterate(v[:B], d, T, verts)
            assert got.shape == single[:B].shape
            for b in range(B):
                assert torch.equal(_bits(got[b]), _bits(single[b])), f"{name} d={d} B={B} column {b}"


def test_batched_iteration_counts_and_the_reset_rows_of_personalized_pagerank():
    g = _device_graph("comorag-shaped")
    resets = _resets(g.n, 7, 11)
    for T in (0, 1, 2):
        v = g.reset_vector(resets)
        got = g.ppr_iterate(v, 0.5, T)
        for b in range(7):
            assert torch.equal(_bits(got[b]), _bits(g.ppr_iterate(v[b], 0.5, T)))
    got = g.personalized_pagerank(resets, 0.5)
    for b in range(7):
        assert torch.equal(_bits(got[b]), _bits(g.personalized_pagerank(resets[b], 0.5)))


def test_bit_identical_across_repeats_and_streams():
    g = _device_graph("power-law")
    v = g.reset_vector(_resets(g.n, 32, 5))
    first = g.ppr_iterate(v, 0.5, 35)
    side = torch.cuda.Stream()
    for st in (None, side, None, side):
        again = g.ppr_iterate(v, 0.5, 35, stream=st)
        torch.cuda.synchronize()
        assert torch.equal(_bits(first), _bits(again))


def test_argument_errors_return_before_any_launch():
    lib = _native.load()
    g = _device_graph("path")
    v = g.reset_vector(_resets(g.n, 4, 1))
    ws_bytes = lib.crag_ppr_batch_workspace_bytes(g.n, g.nnz, 4)
    assert ws_bytes > 0
    ws = torch.empty(ws_bytes + 256, dtype=torch.uint8, device="cuda")
    out = torch.full((4, g.n), -7.0, device="cuda")
    sub = torch.zeros(3, dtype=torch.int32, device="cuda")
    base = dict(row_ptr=g.row_ptr.data_ptr(), col=g.col.data_ptr(), coef=g.coef.data_ptr(), n=g.n, nnz=g.nnz,
                resets=v.data_ptr(), batch=4, d=0.5, T=35, verts=None, n_out=g.n, out=out.data_ptr(), ws=ws.data_ptr(),
                ws_bytes=ws_bytes)

    def call(**kw):
        a = {**base, **kw}
        return lib.crag_ppr_batch(a["row_ptr"], a["col"], a["coef"], a["n"], a["nnz"], a["resets"], a["batch"], a["d"],
                                  a["T"], a["verts"], a["n_out"], a["out"], a["ws"], a["ws_bytes"], None)
    INVALID, WORKSPACE = -1, -3
    for kw, rc in [(dict(batch=0), INVALID), (dict(batch=33), INVALID), (dict(n=0), INVALID), (dict(nnz=-1), INVALID),
                   (dict(d=1.0), INVALID), (dict(d=-0.1), INVALID), (dict(d=float("nan")), INVALID), (dict(T=-1), INVALID),
                   (dict(n_out=3), INVALID), (dict(verts=sub.data_ptr(), n_out=-1), INVALID),
                   (dict(row_ptr=None), INVALID), (dict(col=None), INVALID), (dict(coef=None), INVALID),
                   (dict(resets=None), INVALID), (dict(out=None), INVALID), (dict(ws=None), INVALID),
                   (dict(ws=ws.data_ptr() + 4), INVALID), (dict(ws_bytes=ws_bytes - 1), WORKSPACE)]:
        assert call(**kw) == rc, kw
        assert lib.crag_last_error().decode().startswith("crag_ppr_batch")
    torch.cuda.synchronize()
    assert (out == -7.0).all()                   # nothing was launched
    assert lib.crag_ppr_batch_workspace_bytes(g.n, g.nnz, 0) == 0
    assert lib.crag_ppr_batch_workspace_bytes(g.n, g.nnz, 33) == 0
    assert lib.crag_ppr_batch_workspace_bytes(0, 5, 2) == 0 and lib.crag_ppr_batch_workspace_bytes(5, -1, 2) == 0
    big = _device_graph("power-law")             # wider batches need more workspace once n * W outgrows 256 B
    assert lib.crag_ppr_batch_workspace_bytes(big.n, big.nnz, 32) > lib.crag_ppr_batch_workspace_bytes(big.n, big.nnz, 4)
    assert lib.crag_ppr_batch_workspace_bytes(big.n, big.nnz, 3) == lib.crag_ppr_batch_workspace_bytes(big.n, big.nnz, 4)
    assert lib.crag_version() == 1003
    assert call() == 0
    torch.cuda.synchronize()
    assert torch.allclose(out.sum(1), torch.ones(4, device="cuda"), atol=1e-5)


def test_reset_vector_names_the_row_without_mass():
    g = _device_graph("path")
    r = _resets(g.n, 5, 2)
    r[3] = 0.0
    r[3, 1] = -2.0                               # sanitised to 0
    with pytest.raises(ValueError, match="row 3"):
        g.reset_vector(r)
    r[3, 2] = float("inf")
    with pytest.raises(ValueError, match="row 3"):
        g.personalized_pagerank(r)


def _concurrent(call, inputs, bad=None):
    """call(x) from one thread per input, all released together; returns (results, errors) by index."""
    barrier = threading.Barrier(len(inputs))
    results, errors = {}, {}

    def work(i):
        barrier.wait()
        try:
            results[i] = call(inputs[i]).cpu()
        except Exception as e:              # noqa: BLE001 -- collected and asserted on below
            errors[i] = e
    threads = [threading.Thread(target=work, args=(i,)) for i in range(len(inputs))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    return results, errors


def test_concurrent_calls_coalesce_and_each_gets_its_lone_result():
    n, e, w = GRAPHS["comorag-shaped"]
    g = DeviceGraph.from_edges(n, torch.as_tensor(e, device="cuda"), torch.as_tensor(w, device="cuda"))
    resets = list(_resets(g.n, 16, 21))
    resets[9] = np.zeros(g.n)                    # this caller's reset is invalid: only it may fail
    passages = torch.arange(1200, 4200, device="cuda")
    want = {}
    for i, r in enumerate(resets):
        if i != 9:
            want[i] = g.personalized_pagerank(r, 0.5, vertices=passages).cpu()
    # every call through the Batcher, with a long window: the 15 valid calls all meet in it
    batcher = g.enable_batching(max_wait_s=2.0, lone_calls_direct=False)
    try:
        results, errors = _concurrent(lambda r: g.personalized_pagerank(r, 0.5, vertices=passages), resets)
    finally:
        g.disable_batching()
    assert set(errors) == {9} and isinstance(errors[9], ValueError), errors
    assert set(results) == set(want)
    for i in want:
        assert torch.equal(_bits(results[i]), _bits(want[i])), i
    assert batcher.items == 15 and batcher.batches < batcher.items
    # once closed, calls run directly again
    assert g.batcher is None
    assert torch.equal(_bits(g.personalized_pagerank(resets[0], 0.5, vertices=passages).cpu()), _bits(want[0]))


def test_an_explicit_stream_bypasses_the_batcher():
    g = _device_graph("power-law")
    r = _resets(g.n, 1, 4)[0]
    want = g.personalized_pagerank(r)
    batcher = g.enable_batching(max_wait_s=2.0, lone_calls_direct=False)
    try:
        side = torch.cuda.Stream()
        got = g.personalized_pagerank(r, stream=side)
        side.synchronize()
        assert batcher.items == 0
        assert torch.equal(_bits(got), _bits(want))
    finally:
        g.disable_batching()


def test_a_lone_caller_runs_directly_and_batching_settings_are_not_silently_changed():
    g = _device_graph("comorag-shaped")
    resets = _resets(g.n, 4, 41)
    want = [g.personalized_pagerank(r) for r in resets]
    batcher = g.enable_batching()
    try:
        for r, w in zip(resets, want):
            got = g.personalized_pagerank(r)
            torch.cuda.synchronize()             # nothing is in flight when the next call starts
            assert torch.equal(_bits(got), _bits(w))
        assert batcher.items == 0                # each call found itself alone: crag_ppr on the caller's stream
        assert g.enable_batching() is batcher
        with pytest.raises(ValueError, match="already on"):
            g.enable_batching(max_wait_s=2.0)
        with pytest.raises(ValueError, match="already on"):
            g.enable_batching(lone_calls_direct=False)
    finally:
        g.disable_batching()
    assert g.enable_batching(max_wait_s=2.0) is not batcher
    g.disable_batching()


def test_a_dropped_graph_is_freed_and_its_batcher_closed():
    import gc
    import weakref
    n, e, w = GRAPHS["path"]
    g = DeviceGraph.from_edges(n, torch.as_tensor(e, device="cuda"), torch.as_tensor(w, device="cuda"))
    batcher = g.enable_batching(lone_calls_direct=False)
    g.personalized_pagerank(np.ones(n)).cpu()    # the worker thread has run the graph's batch function
    ref = weakref.ref(g)
    del g
    gc.collect()
    assert ref() is None
    assert batcher._closed and not batcher._t.is_alive()


class _Graph:
    def __init__(self, n, e):
        self.n, self.e = n, e

    def vcount(self):
        return self.n

    def ecount(self):
        return self.e


def test_concurrent_run_ppr_through_the_binding():
    """comorag_methods.run_ppr on a fake rag (as tools/ppr_bench.py builds one): 16 threads at once, with the graph's
    batcher on, each get the ranking run_ppr gives them alone."""
    n, e, w = GRAPHS["comorag-shaped"]
    g = DeviceGraph.from_edges(n, torch.as_tensor(e, device="cuda"), torch.as_tensor(w, device="cuda"))
    rag = type("Rag", (), {})()
    rag.graph = _Graph(n, len(e))
    rag._crag_graph = ((n, len(e)), g)
    rag.passage_node_idxs = list(range(1200, 4200))
    resets = list(_resets(n, 16, 31))
    alone = [cm.run_ppr(rag, r, 0.5) for r in resets]
    batcher = g.enable_batching(max_wait_s=2.0, lone_calls_direct=False)
    try:
        barrier = threading.Barrier(16)
        got = {}

        def work(i):
            barrier.wait()
            got[i] = cm.run_ppr(rag, resets[i], 0.5)
        threads = [threading.Thread(target=work, args=(i,)) for i in range(16)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
    finally:
        g.disable_batching()
    assert batcher.items == 16 and batcher.batches < 16
    for i in range(16):
        np.testing.assert_array_equal(got[i][0], alone[i][0])
        np.testing.assert_array_equal(got[i][1].view(np.uint64), alone[i][1].view(np.uint64))


def test_device_graph_of_the_binding_batches_and_a_rebuild_closes_the_old_batcher():
    n, e, w = GRAPHS["triangle + isolated"]

    class G(_Graph):
        def get_edgelist(self):
            return [tuple(x) for x in e[:self.e]]

        @property
        def es(self):
            return {"weight": list(w[:self.e])}
    rag = type("Rag", (), {})()
    rag.graph = G(n, len(e) - 1)
    first = cm._device_graph(rag)
    assert first.batcher is not None
    rag.graph = G(n, len(e))
    second = cm._device_graph(rag)
    assert second is not first and second.batcher is not None and first.batcher is None
    r = np.ones(n)
    assert torch.equal(_bits(first.personalized_pagerank(r)), _bits(first.ppr_iterate(first.reset_vector(r), 0.5, 35)))
    second.disable_batching()
