"""Multi-source PPR at ComoRAG scale: one crag_ppr_batch call for B resets against B sequential crag_ppr calls, and
16 concurrent graph searches with the graph's Batcher on and off, on the seeded ComoRAG-shaped graphs of
tools/ppr_bench.py.

Per B in {1, 2, 4, 8, 16, 32}: the batched call and the B sequential calls alternate in one process after warm-up;
each side's time is the median over --calls repeats (CUDA events).  Every column of every timed batched call is
compared bit for bit with the sequential outputs.  Algorithmic bytes per iteration: crag_ppr reads col + coef
(8 nnz), gathers y (4 nnz) and reads the reset and writes y (8 n); crag_ppr_batch reads col + coef once
(8 nnz), gathers W floats per nonzero (4 W nnz) and reads V and writes y (8 W n), W the padded batch width; both
against the H100 SXM data-sheet 3.35 TB/s.

Lone calls: one personalized_pagerank at a time with batching off, on (a lone caller runs crag_ppr directly), and
forced through the Batcher (lone_calls_direct=False), wall clock to the result on the host.

End to end: 16 threads each run the rebound graph_search_with_fact_entities (on the fake rag of ppr_bench.py),
started together, wall clock until every thread is done (each ends in a device-to-host copy); the same alone.  With
batching on, the rag's graph comes from comorag_methods._device_graph, which turns batching on as the binding does.

    python tools/ppr_batch_bench.py --passages 1000000 10000000 --out ppr_batch_bench.json
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import threading
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from comorag_b200 import comorag_methods as cm  # noqa: E402
from comorag_b200.embedding_store import compute_mdhash_id  # noqa: E402
from comorag_b200.graph import DeviceGraph, ppr_iterations  # noqa: E402
from ppr_bench import HBM_PEAK, _Graph, card, comorag_graph  # noqa: E402

BATCHES = (1, 2, 4, 8, 16, 32)


def _events_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b), out


def _width(batch):
    w = 2
    while w < batch:
        w *= 2
    return w


def bench_batches(dg, resets, passage_v, T, calls):
    n, nnz = dg.n, dg.nnz
    v = dg.reset_vector(resets)                      # [32, n]
    rows = []
    for B in BATCHES:
        vb = v[:B].contiguous()

        def batched():
            return dg.ppr_iterate(vb, 0.5, T, passage_v)

        def sequential():
            return [dg.ppr_iterate(vb[b], 0.5, T, passage_v) for b in range(B)]
        for _ in range(2):                           # warm-up: allocator, caches, clocks
            batched()
            sequential()
        t_batch, t_seq, identical = [], [], True
        for _ in range(calls):
            ms, got = _events_ms(batched)
            t_batch.append(ms)
            ms, want = _events_ms(sequential)
            t_seq.append(ms)
            for b in range(B):
                identical &= bool(torch.equal(got[b].view(torch.int32), want[b].view(torch.int32)))
        W = _width(B) if B > 1 else 1
        bytes_iter = 8 * nnz + 4 * W * nnz + 8 * W * n if B > 1 else 12 * nnz + 8 * n
        mb, ms_ = float(np.median(t_batch)), float(np.median(t_seq))
        rows.append({"B": B, "width": W, "batched_ms": {"median": mb, "min": float(np.min(t_batch)), "max": float(np.max(t_batch))},
                     "sequential_ms": {"median": ms_, "min": float(np.min(t_seq)), "max": float(np.max(t_seq))},
                     "per_query_ms_batched": mb / B, "per_query_ms_sequential": ms_ / B, "speedup": ms_ / mb,
                     "bytes_per_iteration": bytes_iter,
                     "batched_TBps_per_iteration": bytes_iter * T / (mb * 1e-3) / 1e12 if T else None,
                     "share_of_3.35TBps": bytes_iter * T / (mb * 1e-3) / HBM_PEAK if T else None,
                     "bit_identical": identical})
        print(json.dumps(rows[-1]), flush=True)
    return rows


def fake_rag(dg, n, n_edges, ent, passages, rng):
    rag = type("Rag", (), {})()
    rag.graph = _Graph(n, n_edges)
    rag._crag_graph = ((n, n_edges), dg)
    phrases = [f"entity {i}" for i in range(40)]
    keys = [compute_mdhash_id(p, prefix="entity-") for p in phrases]
    rag.node_name_to_vertex_idx = {k: int(i) for k, i in zip(keys, rng.choice(ent, len(keys), replace=False))}
    rag.ent_node_to_num_chunk = {k: int(c) for k, c in zip(keys, rng.integers(1, 5, len(keys)))}
    rag.passage_node_idxs = list(range(ent, ent + passages))
    rag.run_ppr = lambda reset_prob, damping=0.5: cm.run_ppr(rag, reset_prob, damping)
    dpr_ids = rng.permutation(passages)
    dpr_scores = np.sort(rng.uniform(0, 1, passages).astype(np.float32))[::-1].copy()
    rag.dense_passage_retrieval = lambda query, need_cluster=False: (dpr_ids.copy(), dpr_scores.copy())
    return rag, phrases


def graph_search_kwargs(phrases, rng, i):
    """Thread i's query: its own facts and fact scores, so every graph search has its own reset."""
    order = rng.permutation(len(phrases))
    facts = [(phrases[order[j]], "rel", phrases[order[j + 1]]) for j in range(0, 30, 2)]
    fact_scores = rng.uniform(0.2, 1, 100).astype(np.float32)
    return dict(query=f"q{i}", link_top_k=5, query_fact_scores=fact_scores, top_k_facts=facts,
                top_k_fact_indices=list(range(len(facts))), passage_node_weight=0.005)


def wall_threads(rag, kws, repeats):
    """Wall ms for len(kws) threads running one graph search each, released together; median over repeats."""
    out_ms, results = [], None
    for _ in range(repeats):
        barrier = threading.Barrier(len(kws) + 1)
        res = {}

        def work(i):
            barrier.wait()
            res[i] = cm.graph_search_with_fact_entities(rag, **kws[i])
        threads = [threading.Thread(target=work, args=(i,)) for i in range(len(kws))]
        for t in threads:
            t.start()
        barrier.wait()
        t0 = time.perf_counter()
        for t in threads:
            t.join()
        out_ms.append((time.perf_counter() - t0) * 1e3)
        results = res
    return {"median": float(np.median(out_ms)), "min": float(np.min(out_ms)), "max": float(np.max(out_ms))}, results


def through_device_graph(rag, dg):
    """Let comorag_methods._device_graph build the rag's graph, as the binding does on first use (turning batching
    on), with from_igraph answering with the already-built graph instead of re-reading 19M+ edges."""
    real = DeviceGraph.__dict__["from_igraph"]
    rag._crag_graph = None
    DeviceGraph.from_igraph = classmethod(lambda cls, g, device=None: dg)
    try:
        assert cm._device_graph(rag) is dg and dg.batcher is not None
    finally:
        DeviceGraph.from_igraph = real


def bench_lone_calls(dg, resets, passage_v, T, repeats):
    """One personalized_pagerank call at a time, wall clock to the result on the host: batching off, batching on
    (a lone caller runs directly), and the same call forced through the Batcher's thread and stream."""
    out = {}
    r = resets[0]

    def timed(fn):
        ms = []
        for _ in range(repeats + 1):
            t = time.perf_counter()
            fn().cpu()
            ms.append((time.perf_counter() - t) * 1e3)
        ms = ms[1:]
        return {"median": float(np.median(ms)), "min": float(np.min(ms)), "max": float(np.max(ms))}
    for label in ("off", "on", "through the batcher", "off again", "on again", "through the batcher again"):
        if label.startswith("off"):
            out[f"lone_call_ms_batching_{label}"] = timed(lambda: dg.personalized_pagerank(r, 0.5, vertices=passage_v))
        elif label.startswith("on"):
            b = dg.enable_batching()
            out[f"lone_call_ms_batching_{label}"] = timed(lambda: dg.personalized_pagerank(r, 0.5, vertices=passage_v))
            out[f"lone_call_batcher_items_{label}"] = b.items
            dg.disable_batching()
        else:
            b = dg.enable_batching(lone_calls_direct=False)
            out[f"lone_call_ms_{label}"] = timed(lambda: dg.personalized_pagerank(r, 0.5, vertices=passage_v))
            dg.disable_batching()
    return out


def bench_end_to_end(dg, n, n_edges, ent, passages, seed, repeats):
    rng = np.random.default_rng(seed + 1)
    rag, phrases = fake_rag(dg, n, n_edges, ent, passages, rng)
    kws = [graph_search_kwargs(phrases, rng, i) for i in range(16)]
    out = {}
    for label, on in (("off", False), ("on", True), ("off again", False), ("on again", True)):
        if on:
            through_device_graph(rag, dg)
        wall_threads(rag, kws[:1], 1)               # warm-up
        out[f"16_threads_ms_batching_{label}"], res = wall_threads(rag, kws, repeats)
        out[f"1_thread_ms_batching_{label}"], _ = wall_threads(rag, kws[:1], repeats)
        if on:
            out[f"batcher_{label}"] = {"batches": dg.batcher.batches, "items": dg.batcher.items}
            dg.disable_batching()
            out["identical_with_and_without_batching"] = all(
                np.array_equal(res[i][0], ref[i][0]) and np.array_equal(res[i][1], ref[i][1]) for i in range(16))
        else:
            ref = res
    return out


def bench(passages, calls, seed, repeats, batches=True):
    dev = torch.device("cuda", 0)
    n, ent, edges, weights = comorag_graph(passages, seed, dev)
    dg = DeviceGraph.from_edges(n, edges, weights)
    n_edges = edges.shape[0]
    del edges, weights
    torch.cuda.synchronize()
    rng = np.random.default_rng(seed)
    resets = np.zeros((32, n))
    for b in range(32):
        resets[b, rng.integers(0, ent, 30)] = rng.uniform(0.1, 1.0, 30)
        resets[b, ent:ent + passages] = rng.uniform(0, 1, passages) * 0.005
    passage_v = torch.arange(ent, ent + passages, device=dev)
    T = ppr_iterations(0.5)
    out = {"passages": passages, "vertices": n, "nnz": dg.nnz, "iterations": T}
    if batches:
        out["batches"] = bench_batches(dg, resets, passage_v, T, calls)
    out["lone_calls"] = bench_lone_calls(dg, resets, passage_v, T, repeats)
    print(json.dumps(out["lone_calls"]), flush=True)
    out["end_to_end"] = bench_end_to_end(dg, n, n_edges, ent, passages, seed, repeats)
    print(json.dumps(out["end_to_end"]), flush=True)
    del dg
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, nargs="+", default=[1_000_000, 10_000_000])
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--no-batches", action="store_true", help="skip the batched-vs-sequential sweep")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ppr_batch_bench needs a GPU")
    res = {"card": card(), "torch": torch.__version__, "runs": []}
    for p in a.passages:
        res["runs"].append(bench(p, a.calls, a.seed, a.repeats, not a.no_batches))
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
