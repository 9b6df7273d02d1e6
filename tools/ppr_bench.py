"""Device PPR at ComoRAG scale: crag_ppr per call and per iteration, and the rebound graph_search_with_fact_entities
end to end, on seeded synthetic ComoRAG-shaped graphs generated on the device.

Graph shape (per passage count P): P // 2 entities, P passages each linked to 10-20 random entities, 2P fact edges
between entities in both orientations (ComoRAG.py:641-644 adds both), P // 10 synonymy edges with weights in
[0.8, 1], and P // 100 isolated summary vertices.  Bandwidth is algorithmic: per iteration 8 nnz (col + coef) +
4 nnz (y gathers) + 8 n (reset read, y write) bytes over the measured time, against the H100 SXM data-sheet 3.35 TB/s;
the y gathers may hit L2, so this can exceed what HBM traffic alone would allow.

    python tools/ppr_bench.py --passages 1000000 10000000 --out ppr_bench.json
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from comorag_b200 import comorag_methods as cm  # noqa: E402
from comorag_b200.embedding_store import compute_mdhash_id  # noqa: E402
from comorag_b200.graph import DeviceGraph, ppr_iterations  # noqa: E402

HBM_PEAK = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def comorag_graph(passages: int, seed: int, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    ent = passages // 2
    summaries = passages // 100
    links = torch.randint(10, 21, (passages,), generator=g, device=dev)
    p = torch.repeat_interleave(torch.arange(passages, device=dev), links) + ent
    pe = torch.randint(0, ent, (p.numel(),), generator=g, device=dev)
    fa = torch.randint(0, ent, (2 * passages,), generator=g, device=dev)
    fb = torch.randint(0, ent, (2 * passages,), generator=g, device=dev)
    keep = fa != fb
    fa, fb = fa[keep], fb[keep]
    sa = torch.randint(0, ent, (passages // 10,), generator=g, device=dev)
    sb = torch.randint(0, ent, (passages // 10,), generator=g, device=dev)
    keep = sa != sb
    sa, sb = sa[keep], sb[keep]
    edges = torch.cat([torch.stack([p, pe], 1), torch.stack([fa, fb], 1), torch.stack([fb, fa], 1),
                       torch.stack([sa, sb], 1)])
    weights = torch.cat([torch.ones(p.numel() + 2 * fa.numel(), dtype=torch.float64, device=dev),
                         torch.rand(sa.numel(), generator=g, device=dev, dtype=torch.float64) * 0.2 + 0.8])
    n = ent + passages + summaries
    return n, ent, edges, weights


def time_calls(fn, calls: int, warmup: int = 3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(calls):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), float(np.min(ms)), float(np.max(ms))


class _Graph:
    def __init__(self, n, e):
        self.n, self.e = n, e

    def vcount(self):
        return self.n

    def ecount(self):
        return self.e


def bench(passages: int, calls: int, seed: int):
    dev = torch.device("cuda", 0)
    t0 = time.perf_counter()
    n, ent, edges, weights = comorag_graph(passages, seed, dev)
    dg = DeviceGraph.from_edges(n, edges, weights)
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t0
    n_edges = edges.shape[0]
    del edges, weights
    rng = np.random.default_rng(seed)
    reset = np.zeros(n)
    reset[rng.integers(0, ent, 30)] = rng.uniform(0.1, 1.0, 30)
    reset[ent:ent + passages] = rng.uniform(0, 1, passages) * 0.005
    v = dg.reset_vector(reset)
    passage_v = torch.arange(ent, ent + passages, device=dev)
    T = ppr_iterations(0.5)
    call_ms = time_calls(lambda: dg.ppr_iterate(v, 0.5, T, passage_v), calls)
    t0_ms = time_calls(lambda: dg.ppr_iterate(v, 0.5, 0, passage_v), calls)
    iter_ms = (call_ms[0] - t0_ms[0]) / T
    bytes_iter = 12 * dg.nnz + 8 * n
    out = {"passages": passages, "vertices": n, "edges_in": n_edges, "nnz": dg.nnz, "iterations": T,
           "csr_build_s": round(build_s, 3),
           "crag_ppr_ms": {"median": call_ms[0], "min": call_ms[1], "max": call_ms[2]},
           "crag_ppr_T0_ms": t0_ms[0], "per_iteration_ms": iter_ms,
           "bytes_per_iteration": bytes_iter, "per_iteration_TBps": bytes_iter / (iter_ms * 1e-3) / 1e12,
           "share_of_3.35TBps": bytes_iter / (iter_ms * 1e-3) / HBM_PEAK}

    # the rebound graph search end to end: phrase weights, passage scatter, crag_ppr, device ranking, D2H of the
    # full passage ranking (the DPR ranking comes precomputed, as the retrieval wave hands it over)
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
    facts = [(phrases[i], "rel", phrases[i + 1]) for i in range(0, 30, 2)]
    fact_scores = rng.uniform(0.2, 1, 100).astype(np.float32)
    kw = dict(query="q", link_top_k=5, query_fact_scores=fact_scores, top_k_facts=facts,
              top_k_fact_indices=list(range(len(facts))), passage_node_weight=0.005)
    for _ in range(2):
        cm.graph_search_with_fact_entities(rag, **kw)
    wall = []
    for _ in range(max(5, calls // 4)):
        t = time.perf_counter()
        cm.graph_search_with_fact_entities(rag, **kw)
        wall.append((time.perf_counter() - t) * 1e3)
    out["graph_search_ms"] = {"median": float(np.median(wall)), "min": float(np.min(wall)), "max": float(np.max(wall))}
    del dg, rag
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, nargs="+", default=[1_000_000, 10_000_000])
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ppr_bench needs a GPU")
    res = {"card": card(), "torch": torch.__version__, "runs": []}
    for p in a.passages:
        res["runs"].append(bench(p, a.calls, a.seed))
        print(json.dumps(res["runs"][-1]), flush=True)
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
