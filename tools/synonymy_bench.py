"""The synonymy edges of add_synonymy_edges, old path against new, on one GPU.

Old path: retrieval.retrieve_knn(k = 2047) (crag_knn_topk: 2 047 (id, score) pairs per entity copied to the host and
turned into Python lists) followed by the reference walk over those lists (tests/synonymy_oracle.edges_from_knn).
New path: comorag_methods.add_synonymy_edges (crag_knn_threshold: only the kept edges leave the device).  Both run
in one process, alternating, on planted synonym groups (sizes 1 to 3 000) at N entities and dim 1 024; the edges
must be equal as lists.  Reported per N: wall time of each path, device time of one crag_knn_threshold call against
crag_knn_topk at k = 2047 (CUDA events, same queries and shard), bytes copied device to host, peak host RSS growth,
and the card name and power limit the numbers were taken at.

    python tools/synonymy_bench.py --n 50000 200000 --out /tmp/synonymy_bench.json
"""
from __future__ import annotations

import argparse
import json
import os
import resource
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                               text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        power = f"unknown ({type(e).__name__})"
    return name, power


def planted(n, dim, seed):
    rng = np.random.default_rng(seed)
    sizes = [3000, 1000, 300, 100, 30, 10, 3, 2]
    groups = np.concatenate([np.full(s, g) for g, s in enumerate(sizes)] + [len(sizes) + np.arange(n - sum(sizes))])
    centers = rng.standard_normal((int(groups.max()) + 1, dim)).astype(np.float32)
    return centers[groups] + 0.3 * rng.standard_normal((n, dim)).astype(np.float32)


def rss_mb():
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024.0


class D2HCounter:
    """Counts bytes of device-to-host copies made through Tensor.cpu() while active."""

    def __init__(self):
        self.bytes = 0
        self._real = torch.Tensor.cpu

    def __enter__(self):
        real = self._real

        def cpu(t, *a, **kw):
            if t.is_cuda:
                self.bytes += t.numel() * t.element_size()
            return real(t, *a, **kw)
        torch.Tensor.cpu = cpu
        return self

    def __exit__(self, *exc):
        torch.Tensor.cpu = self._real


def old_path(keys, texts, emb):
    import synonymy_oracle as so
    from comorag_b200.retrieval import retrieve_knn
    lists = retrieve_knn(keys, keys, emb, emb, k=2047)
    stats = {}
    for edge, score in so.edges_from_knn(lists, dict(zip(keys, texts)), 0.8, 101):
        stats[edge] = score
    return stats


def new_path(keys, texts, emb):
    from comorag_b200 import comorag_methods as cm
    store = SimpleNamespace(get_text_for_all_rows=lambda: {h: {"hash_id": h, "content": t} for h, t in zip(keys, texts)},
                            get_embeddings=lambda ks: emb)
    cfg = SimpleNamespace(synonymy_edge_topk=2047, synonymy_edge_sim_threshold=0.8)
    rag = SimpleNamespace(entity_embedding_store=store, global_config=cfg, node_to_node_stats={})
    cm.add_synonymy_edges(rag)
    return rag.node_to_node_stats


def device_times(emb, reps=3):
    """ms of one crag_knn_threshold call and one crag_knn_topk(k = 2047) call over the whole self-join."""
    from comorag_b200.index import fp32_threshold
    from comorag_b200.retrieval import knn_key_index
    index = knn_key_index(emb)
    q = index.matrix().contiguous() if index.dim == index.dim_pad else index._buf[: index.n_rows].contiguous()
    rows = torch.arange(index.n_rows, device=index.device)
    out = {}
    for name, fn in (("threshold", lambda: index.search_threshold_device(q, fp32_threshold(0.8), 101, 2047, self_rows=rows)),
                     ("topk_2047", lambda: index._search_device_knn(q, 2047, None))):
        fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        out[name] = float(np.median(ts))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[50_000, 200_000])
    ap.add_argument("--dim", type=int, default=1024)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "synonymy_bench needs a GPU"
    name, power = card()
    results = {"card": name, "power_limit": power, "dim": args.dim, "runs": []}
    for n in args.n:
        emb = planted(n, args.dim, 1)
        keys = [f"entity-{i:07d}" for i in range(n)]
        texts = [f"entity {i}" for i in range(n)]
        new_path(keys[:2000], texts[:2000], emb[:2000])               # warm-up: library load, kernels, allocator
        row = {"n": n}
        for label, fn in (("new", new_path), ("old", old_path)):   # new first: the peak-RSS growth of each is its own
            rss0 = rss_mb()
            torch.cuda.synchronize()
            with D2HCounter() as d2h:
                t0 = time.perf_counter()
                stats = fn(keys, texts, emb)
                torch.cuda.synchronize()
                row[f"{label}_wall_s"] = time.perf_counter() - t0
            row[f"{label}_d2h_bytes"] = d2h.bytes
            row[f"{label}_peak_rss_growth_mb"] = rss_mb() - rss0
            row[f"{label}_edges"] = len(stats)
            row[f"_{label}"] = stats
        assert list(row.pop("_old").items()) == list(row.pop("_new").items()), "edges differ"
        row.update({f"device_ms_{k}": v for k, v in device_times(emb).items()})
        results["runs"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({"card": name, "power_limit": power}))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
