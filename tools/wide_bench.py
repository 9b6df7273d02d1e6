"""One-bit shards with more than 128 rescored candidates: BinaryIndex.search_device_wide over a candidates sweep.

Shapes: 1M x 1024 and 10M x 1024 rows (bf16), 32 queries, k = 10 and 100, candidates 128, 512, 1024 and 2048, the
seeded randn and planted-neighbour row sets of tools/binary_bench.py, bf16 rows on the device (both sizes) and in
page-locked host memory (1M only, to keep pinned memory modest).  Per cell, ms (CUDA events, median over three
alternating rounds of the median of --reps timed calls):
  stage1   crag_search_topk_b1 (candidates 128) or crag_knn_topk_b1 (above): the score-all pass and the select
  rescore  crag_rescore_topk of stage 1's candidates
  total    BinaryIndex.search_device_wide, query quantisation included
and, from one torch.profiler run of --reps stage-1 calls after the timed rounds, the kernel time of the select
(knn_select_kernel) and of the score-all pass (search_topk_kernel) per call.  recall@k is against the bf16 scan's ids
(crag_search_topk).  The card's name and power limit are read in the same run.

  python tools/wide_bench.py [--sizes 1000000,10000000] [--out DIR]   (one JSON line per cell; --out also writes
  DIR/wide_bench.json)
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from binary_bench import make_rows  # noqa: E402
from quant_bench import card, time_ms  # noqa: E402

CANDIDATES = (128, 512, 1024, 2048)


def kernel_ms(fn, reps):
    """Per-call CUDA time of the select and score-all kernels of `fn`, from one profiler run."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {"select": 0.0, "score_all": 0.0}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if "knn_select_kernel" in e.key:
            out["select"] += us / 1000 / reps
        elif "search_topk_kernel" in e.key:
            out["score_all"] += us / 1000 / reps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000000,10000000")
    ap.add_argument("--dim", type=int, default=1024)
    ap.add_argument("--nq", type=int, default=32)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None, help="directory for wide_bench.json (default: print only)")
    a = ap.parse_args()

    import numpy as np
    import torch

    from comorag_b200 import _native
    from comorag_b200.binary import BinaryIndex
    from comorag_b200.index import DenseIndex, knn_chunk
    from comorag_b200.quantized import quantize_rows

    if not torch.cuda.is_available():
        raise SystemExit("wide_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    lib = _native.load()
    result = {"card": card(), "dim": a.dim, "nq": a.nq, "cells": []}
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    st = torch.cuda.current_stream(dev).cuda_stream
    for n in [int(s) for s in a.sizes.split(",")]:
        for planted in (False, True):
            g = torch.Generator(device=dev).manual_seed(n + planted)
            q = torch.nn.functional.normalize(torch.randn((a.nq, a.dim), generator=g, device=dev), dim=1).bfloat16()
            rows = make_rows(n, a.dim, q, planted, g, dev)
            ix = DenseIndex.from_tensor(rows)
            places = {"device": BinaryIndex.from_dense(ix, "device")}
            if n <= 1_000_000:
                places["host"] = BinaryIndex.from_dense(ix, "host")
            bd = places["device"]
            q8, qs = quantize_rows(q, bd.dim8)
            for k in (10, 100):
                want = ix.search_device(q, k)[0].cpu().numpy()
                for c in CANDIDATES:
                    c_ids = torch.empty((a.nq, c), dtype=torch.int64, device=dev)
                    c_sc = torch.empty((a.nq, c), dtype=torch.float32, device=dev)
                    wide = c > 128
                    if wide:
                        ws_bytes = lib.crag_knn_code_workspace_bytes(n, knn_chunk(a.nq, n))
                    else:
                        ws_bytes = lib.crag_search_workspace_bytes(a.nq, c)
                    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
                    name = "crag_knn_topk_b1" if wide else "crag_search_topk_b1"

                    def stage1():
                        _native.check(getattr(lib, name)(bd._codes.data_ptr(), bd._scales.data_ptr(), n, bd.dim8,
                                                         bd._codes.shape[1], 0, q8.data_ptr(), qs.data_ptr(), a.nq, c,
                                                         c_ids.data_ptr(), c_sc.data_ptr(), 0, ws.data_ptr(), ws.numel(),
                                                         st), name)
                    stage1()
                    out_i = torch.empty((a.nq, k), dtype=torch.int64, device=dev)
                    out_s = torch.empty((a.nq, k), dtype=torch.float32, device=dev)
                    for where, bix in places.items():
                        r = bix._rows

                        def rescore():
                            _native.check(lib.crag_rescore_topk(r.data_ptr(), n, bix.dim_pad, r.stride(0), 0,
                                                                q.data_ptr(), a.nq, c_ids.data_ptr(), c, k,
                                                                out_i.data_ptr(), out_s.data_ptr(), st),
                                          "crag_rescore_topk")

                        paths = {"stage1": stage1, "rescore": rescore, "total": lambda: bix.search_device_wide(q, k, c)}
                        times = {p: [] for p in paths}
                        for _ in range(3):     # alternate the paths: drift of a shared host hits all of them alike
                            for p, fn in paths.items():
                                times[p].append(time_ms(fn, a.warmup, a.reps))
                        ms = {p: float(np.median(v)) for p, v in times.items()}
                        got = bix.search_device_wide(q, k, c)[0].cpu().numpy()
                        rec = {"n": n, "rows": "planted" if planted else "randn", "bf16_rows": where, "k": k,
                               "candidates": c, "ms": ms, "ms_runs": times,
                               "kernel_ms": kernel_ms(stage1, a.reps) if where == "device" else None,
                               f"recall_at_{k}": float(np.mean([len(set(got[j]) & set(want[j])) / k
                                                                 for j in range(a.nq)])),
                               "workspace_bytes": ws_bytes, "q_chunk": knn_chunk(a.nq, n) if wide else None,
                               "rescore_bytes": a.nq * c * bix.dim_pad * 2}
                        print(json.dumps(rec), flush=True)
                        result["cells"].append(rec)
                        if a.out:
                            with open(os.path.join(a.out, "wide_bench.json"), "w") as f:
                                json.dump(result, f, indent=1)
                    del ws, c_ids, c_sc
            del ix, places, bd, rows
            torch.cuda.empty_cache()
    print(json.dumps({"card": result["card"]}))


if __name__ == "__main__":
    main()
