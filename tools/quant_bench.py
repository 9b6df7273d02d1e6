"""Int8 shard search against the bf16 scan, alternating the paths in one process.

Shapes: 1M x 1024 and 10M x 1024 random unit rows (bf16), 32 queries, k = 10 and 100 (candidates min(128, 4 k)).
Per shape, ms per pass (CUDA events, median of --reps timed calls after --warmup):
  bf16        crag_search_topk over the bf16 shard
  i8          crag_search_topk_i8 alone (queries already quantised)
  i8+rescore  query quantisation + crag_search_topk_i8 + crag_rescore_topk, bf16 rows on the device
  i8+host     the same with the bf16 rows in page-locked host memory (1M only, to keep pinned memory modest)
plus algorithmic bytes per pass (bf16: 2 n dim; int8: n dim8 + 4 n) and TB/s, recall@k of the int8 path against the
bf16 scan's ids, and device bytes.  The card's name and power limit are read in the same run.

  python tools/quant_bench.py [--sizes 1000000,10000000] [--out DIR]   (one JSON line per shape; --out also writes
  DIR/quant_bench.json)
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        name, power, clock = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # the measurement itself does not depend on it; say what is missing
        import torch
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"not read ({e})", "max_sm_clock": "not read"}


def time_ms(fn, warmup, reps):
    import torch
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000000,10000000")
    ap.add_argument("--dim", type=int, default=1024)
    ap.add_argument("--nq", type=int, default=32)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--out", default=None, help="directory for quant_bench.json (default: print only)")
    a = ap.parse_args()

    import numpy as np
    import torch

    from comorag_b200 import _native
    from comorag_b200.index import DenseIndex
    from comorag_b200.quantized import QuantizedIndex, quantize_rows

    if not torch.cuda.is_available():
        raise SystemExit("quant_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    lib = _native.load()
    result = {"card": card(), "dim": a.dim, "nq": a.nq, "shapes": []}
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    for n in [int(s) for s in a.sizes.split(",")]:
        g = torch.Generator(device=dev).manual_seed(n)
        rows = torch.empty((n, a.dim), dtype=torch.bfloat16, device=dev)
        for r0 in range(0, n, 500_000):
            c = torch.randn((min(500_000, n - r0), a.dim), generator=g, device=dev)
            rows[r0:r0 + c.shape[0]] = torch.nn.functional.normalize(c, dim=1).bfloat16()
            del c
        ix = DenseIndex.from_tensor(rows)
        qd = QuantizedIndex.from_dense(ix, "device")
        qh = QuantizedIndex.from_dense(ix, "host") if n <= 1_000_000 else None
        q = torch.nn.functional.normalize(torch.randn((a.nq, a.dim), generator=g, device=dev), dim=1).bfloat16()
        q8, qs = quantize_rows(q, qd.dim8)
        for k in (10, 100):
            cand = min(128, 4 * k)
            ws_b = lib.crag_search_workspace_bytes(a.nq, k)
            ws_c = lib.crag_search_workspace_bytes(a.nq, cand)
            ws = torch.empty(max(ws_b, ws_c), dtype=torch.uint8, device=dev)
            ids = torch.empty((a.nq, 128), dtype=torch.int64, device=dev)
            sc = torch.empty((a.nq, 128), dtype=torch.float32, device=dev)
            mm = torch.empty((a.nq, 2), dtype=torch.float32, device=dev)
            st = torch.cuda.current_stream(dev).cuda_stream

            def bf16():
                _native.check(lib.crag_search_topk(rows.data_ptr(), n, a.dim, a.dim, 0, q.data_ptr(), a.nq, k,
                                                   ids.data_ptr(), sc.data_ptr(), mm.data_ptr(), ws.data_ptr(),
                                                   ws.numel(), st), "crag_search_topk")

            def i8():
                _native.check(lib.crag_search_topk_i8(qd._codes.data_ptr(), qd._scales.data_ptr(), n, qd.dim8, qd.dim8, 0,
                                                      q8.data_ptr(), qs.data_ptr(), a.nq, cand, ids.data_ptr(),
                                                      sc.data_ptr(), mm.data_ptr(), ws.data_ptr(), ws.numel(), st),
                              "crag_search_topk_i8")

            paths = {"bf16": bf16, "i8": i8, "i8+rescore": lambda: qd.search_device(q, k)}
            if qh is not None:
                paths["i8+host"] = lambda: qh.search_device(q, k)
            times = {p: [] for p in paths}
            for _ in range(3):                 # alternate the paths: drift of a shared host hits all of them alike
                for p, fn in paths.items():
                    times[p].append(time_ms(fn, a.warmup, a.reps))
            ms = {p: float(np.median(v)) for p, v in times.items()}
            want = ix.search_device(q, k)[0].cpu().numpy()
            got = qd.search_device(q, k)[0].cpu().numpy()
            recall = float(np.mean([len(set(got[j]) & set(want[j])) / k for j in range(a.nq)]))
            if qh is not None:
                assert np.array_equal(qh.search_device(q, k)[0].cpu().numpy(), got), "host rows differ from device rows"
            bytes_bf16 = 2 * n * a.dim
            bytes_i8 = n * qd.dim8 + 4 * n
            rec = {"n": n, "k": k, "candidates": cand, "ms": ms, "ms_runs": times,
                   "bytes_bf16": bytes_bf16, "bytes_i8": bytes_i8,
                   "tbps_bf16": bytes_bf16 / ms["bf16"] / 1e9, "tbps_i8": bytes_i8 / ms["i8"] / 1e9,
                   "speedup_i8_rescore_vs_bf16": ms["bf16"] / ms["i8+rescore"], f"recall_at_{k}": recall,
                   "device_bytes_bf16": bytes_bf16, "device_bytes_i8_rows_device": qd.device_bytes,
                   "device_bytes_i8_rows_host": qh.device_bytes if qh is not None else n * qd.dim8 + 4 * n}
            print(json.dumps(rec), flush=True)
            result["shapes"].append(rec)
            if a.out:
                with open(os.path.join(a.out, "quant_bench.json"), "w") as f:
                    json.dump(result, f, indent=1)
        del ix, qd, qh, rows
        torch.cuda.empty_cache()
    print(json.dumps({"card": result["card"]}))


if __name__ == "__main__":
    main()
