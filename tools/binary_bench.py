"""One-bit shard search against the bf16 and int8 paths, alternating the paths in one process.

Shapes: 1M x 1024 and 10M x 1024 rows (bf16), 32 queries, k = 10 and 100 (candidates min(128, 4 k)).  Two row sets:
seeded randn rows (unit norm), and SURVEY.md section 8d's planted neighbours (2 000 rows per query are
normalise(q + 0.3 noise), the rest randn), where the true top k has wide score gaps.
Per shape, ms per pass (CUDA events, median over three alternating rounds of the median of --reps timed calls):
  bf16        crag_search_topk over the bf16 shard
  i8          crag_search_topk_i8 alone (queries already quantised)      i8+rescore  QuantizedIndex.search_device
  b1          crag_search_topk_b1 alone (queries already quantised)      b1+rescore  BinaryIndex.search_device
  b1+host     BinaryIndex.search_device with the bf16 rows in page-locked host memory (1M only, to keep pinned
              memory modest)
plus algorithmic bytes per pass (bf16 2 n dim, int8 n dim8 + 4 n, b1 n dim8 / 8 + 4 n) and TB/s, device bytes, and
recall@k of the int8 and one-bit paths against the bf16 scan's ids.  The card's name and power limit are read in the
same run.

  python tools/binary_bench.py [--sizes 1000000,10000000] [--out DIR]   (one JSON line per shape; --out also writes
  DIR/binary_bench.json)
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from quant_bench import card, time_ms  # noqa: E402


def make_rows(n, dim, q, planted, gen, dev):
    import torch
    rows = torch.empty((n, dim), dtype=torch.bfloat16, device=dev)
    for r0 in range(0, n, 500_000):
        c = torch.randn((min(500_000, n - r0), dim), generator=gen, device=dev)
        rows[r0:r0 + c.shape[0]] = torch.nn.functional.normalize(c, dim=1).bfloat16()
        del c
    if planted:   # 2 000 neighbours per query, spread over the shard
        nq = q.shape[0]
        idx = torch.randperm(n, generator=gen, device=dev)[: nq * 2000].view(nq, 2000)
        for j in range(nq):
            noise = torch.randn((2000, dim), generator=gen, device=dev)
            rows[idx[j]] = torch.nn.functional.normalize(q[j].float()[None, :] + 0.3 * noise, dim=1).bfloat16()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000000,10000000")
    ap.add_argument("--dim", type=int, default=1024)
    ap.add_argument("--nq", type=int, default=32)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--out", default=None, help="directory for binary_bench.json (default: print only)")
    a = ap.parse_args()

    import numpy as np
    import torch

    from comorag_b200 import _native
    from comorag_b200.binary import BinaryIndex
    from comorag_b200.index import DenseIndex
    from comorag_b200.quantized import QuantizedIndex, quantize_rows

    if not torch.cuda.is_available():
        raise SystemExit("binary_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    lib = _native.load()
    result = {"card": card(), "dim": a.dim, "nq": a.nq, "shapes": []}
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    for n in [int(s) for s in a.sizes.split(",")]:
        for planted in (False, True):
            g = torch.Generator(device=dev).manual_seed(n + planted)
            q = torch.nn.functional.normalize(torch.randn((a.nq, a.dim), generator=g, device=dev), dim=1).bfloat16()
            rows = make_rows(n, a.dim, q, planted, g, dev)
            ix = DenseIndex.from_tensor(rows)
            qd = QuantizedIndex.from_dense(ix, "device")
            bd = BinaryIndex.from_dense(ix, "device")
            bh = BinaryIndex.from_dense(ix, "host") if n <= 1_000_000 else None
            q8, qs = quantize_rows(q, qd.dim8)
            for k in (10, 100):
                cand = min(128, 4 * k)
                ws = torch.empty(max(lib.crag_search_workspace_bytes(a.nq, k), lib.crag_search_workspace_bytes(a.nq, cand)),
                                 dtype=torch.uint8, device=dev)
                ids = torch.empty((a.nq, 128), dtype=torch.int64, device=dev)
                sc = torch.empty((a.nq, 128), dtype=torch.float32, device=dev)
                mm = torch.empty((a.nq, 2), dtype=torch.float32, device=dev)
                st = torch.cuda.current_stream(dev).cuda_stream

                def bf16():
                    _native.check(lib.crag_search_topk(rows.data_ptr(), n, a.dim, a.dim, 0, q.data_ptr(), a.nq, k,
                                                       ids.data_ptr(), sc.data_ptr(), mm.data_ptr(), ws.data_ptr(),
                                                       ws.numel(), st), "crag_search_topk")

                def i8():
                    _native.check(lib.crag_search_topk_i8(qd._codes.data_ptr(), qd._scales.data_ptr(), n, qd.dim8,
                                                          qd.dim8, 0, q8.data_ptr(), qs.data_ptr(), a.nq, cand,
                                                          ids.data_ptr(), sc.data_ptr(), mm.data_ptr(), ws.data_ptr(),
                                                          ws.numel(), st), "crag_search_topk_i8")

                def b1():
                    _native.check(lib.crag_search_topk_b1(bd._codes.data_ptr(), bd._scales.data_ptr(), n, bd.dim8,
                                                          bd._codes.shape[1], 0, q8.data_ptr(), qs.data_ptr(), a.nq,
                                                          cand, ids.data_ptr(), sc.data_ptr(), mm.data_ptr(),
                                                          ws.data_ptr(), ws.numel(), st), "crag_search_topk_b1")

                paths = {"bf16": bf16, "i8": i8, "i8+rescore": lambda: qd.search_device(q, k), "b1": b1,
                         "b1+rescore": lambda: bd.search_device(q, k)}
                if bh is not None:
                    paths["b1+host"] = lambda: bh.search_device(q, k)
                times = {p: [] for p in paths}
                for _ in range(3):             # alternate the paths: drift of a shared host hits all of them alike
                    for p, fn in paths.items():
                        times[p].append(time_ms(fn, a.warmup, a.reps))
                ms = {p: float(np.median(v)) for p, v in times.items()}
                want = ix.search_device(q, k)[0].cpu().numpy()
                got_i8 = qd.search_device(q, k)[0].cpu().numpy()
                got_b1 = bd.search_device(q, k)[0].cpu().numpy()
                if bh is not None:
                    assert np.array_equal(bh.search_device(q, k)[0].cpu().numpy(), got_b1), "host rows differ from device"

                def recall(got):
                    return float(np.mean([len(set(got[j]) & set(want[j])) / k for j in range(a.nq)]))

                bytes_bf16, bytes_i8, bytes_b1 = 2 * n * a.dim, n * qd.dim8 + 4 * n, n * (bd.dim8 // 8) + 4 * n
                rec = {"n": n, "rows": "planted" if planted else "randn", "k": k, "candidates": cand, "ms": ms,
                       "ms_runs": times, "bytes_bf16": bytes_bf16, "bytes_i8": bytes_i8, "bytes_b1": bytes_b1,
                       "tbps_bf16": bytes_bf16 / ms["bf16"] / 1e9, "tbps_i8": bytes_i8 / ms["i8"] / 1e9,
                       "tbps_b1": bytes_b1 / ms["b1"] / 1e9,
                       f"recall_at_{k}_i8": recall(got_i8), f"recall_at_{k}_b1": recall(got_b1),
                       "device_bytes_bf16": bytes_bf16, "device_bytes_i8_rows_device": qd.device_bytes,
                       "device_bytes_b1_rows_device": bd.device_bytes, "device_bytes_b1_rows_host": bytes_b1}
                print(json.dumps(rec), flush=True)
                result["shapes"].append(rec)
                if a.out:
                    with open(os.path.join(a.out, "binary_bench.json"), "w") as f:
                        json.dump(result, f, indent=1)
            del ix, qd, bd, bh, rows
            torch.cuda.empty_cache()
    print(json.dumps({"card": result["card"]}))


if __name__ == "__main__":
    main()
