"""IVF over product-quantized residuals against bf16 and int8 IVF: one rank's share of BASELINE config 4 on one GPU

    python tools/ivf_pq_bench.py [--rows 12500000 --dim 768 --nlist 4096 --nprobe 32 --nq 32 --ks 10,100 --ms 48,96,192]

Synthetic clustered unit vectors (tools/ivf_bench.py's generator), the same share tools/ivf_i8_bench.py measures.
One IVFIndex is built; QuantizedIVF and PQIVF snapshots of it (one set of trained codebooks per m) keep their bf16
residuals on the device and in page-locked host memory.  For each k all searches run in alternating rounds in this
process; each round times `steps` searches of one 32-query block with CUDA events and the median over rounds is
reported.  The fine pass's first-stage bytes are those of the probed tiles: code_stride(m) per stored row for PQ,
dim8 + 4 for int8, 2 dim for bf16.  Recall@k is against bf16 IVF and against the exact flat search of the same bf16
rows.  One JSON object per k, with the card's name and power limit, and one with the build times.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from tools.ivf_bench import clustered  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = (s.strip() for s in out.split(","))
        return name, power
    except Exception as e:   # the numbers stand without it, but say so
        return f"unknown ({e})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=12_500_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--nlist", type=int, default=4096)
    ap.add_argument("--nprobe", type=int, default=32)
    ap.add_argument("--nq", type=int, default=32)
    ap.add_argument("--ks", default="10,100")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--kmeans-iters", type=int, default=6)
    ap.add_argument("--train-rows", type=int, default=1 << 20)
    ap.add_argument("--ms", default="48,96,192")
    ap.add_argument("--pq-iters", type=int, default=8)
    args = ap.parse_args()

    import numpy as np
    import torch
    from comorag_b200.index import DenseIndex
    from comorag_b200.ivf import IVFIndex, QuantizedIVF
    from comorag_b200.pq import PQIVF, code_stride
    import time

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    x, dirs = clustered(args.rows, args.dim, 4 * args.nlist, 1, dev)
    g = torch.Generator(device=dev).manual_seed(2)
    q = torch.nn.functional.normalize(
        dirs[torch.randint(0, dirs.shape[0], (args.nq,), generator=g, device=dev)]
        + (0.5 / args.dim ** 0.5) * torch.randn(args.nq, args.dim, generator=g, device=dev), dim=1).to(torch.bfloat16)
    bf = IVFIndex.build(x, args.nlist, iters=args.kmeans_iters, seed=0, train_rows=args.train_rows)
    ks = [int(k) for k in args.ks.split(",")]
    flat = DenseIndex.from_tensor(x.to(torch.bfloat16))
    del x
    exact = {k: flat.search_device(q, k)[0].cpu().numpy() for k in ks}
    del flat
    torch.cuda.empty_cache()
    qd = QuantizedIVF.from_ivf(bf, "device")
    qh = QuantizedIVF.from_ivf(bf, "host")
    variants = {"bf16": bf, "int8_device_residuals": qd, "int8_host_residuals": qh}
    ms = [int(m) for m in args.ms.split(",")]
    build_s = {}
    for m in ms:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pd = PQIVF.from_ivf(bf, m, train_rows=args.train_rows, iters=args.pq_iters, seed=0)
        build_s[f"pq{m}_train_and_encode"] = round(time.perf_counter() - t0, 2)
        variants[f"pq{m}_device_residuals"] = pd
        variants[f"pq{m}_host_residuals"] = PQIVF(bf, qh._rows, pd.codes, pd.codebooks)   # shares the pinned copy
    name, power = card()

    _, _, _, (p_ids, _) = bf.search_device(q, args.nprobe, 10)
    list_rows = bf.list_rows.cpu().numpy().astype(np.int64)
    probed = np.unique(p_ids.cpu().numpy())
    probed_rows = int(((list_rows[probed[probed >= 0]] + 127) // 128 * 128).sum())   # stored rows of the probed tiles
    fine_bytes = {"bf16": probed_rows * 2 * args.dim, "int8": probed_rows * (qd.dim8 + 4),
                  **{f"pq{m}": probed_rows * code_stride(m) for m in ms}}

    def recall(a, b):
        return float(np.mean([len(set(r[r >= 0].tolist()) & set(s[s >= 0].tolist())) / max(1, (s >= 0).sum())
                              for r, s in zip(a, b)]))

    for k in ks:
        run = {n: (lambda v=v: v.search_device(q, args.nprobe, k)) for n, v in variants.items()}
        for fn in run.values():
            for _ in range(3):
                fn()
        times = {n: [] for n in run}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(args.rounds):
            for n, fn in run.items():
                torch.cuda.synchronize()
                e0.record()
                for _ in range(args.steps):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                times[n].append(e0.elapsed_time(e1) / args.steps)
        ids = {n: fn()[0].cpu().numpy() for n, fn in run.items()}
        med = {n: float(np.median(t)) for n, t in times.items()}
        print(json.dumps({
            "workload": f"IVF-{args.nlist}, {args.rows}x{args.dim}, nprobe {args.nprobe}, top-{k}, {args.nq} queries, "
                        f"1 GPU, candidates {min(128, 4 * k)}",
            "gpu": name, "power_limit": power,
            "median_ms_per_step": {n: round(v, 4) for n, v in med.items()},
            "spread_ms": {n: [round(min(t), 4), round(max(t), 4)] for n, t in times.items()},
            "speedup_vs_bf16": {n: round(med["bf16"] / v, 3) for n, v in med.items() if n != "bf16"},
            "fine_pass_bytes": fine_bytes, "probed_stored_rows": probed_rows,
            f"recall_at_{k}_vs_bf16_ivf": {n: round(recall(ids[n], ids["bf16"]), 4) for n in ids if n != "bf16"},
            f"recall_at_{k}_vs_exact_flat": {n: round(recall(ids[n], exact[k]), 4) for n in ids},
            "device_bytes": {"bf16_residuals": 2 * bf.residuals.numel(),
                             **{n: v.device_bytes for n, v in variants.items() if n != "bf16"}},
            "data": "synthetic clustered unit vectors",
        }), flush=True)
    print(json.dumps({"gpu": name, "power_limit": power, "build_seconds": build_s}), flush=True)


if __name__ == "__main__":
    main()
