"""Wide IVF stage 1 (QuantizedIVF / PQIVF.search_device_wide) against the 128-candidate path, on tools/ivf_pq_bench.py's
share of BASELINE config 4 on one GPU

    python tools/ivf_wide_bench.py [--rows 12500000 --dim 768 --nlist 4096 --nprobe 32 --nq 32 --ks 10,100
                                    --cands 128,512,1024,2048 --ms 48,96,192]

Synthetic clustered unit vectors (tools/ivf_bench.py's generator).  One IVFIndex is built; a QuantizedIVF and one
PQIVF per m snapshot it with their bf16 residuals on the device, and the same codes with the residuals in page-locked
host memory.  For each (k, code) every candidate count runs in alternating rounds in this process, the narrow path at
128 among them; each round times `steps` searches of one 32-query block with CUDA events and the median over rounds
is reported.  A separate torch.profiler pass splits one wide search into its kernels: plan (ivf_plan_kernel,
ivf_wide_plan_kernel), fill (pq_table_kernel, ivf_fill_*), select (ivf_wide_select_kernel, ivf_slot_map_kernel),
rescore (ivf_rescore_*).  Recall@k is against bf16 IVF and against the exact flat search of the same bf16 rows.  One
JSON object per (k, code), with the card's name and power limit.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from tools.ivf_bench import clustered  # noqa: E402
from tools.ivf_pq_bench import card  # noqa: E402

STAGES = {"plan": ("ivf_plan_kernel", "ivf_wide_plan_kernel"), "fill": ("pq_table_kernel", "ivf_fill_"),
          "select": ("ivf_wide_select_kernel", "ivf_slot_map_kernel"), "rescore": ("ivf_rescore_",)}


def stage_split(fn, reps=5):
    """ms per call of each stage of `fn`, from the CUDA kernel times of a torch.profiler run."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {s: 0.0 for s in STAGES}
    for e in prof.key_averages():
        for s, names in STAGES.items():
            if any(n in e.key for n in names):
                out[s] += e.device_time_total / 1000.0 / reps
    return {s: round(v, 4) for s, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=12_500_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--nlist", type=int, default=4096)
    ap.add_argument("--nprobe", type=int, default=32)
    ap.add_argument("--nq", type=int, default=32)
    ap.add_argument("--ks", default="10,100")
    ap.add_argument("--cands", default="128,512,1024,2048")
    ap.add_argument("--ms", default="48,96,192")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--kmeans-iters", type=int, default=6)
    ap.add_argument("--train-rows", type=int, default=1 << 20)
    ap.add_argument("--pq-iters", type=int, default=8)
    args = ap.parse_args()

    import numpy as np
    import torch
    from comorag_b200.index import DenseIndex
    from comorag_b200.ivf import IVFIndex, QuantizedIVF
    from comorag_b200.pq import PQIVF

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    name, power = card()
    x, dirs = clustered(args.rows, args.dim, 4 * args.nlist, 1, dev)
    g = torch.Generator(device=dev).manual_seed(2)
    q = torch.nn.functional.normalize(
        dirs[torch.randint(0, dirs.shape[0], (args.nq,), generator=g, device=dev)]
        + (0.5 / args.dim ** 0.5) * torch.randn(args.nq, args.dim, generator=g, device=dev), dim=1).to(torch.bfloat16)
    bf = IVFIndex.build(x, args.nlist, iters=args.kmeans_iters, seed=0, train_rows=args.train_rows)
    ks = [int(k) for k in args.ks.split(",")]
    cands = [int(c) for c in args.cands.split(",")]
    flat = DenseIndex.from_tensor(x.to(torch.bfloat16))
    del x
    exact = {k: flat.search_device(q, k)[0].cpu().numpy() for k in ks}
    del flat
    torch.cuda.empty_cache()
    qh = QuantizedIVF.from_ivf(bf, "host")
    codes = {"int8": (QuantizedIVF.from_ivf(bf, "device"), qh)}
    for m in (int(m) for m in args.ms.split(",")):
        pd = PQIVF.from_ivf(bf, m, train_rows=args.train_rows, iters=args.pq_iters, seed=0)
        codes[f"pq{m}"] = (pd, PQIVF(bf, qh._rows, pd.codes, pd.codebooks))   # shares the pinned copy
    bound = codes["int8"][0].probe_rows_bound(args.nprobe)
    print(json.dumps({"gpu": name, "power_limit": power, "max_probe_rows": bound,
                      "s1_block_bytes": 32 * ((bound + 3) // 4 * 4) * 4}), flush=True)

    def recall(a, b):
        return float(np.mean([len(set(r[r >= 0].tolist()) & set(s[s >= 0].tolist())) / max(1, (s >= 0).sum())
                              for r, s in zip(a, b)]))

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for k in ks:
        ref = bf.search_device(q, args.nprobe, k)[0].cpu().numpy()
        for cname, (d, h) in codes.items():
            run = {}
            for c in cands:
                if c < k:
                    continue
                run[f"{c}_device"] = lambda d=d, c=c: d.search_device_wide(q, args.nprobe, k, c)
                run[f"{c}_host"] = lambda h=h, c=c: h.search_device_wide(q, args.nprobe, k, c)
            for fn in run.values():
                for _ in range(2):
                    fn()
            times = {n: [] for n in run}
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
            split = {c: stage_split(run[f"{c}_device"]) for c in cands if c > 128 and f"{c}_device" in run}
            split_host = {c: stage_split(run[f"{c}_host"])["rescore"] for c in cands if c > 128 and f"{c}_host" in run}
            print(json.dumps({
                "workload": f"IVF-{args.nlist}, {args.rows}x{args.dim}, nprobe {args.nprobe}, top-{k}, {args.nq} "
                            f"queries, 1 GPU, {cname}",
                "gpu": name, "power_limit": power,
                "median_ms_per_step": {n: round(float(np.median(t)), 4) for n, t in times.items()},
                "spread_ms": {n: [round(min(t), 4), round(max(t), 4)] for n, t in times.items()},
                "wide_stage_ms_device_residuals": split, "wide_rescore_ms_host_residuals": split_host,
                f"recall_at_{k}_vs_bf16_ivf": {n: round(recall(ids[n], ref), 4) for n in ids if n.endswith("device")},
                f"recall_at_{k}_vs_exact_flat": {n: round(recall(ids[n], exact[k]), 4) for n in ids
                                                 if n.endswith("device")},
                "data": "synthetic clustered unit vectors",
            }), flush=True)


if __name__ == "__main__":
    main()
