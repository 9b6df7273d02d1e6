"""First-light / regression check of the search kernel on a real H100.

Each case runs in its own subprocess with a timeout, so a trap or hang in one
case cannot take the others (or the box) down.  Usage (on the GPU box):
    python tools/gpu_check_search.py            # all cases
    python tools/gpu_check_search.py --case N   # one case, in-process
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

# (n_rows, dim, nq, k, seed, note)
CASES = [
    (128, 64, 32, 10, 1, "one full tile"),
    (1000, 64, 1, 5, 2, "single query, ragged last tile"),
    (100, 128, 3, 10, 3, "n_rows < tile"),
    (7, 64, 2, 10, 4, "n_rows < k"),
    (5000, 384, 7, 50, 5, "bge-small width, k=50"),
    (40000, 768, 40, 100, 6, "two query passes, k=100 (large-k kernel)"),
    (200000, 1024, 32, 10, 7, "1024-d, many tiles per CTA"),
    (3000, 256, 32, 10, 8, "duplicate rows (exact ties)"),
    (1000000, 1024, 32, 10, 9, "config 2 size"),
]


def run_case(i: int) -> dict:
    import numpy as np
    import torch
    from comorag_b200.index import DenseIndex
    from oracle.search_oracle import assert_topk_matches
    from util_search import make_unit_rows, torch_reference_topk

    n, dim, nq, k, seed, note = CASES[i]
    dev = torch.device("cuda:0")
    corpus = make_unit_rows(n, dim, 1000 + seed, device=dev)
    if "duplicate" in note:
        corpus[n // 2:] = corpus[: n - n // 2]
    queries = make_unit_rows(nq, dim, 2000 + seed, device=dev)
    index = DenseIndex.from_tensor(corpus.contiguous())
    t0 = time.time()
    ids, scores, minmax = index.search_device(queries.contiguous(), k)
    torch.cuda.synchronize()
    t_first = time.time() - t0
    want_i, want_s, want_mm, gaps = torch_reference_topk(corpus, queries, k)
    got_i, got_s, got_mm = ids.cpu().numpy(), scores.cpu().numpy().astype(np.float64), minmax.cpu().numpy()
    res = {"case": i, "note": note, "shape": [n, dim, nq, k], "first_call_s": round(t_first, 4)}
    try:
        assert_topk_matches(got_i, got_s, want_i, want_s, gaps)
        exact = float((got_i == want_i).mean())
        mm_err = float(np.abs(got_mm - want_mm).max())
        assert mm_err < 1e-3, f"minmax err {mm_err}"
        res.update(ok=True, exact_id_frac=exact, max_score_err=float(np.abs(got_s - want_s)[want_i >= 0].max()) if (want_i >= 0).any() else 0.0,
                   minmax_err=mm_err)
    except AssertionError as e:
        res.update(ok=False, error=str(e)[:500], got_ids=got_i[:2].tolist(), want_ids=want_i[:2].tolist(),
                   got_scores=got_s[:2].tolist(), want_scores=want_s[:2].tolist())
    # timing (device, CUDA events) for the bigger cases
    if n >= 200000:
        st = torch.cuda.current_stream()
        for _ in range(3):
            index.search_device(queries, k)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 10
        e0.record(st)
        for _ in range(reps):
            index.search_device(queries, k)
        e1.record(st)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        res.update(ms_per_pass=ms, gbps=n * dim * 2 / ms / 1e6, qps=nq / ms * 1e3)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", type=int, default=None)
    ap.add_argument("--timeout", type=int, default=240)
    args = ap.parse_args()
    if args.case is not None:
        print("RESULT " + json.dumps(run_case(args.case)))
        return
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    results = []
    for i in range(len(CASES)):
        try:
            p = subprocess.run([sys.executable, __file__, "--case", str(i)], capture_output=True, text=True,
                               timeout=args.timeout)
            line = [l for l in p.stdout.splitlines() if l.startswith("RESULT ")]
            if line:
                results.append(json.loads(line[-1][7:]))
            else:
                results.append({"case": i, "ok": False, "rc": p.returncode, "stderr": p.stderr[-1500:]})
        except subprocess.TimeoutExpired:
            results.append({"case": i, "ok": False, "error": "timeout"})
        print(json.dumps(results[-1]), flush=True)
    with open(os.path.join(ROOT, "gpurun_out", "check_search.json"), "w") as f:
        json.dump(results, f, indent=1)
    print("SUMMARY", sum(1 for r in results if r.get("ok")), "/", len(results), "ok")


if __name__ == "__main__":
    main()
