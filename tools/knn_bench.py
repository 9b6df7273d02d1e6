"""crag_knn_topk (score-block GEMM + per-query radix select) against the scan path it replaces, on one GPU

    python tools/knn_bench.py --out DIR [--shapes selfjoin,few] [--max-rows N]

Today's path is what DenseIndex ran before crag_knn_topk existed: crag_search_topk for k <= 128, and for k > 128 a
chain of ceil(k/128) crag_search_topk_after calls, each one more pass over the shard per block of 32 queries.
Shapes:
  selfjoin  N = nq in {10 000, 50 000, 200 000}, dim in {384, 1024}, k in {10, 100, 2047}: the entities-against-
            themselves retrieve_knn of add_synonymy_edges (ComoRAG.py:670-684, embed_utils.py:8-97)
  few       N = 10M, dim 1024, nq in {1, 32, 256}, k in {10, 2047}: a few queries over a large shard
Per shape, in the same process: both paths warmed, then timed alternately with CUDA events (end-to-end call time);
one extra run of the new path under torch.profiler gives the GEMM and select kernel times, hence the GEMM's share,
its TFLOP/s (2 nq N dim / GEMM time) and the select kernel's bytes/s (4 reads of the nq x N fp32 block when N > k:
three radix passes and the gather).  The ids of both paths are compared on the timed inputs, ranks inside near-tie
runs (neighbouring scores closer than 2e-6) excepted, and the share of bit-identical scores is recorded.  The card
name and power limit are read in the same run.  Writes DIR/knn_bench.json (rewritten after every shape).
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

TIE_TOL = 2e-6


def unit_rows(n, dim, seed, device):
    import torch
    g = torch.Generator(device=device).manual_seed(seed)
    out = torch.empty((n, dim), dtype=torch.bfloat16, device=device)
    slab = max(1, (1 << 28) // dim)
    for s0 in range(0, n, slab):
        x = torch.randn((min(slab, n - s0), dim), generator=g, device=device, dtype=torch.float32)
        out[s0:s0 + x.shape[0]] = torch.nn.functional.normalize(x, dim=1).to(torch.bfloat16)
    return out


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        name, power, clock = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # the measurement itself does not depend on it; say what is missing
        import torch
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"not read ({e})", "max_sm_clock": "not read"}


class Paths:
    def __init__(self, corpus, queries, k):
        import torch
        from comorag_b200 import _native
        from comorag_b200.index import knn_chunk
        self.lib, self.corpus, self.queries, self.k = _native.load(), corpus, queries, k
        self.n, self.dim = corpus.shape
        self.nq = queries.shape[0]
        dev = corpus.device
        self.stream = torch.cuda.current_stream(dev).cuda_stream
        self.knn_ws_bytes = self.lib.crag_knn_workspace_bytes(self.n, knn_chunk(self.nq, self.n))
        self.knn_ws = torch.empty((self.knn_ws_bytes,), dtype=torch.uint8, device=dev)
        kk = min(k, 128)
        self.scan_ws_bytes = self.lib.crag_search_workspace_bytes(self.nq, kk)
        self.scan_ws = torch.empty((self.scan_ws_bytes,), dtype=torch.uint8, device=dev)
        self.out = {}
        for name in ("new", "old"):
            self.out[name] = (torch.empty((self.nq, k), dtype=torch.int64, device=dev),
                              torch.empty((self.nq, k), dtype=torch.float32, device=dev),
                              torch.empty((self.nq, 2), dtype=torch.float32, device=dev))
        if k > 128:
            self.pages = [(p0, min(128, k - p0)) for p0 in range(0, k, 128)]
            self.page_ids = [torch.empty((self.nq, kk), dtype=torch.int64, device=dev) for _, kk in self.pages]
            self.page_sc = [torch.empty((self.nq, kk), dtype=torch.float32, device=dev) for _, kk in self.pages]
            self.last = [torch.empty((self.nq,), dtype=torch.int64, device=dev) for _ in self.pages]

    def new(self):
        from comorag_b200 import _native
        ids, sc, mm = self.out["new"]
        rc = self.lib.crag_knn_topk(self.corpus.data_ptr(), self.n, self.dim, self.corpus.stride(0), 0,
                                    self.queries.data_ptr(), self.nq, self.k, ids.data_ptr(), sc.data_ptr(), mm.data_ptr(),
                                    self.knn_ws.data_ptr(), self.knn_ws_bytes, self.stream)
        _native.check(rc, "crag_knn_topk")

    def old(self):
        from comorag_b200 import _native
        ids, sc, mm = self.out["old"]
        if self.k <= 128:
            rc = self.lib.crag_search_topk(self.corpus.data_ptr(), self.n, self.dim, self.corpus.stride(0), 0,
                                           self.queries.data_ptr(), self.nq, self.k, ids.data_ptr(), sc.data_ptr(),
                                           mm.data_ptr(), self.scan_ws.data_ptr(), self.scan_ws_bytes, self.stream)
            _native.check(rc, "crag_search_topk")
            return
        after = 0
        for i, (p0, kk) in enumerate(self.pages):
            rc = self.lib.crag_search_topk_after(self.corpus.data_ptr(), self.n, self.dim, self.corpus.stride(0), 0,
                                                 self.queries.data_ptr(), self.nq, kk, after, self.page_ids[i].data_ptr(),
                                                 self.page_sc[i].data_ptr(), mm.data_ptr(), self.last[i].data_ptr(),
                                                 self.scan_ws.data_ptr(), self.scan_ws_bytes, self.stream)
            _native.check(rc, "crag_search_topk_after")
            after = self.last[i].data_ptr()
            ids[:, p0:p0 + kk].copy_(self.page_ids[i])
            sc[:, p0:p0 + kk].copy_(self.page_sc[i])


def timed(fn):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def kernel_times(fn, out_dir, tag):
    """GEMM and select kernel time (ms) of one call, from torch.profiler's CUDA activity."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    gemm = sel = 0.0
    for e in prof.key_averages():
        t = e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
        if "gemm_bf16_kernel" in e.key:
            gemm += t
        elif "knn_select_kernel" in e.key:
            sel += t
    return gemm, sel


def compare(p):
    import torch
    ni, ns, nm = p.out["new"]
    oi, os_, om = p.out["old"]
    s = os_.double()
    gap = torch.full_like(s, float("inf"))
    gap[:, :-1] = s[:, :-1] - s[:, 1:]
    near = gap < TIE_TOL
    near[:, 1:] |= gap[:, :-1] < TIE_TOL
    near[:, -1] = True
    diff = ni != oi
    return {"ranks_differing": int(diff.sum()), "ranks_differing_outside_near_ties": int((diff & ~near).sum()),
            "max_abs_score_diff": float((ns - os_).abs().max()),
            "scores_bit_identical_share": float((ns.view(torch.int32) == os_.view(torch.int32)).double().mean()),
            "minmax_equal": bool(torch.equal(nm, om))}


def run_shape(kind, n, dim, nq, k, seed, out_dir):
    import torch
    dev = torch.device("cuda:0")
    corpus = unit_rows(n, dim, seed, dev)
    queries = corpus if kind == "selfjoin" else unit_rows(nq, dim, seed + 1, dev)
    p = Paths(corpus, queries, k)
    # warm both paths; shapes whose calls take seconds get one timed repetition each
    first = {"new": timed(p.new), "old": timed(p.old)}
    reps = 5 if max(first.values()) < 300 else (2 if max(first.values()) < 3000 else 1)
    times = {"new": [], "old": []}
    for _ in range(reps):
        for name in ("old", "new"):
            times[name].append(timed(getattr(p, name)))
    res = compare(p)
    gemm_ms, sel_ms = kernel_times(p.new, out_dir, f"{kind}_{n}_{dim}_{nq}_{k}")
    if gemm_ms == 0.0 and sel_ms == 0.0:    # the profiler returned no kernel events: not measured
        gemm_ms = sel_ms = None
    med = {name: sorted(v)[len(v) // 2] for name, v in times.items()}
    passes = 4 if n > k else 1
    out = {"shape": kind, "n_rows": n, "dim": dim, "nq": nq, "k": k, "reps": reps,
           "new_ms": med["new"], "old_ms": med["old"], "new_ms_all": times["new"], "old_ms_all": times["old"],
           "speedup": med["old"] / med["new"],
           "gemm_ms": gemm_ms, "select_ms": sel_ms,
           "gemm_share_of_new": gemm_ms / med["new"] if gemm_ms else None,
           "gemm_tflops": 2.0 * nq * n * dim / (gemm_ms * 1e-3) / 1e12 if gemm_ms else None,
           "select_gbps": passes * 4.0 * nq * n / (sel_ms * 1e-3) / 1e9 if sel_ms else None,
           "knn_workspace_bytes": p.knn_ws_bytes, **res}
    del p, corpus, queries
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--shapes", default="selfjoin,few")
    ap.add_argument("--max-rows", type=int, default=10_000_000)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("knn_bench measures on a GPU; none is visible")
    os.makedirs(args.out, exist_ok=True)
    grid = []
    if "selfjoin" in args.shapes:
        grid += [("selfjoin", n, dim, n, k) for n in (10_000, 50_000, 200_000) for dim in (384, 1024) for k in (10, 100, 2047)]
    if "few" in args.shapes:
        grid += [("few", 10_000_000, 1024, nq, k) for nq in (1, 32, 256) for k in (10, 2047)]
    grid = [g for g in grid if g[1] <= args.max_rows]
    doc = {"card": card(), "torch": torch.__version__, "tie_tol": TIE_TOL, "results": []}
    path = os.path.join(args.out, "knn_bench.json")
    for i, (kind, n, dim, nq, k) in enumerate(grid):
        t0 = time.time()
        r = run_shape(kind, n, dim, nq, k, 1000 + i, args.out)
        r["wall_s"] = time.time() - t0
        doc["results"].append(r)
        print(json.dumps({key: r[key] for key in ("shape", "n_rows", "dim", "nq", "k", "new_ms", "old_ms", "speedup",
                                                   "gemm_tflops", "select_gbps", "ranks_differing_outside_near_ties")}),
              flush=True)
        with open(path, "w") as f:
            json.dump(doc, f, indent=1)
    print(path)


if __name__ == "__main__":
    main()
