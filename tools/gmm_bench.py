"""The BIC sweep of ComoRAG's soft clustering on the device (crag_gmm_sweep through cluster.gmm_sweep) against
scikit-learn's sweep as the reference calls it (GaussianMixture(n, random_state=224).fit + bic for n = 1..M, then
the winner's predict_proba), on the same float64 input: seeded mixtures of 8 Gaussians in d = 10, the dimension the
reference's UMAP reduces to, at N rows.

Reported per N: median wall time of the device sweep to the result on the host (a host clock around the call, which
ends in a device synchronise and the copies back), scikit-learn's wall time (one run: a sweep takes minutes), both
chosen n, and the largest membership difference.  The card's name and power limit are read in the same run.

    python tools/gmm_bench.py --n 2000 8000 32000 --out gmm_bench.json
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from comorag_b200.cluster import gmm_sweep  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def data(n, d, seed=0):
    rng = np.random.default_rng(seed)
    centres = rng.normal(0, 4.0, size=(8, d))
    return centres[rng.integers(0, 8, n)] + rng.normal(0, 1.0, size=(n, d))


def sklearn_sweep(X, M):
    from sklearn.mixture import GaussianMixture
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        bics = [GaussianMixture(m, random_state=224).fit(X).bic(X) for m in range(1, M + 1)]
        best = int(np.argmin(bics)) + 1
        memb = GaussianMixture(best, random_state=224, covariance_type="full").fit(X).predict_proba(X)
    return best, memb


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[2000, 8000, 32000])
    ap.add_argument("--d", type=int, default=10)
    ap.add_argument("--M", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sklearn-max-n", type=int, default=1 << 30, help="skip scikit-learn above this N")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gmm_bench: needs a GPU")
    rows = []
    for n in a.n:
        X = data(n, a.d)
        r = gmm_sweep(X, a.M)                          # warm-up: module load, allocator
        times = []
        for _ in range(a.reps):
            torch.cuda.synchronize()
            t = time.perf_counter()
            r = gmm_sweep(X, a.M)
            times.append(time.perf_counter() - t)
        row = {"n": n, "d": a.d, "M": a.M, "device_s_median": float(np.median(times)),
               "device_s_all": [round(t, 4) for t in times], "device_n": r.n_components,
               "device_em_iters_total": int(r.iterations.sum())}
        if n <= a.sklearn_max_n:
            t = time.perf_counter()
            best, memb = sklearn_sweep(X, a.M)
            row["sklearn_s"] = time.perf_counter() - t
            row["sklearn_n"] = best
            row["speedup"] = row["sklearn_s"] / row["device_s_median"]
            if best == r.n_components:
                row["max_membership_diff"] = float(np.abs(memb - r.memberships).max())
        rows.append(row)
        print(json.dumps(row), flush=True)
    out = {"card": card(), "rows": rows}
    print(json.dumps(out))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
