"""UMAP on the device (comorag_b200.umap_layout.umap_reduce) on planted clusters of 1024-d rows.

For each N: per-stage device time from CUDA events (k-NN self-join, fuzzy graph + symmetric CSR, spectral start,
layout epochs), the median wall time of umap_reduce to the host result, trustworthiness (15 neighbours, cosine) on a
1000-row subsample, and the ARI of the device GMM sweep's labels.  umap-learn is timed in the same run only if it
imports.  Prints one JSON line per N, with the card's name and power limit.

    python tools/umap_bench.py [--sizes 2000,8000,32000] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from comorag_b200 import umap_layout as ul  # noqa: E402
from comorag_b200.cluster import gmm_sweep  # noqa: E402
from umap_oracle import planted  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(), "unknown"


def staged(X, k, d):
    """One reduction with CUDA events between the stages: {stage: ms}."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
    n = len(X)
    x = torch.as_tensor(X).cuda()
    torch.cuda.synchronize()
    ev[0].record()
    ids, scores = ul.knn_self_join(x, k)
    ev[1].record()
    nbr, dist, rho, sigma, memb = ul.fuzzy_graph(ids, scores)
    indptr, indices, w, eps = ul.symmetric_graph(nbr, memb, ul.default_epochs(n))
    ev[2].record()
    y0 = ul.spectral_init(indptr, indices, w, d)
    ev[3].record()
    a, b = ul.find_ab_params()
    ul.optimize(indptr, indices, eps, y0, a, b, ul.default_epochs(n))
    ev[4].record()
    torch.cuda.synchronize()
    names = ["knn", "graph", "start", "epochs"]
    return {nm: ev[i].elapsed_time(ev[i + 1]) for i, nm in enumerate(names)}, int(indices.numel())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="2000,8000,32000")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--clusters", type=int, default=8)
    args = ap.parse_args()
    from sklearn.manifold import trustworthiness
    from sklearn.metrics import adjusted_rand_score
    name, power = card()
    try:
        import umap as umap_learn
        have_umap = hasattr(umap_learn, "UMAP")
    except Exception:
        have_umap = False
    for n in [int(s) for s in args.sizes.split(",")]:
        X, labels = planted(n, 1024, args.clusters, seed=11)
        k = min(30, max(5, int(n * 0.2)))
        d = 10
        ul.umap_reduce(X[:256], 15, d)                      # warm-up: module load, allocator, a and b
        staged(X, k, d)                                    # every shape of this N once
        stages, nnz = staged(X, k, d)
        walls = []
        for _ in range(args.reps):
            t = time.perf_counter()
            Y = ul.umap_reduce(X, k, d)
            walls.append(time.perf_counter() - t)
        sub = np.random.RandomState(0).choice(n, min(n, 1000), replace=False)
        tw = float(trustworthiness(X[sub], Y[sub], n_neighbors=15, metric="cosine"))
        r = gmm_sweep(Y, 2 * args.clusters)
        ari = float(adjusted_rand_score(labels, r.memberships.argmax(axis=1)))
        rec = dict(tool="umap_bench", gpu=name, power_limit=power, n=n, dim=1024, n_neighbors=k, d=d,
                   n_epochs=ul.default_epochs(n), nnz=nnz, stage_ms={s: round(v, 3) for s, v in stages.items()},
                   wall_s_median=round(float(np.median(walls)), 4), wall_s=[round(w, 4) for w in walls],
                   finite=bool(np.isfinite(Y).all()), trustworthiness=round(tw, 4), gmm_n=int(r.n_components),
                   ari=round(ari, 4))
        if have_umap:
            t = time.perf_counter()
            umap_learn.UMAP(n_neighbors=k, n_components=d, metric="cosine", random_state=224).fit_transform(X)
            rec["umap_learn_s"] = round(time.perf_counter() - t, 3)
        else:
            rec["umap_learn_s"] = "not available"
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
