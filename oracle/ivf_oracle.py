"""CPU statement (numpy) of the IVF residual inner-product search BASELINE config 4 names
("100M x 768, IVF-4096 coarse quantizer + fused residual-IP top-100").

TEST INFRASTRUCTURE ONLY: the product path never imports this module.

PARITY UNPINNED: the reference has no IVF / ANN code at all (faiss-cpu is pinned in requirements.txt:34 but never
imported; SURVEY.md section 1), so there is nothing of the reference's to check this against.  It is our own
definition of the search the engine's IVF path must reproduce, written down before the kernel so that the kernel
is tested against a fixed semantic:

  build   rows x (unit-norm fp32) are assigned to the coarse centroid of largest inner product (ties: smaller list
          id); the index stores, per list, the residuals r = bf16(x - c_l) and the rows' original ids, lists laid
          out back to back in list order (ascending original id inside a list).
  search  for a query q (rounded to bf16, like the flat path): the `nprobe` lists of largest q.c_l (centroids
          rounded to bf16; ties: smaller list id) are probed; a row's score is  q.c_l + q.r  -- the coarse term is
          shared by the whole list and the fine term runs over the bf16 residuals, which is why the residual form
          is more accurate than scoring bf16(x) directly (|r| << |x|); the answer is the k best among the probed
          lists only, ranked by score descending, then by STORED POSITION ascending -- list id first, then original
          id inside the list (the kernel keys on the position, a 32-bit word, and maps positions to 64-bit ids
          afterwards).  So an exact tie between rows of two lists goes to the row of the smaller list id.

`nprobe == nlist` degenerates to exact search over the reconstructed rows c_l + r.
"""
from __future__ import annotations

from typing import List, Tuple

import numpy as np


def bf16_round(x: np.ndarray) -> np.ndarray:
    """fp32 -> nearest-even bf16 -> fp32 (numpy has no bf16; same rounding torch's .bfloat16() applies)."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32).reshape(np.shape(x))


def spherical_kmeans(x: np.ndarray, nlist: int, iters: int = 10, seed: int = 0) -> np.ndarray:
    """Lloyd iterations on the unit sphere: assign by largest inner product, centroid = normalised mean of its rows;
    an empty list is re-seeded with the row that is worst served by its current centroid.  Deterministic."""
    x = np.asarray(x, dtype=np.float32)
    n = x.shape[0]
    if not 1 <= nlist <= n:
        raise ValueError("need 1 <= nlist <= rows")
    rng = np.random.default_rng(seed)
    c = x[rng.choice(n, size=nlist, replace=False)].astype(np.float64)
    for _ in range(iters):
        sims = x.astype(np.float64) @ c.T
        a = np.argmax(sims, axis=1)
        best = sims[np.arange(n), a]
        for l in range(nlist):
            rows = np.nonzero(a == l)[0]
            if rows.size == 0:
                worst = int(np.argmin(best))
                c[l], best[worst] = x[worst], np.inf
                continue
            m = x[rows].astype(np.float64).mean(axis=0)
            c[l] = m / max(np.linalg.norm(m), 1e-12)
    return c.astype(np.float32)


def assign(x: np.ndarray, centroids: np.ndarray) -> np.ndarray:
    """List of every row: argmax_l bf16(x).bf16(c_l) in float64, ties to the smaller list id (what a top-1 pass of
    the flat search kernel over the centroid table returns)."""
    s = bf16_round(x).astype(np.float64) @ bf16_round(centroids).astype(np.float64).T
    return np.argmax(s, axis=1).astype(np.int64)      # np.argmax returns the first maximum = the smaller id


class IVFLists:
    """The layout the engine's IVF shard uses: rows grouped by list, back to back."""

    def __init__(self, x: np.ndarray, centroids: np.ndarray, assignment: np.ndarray = None):
        """`assignment` overrides assign(): parity tests of the SEARCH pass it the engine's own row -> list map, so
        that a row sitting on a float tie between two centroids does not turn into a search mismatch."""
        x = np.asarray(x, dtype=np.float32)
        self.centroids = bf16_round(centroids)                     # what the coarse pass sees
        a = assign(x, centroids) if assignment is None else np.asarray(assignment, dtype=np.int64)
        order = np.lexsort((np.arange(x.shape[0]), a))             # list id, then original id
        self.ids = order.astype(np.int64)                          # original id of each stored row
        self.list_of_row = a[order]
        counts = np.bincount(a, minlength=centroids.shape[0])
        self.offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        self.residuals = bf16_round(x[order] - self.centroids[self.list_of_row])

    @property
    def nlist(self) -> int:
        return self.centroids.shape[0]

    def reconstructed(self) -> np.ndarray:
        """c_l + r in float64, in STORED order (what nprobe == nlist searches exactly)."""
        return self.centroids[self.list_of_row].astype(np.float64) + self.residuals.astype(np.float64)


def probe_lists(lists: IVFLists, queries: np.ndarray, nprobe: int) -> Tuple[np.ndarray, np.ndarray]:
    """Coarse pass: (list ids int64 [nq, nprobe] best first, their q.c_l float64)."""
    q = bf16_round(queries).astype(np.float64)
    s = q @ lists.centroids.astype(np.float64).T
    order = np.stack([np.lexsort((np.arange(lists.nlist), -s[i]))[:nprobe] for i in range(q.shape[0])])
    return order.astype(np.int64), np.take_along_axis(s, order, axis=1)


def search(lists: IVFLists, queries: np.ndarray, nprobe: int, k: int, probed=None):
    """-> (ids int64 [nq, k], scores float64 [nq, k], gaps float64 [nq, k]); id -1 / score -inf where the probed
    lists hold fewer than k rows.  gaps as in search_oracle.topk_exact (near ties are compared as sets).  Exact ties
    go to the smaller stored position (list id, then original id).
    `probed = (list ids [nq, nprobe], coarse scores)` replaces the coarse pass: the fine pass can then be checked on
    exactly the lists, and with exactly the fp32 coarse terms, the engine used.  A list id < 0 or >= nlist is
    absent, and a list probed twice counts once (with its first coarse score)."""
    q = bf16_round(queries).astype(np.float64)
    nq = q.shape[0]
    probed, coarse = probe_lists(lists, queries, min(nprobe, lists.nlist)) if probed is None else probed
    out_i = np.full((nq, k), -1, dtype=np.int64)
    out_s = np.full((nq, k), -np.inf)
    gaps = np.full((nq, k), np.inf)
    for i in range(nq):
        cand_p: List[np.ndarray] = []
        cand_s: List[np.ndarray] = []
        seen = set()
        for l, cs in zip(probed[i], coarse[i]):
            l = int(l)
            if l < 0 or l >= lists.nlist or l in seen:
                continue
            seen.add(l)
            a, b = lists.offsets[l], lists.offsets[l + 1]
            if b > a:
                cand_p.append(np.arange(a, b))                     # stored positions: list order, then id
                cand_s.append(np.float32(cs).astype(np.float64) + lists.residuals[a:b].astype(np.float64) @ q[i])
        if not cand_p:
            continue
        cp, cs_ = np.concatenate(cand_p), np.concatenate(cand_s)
        order = np.lexsort((cp, -cs_))[:k + 1]
        ci = lists.ids[cp]
        m = min(k, order.size)
        out_i[i, :m], out_s[i, :m] = ci[order[:m]], cs_[order[:m]]
        d = cs_[order[:-1]] - cs_[order[1:]]
        gaps[i, :min(k, d.size)] = d[:k]
    return out_i, out_s, gaps


def recall_at_k(got_ids: np.ndarray, exact_ids: np.ndarray) -> float:
    """Mean fraction of the exact top-k ids that the IVF answer contains."""
    hits = [len(set(g[g >= 0].tolist()) & set(e.tolist())) / max(len(e), 1) for g, e in zip(got_ids, exact_ids)]
    return float(np.mean(hits))
