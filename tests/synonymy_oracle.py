"""The synonymy-edge walk of add_synonymy_edges, restated in numpy (test infrastructure).

For query q over fp32 scores S[q, :] (key rows 0 .. n - 1):
  1. L = the first min(limit, n) rows in crag_knn_topk's order: score descending by the orderable key (so -0.0 ranks
     below +0.0 and a positive NaN above +inf), then row ascending;
  2. walk L: stop at the first entry with !(S >= threshold) compared as fp32, skip self_rows[q] and every row of
     exclude_rows, accept the others until `cap` are accepted;
  3. (count, ids [cap], scores [cap]) with -1 / -inf past the count.
`fp32_threshold` turns the configured double threshold into the smallest fp32 >= it, which makes the fp32 compare of
step 2 the double compare the reference makes (a Python float from the fp32 score against a Python float)."""
from __future__ import annotations

import numpy as np


def orderable(s: np.ndarray) -> np.ndarray:
    """orderable_f32 of fp32 scores, as uint64."""
    u = np.ascontiguousarray(s, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return np.where(u & 0x80000000, (~u) & 0xFFFFFFFF, u | 0x80000000)


def rank_order(s: np.ndarray, limit: int) -> np.ndarray:
    """The first min(limit, n) rows of one score row in crag_knn_topk's order."""
    n = s.shape[0]
    order = np.lexsort((np.arange(n), -orderable(s).astype(np.int64)))
    return order[: min(limit, n)]


def fp32_threshold(t: float) -> np.float32:
    """The smallest fp32 >= the double t."""
    f = np.float32(t)
    if float(f) < float(t):
        f = np.nextafter(f, np.float32(np.inf))
    return f


def walk(s: np.ndarray, threshold: np.float32, limit: int, cap: int, self_row: int = -1, exclude_rows=()):
    """One query: (count, ids int64 [cap], scores fp32 [cap])."""
    s = np.asarray(s, dtype=np.float32)
    skip = set(int(r) for r in exclude_rows) | {int(self_row)}
    ids = np.full(cap, -1, dtype=np.int64)
    sc = np.full(cap, -np.inf, dtype=np.float32)
    count = 0
    t = np.float32(threshold)
    for r in rank_order(s, limit):
        if count == cap or not (s[r] >= t):
            break
        if int(r) in skip:
            continue
        ids[count], sc[count] = r, s[r]
        count += 1
    return count, ids, sc


def walk_all(S: np.ndarray, threshold, limit: int, cap: int, self_rows=None, exclude_rows=()):
    """Every query of S [nq, n]: (counts int32 [nq], ids int64 [nq, cap], scores fp32 [nq, cap])."""
    S = np.asarray(S, dtype=np.float32)
    nq = S.shape[0]
    counts = np.zeros(nq, dtype=np.int32)
    ids = np.full((nq, cap), -1, dtype=np.int64)
    sc = np.full((nq, cap), -np.inf, dtype=np.float32)
    for q in range(nq):
        counts[q], ids[q], sc[q] = walk(S[q], threshold, limit, cap, -1 if self_rows is None else int(self_rows[q]),
                                        exclude_rows)
    return counts, ids, sc


def edges_from_knn(knn: dict, contents: dict, threshold: float, cap: int = 101):
    """The add_synonymy_edges loop over a retrieve_knn-shaped dict {key: (neighbour keys, scores)}: eligible query keys
    (more than 2 alphanumerics) in the dict's order, each walked in list order -- stop at the first score below the
    double threshold, skip the key itself and keys whose content is '', accept up to cap.  Returns the list of
    ((key, nn), score) assignments in the order they are made."""
    import re
    out = []
    for key, (nns, scores) in knn.items():
        if len(re.sub('[^A-Za-z0-9]', '', contents[key])) <= 2:
            continue
        taken = 0
        for nn, score in zip(nns, scores):
            if score < threshold or taken >= cap:
                break
            if nn != key and contents[nn] != '':
                out.append(((key, nn), score))
                taken += 1
    return out
