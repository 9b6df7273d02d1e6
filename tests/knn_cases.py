"""Case builders for the exact tests of crag_knn_topk (test infrastructure: seeded, built on any device).

crag_knn_topk writes an fp32 score block with the wgmma GEMM and then selects each query's k best rows with
csrc/knn_select.cuh: three radix passes over orderable_f32(score) with 11/11/10-bit digits find the k-th best score
word T and `quota`, how many of the k kept rows score exactly T; a gather in row order, 2 048 rows per iteration (512
threads x one float4), keeps every row above T and the FIRST `quota` rows equal to T; a bitonic sort orders them.

The random kinds of the scan family (unit, scaled, dyadic, near_dup rows, strided views) are re-exported from
test_scan_exact_gpu.py.  The integer-score corpora added here pin the select's hard regimes with answers that need no
kernel: every bf16 entry is a small integer or a power of two, and sum_i |q_i x_i| < 2^24 (times the query's
power-of-two scale), so every partial sum is exact in fp32 whatever the summation order, and the score of row r is
exactly its planned integer.  The rows hold that integer as balanced base-128 digits in one column of each of the
first four 64-wide K blocks, against query weights 1, 2^7, 2^14 and 2^21; the other columns carry pairs of entries
that cancel (u against one query weight, -u against the same weight), so every K block adds to the sum.

regime(scores, k) states where a case lands in knn_select.cuh's plan, and two deliberately wrong selectors show that
the exact reference can tell a case's answer from theirs."""
from __future__ import annotations

import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import scan_reference as sr  # noqa: E402
from test_scan_exact_gpu import corpus, queries_for, scaled, strided  # noqa: E402,F401

GATHER_ROWS = 2048                              # rows per gather iteration: 512 threads x 4 scores
DIGITS = ((21, 11), (10, 11), (0, 10))          # (shift, bits) of radix passes 0, 1, 2
INT_DIM = 256
DIGIT_COLS = (3, 70, 141, 200)                  # one column in each of the first four K blocks
DIGIT_WEIGHTS = (1, 1 << 7, 1 << 14, 1 << 21)
QUERY_SCALES = (1.0, 2.0 ** -12, -(2.0 ** 6))   # query j is the weight vector times QUERY_SCALES[j]
EXACT_LIMIT = 2 ** 24


# ------------------------------------------------------------------------------------------------- integer corpora
def _digits(s: torch.Tensor) -> torch.Tensor:
    """Balanced base-128 digits [n, 4] of int64 s: s = sum_j d_j * DIGIT_WEIGHTS[j], |d_0..2| <= 64, |d_3| <= 4."""
    out, rest = [], s.clone()
    for _ in range(3):
        d = torch.remainder(rest + 64, 128) - 64
        out.append(d)
        rest = (rest - d) // 128
    assert bool((rest.abs() <= 4).all()), "score outside the representable range"
    out.append(rest)
    return torch.stack(out, dim=1)


def int_rows(s: torch.Tensor, seed: int, identical_noise: bool = False) -> torch.Tensor:
    """bf16 [n, INT_DIM] rows whose dot product with int_queries()[0] is exactly s (int64 [n])."""
    n = s.numel()
    g = torch.Generator().manual_seed(seed)
    x = torch.zeros((n, INT_DIM), dtype=torch.float32)
    x[:, list(DIGIT_COLS)] = _digits(s.to(torch.int64)).float()
    noise = [c for c in range(INT_DIM) if c not in DIGIT_COLS]
    a, b = torch.tensor(noise[0::2]), torch.tensor(noise[1::2][: len(noise[0::2])])
    u = torch.randint(-8, 9, (1 if identical_noise else n, a.numel()), generator=g).float().expand(n, -1)
    x[:, a], x[:, b] = u, -u
    return x.bfloat16()


def int_queries() -> torch.Tensor:
    """bf16 [len(QUERY_SCALES), INT_DIM]: the digit weights, the noise columns' weights, times each scale."""
    w = torch.zeros(INT_DIM, dtype=torch.float32)
    noise = [c for c in range(INT_DIM) if c not in DIGIT_COLS]
    m = min(len(noise[0::2]), len(noise[1::2]))
    wn = torch.tensor([1.0, 2.0, -1.0, 4.0])[torch.arange(m) % 4]
    w[torch.tensor(noise[0::2][:m])], w[torch.tensor(noise[1::2][:m])] = wn, wn
    w[list(DIGIT_COLS)] = torch.tensor([float(v) for v in DIGIT_WEIGHTS])
    return (torch.tensor(QUERY_SCALES)[:, None] * w[None, :]).bfloat16()


def _perm(n, g):
    return torch.randperm(n, generator=g)


def _planted_ties(n, k, quota, t, above, below, tie_rows, g):
    """Scores with exactly k - quota rows above t (values drawn from `above`), t on tie_rows, `below` elsewhere."""
    s = torch.tensor(below, dtype=torch.int64)[torch.randint(len(below), (n,), generator=g)]
    s[tie_rows] = t
    free = torch.ones(n, dtype=torch.bool)
    free[tie_rows] = False
    cand = free.nonzero()[:, 0]
    top = cand[_perm(cand.numel(), g)[: k - quota]]
    s[top] = torch.tensor(above, dtype=torch.int64)[torch.randint(len(above), (top.numel(),), generator=g)]
    return s


def _spread_ties(n, quota, g, iters=4.5):
    """Tie rows at a density that meets the quota about `iters` gather iterations in: a run of thousands overall."""
    p = quota / (iters * GATHER_ROWS)
    return (torch.rand(n, generator=g) < p).nonzero()[:, 0]


def _scores(name: str, g: torch.Generator):
    """(k, planned int64 scores [n]) of a named case."""
    if name == "pass0":                        # k-th 2^20, (k+1)-th below 2^19: the exponents differ
        n, k = 4097, 1000
        s = torch.cat([(1 << 20) + 3 * torch.arange(k), (1 << 18) + 5 * torch.arange(n - k)])
        return k, s[_perm(n, g)]
    if name == "pass1":                        # 2^22 + 512 j: mantissas apart in bits 10..20 only
        n, k = 4097, 1000
        return k, (1 << 22) + 512 * _perm(n, g).to(torch.int64)
    if name == "pass2":                        # 2^23 + j, j < 1024: one fp32 ulp apart, only the low 10-bit digit
        n, k = 4097, 1000                      # j = 1023 - r // 4 at sorted rank r: ranks 999 and 1000 differ
        s = (1 << 23) + 1023 - torch.arange(n).clamp(max=4095) // 4
        return k, s[_perm(n, g)]
    if name == "ulp_ties":                     # 2^23 + j again, ~98 rows per value: a tie decided in the last digit
        n, k = 100_003, 1000
        return k, (1 << 23) + torch.randint(0, 1024, (n,), generator=g)
    if name.startswith("long_tie_"):           # narrow range 0..7, the tie run at 3 spans 4-5 iterations to the quota
        k = int(name.rsplit("_", 1)[1])
        n, quota = 100_003, k - k // 3
        return k, _planted_ties(n, k, quota, 3, [4, 5, 6, 7], [0, 1, 2], _spread_ties(n, quota, g), g)
    if name == "all_negative":                 # every score negative, the tie run as above
        n, k = 20_001, 1000
        quota = 600
        return k, _planted_ties(n, k, quota, -5, [-4, -3, -2, -1], [-9, -8, -7, -6], _spread_ties(n, quota, g), g)
    if name == "tie_from_row0":                # ties are rows 0 .. 599, score 0
        n, k = 4097, 129
        return k, _planted_ties(n, k, 100, 0, [1, 2], [-2, -1], torch.arange(600), g)
    if name == "tie_to_last_row":              # every 7th row up to the last one ties at 0 and all of them are kept;
        n, k = 4097, 700                       # n % 4 == 1, so the last row shares its float4 with three dead lanes
        ties = torch.arange(n - 1, -1, -7)
        return k, _planted_ties(n, k, ties.numel(), 0, [1, 2, 3], [-3, -2, -1], ties, g)
    if name == "constant":                     # identical rows: n_eq = n
        return 2047, torch.full((10_001,), 7, dtype=torch.int64)
    if name == "dup_2048":                     # row r repeats row r mod 2048: copies 2 048 j rows apart
        n, k = 6 * GATHER_ROWS + 5, 129
        base = (_perm(GATHER_ROWS, g).to(torch.int64) - 1000) * 3
        return k, base[torch.arange(n) % GATHER_ROWS]
    if name == "take_all":                     # n <= k with ties: the sort-only path
        return 2048, torch.randint(-3, 4, (2000,), generator=g)
    raise KeyError(name)


# name -> (regime fields the case must land in, wrong selectors whose answer must differ from the reference's)
INT_CASES = {
    "pass0": ({"pass": 0, "ordered_ties": False}, ()),
    "pass1": ({"pass": 1, "ordered_ties": False}, ()),
    "pass2": ({"pass": 2, "ordered_ties": False}, ()),
    "ulp_ties": ({"pass": "tie", "ordered_ties": True}, ("last_ties",)),
    "long_tie_129": ({"pass": "tie", "ordered_ties": True, "long": True}, ("last_ties",)),
    "long_tie_1000": ({"pass": "tie", "ordered_ties": True, "long": True}, ("last_ties",)),
    "long_tie_2048": ({"pass": "tie", "ordered_ties": True, "long": True}, ("last_ties",)),
    "all_negative": ({"pass": "tie", "ordered_ties": True, "long": True, "all_negative": True}, ("last_ties",)),
    "tie_from_row0": ({"pass": "tie", "ordered_ties": True, "first_tie_row": 0}, ("last_ties",)),
    "tie_to_last_row": ({"ordered_ties": False, "last_tie_row": -1, "take_all": False}, ("trailing_row",)),
    "constant": ({"pass": "tie", "ordered_ties": True, "n_eq": "n"}, ("last_ties",)),
    "dup_2048": ({"pass": "tie", "ordered_ties": True, "dup_stride": GATHER_ROWS}, ("last_ties",)),
    "take_all": ({"take_all": True}, ()),
}
LONG_TIE_CASES = [c for c, (want, _) in INT_CASES.items() if want.get("long")]


def int_case(name: str, seed: int = 0, device="cpu"):
    """(rows bf16 [n, INT_DIM], queries bf16 [3, INT_DIM], S float64 [3, n] exact scores, k, planned int64 [n])."""
    g = torch.Generator().manual_seed(1000 + seed + sum(map(ord, name)))
    k, s = _scores(name, g)
    rows = int_rows(s, seed=seed + 7, identical_noise=name in ("constant", "dup_2048"))
    if name == "dup_2048":
        rows = rows[torch.arange(s.numel()) % GATHER_ROWS]
    q = int_queries()
    # + 0.0: an exact zero is +0, as a sum that starts from a +0 accumulator ends (-64 * 0 alone would be -0)
    S = torch.tensor(QUERY_SCALES, dtype=torch.float64)[:, None] * s.double()[None, :] + 0.0
    return rows.to(device), q.to(device), S.to(device), k, s


def exactness(rows: torch.Tensor, queries: torch.Tensor):
    """(float64 q . x, max over the block of sum_i |q_i x_i| / |scale|): the score is exact in fp32 under any
    summation order when the second is below EXACT_LIMIT."""
    ref, mag = sr.score_reference(queries.cpu(), rows.cpu())
    scale = torch.tensor(QUERY_SCALES, dtype=torch.float64).abs()[:, None]
    return ref, float((mag / scale).max())


# ----------------------------------------------------------------------------------------------------------- regime
def regime(scores: torch.Tensor, k: int) -> dict:
    """Where one query's fp32 scores [n] land in knn_select.cuh's plan at this k:
      take_all      n <= k (no radix select: every row is sorted)
      pass          the radix pass (0, 1, 2) whose digit first tells the k-th key's score word from the (k+1)-th's,
                    or "tie" when the two score words are equal
      T_score, quota, n_eq, ordered_ties     as the kernel computes them (ordered_ties: quota < n_eq)
      tie_rows      the rows scoring exactly T, ascending
      tie_iters     the gather iterations (row // 2048) holding tie rows
      iters_to_quota  how many of those iterations hold one of the first `quota` ties
      quota_row, quota_iter, quota_pos      the quota-th tie row, its iteration and its place inside it
      ties_after_in_iter   tie rows after quota_row in the same iteration (left out by the same block scan)"""
    s = scores.detach().to(torch.float32).cpu().reshape(-1)
    n = s.numel()
    out = {"n": n, "k": k, "take_all": n <= k}
    if n <= k:
        return out
    o = sr.orderable(s)
    desc = torch.sort(o, descending=True, stable=True).values
    t, nxt = int(desc[k - 1]), int(desc[k])
    if t == nxt:
        p = "tie"
    else:
        p = next(i for i, (sh, _) in enumerate(DIGITS) if (t >> sh) != (nxt >> sh))
    ties = (o == t).nonzero()[:, 0]
    quota = k - int((o > t).sum())
    qrow = int(ties[quota - 1])
    out.update({
        "pass": p, "T_score": float(s[ties[0]]), "quota": quota, "n_eq": ties.numel(), "ordered_ties": quota < ties.numel(),
        "tie_rows": ties, "tie_iters": sorted(set((ties // GATHER_ROWS).tolist())),
        "iters_to_quota": len(set((ties[:quota] // GATHER_ROWS).tolist())),
        "quota_row": qrow, "quota_iter": qrow // GATHER_ROWS, "quota_pos": qrow % GATHER_ROWS,
        "ties_after_in_iter": int(((ties > qrow) & (ties // GATHER_ROWS == qrow // GATHER_ROWS)).sum()),
    })
    return out


# ------------------------------------------------------------------------------------------------- wrong selectors
def topk_keep_last_ties(S: torch.Tensor, k: int, row_offset: int = 0):
    """A gather that keeps the LAST `quota` rows equal to T instead of the first: (ids, scores) [nq, k]."""
    S = S.to(torch.float32)
    nq, n = S.shape
    ids, sc = [], []
    for q in range(nq):
        if n <= k:
            i, v, _, _ = sr.topk_from_scores(S[q:q + 1], k, row_offset)
            ids.append(i[0]), sc.append(v[0])
            continue
        r = regime(S[q], k)
        o = sr.orderable(S[q])
        t = int(sr.orderable(torch.tensor([r["T_score"]]))[0])
        kept = torch.cat([(o > t).nonzero()[:, 0], r["tie_rows"][r["n_eq"] - r["quota"]:]])
        sub = S[q:q + 1, kept]
        i, v, _, _ = sr.topk_from_scores(sub, k)
        # ranks among the kept rows keep their (score desc, row asc) order: map the columns back to rows
        ids.append(kept[i[0]] + row_offset), sc.append(v[0])
    return torch.stack(ids), torch.stack(sc)


def topk_drop_trailing(S: torch.Tensor, k: int, row_offset: int = 0):
    """A select that reads n // 4 whole float4s and so ignores the last n % 4 rows: (ids, scores, minmax)."""
    n = S.shape[1]
    ids, sc, mm, _ = sr.topk_from_scores(S[:, : n - n % 4], k, row_offset)
    return ids, sc, mm
