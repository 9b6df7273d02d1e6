"""Exact reference of the bf16 scan family, built from a score matrix (torch, CPU or CUDA; test infrastructure).

Every bf16 scan variant -- the flat top-k (crag_search_topk / _after), the IVF fine pass (crag_ivf_search) and the IVF
assignment (crag_ivf_assign) -- runs the score-all pass's main loop: the same TMA boxes, K-block order, m64n32k16
instructions and query slot per 32-query pass.  So the fp32 scores that crag_search_scores writes for a (rows,
queries) pair are the scores every other variant ranks, and what those variants return is a function of that matrix:

  keys      key = orderable(score) << 32 | (0xFFFFFFFF - row), compared as unsigned 64-bit (topk.cuh): score
            descending, then row ascending; +0 ranks above -0.  `row` is the local row (flat) or the stored position
            (IVF), below 2^31.
  flat      the first k keys of each query's row of S; ids = row + row_offset; -1 / -inf past n_rows; (min, max) of the
            row, ordered as the keys order scores; the k-th key (0 when fewer than k rows) continues a page: the next
            page takes keys strictly below it.
  IVF       S_res = score-all over the padded residual matrix.  A real position p of a list l that query q probes
            scores fp32(S_res[q, p] + coarse[q, l]); a probe id -1 or >= nlist is absent and a repeated probe counts
            once.  Top k by (score desc, position asc), positions mapped to ids through row_ids; (min, max) over the
            probed real rows, (+inf, -inf) when there are none.
  assign    the first argmax over the centroids in ascending list id, and its score.

The score-all pass itself is held to float64 under SCORE_BOUND (see score_bound).
"""
from __future__ import annotations

import torch

SIGN = -(1 << 63)           # int64 with only bit 63 set: x ^ SIGN maps unsigned order onto signed order
TILE_ROWS = 128
# |s - ref| <= 2^-16 sum_i |q_i x_i|.  A bf16 x bf16 product is exact in fp32, so all error is accumulation: at most
# 1024 / 16 = 64 k16 steps, each adding one fp32 rounding (or truncation, 2^-23) relative to a partial sum bounded by
# sum |q_i x_i|: 64 * 2^-23 = 2^-17.  The other factor of 2 covers the alignment inside one k16 step.  The score is
# stored as the fp32 accumulator: no output rounding.
SCORE_BOUND = 2.0 ** -16


# ------------------------------------------------------------------------------------------------------------- keys
def orderable(scores: torch.Tensor) -> torch.Tensor:
    """orderable_f32 of fp32 scores as int64 in [0, 2^32)."""
    u = scores.contiguous().to(torch.float32).view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    return torch.where((u & 0x80000000) != 0, (~u) & 0xFFFFFFFF, u | 0x80000000)


def _rank(scores: torch.Tensor, rows: torch.Tensor) -> torch.Tensor:
    """Signed int64 with the order of the unsigned keys (key ^ SIGN), computed without overflow."""
    return (orderable(scores) - (1 << 31)) * (1 << 32) + (0xFFFFFFFF - rows.to(torch.int64))


def keys(scores: torch.Tensor, rows: torch.Tensor) -> torch.Tensor:
    """The kernels' 64-bit keys, as the bit patterns of an int64 tensor (what crag_search_topk_after's last_keys
    holds).  Compare them as unsigned, or through key ^ SIGN as signed."""
    return _rank(scores, rows) ^ SIGN


def ordered_minmax(s: torch.Tensor, valid: torch.Tensor):
    """(min, max) of each row of s over `valid`, ordered as the keys order scores; (+inf, -inf) where none is valid."""
    o = orderable(s)
    lo = torch.where(valid, o, torch.full_like(o, 1 << 33)).argmin(dim=1, keepdim=True)
    hi = torch.where(valid, o, torch.full_like(o, -1)).argmax(dim=1, keepdim=True)
    any_ = valid.any(dim=1)
    mn = torch.where(any_, s.gather(1, lo)[:, 0], torch.full_like(s[:, 0], float("inf")))
    mx = torch.where(any_, s.gather(1, hi)[:, 0], torch.full_like(s[:, 0], float("-inf")))
    return torch.stack([mn, mx], dim=1)


def _select(rank: torch.Tensor, valid: torch.Tensor, k: int):
    """The k largest ranks of each row among `valid`: (rank [nq, k], column [nq, k], present [nq, k])."""
    nq, n = rank.shape
    r = torch.where(valid, rank, torch.full_like(rank, SIGN))
    if n < k:
        r = torch.cat([r, torch.full((nq, k - n), SIGN, dtype=torch.int64, device=r.device)], dim=1)
    top, col = torch.topk(r, k, dim=1, largest=True, sorted=True)
    return top, col, top != SIGN


# ------------------------------------------------------------------------------------------------------------- flat
def topk_from_scores(S: torch.Tensor, k: int, row_offset: int = 0, after_keys: torch.Tensor = None):
    """Flat top-k of the score matrix S fp32 [nq, n_rows]: (ids int64 [nq, k], scores fp32 [nq, k], minmax fp32
    [nq, 2], last_keys int64 [nq]).  after_keys (key bits [nq], as last_keys) admits only keys strictly below."""
    S = S.to(torch.float32)
    nq, n = S.shape
    rows = torch.arange(n, device=S.device, dtype=torch.int64).expand(nq, n)
    rank = _rank(S, rows)
    valid = torch.ones_like(rank, dtype=torch.bool)
    if after_keys is not None:
        valid = rank < (after_keys.to(S.device).to(torch.int64) ^ SIGN)[:, None]
    top, col, present = _select(rank, valid, k)
    colc = col.clamp(max=max(n - 1, 0))
    ids = torch.where(present, colc + int(row_offset), torch.full_like(col, -1))
    sc = torch.where(present, S.gather(1, colc) if n else torch.zeros_like(top, dtype=torch.float32),
                     torch.full(top.shape, float("-inf"), device=S.device))
    last = torch.where(present[:, -1], top[:, -1] ^ SIGN, torch.zeros_like(top[:, -1]))
    return ids, sc, ordered_minmax(S, torch.ones_like(rank, dtype=torch.bool)), last


# -------------------------------------------------------------------------------------------------------------- IVF
def list_of_positions(list_tile_start: torch.Tensor, n_pos: int) -> torch.Tensor:
    """The list owning each stored position 0 .. n_pos - 1 (empty lists own no tile)."""
    starts = list_tile_start.to(torch.int64)
    tiles = torch.arange(n_pos, device=starts.device, dtype=torch.int64) // TILE_ROWS
    return torch.searchsorted(starts[1:].contiguous(), tiles, right=True)


def probe_table(probed_ids: torch.Tensor, probed_scores: torch.Tensor, nlist: int):
    """(mask bool [nq, nlist], coarse fp32 [nq, nlist]) of the caller's probes: ids -1 or >= nlist are absent, a
    repeated probe counts once and must repeat its coarse score (the plan keeps one of them)."""
    ids = probed_ids.cpu().to(torch.int64)
    sbits = probed_scores.cpu().to(torch.float32).contiguous().view(torch.int32)
    nq, nprobe = ids.shape
    mask = torch.zeros((nq, nlist), dtype=torch.bool)
    cbits = torch.zeros((nq, nlist), dtype=torch.int32)
    for q in range(nq):
        for j in range(nprobe):
            l = int(ids[q, j])
            if 0 <= l < nlist:
                assert not mask[q, l] or cbits[q, l] == sbits[q, j], "a repeated probe needs one coarse score"
                mask[q, l], cbits[q, l] = True, sbits[q, j]
    return mask, cbits.view(torch.float32)


def ivf_from_scores(S_res: torch.Tensor, probed_ids: torch.Tensor, probed_scores: torch.Tensor,
                    list_tile_start: torch.Tensor, list_rows: torch.Tensor, row_ids: torch.Tensor, k: int):
    """crag_ivf_search from the score-all matrix S_res fp32 [nq, n_rows_padded] of the queries against the padded
    residuals: (ids int64 [nq, k], scores fp32 [nq, k], minmax fp32 [nq, 2])."""
    dev = S_res.device
    S_res = S_res.to(torch.float32)
    nq, n_pos = S_res.shape
    nlist = list_rows.numel()
    mask, coarse = (t.to(dev) for t in probe_table(probed_ids, probed_scores, nlist))
    lst = list_of_positions(list_tile_start.to(dev), n_pos)
    starts = list_tile_start.to(dev).to(torch.int64)
    pos = torch.arange(n_pos, device=dev, dtype=torch.int64)
    real = (pos - starts[lst] * TILE_ROWS) < list_rows.to(dev).to(torch.int64)[lst]
    valid = mask[:, lst] & real[None, :]
    s = S_res + coarse[:, lst]                                     # fp32 + fp32, rounded to nearest
    top, col, present = _select(_rank(s, pos.expand(nq, n_pos)), valid, k)
    colc = col.clamp(max=max(n_pos - 1, 0))
    ids = torch.where(present, row_ids.to(dev).to(torch.int64)[colc], torch.full_like(col, -1))
    sc = torch.where(present, s.gather(1, colc), torch.full(top.shape, float("-inf"), device=dev))
    return ids, sc, ordered_minmax(s, valid)


# ----------------------------------------------------------------------------------------------------------- assign
def assign_from_scores(S_cent: torch.Tensor):
    """crag_ivf_assign from the score-all matrix S_cent fp32 [nlist, n_rows] of the centroids (as queries) against
    the rows: (list id int32 [n_rows], its score fp32 [n_rows]); ties to the smaller list id."""
    S_cent = S_cent.to(torch.float32)
    nlist, n = S_cent.shape
    best = torch.full((n,), float("-inf"), device=S_cent.device)
    ids = torch.zeros(n, dtype=torch.int32, device=S_cent.device)
    for l in range(nlist):                 # strict >: a later list must beat the best so far, as the kernel's update
        s = S_cent[l]
        take = s > best
        best = torch.where(take, s, best)
        ids = torch.where(take, torch.full_like(ids, l), ids)
    return ids, best


# ------------------------------------------------------------------------------------------------- bound and checks
def score_reference(queries_bf16: torch.Tensor, rows_bf16: torch.Tensor):
    """(float64 q . x [nq, n], sum_i |q_i x_i| [nq, n]) on the tensors' device."""
    q, x = queries_bf16.double(), rows_bf16.double()
    return q @ x.T, q.abs() @ x.abs().T


def err_over_bound(S: torch.Tensor, ref: torch.Tensor, mag: torch.Tensor) -> float:
    """Worst |S - ref| / (SCORE_BOUND * mag); an exact zero error counts 0 even where the bound is 0."""
    err = (S.double() - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / (SCORE_BOUND * mag))
    return float(torch.nan_to_num(r, nan=float("inf")).max()) if r.numel() else 0.0


def assert_bits(got: torch.Tensor, want: torch.Tensor, what: str = "") -> None:
    """Bit-for-bit equality (fp32 compared as their bit patterns, so -0 != +0 and NaN payloads count)."""
    got, want = got.detach().cpu(), want.detach().cpu()
    assert got.shape == want.shape, (what, tuple(got.shape), tuple(want.shape))
    if got.dtype == torch.float32:
        got, want = got.view(torch.int32), want.view(torch.int32)
    assert got.dtype == want.dtype, (what, got.dtype, want.dtype)
    bad = (got != want).nonzero()
    assert bad.numel() == 0, f"{what}: {bad.shape[0]} mismatches, first at {bad[:5].tolist()}"
