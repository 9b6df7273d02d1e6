"""numpy restatement of the IVF search over int8 residuals (crag_ivf_search_i8, QuantizedIVF), bit for bit.
DESIGN.md section 7 states the semantics; this module builds them from oracle/quant_oracle.py's quantiser, S1, S2
and key order, over the padded stored positions of an index laid out as the engine lays it out (ivf.ivf_layout).

  index     residuals bf16 [total_tiles * 128, dim] (zero padding rows), row_ids (-1 on padding), list_tile_start
            [nlist + 1], list_rows [nlist].  Every stored row is quantised (padding: scale 0), queries too.
  stage 1   for a row at position p of list l probed by query q:  S1 = fp32(fp32(acc) * fp32(s_q * s_p)) + coarse[q][l]
            over the list's real rows; the top n_cand by (S1 descending, position ascending), and (min, max) of S1.
  stage 2   S2 = fp32(dot + coarse[q][l]), dot = quant_oracle.s2_scores of the bf16 residual row and bf16 query; the
            top k by (S2 descending, position ascending), positions mapped to ids through row_ids; -1 / -inf past the
            valid candidates.

Test infrastructure only: the product path never imports this module.
"""
from __future__ import annotations

import numpy as np

from oracle import quant_oracle as qo

F32 = np.float32
TILE_ROWS = 128


def list_of_positions(list_tile_start: np.ndarray, p: np.ndarray) -> np.ndarray:
    """List l with list_tile_start[l] <= p // 128 < list_tile_start[l + 1] (empty lists own no tile)."""
    starts = np.asarray(list_tile_start, np.int64)
    return np.searchsorted(starts[1:], np.asarray(p, np.int64) // TILE_ROWS, side="right").astype(np.int64)


def rescore(residuals_f32: np.ndarray, list_tile_start: np.ndarray, coarse, queries_f32: np.ndarray,
            cand_pos: np.ndarray, k: int):
    """Stage 2 on positions: (positions [nq, k], S2 [nq, k]).  coarse(q, l) -> the fp32 coarse term; candidates
    outside [0, n_rows_padded) (-1 among them) are skipped."""
    nq = queries_f32.shape[0]
    n = residuals_f32.shape[0]
    pos = np.full((nq, k), -1, np.int64)
    sc = np.full((nq, k), -np.inf, F32)
    for j in range(nq):
        p = cand_pos[j].astype(np.int64)
        p = p[(p >= 0) & (p < n)]
        if p.size == 0:
            continue
        dot = qo.s2_scores(residuals_f32[p], queries_f32[j])
        lists = list_of_positions(list_tile_start, p)
        s2 = (dot + np.array([coarse(j, l) for l in lists], F32)).astype(F32)
        pos[j], sc[j] = qo.topk_keys(s2, p, k)
    return pos, sc


def _probed_of(probed, nq, nlist):
    ids, scores = (np.asarray(a) for a in probed)
    out = []
    for i in range(nq):
        d = {}
        for l, s in zip(ids[i], scores[i]):
            if 0 <= l < nlist:
                d[int(l)] = F32(s)
        out.append(d)
    return out


def search_i8(residuals_f32: np.ndarray, row_ids: np.ndarray, list_tile_start: np.ndarray, list_rows: np.ndarray,
              queries_f32: np.ndarray, probed, k: int, n_cand: int):
    """(ids [nq, k], S2 [nq, k], S1 minmax [nq, 2], (candidate positions [nq, n_cand], their S1)).  residuals_f32 /
    queries_f32 hold bf16 values; probed = (list ids [nq, nprobe] (-1 = none), fp32 coarse scores), as the coarse
    pass returns them."""
    residuals_f32 = np.asarray(residuals_f32, F32)
    queries_f32 = np.asarray(queries_f32, F32)
    nq, dim = queries_f32.shape
    nlist = len(list_rows)
    dim8 = qo.dim8_of(dim)
    r8, rs = qo.quantize(residuals_f32, dim8)
    q8, qs = qo.quantize(queries_f32, dim8)
    starts = np.asarray(list_tile_start, np.int64)
    lrows = np.asarray(list_rows, np.int64)
    per_q = _probed_of(probed, nq, nlist)
    c_pos = np.full((nq, n_cand), -1, np.int64)
    c_sc = np.full((nq, n_cand), -np.inf, F32)
    mm = np.tile(np.array([np.inf, -np.inf], F32), (nq, 1))
    for i in range(nq):
        pos, s1 = [], []
        for l, cs in sorted(per_q[i].items()):
            if lrows[l] <= 0:
                continue
            p = starts[l] * TILE_ROWS + np.arange(lrows[l], dtype=np.int64)
            s = qo.s1_scores(r8[p], rs[p], q8[i:i + 1], qs[i:i + 1])[0]
            pos.append(p)
            s1.append((s + cs).astype(F32))
        if not pos:
            continue
        p, s = np.concatenate(pos), np.concatenate(s1)
        c_pos[i], c_sc[i] = qo.topk_keys(s, p, n_cand)
        o = qo.orderable(s)
        mm[i] = s[np.argmin(o)], s[np.argmax(o)]
    pos, sc = rescore(residuals_f32, starts, lambda j, l: per_q[j][int(l)], queries_f32, c_pos, k)
    ids = np.where(pos >= 0, np.asarray(row_ids, np.int64)[np.maximum(pos, 0)], -1)
    return ids, sc, mm, (c_pos, c_sc)


def padded_layout(lists, row_offset: int = 0):
    """ivf_oracle.IVFLists -> the engine's padded layout: (residuals float32 [total_tiles * 128, dim] with zero padding,
    row_ids int64 (-1 on padding), list_tile_start int32 [nlist + 1], list_rows int32 [nlist])."""
    counts = np.diff(lists.offsets)
    tiles = (counts + TILE_ROWS - 1) // TILE_ROWS
    starts = np.concatenate([[0], np.cumsum(tiles)]).astype(np.int64)
    n = int(starts[-1]) * TILE_ROWS
    res = np.zeros((n, lists.residuals.shape[1]), F32)
    row_ids = np.full(n, -1, np.int64)
    for l in range(lists.nlist):
        a, b = lists.offsets[l], lists.offsets[l + 1]
        p = starts[l] * TILE_ROWS + np.arange(b - a)
        res[p] = lists.residuals[a:b]
        row_ids[p] = lists.ids[a:b] + row_offset
    return res, row_ids, starts.astype(np.int32), counts.astype(np.int32)
