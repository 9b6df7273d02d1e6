"""numpy restatement of the int8 shard search (crag_quantize_rows_i8 -> crag_search_topk_i8 -> crag_rescore_topk):
quantise -> S1 -> top k' -> S2 -> top k, bit for bit.  DESIGN.md section 3e states the semantics.

  quantise  s = float32(amax) / 127 (float32 division, round to nearest); x^ = clip(rint(x / s), -127, 127) with rint
            rounding half to even; a zero row has s = 0 and x^ = 0.  Columns dim .. dim8 - 1 are zero.
  S1        float32(sum q^ x^) * float32(s_q * s_row): the integer dot is exact (|acc| <= 127^2 * 1024 < 2^24, so every
            float32 partial sum and the conversion are exact too).
  S2        the fp32 dot of the bf16 row and query in the kernel's order: 8-element chunks dealt to 32 lanes
            round-robin, each lane adding its products in element order from 0, then an xor tree over 16, 8, 4, 2, 1.
  ranking   (score descending, row ascending), with scores ordered as their orderable_f32 keys order them (-0 < +0).
"""
from __future__ import annotations

import numpy as np

F32 = np.float32


def dim8_of(dim: int) -> int:
    return (dim + 127) // 128 * 128


def quant_value(x: np.ndarray, s: np.ndarray) -> np.ndarray:
    """clamp(rint(x / s), -127, 127) in float32 (s != 0)."""
    return np.clip(np.rint(np.asarray(x, F32) / np.asarray(s, F32)), -127, 127).astype(np.int8)


def quantize(x: np.ndarray, dim8: int | None = None) -> tuple[np.ndarray, np.ndarray]:
    """float32 rows [n, dim] (bf16 values) -> (int8 [n, dim8], float32 scales [n])."""
    x = np.asarray(x, F32)
    n, dim = x.shape
    dim8 = dim8_of(dim) if dim8 is None else dim8
    amax = np.abs(x).max(axis=1) if dim else np.zeros(n, F32)
    s = (amax / F32(127)).astype(F32)
    q = np.zeros((n, dim8), np.int8)
    nz = s != 0
    if nz.any():
        q[nz, :dim] = quant_value(x[nz], s[nz, None])
    return q, s


def s1_scores(rows_i8: np.ndarray, row_scales: np.ndarray, q_i8: np.ndarray, q_scales: np.ndarray) -> np.ndarray:
    """S1 [nq, n] of int8 rows and queries."""
    # exact: every partial sum is an integer below 127^2 * 1024 < 2^24, which float32 holds exactly in any order
    acc = q_i8.astype(F32) @ rows_i8.astype(F32).T
    scale = (q_scales.astype(F32)[:, None] * row_scales.astype(F32)[None, :]).astype(F32)
    return (acc.astype(F32) * scale).astype(F32)


def orderable(s: np.ndarray) -> np.ndarray:
    u = np.ascontiguousarray(s, F32).view(np.uint32).astype(np.uint64)
    return np.where(u & 0x80000000, (~u) & 0xFFFFFFFF, u | 0x80000000)


def topk_keys(scores: np.ndarray, rows: np.ndarray, k: int) -> tuple[np.ndarray, np.ndarray]:
    """Top k of one query's (score, row) pairs by (score desc, row asc): (rows [k], scores [k]), -1 / -inf padded."""
    key = (orderable(scores) << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - rows.astype(np.uint64))
    m = min(k, key.size)
    if key.size > m:
        part = np.argpartition(key, key.size - m)[key.size - m:]
    else:
        part = np.arange(key.size)
    order = part[np.argsort(key[part])[::-1]]
    ids = np.full(k, -1, np.int64)
    sc = np.full(k, -np.inf, F32)
    ids[:m] = rows[order]
    sc[:m] = scores[order]
    return ids, sc


def search_i8(rows_i8, row_scales, q_i8, q_scales, k: int, row_offset: int = 0):
    """crag_search_topk_i8: (ids [nq, k], S1 [nq, k], minmax [nq, 2])."""
    n = rows_i8.shape[0]
    nq = q_i8.shape[0]
    ids = np.full((nq, k), -1, np.int64)
    sc = np.full((nq, k), -np.inf, F32)
    mm = np.tile(np.array([np.inf, -np.inf], F32), (nq, 1))
    if n == 0:
        return ids, sc, mm
    rows = np.arange(n, dtype=np.int64)
    for q0 in range(0, nq, 32):
        s1 = s1_scores(rows_i8, row_scales, q_i8[q0:q0 + 32], q_scales[q0:q0 + 32])
        for j in range(s1.shape[0]):
            i, s = topk_keys(s1[j], rows, k)
            ids[q0 + j] = np.where(i >= 0, i + row_offset, -1)
            sc[q0 + j] = s
            o = orderable(s1[j])
            mm[q0 + j] = s1[j][np.argmin(o)], s1[j][np.argmax(o)]
    return ids, sc, mm


def s2_scores(rows: np.ndarray, q: np.ndarray) -> np.ndarray:
    """The rescore kernel's fp32 dot of each row of `rows` [m, dim] with q [dim] (bf16 values as float32)."""
    rows = np.asarray(rows, F32)
    q = np.asarray(q, F32)
    m, dim = rows.shape
    assert dim % 8 == 0
    n_chunks = dim // 8
    rounds = (n_chunks + 31) // 32
    prod = np.zeros((m, rounds * 32, 8), F32)
    prod[:, :n_chunks] = (rows * q[None, :]).astype(F32).reshape(m, n_chunks, 8)
    prod = prod.reshape(m, rounds, 32, 8)          # [m, round, lane, element]
    partial = np.zeros((m, 32), F32)
    for r in range(rounds):
        for e in range(8):
            partial = (partial + prod[:, r, :, e]).astype(F32)
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        partial = (partial + partial[:, lanes ^ o]).astype(F32)
    return partial[:, 0]


def rescore(rows_f32: np.ndarray, n_rows: int, row_offset: int, queries_f32: np.ndarray, cand_ids: np.ndarray, k: int):
    """crag_rescore_topk: (ids [nq, k], S2 [nq, k]).  Ids outside [row_offset, row_offset + n_rows) are skipped."""
    nq = queries_f32.shape[0]
    ids = np.full((nq, k), -1, np.int64)
    sc = np.full((nq, k), -np.inf, F32)
    for j in range(nq):
        local = cand_ids[j].astype(np.int64) - row_offset
        local = local[(local >= 0) & (local < n_rows)]
        if local.size == 0:
            continue
        s2 = s2_scores(rows_f32[local], queries_f32[j])
        i, s = topk_keys(s2, local, k)
        ids[j] = np.where(i >= 0, i + row_offset, -1)
        sc[j] = s
    return ids, sc


def quantized_search(rows_f32: np.ndarray, queries_f32: np.ndarray, k: int, candidates: int, row_offset: int = 0):
    """The whole pipeline: (ids [nq, k], S2 [nq, k]) and the stage-1 (ids, S1, minmax)."""
    dim8 = dim8_of(rows_f32.shape[1])
    r8, rs = quantize(rows_f32, dim8)
    q8, qs = quantize(queries_f32, dim8)
    c_ids, c_sc, c_mm = search_i8(r8, rs, q8, qs, candidates, row_offset)
    ids, sc = rescore(rows_f32, rows_f32.shape[0], row_offset, queries_f32, c_ids, k)
    return ids, sc, (c_ids, c_sc, c_mm)
