"""numpy restatement of the one-bit shard search (crag_binarize_rows -> crag_search_topk_b1 -> crag_rescore_topk):
binarize -> S1 -> top k' -> S2 -> top k, bit for bit.  DESIGN.md section 3f states the semantics.

  binarize  dim8 = ceil(dim / 128) * 128 columns, bit j of byte b = column 8 b + j, set iff x > 0 (zero, -0 and padding
            give 0, read as -1); alpha = float32(sum |x_i|) / float32(dim), the sum in the rescore's pinned order (the
            rescore's dot of |x| with a row of ones, which is exact product by product).
  S1        float32(sum_i q^_i b_i) * float32(s_q * alpha), b_i = +-1, q^ / s_q from crag_quantize_rows_i8 at dim8: the
            integer dot is exact (|acc| <= 127 * 1024 < 2^24).
  S2 / top k  crag_rescore_topk, as oracle/quant_oracle.py restates it.
"""
from __future__ import annotations

import numpy as np

from oracle import quant_oracle as qo

F32 = np.float32
dim8_of = qo.dim8_of


def binarize(x: np.ndarray, dim8: int | None = None) -> tuple[np.ndarray, np.ndarray]:
    """float32 rows [n, dim] (bf16 values) -> (uint8 codes [n, dim8 / 8], float32 alpha [n])."""
    x = np.asarray(x, F32)
    n, dim = x.shape
    dim8 = dim8_of(dim) if dim8 is None else dim8
    pos = np.zeros((n, dim8), bool)
    pos[:, :dim] = x > 0
    codes = np.packbits(pos, axis=1, bitorder="little")
    width = (dim + 7) // 8 * 8
    abs_sum = np.zeros(n, F32)
    for r0 in range(0, n, 1 << 15):
        a = np.zeros((min(n - r0, 1 << 15), width), F32)
        a[:, :dim] = np.abs(x[r0:r0 + a.shape[0]])
        abs_sum[r0:r0 + a.shape[0]] = qo.s2_scores(a, np.ones(width, F32))
    return codes, (abs_sum / F32(dim)).astype(F32)


def signs(codes: np.ndarray) -> np.ndarray:
    """uint8 codes [n, dim8 / 8] -> float32 +-1 [n, dim8]."""
    b = np.unpackbits(np.asarray(codes, np.uint8), axis=1, bitorder="little")
    return (2 * b.astype(F32) - 1).astype(F32)


def s1_scores(codes: np.ndarray, alpha: np.ndarray, q_i8: np.ndarray, q_scales: np.ndarray,
              block: int = 1 << 16) -> np.ndarray:
    """S1 [nq, n] of one-bit rows and int8 queries."""
    n = codes.shape[0]
    out = np.empty((q_i8.shape[0], n), F32)
    q = q_i8.astype(F32)
    qs = q_scales.astype(F32)[:, None]
    for r0 in range(0, n, block):
        # exact: every partial sum is an integer below 127 * 1024 < 2^24
        acc = q @ signs(codes[r0:r0 + block]).T
        scale = (qs * alpha[r0:r0 + block].astype(F32)[None, :]).astype(F32)
        out[:, r0:r0 + block] = (acc.astype(F32) * scale).astype(F32)
    return out


def search_b1(codes, alpha, q_i8, q_scales, k: int, row_offset: int = 0):
    """crag_search_topk_b1: (ids [nq, k], S1 [nq, k], minmax [nq, 2])."""
    n = codes.shape[0]
    nq = q_i8.shape[0]
    ids = np.full((nq, k), -1, np.int64)
    sc = np.full((nq, k), -np.inf, F32)
    mm = np.tile(np.array([np.inf, -np.inf], F32), (nq, 1))
    if n == 0:
        return ids, sc, mm
    rows = np.arange(n, dtype=np.int64)
    for q0 in range(0, nq, 32):
        s1 = s1_scores(codes, alpha, q_i8[q0:q0 + 32], q_scales[q0:q0 + 32])
        for j in range(s1.shape[0]):
            i, s = qo.topk_keys(s1[j], rows, k)
            ids[q0 + j] = np.where(i >= 0, i + row_offset, -1)
            sc[q0 + j] = s
            o = qo.orderable(s1[j])
            mm[q0 + j] = s1[j][np.argmin(o)], s1[j][np.argmax(o)]
    return ids, sc, mm


def binary_search(rows_f32: np.ndarray, queries_f32: np.ndarray, k: int, candidates: int, row_offset: int = 0):
    """The whole pipeline: (ids [nq, k], S2 [nq, k]) and the stage-1 (ids, S1, minmax)."""
    dim8 = dim8_of(rows_f32.shape[1])
    codes, alpha = binarize(rows_f32, dim8)
    q8, qs = qo.quantize(queries_f32, dim8)
    c_ids, c_sc, c_mm = search_b1(codes, alpha, q8, qs, candidates, row_offset)
    ids, sc = qo.rescore(rows_f32, rows_f32.shape[0], row_offset, queries_f32, c_ids, k)
    return ids, sc, (c_ids, c_sc, c_mm)
