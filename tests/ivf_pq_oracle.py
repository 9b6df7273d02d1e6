"""numpy restatement of the IVF search over product-quantized residuals (crag_ivf_search_pq, crag_pq_encode, PQIVF),
bit for bit.  DESIGN.md section 7 states the semantics; the layout, the probes, the candidate keys and the exact
rescore are tests/ivf_i8_oracle.py's and oracle/quant_oracle.py's.  Every fp32 operation below is one numpy float32
elementwise operation, i.e. one correctly rounded __f*_rn (nothing is contracted into an FMA).

  codebooks  fp32 [m, 256, dsub], dsub = dim / m
  encode     code_j(r) = argmin_c sum_t (r_{j,t} - C_j[c][t])^2, the sum in t order starting from the t = 0 term;
             equal distances go to the smaller c
  table      LUT_q[j][c] = sum_t q_{j,t} * C_j[c][t], in t order starting from the t = 0 product
  stage 1    S1 = (sum_j LUT_q[j][code_j(p)]) + coarse[q][l], the sum in j order starting from j = 0; the top n_cand
             by (S1 descending, position ascending) and (min, max) of S1 over the probed lists' real rows
  stage 2    ivf_i8_oracle.rescore of the candidates, positions mapped to ids through row_ids

Test infrastructure only: the product path never imports this module.
"""
from __future__ import annotations

import numpy as np

import ivf_i8_oracle as io
from oracle import quant_oracle as qo

F32 = np.float32
TILE_ROWS = io.TILE_ROWS


def encode(residuals_f32: np.ndarray, codebooks: np.ndarray) -> np.ndarray:
    """uint8 [n, m] codes of float32 rows [n, dim] (bf16 values)."""
    x = np.asarray(residuals_f32, F32)
    cb = np.asarray(codebooks, F32)
    m, _, dsub = cb.shape
    out = np.empty((x.shape[0], m), np.uint8)
    for j in range(m):
        d = None
        for t in range(dsub):
            diff = (x[:, j * dsub + t, None] - cb[j, None, :, t]).astype(F32)
            sq = (diff * diff).astype(F32)
            d = sq if d is None else (d + sq).astype(F32)
        out[:, j] = np.argmin(d, axis=1)                        # the first minimum: the smaller codeword
    return out


def table(queries_f32: np.ndarray, codebooks: np.ndarray) -> np.ndarray:
    """fp32 [nq, m, 256]: LUT_q[j][c]."""
    q = np.asarray(queries_f32, F32)
    cb = np.asarray(codebooks, F32)
    m, _, dsub = cb.shape
    qs = q.reshape(q.shape[0], m, dsub)
    acc = None
    for t in range(dsub):
        prod = (qs[:, :, t, None] * cb[None, :, :, t]).astype(F32)
        acc = prod if acc is None else (acc + prod).astype(F32)
    return acc


def pq_sums(lut_q: np.ndarray, codes: np.ndarray) -> np.ndarray:
    """sum_j LUT_q[j][codes[:, j]] in j order, fp32 [n]."""
    acc = lut_q[0, codes[:, 0]]
    for j in range(1, lut_q.shape[0]):
        acc = (acc + lut_q[j, codes[:, j]]).astype(F32)
    return acc


def search_pq(residuals_f32: np.ndarray, codes: np.ndarray, codebooks: np.ndarray, row_ids: np.ndarray,
              list_tile_start: np.ndarray, list_rows: np.ndarray, queries_f32: np.ndarray, probed, k: int, n_cand: int):
    """(ids [nq, k], S2 [nq, k], S1 minmax [nq, 2], (candidate positions [nq, n_cand], their S1)).  residuals_f32 /
    queries_f32 hold bf16 values, codes uint8 [n_rows_padded, >= m] the stored codes; probed = (list ids [nq, nprobe]
    (-1 = none), fp32 coarse scores), as the coarse pass returns them."""
    residuals_f32 = np.asarray(residuals_f32, F32)
    queries_f32 = np.asarray(queries_f32, F32)
    nq = queries_f32.shape[0]
    nlist = len(list_rows)
    m = codebooks.shape[0]
    codes = np.asarray(codes)[:, :m]
    lut = table(queries_f32, codebooks)
    starts = np.asarray(list_tile_start, np.int64)
    lrows = np.asarray(list_rows, np.int64)
    per_q = io._probed_of(probed, nq, nlist)
    c_pos = np.full((nq, n_cand), -1, np.int64)
    c_sc = np.full((nq, n_cand), -np.inf, F32)
    mm = np.tile(np.array([np.inf, -np.inf], F32), (nq, 1))
    for i in range(nq):
        pos, s1 = [], []
        for l, cs in sorted(per_q[i].items()):
            if lrows[l] <= 0:
                continue
            p = starts[l] * TILE_ROWS + np.arange(lrows[l], dtype=np.int64)
            pos.append(p)
            s1.append((pq_sums(lut[i], codes[p]) + F32(cs)).astype(F32))
        if not pos:
            continue
        p, s = np.concatenate(pos), np.concatenate(s1)
        c_pos[i], c_sc[i] = qo.topk_keys(s, p, n_cand)
        o = qo.orderable(s)
        mm[i] = s[np.argmin(o)], s[np.argmax(o)]
    pos, sc = io.rescore(residuals_f32, starts, lambda j, l: per_q[j][int(l)], queries_f32, c_pos, k)
    ids = np.where(pos >= 0, np.asarray(row_ids, np.int64)[np.maximum(pos, 0)], -1)
    return ids, sc, mm, (c_pos, c_sc)
