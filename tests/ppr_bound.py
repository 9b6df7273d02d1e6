"""Error bound of crag_ppr's fp32 output against the float64 oracle (oracle/ppr_oracle.py), per entry.

With u = 2^-24 and gamma_m = m u / (1 - m u):
  * Row i of a step is a sum of deg_i + 1 nonnegative terms: d * coef_ij * y_j for its deg_i neighbours and
    (1 - d) * v_i.  Each is a product of fp32-rounded factors (coef and v are rounded once from float64, d * (.) and
    (1 - d) * v once more), and any summation order of the row adds at most deg_i roundings, so the row's relative
    error against exact arithmetic on the same y_t is <= gamma_{deg_i + 3}.
  * y_t increases to y* (every term is nonnegative), so the rounding of step t is <= gamma (.) y* entrywise, and
    through the contraction e_{t+1} = d A e_t + r_t the accumulated error is <= b = (I - d A)^-1 (gamma (.) y*):
    one more float64 solve.
  * Truncation: ||y_T - y*||_1 <= d^(T+1), which bounds every entry too (0 when comparing with the exact T-step
    iterate).
  * Normalisation: sum(y_T) is a fixed-shape tree of depth D (finalize_depth) in fp32, relative error gamma_D, and
    the division rounds once more.
Writing S = sum(y_ref), E = sum(b) + trunc, s_lo = (S - E)(1 - gamma_D) and x = y_ref / S:
    |x_hat_p - x_p| <= num_p / s_lo + u (x_p + num_p / s_lo),  num_p = b_p + trunc + x_p (E + gamma_D (S + E)).
"""
from __future__ import annotations

import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from oracle import ppr_oracle as O  # noqa: E402

U = 2.0 ** -24
SUM_THREADS, MAX_SUM_BLOCKS = 256, 1024      # ppr_kernels.cuh: kPprThreads, kPprMaxSumBlocks


def gamma(m):
    m = np.asarray(m, dtype=np.float64)
    return m * U / (1.0 - m * U)


def finalize_depth(n: int) -> int:
    """Additions on the longest path of the finalize's sum: grid-stride accumulation, block tree, then the partials
    (each thread of the gather block adds <= 4 of them) and the same block tree."""
    blocks = min(max(math.ceil(n / SUM_THREADS), 1), MAX_SUM_BLOCKS)
    per_thread = math.ceil(n / (blocks * SUM_THREADS))
    tree = int(math.log2(SUM_THREADS))
    return per_thread + tree + math.ceil(blocks / SUM_THREADS) + tree


def bound(n: int, edges, weights, reset, damping: float, iterations: int, exact_iterate: bool):
    """(x_ref over all vertices, per-entry bound).  exact_iterate: compare with the float64 T-step iterate (no
    truncation term); otherwise with the exact PPR."""
    d = float(damping)
    A = O.transition(O.adjacency(n, edges, weights))
    deg = np.diff(A.indptr)
    v = O.sanitize_reset(reset)
    y_star = O.solve(A, v, d)
    b = O.solve(A, gamma(deg + 3) * y_star / (1.0 - d), d)
    y_ref = O.iterate(A, v, d, iterations) if exact_iterate else y_star
    trunc = 0.0 if exact_iterate else d ** (iterations + 1)
    S = y_ref.sum()
    E = b.sum() + trunc
    gd = float(gamma(finalize_depth(n)))
    s_lo = (S - E) * (1.0 - gd)
    x = y_ref / S
    num = b + trunc + x * (E + gd * (S + E))
    return x, num / s_lo + U * (x + num / s_lo)
