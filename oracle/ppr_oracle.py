"""Float64 Personalized PageRank with the semantics crag_ppr implements (DESIGN.md section 2), on scipy.sparse.

Undirected graph on n vertices from edges (a, b, w), w finite > 0; parallel edges and both orientations add up
(W_ab = sum of the weights joining a and b); self-loops are rejected.  s_a = sum_b W_ab; a vertex with s_a = 0 is
dangling and restarts by the reset v.  x solves
    x = d * sum_{a: s_a > 0} x_a W_ab / s_a  +  d * (sum_{a: s_a = 0} x_a) * v  +  (1 - d) * v,   sum(x) = 1,
which is y* / sum(y*) for y* = (1 - d) (I - d A)^-1 v with A[b, a] = W_ab / s_a (dangling columns zero).

Parity with igraph's prpack is not pinned here (igraph is not installed where the tests run); the chain is: this
oracle == the end-to-end harness's igraph stand-in (tests/test_oracle_ppr.py) == what produced the committed golden
trace of the cinderella run.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla


def sanitize_reset(reset) -> np.ndarray:
    """run_ppr's rule (ComoRAG.py:1091): NaN or negative entries become 0; then divided by the sum, which must be > 0."""
    r = np.asarray(reset, dtype=np.float64).reshape(-1)
    r = np.where(np.isnan(r) | (r < 0), 0.0, r)
    total = r.sum()
    if not (total > 0 and np.isfinite(total)):
        raise ValueError(f"reset must have a positive, finite sum after sanitising (sum = {total})")
    return r / total


def adjacency(n: int, edges, weights) -> sp.csr_matrix:
    """W, symmetrised and coalesced (sorted indices, duplicates summed)."""
    e = np.asarray(edges, dtype=np.int64).reshape(-1, 2)
    w = np.asarray(weights, dtype=np.float64).reshape(-1)
    if len(w) != len(e):
        raise ValueError("one weight per edge")
    if len(e) and ((e < 0).any() or (e >= n).any()):
        raise ValueError("edge endpoint out of range")
    if (e[:, 0] == e[:, 1]).any():
        raise ValueError("self-loops are not supported")
    if not np.isfinite(w).all() or (w <= 0).any():
        raise ValueError("edge weights must be finite and > 0")
    rows = np.concatenate([e[:, 0], e[:, 1]])
    cols = np.concatenate([e[:, 1], e[:, 0]])
    W = sp.csr_matrix((np.concatenate([w, w]), (rows, cols)), shape=(n, n))
    W.sum_duplicates()
    W.sort_indices()
    return W


def transition(W: sp.csr_matrix) -> sp.csr_matrix:
    """A in pull form: A[i, j] = W_ij / s_j, zero columns for dangling j."""
    s = np.asarray(W.sum(axis=1)).reshape(-1)
    inv = np.divide(1.0, s, out=np.zeros_like(s), where=s > 0)
    A = (W @ sp.diags(inv)).tocsr()
    A.sort_indices()
    return A


def iterate(A: sp.csr_matrix, v: np.ndarray, damping: float, iterations: int) -> np.ndarray:
    """y_T of y_0 = (1 - d) v, y_{t+1} = (1 - d) v + d A y_t (unnormalised)."""
    y = (1.0 - damping) * v
    for _ in range(iterations):
        y = (1.0 - damping) * v + damping * (A @ y)
    return y


def solve(A: sp.csr_matrix, v: np.ndarray, damping: float) -> np.ndarray:
    """y* = (1 - d) (I - d A)^-1 v: a direct solve for small graphs, else the iteration run to an L1 change < 1e-15."""
    n = A.shape[0]
    if n <= 4000:
        return spla.spsolve((sp.identity(n, format="csc") - damping * A.tocsc()), (1.0 - damping) * v)
    y = (1.0 - damping) * v
    for _ in range(100000):
        y_new = (1.0 - damping) * v + damping * (A @ y)
        if np.abs(y_new - y).sum() < 1e-15:
            return y_new
        y = y_new
    return y


def ppr(n: int, edges, weights, reset, damping: float = 0.5, iterations: Optional[int] = None) -> np.ndarray:
    """x over all n vertices (sum 1).  iterations=None: the exact PPR; an int T: y_T / sum(y_T), the iterate crag_ppr
    computes in fp32."""
    A = transition(adjacency(n, edges, weights))
    v = sanitize_reset(reset)
    y = solve(A, v, damping) if iterations is None else iterate(A, v, damping, iterations)
    return y / y.sum()
