"""The passage graph on the device and Personalized PageRank over it (crag_ppr): what the reference's run_ppr asks
of igraph (ComoRAG.py:1086-1105, `personalized_pagerank(directed=False, weights='weight', reset=...)`).

Semantics (DESIGN.md section 2a): an undirected graph on n vertices from edges (a, b, w) with finite w > 0; parallel
edges and both orientations of a pair add up (W_ab = sum of the weights joining a and b); self-loops are rejected.
s_a = sum_b W_ab; a vertex with s_a = 0 is dangling and restarts by the reset v.  PPR x solves
    x = d * sum_{a: s_a > 0} x_a W_ab / s_a  +  d * (sum_{a: s_a = 0} x_a) * v  +  (1 - d) * v,   sum(x) = 1
and the device computes it as y_T / sum(y_T) with y_0 = (1 - d) v, y_{t+1} = (1 - d) v + d A y_t, T chosen before
launch so that the L1 error 2 d^(T+1) / (1 - d) is below `tol`.
"""
from __future__ import annotations

import math
from typing import Optional

import numpy as np
import torch

from . import _native


def ppr_iterations(damping: float, tol: float = 1e-10) -> int:
    """Smallest T with 2 d^(T+1) / (1 - d) <= tol: ||x_T - x||_1 <= that bound (DESIGN.md section 2a)."""
    if not 0.0 <= damping < 1.0:
        raise ValueError(f"damping must be in [0, 1), got {damping}")
    if not tol > 0:
        raise ValueError(f"tol must be > 0, got {tol}")
    if damping == 0.0:
        return 0
    t = 0
    while 2.0 * damping ** (t + 1) / (1.0 - damping) > tol:
        t += 1
    return t


def _segment_sums(values: torch.Tensor, counts: torch.Tensor) -> torch.Tensor:
    """Sum of each run of `values` (runs given by `counts`, all >= 1) as a fixed pairwise tree inside the run:
    the same bits on every run, unlike index_add_ / scatter_add_, whose CUDA kernels add in arrival order."""
    v = values.clone()
    if v.numel() == 0:
        return v
    starts = torch.cumsum(counts, 0) - counts
    rank = torch.arange(v.numel(), device=v.device) - torch.repeat_interleave(starts, counts)
    size = torch.repeat_interleave(counts, counts)
    h = 1
    longest = int(counts.max())
    while h < longest:
        idx = torch.nonzero((rank % (2 * h) == 0) & (rank + h < size)).squeeze(1)
        v[idx] = v[idx] + v[idx + h]
        h *= 2
    return v[starts]


class DeviceGraph:
    """CSR "pull" form of the graph: row i lists every neighbour j once, ascending, with coef_ij = W_ij / s_j
    (computed in float64, rounded once to fp32).  row_ptr int64 [n + 1], col int32 [nnz], coef fp32 [nnz].
    Dangling vertices have empty rows."""

    def __init__(self, n: int, row_ptr: torch.Tensor, col: torch.Tensor, coef: torch.Tensor):
        self.n = int(n)
        self.row_ptr, self.col, self.coef = row_ptr, col, coef
        self.device = row_ptr.device

    @property
    def nnz(self) -> int:
        return int(self.col.numel())

    @classmethod
    def from_edges(cls, n: int, edges, weights, device=None) -> "DeviceGraph":
        """edges [E, 2] (vertex ids), weights [E]; built with torch on `device` (default: the edges' device)."""
        n = int(n)
        if n < 1 or n >= 2 ** 31:
            raise ValueError(f"n must be in [1, 2^31), got {n}")
        e = torch.as_tensor(edges, device=device)
        dev = e.device
        e = e.to(torch.int64).reshape(-1, 2)
        w = torch.as_tensor(weights, device=dev).to(torch.float64).reshape(-1)
        if w.numel() != e.shape[0]:
            raise ValueError(f"{e.shape[0]} edges but {w.numel()} weights")
        a, b = e[:, 0], e[:, 1]
        if e.numel() and bool(((a < 0) | (a >= n) | (b < 0) | (b >= n)).any()):
            raise ValueError(f"edge endpoint outside [0, {n})")
        if bool((a == b).any()):
            raise ValueError("self-loops are not supported")
        if not bool(torch.isfinite(w).all()):
            raise ValueError("edge weights must be finite")
        if bool((w <= 0).any()):
            raise ValueError("edge weights must be > 0")
        # symmetrise, then coalesce (row, col) pairs: sort by row * n + col, sum each run in a fixed order
        key = torch.cat([a * n + b, b * n + a])
        w2 = torch.cat([w, w])
        key, perm = torch.sort(key, stable=True)
        uniq, counts = torch.unique_consecutive(key, return_counts=True)
        W = _segment_sums(w2[perm], counts)
        row, col = uniq // n, uniq % n
        row_counts = torch.bincount(row, minlength=n)
        s = torch.zeros(n, dtype=torch.float64, device=dev)
        if uniq.numel():
            nonempty = row_counts > 0
            s[nonempty] = _segment_sums(W, row_counts[nonempty])
        coef = (W / s[col]).to(torch.float32)
        row_ptr = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        row_ptr[1:] = torch.cumsum(row_counts, 0)
        return cls(n, row_ptr, col.to(torch.int32), coef)

    @classmethod
    def from_igraph(cls, g, device=None) -> "DeviceGraph":
        """g.vcount(), g.get_edgelist() and g.es["weight"] of an igraph.Graph (or anything with those three)."""
        edges = np.asarray(g.get_edgelist(), dtype=np.int64).reshape(-1, 2)
        weights = np.asarray(g.es["weight"] if len(edges) else [], dtype=np.float64)
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        return cls.from_edges(g.vcount(), torch.from_numpy(edges).to(dev), torch.from_numpy(weights).to(dev))

    def reset_vector(self, reset) -> torch.Tensor:
        """run_ppr's sanitising (ComoRAG.py:1091: NaN or negative entries become 0), then v = reset / sum(reset),
        fp32 on the device.  Raises on a zero or non-finite sum."""
        r = torch.as_tensor(reset, dtype=torch.float64, device=self.device).reshape(-1)
        if r.numel() != self.n:
            raise ValueError(f"reset has {r.numel()} entries, the graph {self.n} vertices")
        r = torch.where(torch.isnan(r) | (r < 0), torch.zeros_like(r), r)
        total = float(r.sum())
        if not (total > 0 and math.isfinite(total)):
            raise ValueError(f"reset must have a positive, finite sum after sanitising (sum = {total})")
        return (r / total).to(torch.float32)

    def personalized_pagerank(self, reset, damping: float = 0.5, tol: float = 1e-10,
                              vertices: Optional[torch.Tensor] = None,
                              stream: Optional[torch.cuda.Stream] = None) -> torch.Tensor:
        """x[vertices] (all vertices if None) as device fp32, sum(x) = 1 over all vertices."""
        damping = float(damping)
        iterations = ppr_iterations(damping, tol)
        return self.ppr_iterate(self.reset_vector(reset), damping, iterations, vertices, stream)

    def ppr_iterate(self, v: torch.Tensor, damping: float, iterations: int, vertices: Optional[torch.Tensor] = None,
                    stream: Optional[torch.cuda.Stream] = None) -> torch.Tensor:
        """One crag_ppr call: y_T / sum(y_T) for a device fp32 reset `v` (>= 0, sum 1) and a fixed T."""
        if vertices is not None:
            vertices = torch.as_tensor(vertices, device=self.device).to(torch.int64).reshape(-1)
            if vertices.numel() and bool(((vertices < 0) | (vertices >= self.n)).any()):
                raise ValueError(f"vertices must lie in [0, {self.n})")
            vertices = vertices.to(torch.int32)
        lib = _native.load()
        dev = self.device
        with torch.cuda.device(dev):
            st = stream if stream is not None else torch.cuda.current_stream(dev)
            with torch.cuda.stream(st):
                n_out = self.n if vertices is None else vertices.numel()
                out = torch.empty((n_out,), dtype=torch.float32, device=dev)
                ws_bytes = lib.crag_ppr_workspace_bytes(self.n, self.nnz)
                ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
                rc = lib.crag_ppr(self.row_ptr.data_ptr(), self.col.data_ptr() if self.nnz else 0,
                                  self.coef.data_ptr() if self.nnz else 0, self.n, self.nnz, v.data_ptr(),
                                  float(damping), int(iterations), _native.ptr(vertices), n_out, out.data_ptr(),
                                  ws.data_ptr(), ws_bytes, st.cuda_stream)
                _native.check(rc, "crag_ppr")
        return out

