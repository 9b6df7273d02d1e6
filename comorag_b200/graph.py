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
import threading
import weakref
from typing import Optional

import numpy as np
import torch

from . import _native
from .coalescer import Batcher, BatcherClosed

MAX_PPR_BATCH = 32          # resets per crag_ppr_batch call


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
        self._batcher: Optional[Batcher] = None
        self._lane_lock = threading.Lock()
        self._active = 0                  # coalesced calls that have not returned yet (direct or through the batcher)
        self._pending = []                # events after the launches of recent calls (direct or batched)

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
        fp32 on the device.  Raises on a zero or non-finite sum.  A 2-D reset [B, n] is B resets, each sanitised and
        normalised exactly as it would be alone; a row with a zero or non-finite sum raises naming the row."""
        r = torch.as_tensor(reset, dtype=torch.float64, device=self.device)
        if r.dim() == 2:
            if r.shape[1] != self.n:
                raise ValueError(f"reset has rows of {r.shape[1]} entries, the graph {self.n} vertices")
            if r.shape[0] < 1:
                raise ValueError("reset has no rows")
            r = torch.where(torch.isnan(r) | (r < 0), torch.zeros_like(r), r)
            rows = []
            for i in range(r.shape[0]):
                total = float(r[i].sum())
                if not (total > 0 and math.isfinite(total)):
                    raise ValueError(f"reset row {i} must have a positive, finite sum after sanitising (sum = {total})")
                rows.append((r[i] / total).to(torch.float32))
            return torch.stack(rows)
        r = r.reshape(-1)
        if r.numel() != self.n:
            raise ValueError(f"reset has {r.numel()} entries, the graph {self.n} vertices")
        r = torch.where(torch.isnan(r) | (r < 0), torch.zeros_like(r), r)
        total = float(r.sum())
        if not (total > 0 and math.isfinite(total)):
            raise ValueError(f"reset must have a positive, finite sum after sanitising (sum = {total})")
        return (r / total).to(torch.float32)

    # ------------------------------------------------------------------------------------------ coalescing
    @property
    def batcher(self) -> Optional[Batcher]:
        """The Batcher that coalesces concurrent 1-D personalized_pagerank calls, or None (the default)."""
        return self._batcher

    def enable_batching(self, max_items: int = MAX_PPR_BATCH, max_wait_s: float = 2e-4,
                        lone_calls_direct: bool = True) -> Batcher:
        """From now on, 1-D personalized_pagerank calls without an explicit stream are coalesced: concurrent callers
        with the same (damping, T, vertices object) share one crag_ppr_batch pass of up to `max_items` resets.  Each
        caller still gets its own row, bit-identical to running alone.  With lone_calls_direct (the default), a
        caller that finds no other call in flight (none returning, none whose device work is still running) runs
        crag_ppr directly on its own stream, exactly as with batching off, and the calls that arrive meanwhile are
        coalesced; without it every call goes through the Batcher.  Returns the Batcher; calling this again with
        other settings than the running Batcher's raises ValueError.

        The Batcher's worker thread holds the graph only weakly: a graph dropped without disable_batching() is
        freed, and its Batcher is closed when it is."""
        if self.device.type != "cuda":
            raise ValueError("batching needs the graph on a CUDA device")
        if not 1 <= max_items <= MAX_PPR_BATCH:
            raise ValueError(f"max_items must be in [1, {MAX_PPR_BATCH}], got {max_items}")
        settings = (int(max_items), float(max_wait_s), bool(lone_calls_direct))
        if self._batcher is not None:
            if settings != self._batch_settings:
                raise ValueError(f"batching is already on with (max_items, max_wait_s, lone_calls_direct) = "
                                 f"{self._batch_settings}, "
                                 f"not {settings}; disable_batching() first")
            return self._batcher
        run = weakref.WeakMethod(self._run_batch)

        def run_batch(key, payloads):
            return run()(key, payloads)     # a queued call's caller holds the graph, so it is alive here
        self._batch_stream = torch.cuda.Stream(self.device)
        self._batcher = Batcher(run_batch, max_items=settings[0], max_wait_s=settings[1], name="crag-ppr-batcher")
        self._batch_settings = settings
        self._close_batcher = weakref.finalize(self, self._batcher.close)
        return self._batcher

    def disable_batching(self) -> None:
        """Close the Batcher: queued calls are still served, later calls run directly."""
        if self._batcher is not None:
            self._batcher = None
            self._close_batcher()

    def _coalesced(self, b: Batcher, v: torch.Tensor, damping: float, iterations: int, vertices) -> torch.Tensor:
        # Alone: nothing queued for the batcher and no earlier call's device work pending (its event not yet
        # reached), so there is nothing to share a pass with -- run on the caller's stream, as without batching.
        with self._lane_lock:
            self._pending = [e for e in self._pending if not e.query()]
            alone = self._batch_settings[2] and self._active == 0 and not self._pending
            self._active += 1
        done = None
        try:
            with torch.cuda.device(self.device):
                if alone:
                    out = self.ppr_iterate(v, damping, iterations, vertices)
                    done = torch.cuda.Event()
                    done.record(torch.cuda.current_stream(self.device))
                else:
                    out, done = self._submit(b, v, damping, iterations, vertices)
        finally:
            with self._lane_lock:
                self._active -= 1
                if done is not None:
                    self._pending.append(done)
        return out

    def _submit(self, b: Batcher, v: torch.Tensor, damping: float, iterations: int, vertices):
        # Stream order: the batcher's stream waits for the caller's reset (event `ready`), the caller's stream waits
        # for the batch's result (event `done`); record_stream keeps each tensor's memory until the other stream is
        # done with it.
        caller = torch.cuda.current_stream(self.device)
        ready = torch.cuda.Event()
        ready.record(caller)
        key = (damping, iterations, None if vertices is None else id(vertices))
        try:
            row, done = b.call(key, (v, ready, vertices))
        except BatcherClosed:            # the graph's batcher was closed (graph rebuilt) between the check and here
            row = self.ppr_iterate(v, damping, iterations, vertices)
            done = torch.cuda.Event()
            done.record(caller)
            return row, done
        caller.wait_event(done)
        row.record_stream(caller)
        return row, done

    def _run_batch(self, key, payloads):
        damping, iterations, _ = key
        vertices = payloads[0][2]               # the same object for the whole group (it is part of the key)
        st = self._batch_stream
        with torch.cuda.device(self.device), torch.cuda.stream(st):
            for v, ready, _ in payloads:
                st.wait_event(ready)
                v.record_stream(st)
            if len(payloads) == 1:
                out = self.ppr_iterate(payloads[0][0], damping, iterations, vertices, stream=st)
                rows = [out]
            else:
                out = self.ppr_iterate(torch.stack([p[0] for p in payloads]), damping, iterations, vertices, stream=st)
                rows = list(out.unbind(0))
            done = torch.cuda.Event()
            done.record(st)
        return [(r, done) for r in rows]

    # ------------------------------------------------------------------------------------------ PPR
    def personalized_pagerank(self, reset, damping: float = 0.5, tol: float = 1e-10,
                              vertices: Optional[torch.Tensor] = None,
                              stream: Optional[torch.cuda.Stream] = None) -> torch.Tensor:
        """x[vertices] (all vertices if None) as device fp32, sum(x) = 1 over all vertices.  reset [n] gives [n_out];
        reset [B, n] gives [B, n_out], row b the PPR of reset row b.  With batching enabled, a 1-D call without an
        explicit stream is coalesced with concurrent ones (enable_batching; same result, bit for bit)."""
        damping = float(damping)
        iterations = ppr_iterations(damping, tol)
        v = self.reset_vector(reset)           # in the caller's thread: a bad reset raises for its own caller only
        b = self.batcher
        if b is not None and v.dim() == 1 and stream is None:
            return self._coalesced(b, v, damping, iterations, vertices)
        return self.ppr_iterate(v, damping, iterations, vertices, stream)

    def ppr_iterate(self, v: torch.Tensor, damping: float, iterations: int, vertices: Optional[torch.Tensor] = None,
                    stream: Optional[torch.cuda.Stream] = None) -> torch.Tensor:
        """y_T / sum(y_T) for a device fp32 reset `v` (>= 0, each row summing to 1) and a fixed T.  v [n]: one
        crag_ppr call, [n_out].  v [B, n]: crag_ppr_batch on chunks of up to 32 rows (a chunk of one row: crag_ppr),
        [B, n_out]; row b is bit-identical to ppr_iterate(v[b], ...)."""
        if vertices is not None:
            vertices = torch.as_tensor(vertices, device=self.device).to(torch.int64).reshape(-1)
            if vertices.numel() and bool(((vertices < 0) | (vertices >= self.n)).any()):
                raise ValueError(f"vertices must lie in [0, {self.n})")
            vertices = vertices.to(torch.int32)
        if v.dim() == 2 and v.shape[1] != self.n:
            raise ValueError(f"v has rows of {v.shape[1]} entries, the graph {self.n} vertices")
        lib = _native.load()
        dev = self.device
        col = self.col.data_ptr() if self.nnz else 0
        coef = self.coef.data_ptr() if self.nnz else 0
        with torch.cuda.device(dev):
            st = stream if stream is not None else torch.cuda.current_stream(dev)
            with torch.cuda.stream(st):
                n_out = self.n if vertices is None else vertices.numel()
                if v.dim() == 2:
                    v = v.contiguous()
                    out = torch.empty((v.shape[0], n_out), dtype=torch.float32, device=dev)
                    for s in range(0, v.shape[0], MAX_PPR_BATCH):
                        rows = min(MAX_PPR_BATCH, v.shape[0] - s)
                        if rows == 1:
                            self._crag_ppr(lib, v[s], damping, iterations, vertices, n_out, out[s], st)
                            continue
                        ws_bytes = lib.crag_ppr_batch_workspace_bytes(self.n, self.nnz, rows)
                        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
                        rc = lib.crag_ppr_batch(self.row_ptr.data_ptr(), col, coef, self.n, self.nnz, v[s].data_ptr(),
                                                rows, float(damping), int(iterations), _native.ptr(vertices), n_out,
                                                out[s].data_ptr(), ws.data_ptr(), ws_bytes, st.cuda_stream)
                        _native.check(rc, "crag_ppr_batch")
                    return out
                out = torch.empty((n_out,), dtype=torch.float32, device=dev)
                self._crag_ppr(lib, v, damping, iterations, vertices, n_out, out, st)
        return out

    def _crag_ppr(self, lib, v, damping, iterations, vertices, n_out, out, st) -> None:
        ws_bytes = lib.crag_ppr_workspace_bytes(self.n, self.nnz)
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=self.device)
        rc = lib.crag_ppr(self.row_ptr.data_ptr(), self.col.data_ptr() if self.nnz else 0,
                          self.coef.data_ptr() if self.nnz else 0, self.n, self.nnz, v.data_ptr(),
                          float(damping), int(iterations), _native.ptr(vertices), n_out, out.data_ptr(),
                          ws.data_ptr(), ws_bytes, st.cuda_stream)
        _native.check(rc, "crag_ppr")
