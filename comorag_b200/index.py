"""Device-resident bf16 corpus shard + fused top-k search (host side of K4).

The reference keeps its index as a host fp32 matrix rebuilt from the
EmbeddingStore (ComoRAG.py:876-907) and scores one query at a time with
np.dot + min_max_normalize + np.argsort (ComoRAG.py:937-967).  Here the matrix
lives in HBM as bf16 [n_rows, dim_pad] and a whole query block is scored per
pass by libcomorag_b200's crag_search_topk.
"""
from __future__ import annotations

import threading
from typing import Optional, Tuple

import numpy as np
import torch

from . import _native

MAX_DIM = 1024
MAX_K = 128            # the shard scan (crag_search_topk) and everything built on it
KNN_MAX_K = 2048       # crag_knn_topk: score-block GEMM + per-query radix select
# Score-block budget of crag_knn_topk: a chunk holds this many bytes of fp32 scores (4 * round_up(n_rows, 4) per query)
KNN_WORKSPACE_BYTES = 1 << 30
# Routing between crag_knn_topk and the shard scan, from tools/knn_bench.py on an NVIDIA H100 80GB HBM3 at a 700 W
# power limit (new path vs scan path, ms per call):
#   self-join, N = nq = 10k / 50k / 200k, dim 384 and 1024: the new path wins at every k -- k = 10: 0.78 vs 14.0,
#     23.0 vs 175, 389 vs 1329 (dim 1024, 200k); k = 2047: 1.97 vs 763, 26.2 vs 7326, 402 vs 54160 (dim 1024).
#     The smallest winning batch is nq = 10 000; the smallest winning chunk holds 1 280 queries (N = 200k).
#   N = 10M, dim 1024, nq = 1 / 32 / 256: k = 10 loses (16.6 vs 6.9, 33.5 vs 6.8, 165 vs 53), k = 2047 wins (16.6 vs
#     114, 33.4 vs 119, 165 vs 937).  There one call of the new path costs what 2.4 / 4.9 / 3.1 scan passes cost, and
#     the scan needs ceil(k/128) passes, so k > 640 (>= 6 passes) is on the winning side for every measured nq.
KNN_MIN_QUERIES = 10_000    # many queries: the GEMM path for any k <= 2048 ...
KNN_MIN_CHUNK = 1_280       # ... when a chunk of the workspace budget holds at least this many of them
KNN_MIN_K_FEW = 641         # few queries: the GEMM path from this k on


def _pad_dim(dim: int) -> int:
    return (dim + 63) // 64 * 64


def knn_chunk(nq: int, n_rows: int, budget: int = KNN_WORKSPACE_BYTES) -> int:
    """Queries per crag_knn_topk chunk whose score rows fit `budget` bytes: at least 1, at most nq, and a multiple of
    the GEMM's 128-row tile wherever nq and the budget allow."""
    per_query = 4 * ((max(n_rows, 1) + 3) // 4 * 4)
    c = min(nq, max(1, budget // per_query))
    if 128 <= c < nq:
        c = c // 128 * 128
    return c


def fp32_threshold(t: float) -> float:
    """The smallest fp32 value >= the double t.  A score s (fp32) passes `s >= t` compared as doubles exactly when it
    passes `s >= fp32_threshold(t)` compared as fp32 -- the form crag_knn_threshold takes its threshold in.  At 0.8
    this is float32(0.8), which rounds up; at 0.7 float32(0.7) rounds down and the next fp32 above it is returned."""
    f = np.float32(t)
    if float(f) < float(t):
        f = np.nextafter(f, np.float32(np.inf))
    return float(f)


def use_knn(nq: int, n_rows: int, k: int) -> bool:
    """Route a search to crag_knn_topk (True) or to the shard scan (False): for k <= 2048, the GEMM path for large
    query batches whose chunks stay large, or for k >= KNN_MIN_K_FEW; the scan otherwise and always beyond k = 2048."""
    if k > KNN_MAX_K:
        return False
    if nq >= KNN_MIN_QUERIES and knn_chunk(nq, n_rows) >= KNN_MIN_CHUNK:
        return True
    return k >= KNN_MIN_K_FEW


class _GrowableRows:
    """bf16 [rows, dim_pad] storage whose address never changes: virtual address space reserved once
    (crag_vmem_reserve), physical memory mapped behind it in `step`-sized pieces as rows arrive (crag_vmem_grow).
    Growth copies nothing, and tensor maps / captured graphs that point at the shard stay valid."""

    STEP_BYTES = 64 << 20

    def __init__(self, device: torch.device, dim_pad: int, max_bytes: Optional[int] = None):
        import ctypes as C
        self.device, self.dim_pad = device, dim_pad
        self._lib = _native.load()
        with torch.cuda.device(device):
            if max_bytes is None:
                max_bytes = int(torch.cuda.get_device_properties(device).total_memory)
            base, gran = C.c_uint64(0), C.c_size_t(0)
            _native.check(self._lib.crag_vmem_reserve(int(max_bytes), C.byref(base), C.byref(gran)), "crag_vmem_reserve")
        self.base, self.gran = int(base.value), int(gran.value)
        self.reserved = (int(max_bytes) + self.gran - 1) // self.gran * self.gran
        self.mapped = 0
        self._view: Optional[torch.Tensor] = None

    @property
    def row_bytes(self) -> int:
        return self.dim_pad * 2

    def capacity_rows(self) -> int:
        return self.mapped // self.row_bytes

    def ensure_rows(self, rows: int) -> None:
        need = rows * self.row_bytes
        if need <= self.mapped:
            return
        step = max(self.gran, self.STEP_BYTES // self.gran * self.gran)
        new = min(self.reserved, (need + step - 1) // step * step)
        if new < need:
            raise MemoryError(f"corpus shard would exceed its {self.reserved >> 30} GiB address reservation")
        with torch.cuda.device(self.device):
            _native.check(self._lib.crag_vmem_grow(self.base, self.mapped, new), "crag_vmem_grow")
        # fresh pages: zero them once so the dim..dim_pad padding columns read as 0
        fresh = self._alias(self.mapped, new - self.mapped)
        fresh.zero_()
        self.mapped = new
        self._view = None

    def _alias(self, offset: int, nbytes: int) -> torch.Tensor:
        holder = type("_Mem", (), {"__cuda_array_interface__": {
            "shape": (nbytes // 2,), "typestr": "<i2", "data": (self.base + offset, False), "version": 3, "strides": None}})()
        holder.owner = self        # torch keeps the holder alive for the tensor's lifetime: so the mapping outlives every alias
        return torch.as_tensor(holder, device=self.device)

    def tensor(self) -> torch.Tensor:
        """bf16 [capacity_rows, dim_pad] view of everything mapped so far (same address after every growth)."""
        if self._view is None:
            rows = self.capacity_rows()
            self._view = self._alias(0, rows * self.row_bytes).view(torch.bfloat16).view(rows, self.dim_pad) if rows else \
                torch.zeros((0, self.dim_pad), dtype=torch.bfloat16, device=self.device)
        return self._view

    def close(self) -> None:
        if self.base:
            with torch.cuda.device(self.device):
                torch.cuda.synchronize(self.device)
                self._view = None
                self._lib.crag_vmem_release(self.base, self.mapped, self.reserved)
            self.base, self.mapped = 0, 0

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DenseIndex:
    """One corpus shard in HBM.

    ``row_offset`` is the global id of local row 0 (rank r of a row-sharded
    index owns ids [row_offset, row_offset + n_rows)).
    """

    def __init__(self, dim: int, device: Optional[torch.device] = None, capacity: int = 0, row_offset: int = 0,
                 _adopt: Optional[torch.Tensor] = None):
        if dim < 1:
            raise ValueError("dim must be positive")
        self.dim = int(dim)
        self.dim_pad = _pad_dim(self.dim)
        if self.dim_pad > MAX_DIM:
            raise ValueError(f"dim {dim} > {MAX_DIM} is not supported by the sm_90a search kernel")
        if device is None:
            if not torch.cuda.is_available():
                raise _native.NativeError("DenseIndex needs a CUDA device (no CPU fallback)")
            device = torch.device("cuda", torch.cuda.current_device())
        self.device = torch.device(device)
        self.row_offset = int(row_offset)
        self._n = 0
        _native.load()
        # rows appended with add() live behind a fixed virtual address and grow without reallocation (_GrowableRows);
        # from_tensor() adopts a caller's tensor instead
        self._rows: Optional[_GrowableRows] = None
        if _adopt is not None:
            self._buf = _adopt
        else:
            self._rows = _GrowableRows(self.device, self.dim_pad)
            self._rows.ensure_rows(max(int(capacity), 0))
            self._buf = self._rows.tensor()
        self._lock = threading.Lock()

    # ------------------------------------------------------------------ build
    @classmethod
    def from_tensor(cls, rows: torch.Tensor, row_offset: int = 0) -> "DenseIndex":
        """Adopt a device bf16 [n, dim] tensor (dim % 64 == 0) without copying."""
        if rows.dtype != torch.bfloat16 or rows.dim() != 2 or not rows.is_cuda:
            raise ValueError("from_tensor expects a CUDA bf16 [n, dim] tensor")
        if rows.shape[1] % 64 != 0 or rows.stride(1) != 1 or rows.stride(0) % 8 != 0:
            raise ValueError("from_tensor needs dim % 64 == 0 and a row stride that is a multiple of 8")
        self = cls(rows.shape[1], device=rows.device, row_offset=row_offset, _adopt=rows)
        self._n = rows.shape[0]
        return self

    @property
    def n_rows(self) -> int:
        return self._n

    def matrix(self) -> torch.Tensor:
        """bf16 view [n_rows, dim] of the stored rows."""
        return self._buf[: self._n, : self.dim]

    def _snapshot(self) -> Tuple[torch.Tensor, int]:
        """(buffer, row count) as one consistent pair: add() may swap the buffer for a larger one while another
        thread searches (ComoRAG.py:436-441 runs 16 threads), and reading the two fields separately could pair the
        old pointer with the new count.  The caller's reference keeps the storage from being recycled before its
        launch is enqueued (torch's caching allocator then orders any reuse after it on the same stream)."""
        with self._lock:
            return self._buf, self._n

    def _reserve(self, n: int) -> None:
        if n <= self._buf.shape[0]:
            return
        if self._rows is None:
            # an adopted tensor (from_tensor) that now has to grow: move it behind a growable reservation once
            self._rows = _GrowableRows(self.device, self.dim_pad)
            self._rows.ensure_rows(n)
            self._rows.tensor()[: self._n] = self._buf[: self._n]
        else:
            self._rows.ensure_rows(n)       # maps more pages behind the same address; nothing is copied
        self._buf = self._rows.tensor()

    def add(self, vectors) -> None:
        """Append rows (numpy / torch, any float dtype, [n, dim]); stored as bf16."""
        v = torch.as_tensor(vectors)
        if v.dim() == 1:
            v = v[None, :]
        if v.shape[1] != self.dim:
            raise ValueError(f"expected [n, {self.dim}] vectors, got {tuple(v.shape)}")
        with torch.cuda.device(self.device):
            vb = v.to(self.device, non_blocking=True).to(torch.bfloat16)   # H2D + cast before the lock: searches keep running
            with self._lock:
                n0, n1 = self._n, self._n + vb.shape[0]
                self._reserve(n1)
                self._buf[n0:n1, : self.dim] = vb
                self._n = n1

    def add_bf16_file(self, path: str, n_rows: int) -> None:
        """Append n_rows raw bf16 [*, dim_pad] rows from a file written by EmbeddingStore's append-only persistence."""
        raw = np.fromfile(path, dtype=np.int16, count=n_rows * self.dim_pad)
        if raw.size != n_rows * self.dim_pad:
            raise ValueError(f"{path}: expected {n_rows} rows of {self.dim_pad} bf16")
        with torch.cuda.device(self.device):
            rows = torch.from_numpy(raw).view(torch.bfloat16).view(n_rows, self.dim_pad).to(self.device, non_blocking=True)
            with self._lock:
                n0, n1 = self._n, self._n + n_rows
                self._reserve(n1)
                self._buf[n0:n1] = rows
                self._n = n1

    def save(self, path: str) -> None:
        """Raw bf16 [n_rows, dim_pad] dump + json meta (per-rank shard file for a sharded index)."""
        import json
        self._buf[: self._n].cpu().view(torch.int16).numpy().tofile(path)
        with open(path + ".meta.json", "w") as f:
            json.dump({"dim": self.dim, "dim_pad": self.dim_pad, "rows": self._n, "row_offset": self.row_offset,
                       "format": "comorag_b200.raw.v1"}, f)

    @classmethod
    def load(cls, path: str, device: Optional[torch.device] = None) -> "DenseIndex":
        import json
        meta = json.load(open(path + ".meta.json"))
        self = cls(meta["dim"], device=device, capacity=meta["rows"], row_offset=meta.get("row_offset", 0))
        self.add_bf16_file(path, meta["rows"])
        return self

    # ----------------------------------------------------------------- search
    def search_device(self, queries: torch.Tensor, k: int, stream: Optional[torch.cuda.Stream] = None,
                      out: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = None
                      ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Top-k of a device bf16 [nq, dim_pad] query block.

        Returns (ids int64 [nq, k], scores fp32 [nq, k], minmax fp32 [nq, 2]),
        all on the device, enqueued on ``stream`` (default: current stream).
        Scores are raw inner products sorted descending (ties: ascending id);
        missing entries (n_rows < k) have id -1 / score -inf.
        """
        if k < 1:
            raise ValueError("k must be >= 1")
        if k > MAX_K and out is not None:
            raise ValueError(f"out= is only supported for k <= {MAX_K}")
        if use_knn(queries.shape[0], self._n, k):
            return self._search_device_knn(queries, k, stream, out)
        if k > MAX_K:
            return self._search_device_paged(queries, k, stream)
        if queries.dtype != torch.bfloat16 or queries.dim() != 2 or queries.shape[1] != self.dim_pad:
            raise ValueError(f"queries must be bf16 [nq, {self.dim_pad}]")
        if not queries.is_contiguous():
            queries = queries.contiguous()
        nq = queries.shape[0]
        lib = _native.load()
        dev = self.device
        buf, n_rows = self._snapshot()
        with torch.cuda.device(dev):
            st = stream if stream is not None else torch.cuda.current_stream(dev)
            with torch.cuda.stream(st):
                if out is not None:
                    ids, scores, minmax = out   # caller-provided (e.g. views of one packed send buffer)
                else:
                    ids = torch.empty((nq, k), dtype=torch.int64, device=dev)
                    scores = torch.empty((nq, k), dtype=torch.float32, device=dev)
                    minmax = torch.empty((nq, 2), dtype=torch.float32, device=dev)
                ws_bytes = lib.crag_search_workspace_bytes(nq, k)
                ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
                rc = lib.crag_search_topk(
                    buf.data_ptr() if n_rows else 0, n_rows, self.dim_pad,
                    buf.stride(0) if buf.shape[0] else self.dim_pad,
                    self.row_offset, queries.data_ptr(), nq, k, ids.data_ptr(), scores.data_ptr(),
                    minmax.data_ptr(), ws.data_ptr(), ws_bytes, st.cuda_stream)
                _native.check(rc, "crag_search_topk")
        return ids, scores, minmax

    def _search_device_knn(self, queries: torch.Tensor, k: int, stream: Optional[torch.cuda.Stream], out=None):
        """crag_knn_topk: per chunk of queries one wgmma GEMM writes the fp32 score block, one CTA per query
        radix-selects its k best.  Same outputs as the scan path."""
        if queries.dtype != torch.bfloat16 or queries.dim() != 2 or queries.shape[1] != self.dim_pad:
            raise ValueError(f"queries must be bf16 [nq, {self.dim_pad}]")
        queries = queries.contiguous()
        nq = queries.shape[0]
        lib = _native.load()
        dev = self.device
        buf, n_rows = self._snapshot()
        with torch.cuda.device(dev):
            st = stream if stream is not None else torch.cuda.current_stream(dev)
            with torch.cuda.stream(st):
                if out is not None:
                    ids, scores, minmax = out
                else:
                    ids = torch.empty((nq, k), dtype=torch.int64, device=dev)
                    scores = torch.empty((nq, k), dtype=torch.float32, device=dev)
                    minmax = torch.empty((nq, 2), dtype=torch.float32, device=dev)
                ws_bytes = lib.crag_knn_workspace_bytes(n_rows, knn_chunk(nq, n_rows))
                ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
                rc = lib.crag_knn_topk(
                    buf.data_ptr() if n_rows else 0, n_rows, self.dim_pad,
                    buf.stride(0) if buf.shape[0] else self.dim_pad,
                    self.row_offset, queries.data_ptr(), nq, k, ids.data_ptr(), scores.data_ptr(),
                    minmax.data_ptr(), ws.data_ptr(), ws_bytes, st.cuda_stream)
                _native.check(rc, "crag_knn_topk")
        return ids, scores, minmax

    def search_threshold_device(self, queries: torch.Tensor, threshold: float, cap: int, limit: int,
                                self_rows: Optional[torch.Tensor] = None, exclude_rows=None,
                                stream: Optional[torch.cuda.Stream] = None
                                ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Threshold join (crag_knn_threshold) of a device bf16 [nq, dim_pad] query block: for each query, walk the
        first `limit` rows of its crag_knn_topk list, stop at the first scoring below `threshold` (an fp32 value: see
        fp32_threshold), skip self_rows[q] (int64 [nq] local rows, -1 for none) and `exclude_rows` (at most 64 local
        rows), and keep the others, at most `cap`.  Returns (counts int32 [nq], ids int64 [nq, cap] local rows,
        scores fp32 [nq, cap]) on the device, -1 / -inf past each count.  Single shard; chunks queries as
        _search_device_knn does."""
        if queries.dtype != torch.bfloat16 or queries.dim() != 2 or queries.shape[1] != self.dim_pad:
            raise ValueError(f"queries must be bf16 [nq, {self.dim_pad}]")
        queries = queries.contiguous()
        nq = queries.shape[0]
        lib = _native.load()
        dev = self.device
        buf, n_rows = self._snapshot()
        with torch.cuda.device(dev):
            st = stream if stream is not None else torch.cuda.current_stream(dev)
            with torch.cuda.stream(st):
                excl = torch.as_tensor(list(exclude_rows) if exclude_rows is not None else [], dtype=torch.int64)
                excl = excl.to(dev, non_blocking=True)
                selfr = None
                if self_rows is not None:
                    selfr = torch.as_tensor(self_rows, dtype=torch.int64).to(dev, non_blocking=True).contiguous()
                    if selfr.shape != (nq,):
                        raise ValueError(f"self_rows must hold one row per query ({nq})")
                counts = torch.empty((nq,), dtype=torch.int32, device=dev)
                ids = torch.empty((nq, cap), dtype=torch.int64, device=dev)
                scores = torch.empty((nq, cap), dtype=torch.float32, device=dev)
                ws_bytes = lib.crag_knn_workspace_bytes(n_rows, knn_chunk(max(nq, 1), n_rows))
                ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
                rc = lib.crag_knn_threshold(
                    buf.data_ptr() if n_rows else 0, n_rows, self.dim_pad,
                    buf.stride(0) if buf.shape[0] else self.dim_pad, queries.data_ptr(), nq, float(threshold),
                    int(limit), int(cap), _native.ptr(selfr), excl.data_ptr() if excl.numel() else 0, excl.numel(),
                    counts.data_ptr(), ids.data_ptr(), scores.data_ptr(), ws.data_ptr(), ws_bytes, st.cuda_stream)
                _native.check(rc, "crag_knn_threshold")
        return counts, ids, scores

    def _search_device_paged(self, queries: torch.Tensor, k: int, stream: Optional[torch.cuda.Stream]):
        """k > 128 where crag_knn_topk does not pay off (few queries, or k > 2048): ceil(k/128) passes chained with
        crag_search_topk_after (exact rank continuation)."""
        if queries.dtype != torch.bfloat16 or queries.dim() != 2 or queries.shape[1] != self.dim_pad:
            raise ValueError(f"queries must be bf16 [nq, {self.dim_pad}]")
        queries = queries.contiguous()
        nq = queries.shape[0]
        lib = _native.load()
        dev = self.device
        buf, n_rows = self._snapshot()
        with torch.cuda.device(dev):
            st = stream if stream is not None else torch.cuda.current_stream(dev)
            with torch.cuda.stream(st):
                ids = torch.empty((nq, k), dtype=torch.int64, device=dev)
                scores = torch.empty((nq, k), dtype=torch.float32, device=dev)
                minmax = torch.empty((nq, 2), dtype=torch.float32, device=dev)
                ws_bytes = lib.crag_search_workspace_bytes(nq, MAX_K)
                ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
                after = None
                for p0 in range(0, k, MAX_K):
                    kk = min(MAX_K, k - p0)
                    p_ids = torch.empty((nq, kk), dtype=torch.int64, device=dev)
                    p_sc = torch.empty((nq, kk), dtype=torch.float32, device=dev)
                    last = torch.empty((nq,), dtype=torch.int64, device=dev)   # opaque u64 positions
                    rc = lib.crag_search_topk_after(
                        buf.data_ptr() if n_rows else 0, n_rows, self.dim_pad,
                        buf.stride(0) if buf.shape[0] else self.dim_pad, self.row_offset,
                        queries.data_ptr(), nq, kk, _native.ptr(after), p_ids.data_ptr(), p_sc.data_ptr(),
                        minmax.data_ptr(), last.data_ptr(), ws.data_ptr(), ws_bytes, st.cuda_stream)
                    _native.check(rc, "crag_search_topk_after")
                    ids[:, p0:p0 + kk], scores[:, p0:p0 + kk] = p_ids, p_sc
                    after = last
        return ids, scores, minmax

    # ------------------------------------------------- full-array contracts
    def scores_device(self, queries: torch.Tensor, stream: Optional[torch.cuda.Stream] = None
                      ) -> Tuple[torch.Tensor, torch.Tensor]:
        """Raw inner products of EVERY row for a device bf16 [nq, dim_pad] query block (crag_search_scores): the
        np.dot(E, q.T) of ComoRAG.py:944 / :958-960 when a caller needs the whole array.  Returns (scores fp32
        [nq, n_rows], minmax fp32 [nq, 2]) on the device."""
        if queries.dtype != torch.bfloat16 or queries.dim() != 2 or queries.shape[1] != self.dim_pad:
            raise ValueError(f"queries must be bf16 [nq, {self.dim_pad}]")
        queries = queries.contiguous()
        nq = queries.shape[0]
        lib = _native.load()
        dev = self.device
        buf, n_rows = self._snapshot()
        with torch.cuda.device(dev):
            st = stream if stream is not None else torch.cuda.current_stream(dev)
            with torch.cuda.stream(st):
                ld = max(n_rows, 1)
                scores = torch.empty((nq, ld), dtype=torch.float32, device=dev)
                minmax = torch.empty((nq, 2), dtype=torch.float32, device=dev)
                ws_bytes = lib.crag_search_workspace_bytes(nq, 1)
                ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
                rc = lib.crag_search_scores(buf.data_ptr() if n_rows else 0, n_rows, self.dim_pad,
                                            buf.stride(0) if buf.shape[0] else self.dim_pad, queries.data_ptr(), nq,
                                            scores.data_ptr(), ld, minmax.data_ptr(), ws.data_ptr(), ws_bytes,
                                            st.cuda_stream)
                _native.check(rc, "crag_search_scores")
        return scores[:, :n_rows], minmax

    def rank_device(self, scores_row: torch.Tensor, stream: Optional[torch.cuda.Stream] = None
                    ) -> Tuple[torch.Tensor, torch.Tensor]:
        """rank_scores() of one fp32 score row of this index (np.argsort(scores)[::-1] + the gather of
        ComoRAG.py:965-966)."""
        return rank_scores(scores_row, stream)

    def session(self, nq: int, k: int, use_graph: bool = True) -> "SearchSession":
        """A reusable, CUDA-graph-captured search step for (nq, k); see SearchSession."""
        return SearchSession(self, nq, k, use_graph=use_graph)

    def prepare_queries(self, queries) -> torch.Tensor:
        """Host/device float [nq, dim] -> device bf16 [nq, dim_pad]."""
        q = torch.as_tensor(queries)
        if q.dim() == 1:
            q = q[None, :]
        if q.shape[1] != self.dim:
            raise ValueError(f"expected [nq, {self.dim}] queries, got {tuple(q.shape)}")
        if not q.is_cuda:
            q = q.pin_memory() if q.dtype in (torch.float32, torch.bfloat16, torch.float16) else q
        q = q.to(self.device, non_blocking=True).to(torch.bfloat16)
        if self.dim_pad != self.dim:
            qp = torch.zeros((q.shape[0], self.dim_pad), dtype=torch.bfloat16, device=self.device)
            qp[:, : self.dim] = q
            q = qp
        return q

    def search(self, queries, k: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """Host-buffer entry point: numpy in, numpy out (ids int64 [nq,k], scores fp32 [nq,k], minmax fp32 [nq,2])."""
        q = self.prepare_queries(queries)
        nq = q.shape[0]
        if k <= MAX_K:
            # the kernel writes straight into one packed record, which comes back in a single device->host copy
            rec = torch.empty(packed_record_bytes(nq, k), dtype=torch.uint8, device=self.device)
            self.search_device(q, k, out=packed_views(rec, nq, k))
            host = rec.cpu()
            ids, scores, minmax = packed_views(host, nq, k)
            return ids.numpy().copy(), scores.numpy().copy(), minmax.numpy().copy()
        ids, scores, minmax = self.search_device(q, k)
        return ids.cpu().numpy(), scores.cpu().numpy(), minmax.cpu().numpy()


class SearchSession:
    """One search step for a fixed (nq <= 32, k <= 128) over static buffers, captured in a CUDA graph: what a serving
    loop (the probe batches of ComoRAG's meta loop, ComoRAG.py:354-358) calls again and again.  The step is
    pool-memset + scan kernel + finalize kernel; with `exchange` (a dist.PeerExchange) the finalize is the fused
    finalize + cross-rank exchange + merge kernel and every rank ends with the global answer; with `gather` (a
    callable doing the NCCL all-gather of the packed record) the step is scan + finalize + all-gather + merge.

    run(queries) returns views of the session's output buffers -- valid until the next run()."""

    def __init__(self, index: "DenseIndex", nq: int, k: int, exchange=None, gather=None, world: int = 1,
                 use_graph: bool = True):
        if not (1 <= nq <= 32 and 1 <= k <= MAX_K):
            raise ValueError("SearchSession needs 1 <= nq <= 32 and 1 <= k <= 128")
        self.index, self.nq, self.k = index, nq, k
        self.exchange, self.gather, self.world = exchange, gather, world
        dev = index.device
        self._lib = _native.load()
        self._buf, self._n = index._snapshot()
        with torch.cuda.device(dev):
            self.queries = torch.zeros((nq, index.dim_pad), dtype=torch.bfloat16, device=dev)
            self.record = torch.zeros(packed_record_bytes(nq, k), dtype=torch.uint8, device=dev)
            self.ids, self.scores, self.minmax = packed_views(self.record, nq, k)
            self._ws_bytes = self._lib.crag_search_workspace_bytes(nq, k)
            self._ws = torch.zeros((self._ws_bytes,), dtype=torch.uint8, device=dev)
            if gather is not None:
                self._gathered = torch.zeros(world * self.record.numel(), dtype=torch.uint8, device=dev)
                self._local = torch.zeros_like(self.record)
            self.graph = None
            if use_graph:
                side = torch.cuda.Stream(dev)
                side.wait_stream(torch.cuda.current_stream(dev))
                with torch.cuda.stream(side):
                    self._enqueue(side)                      # warm-up outside capture (also a collective when sharded)
                side.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, capture_error_mode="thread_local"):
                    self._enqueue(torch.cuda.current_stream(dev))
                self.graph = g

    def _enqueue(self, st) -> None:
        lib, ix = self._lib, self.index
        buf, n = self._buf, self._n
        rc = lib.crag_search_scan(buf.data_ptr() if n else 0, n, ix.dim_pad, buf.stride(0) if buf.shape[0] else ix.dim_pad,
                                  self.queries.data_ptr(), self.nq, self.k, self._ws.data_ptr(), self._ws_bytes, st.cuda_stream)
        _native.check(rc, "crag_search_scan")
        if self.exchange is not None:
            x = self.exchange
            rc = lib.crag_search_finalize_exchange(self._ws.data_ptr(), self._ws_bytes, n, self.nq, self.k, ix.row_offset,
                                                   x.peer_ptrs, x.rank, x.world, x.epochs.data_ptr(), x.status.data_ptr(),
                                                   self.ids.data_ptr(), self.scores.data_ptr(), self.minmax.data_ptr(),
                                                   st.cuda_stream)
            _native.check(rc, "crag_search_finalize_exchange")
            return
        out = packed_views(self._local, self.nq, self.k) if self.gather is not None else (self.ids, self.scores, self.minmax)
        rc = lib.crag_search_finalize(self._ws.data_ptr(), self._ws_bytes, n, self.nq, self.k, ix.row_offset,
                                      out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(), st.cuda_stream)
        _native.check(rc, "crag_search_finalize")
        if self.gather is not None:
            self.gather(self._gathered, self._local)
            per = self._local.numel()
            rc = lib.crag_merge_topk_packed(self._gathered.data_ptr(), per, self.world, self.nq, self.k, self.ids.data_ptr(),
                                            self.scores.data_ptr(), self.minmax.data_ptr(), st.cuda_stream)
            _native.check(rc, "crag_merge_topk_packed")

    def stale(self) -> bool:
        """True when the index grew or moved since the session was built (the tensor maps in the graph are baked)."""
        buf, n = self.index._snapshot()
        return n != self._n or buf.data_ptr() != self._buf.data_ptr()

    def run(self, queries: torch.Tensor):
        """queries: bf16 [nq, dim_pad] (device) or anything DenseIndex.prepare_queries accepts."""
        if self.stale():
            raise RuntimeError("the index changed since this SearchSession was built; build a new one")
        if not (queries.is_cuda and queries.dtype == torch.bfloat16):
            queries = self.index.prepare_queries(queries)
        dev = self.index.device
        with torch.cuda.device(dev):
            if queries.data_ptr() != self.queries.data_ptr():
                self.queries.copy_(queries, non_blocking=True)
            if self.graph is not None:
                self.graph.replay()
            else:
                self._enqueue(torch.cuda.current_stream(dev))
        return self.ids, self.scores, self.minmax


def rank_scores(scores_row: torch.Tensor, stream: Optional[torch.cuda.Stream] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Full descending ranking of one device fp32 score vector (crag_rank_scores; ties by ascending row):
    np.argsort(scores)[::-1] + the gather of ComoRAG.py:965-966 for passage scores, and of ComoRAG.py:1101-1102 for
    PPR scores.  Returns (ids int64 [n], scores fp32 [n]) on the vector's device."""
    if scores_row.dtype != torch.float32 or scores_row.dim() != 1 or not scores_row.is_contiguous():
        raise ValueError("scores_row must be a contiguous fp32 vector")
    n = scores_row.shape[0]
    lib = _native.load()
    dev = scores_row.device
    with torch.cuda.device(dev):
        st = stream if stream is not None else torch.cuda.current_stream(dev)
        with torch.cuda.stream(st):
            ids = torch.empty((n,), dtype=torch.int64, device=dev)
            out = torch.empty((n,), dtype=torch.float32, device=dev)
            if n:
                ws_bytes = lib.crag_rank_workspace_bytes(n)
                ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
                rc = lib.crag_rank_scores(scores_row.data_ptr(), n, ids.data_ptr(), out.data_ptr(), ws.data_ptr(),
                                          ws_bytes, st.cuda_stream)
                _native.check(rc, "crag_rank_scores")
    return ids, out


def merge_topk(scores: torch.Tensor, ids: torch.Tensor, minmax: Optional[torch.Tensor]):
    """Merge [parts, nq, k] per-shard results into the global top-k (device)."""
    if scores.dim() != 3 or ids.shape != scores.shape:
        raise ValueError("scores/ids must be [parts, nq, k]")
    parts, nq, k = scores.shape
    lib = _native.load()
    dev = scores.device
    scores = scores.contiguous().to(torch.float32)
    ids = ids.contiguous().to(torch.int64)
    mm = minmax.contiguous().to(torch.float32) if minmax is not None else None
    out_ids = torch.empty((nq, k), dtype=torch.int64, device=dev)
    out_scores = torch.empty((nq, k), dtype=torch.float32, device=dev)
    out_mm = torch.empty((nq, 2), dtype=torch.float32, device=dev) if mm is not None else None
    with torch.cuda.device(dev):
        rc = lib.crag_merge_topk(scores.data_ptr(), ids.data_ptr(), _native.ptr(mm), parts, nq, k,
                                 out_ids.data_ptr(), out_scores.data_ptr(), _native.ptr(out_mm),
                                 torch.cuda.current_stream(dev).cuda_stream)
        _native.check(rc, "crag_merge_topk")
    return out_ids, out_scores, out_mm


def packed_record_bytes(nq: int, k: int) -> int:
    """Bytes of one shard's packed (ids | scores | minmax) record (crag_merge_topk_packed layout)."""
    return (nq * k * 8 + nq * k * 4 + nq * 2 * 4 + 15) // 16 * 16   # padded so consecutive records stay 8-byte aligned


def packed_views(buf: torch.Tensor, nq: int, k: int):
    """Three typed views (ids int64 [nq,k], scores fp32 [nq,k], minmax fp32 [nq,2]) of one uint8 record buffer."""
    a, b = nq * k * 8, nq * k * 8 + nq * k * 4
    return (buf[:a].view(torch.int64).view(nq, k), buf[a:b].view(torch.float32).view(nq, k),
            buf[b:b + nq * 8].view(torch.float32).view(nq, 2))


def merge_topk_packed(records: torch.Tensor, parts: int, nq: int, k: int):
    """Merge `parts` packed records laid out back to back in one uint8 buffer (the all-gather output)."""
    lib = _native.load()
    dev = records.device
    per = packed_record_bytes(nq, k)
    if records.dtype != torch.uint8 or records.numel() < parts * per or not records.is_contiguous():
        raise ValueError("records must be a contiguous uint8 buffer of parts * record bytes")
    out_ids = torch.empty((nq, k), dtype=torch.int64, device=dev)
    out_scores = torch.empty((nq, k), dtype=torch.float32, device=dev)
    out_mm = torch.empty((nq, 2), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        rc = lib.crag_merge_topk_packed(records.data_ptr(), per, parts, nq, k, out_ids.data_ptr(), out_scores.data_ptr(),
                                        out_mm.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
        _native.check(rc, "crag_merge_topk_packed")
    return out_ids, out_scores, out_mm
