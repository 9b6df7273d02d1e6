"""Int8 snapshot of a DenseIndex: a scan that reads half the bytes of the bf16 shard, then an exact bf16 rescore.

A search runs crag_search_topk_i8 over the int8 rows for `candidates` rows per query, then crag_rescore_topk
recomputes each candidate's score from its bf16 row and the bf16 query and keeps the best k.  search_wide takes up to
2048 candidates: above 128 its stage 1 is crag_knn_topk_i8, a score-all pass over the codes and a per-query select.  The returned scores are
those exact fp32 dots; only the choice of candidates comes from the int8 scores.  The bf16 rows are read for the
candidates only, so they may live in page-locked host memory (rows="host"), which halves the device footprint again.
Semantics: DESIGN.md section 3e and oracle/quant_oracle.py.
"""
from __future__ import annotations

from typing import Callable, Optional, Tuple

import numpy as np
import torch

from . import _native
from .index import KNN_MAX_K, MAX_K, DenseIndex, knn_chunk


def _dim8(dim: int) -> int:
    return (dim + 127) // 128 * 128


def _encode_rows(name: str, fn: str, rows: torch.Tensor, width: Callable[[int], int], dtype: torch.dtype,
                 stream: Optional[torch.cuda.Stream]) -> Tuple[torch.Tensor, torch.Tensor]:
    """The C row encoder `fn` behind the public `name` of a device bf16 [n, dim] tensor (unit inner stride): (codes
    `dtype` [n, width(dim)], fp32 per-row scales [n])."""
    if rows.dtype != torch.bfloat16 or rows.dim() != 2 or not rows.is_cuda or (rows.shape[0] > 1 and rows.stride(1) != 1):
        raise ValueError(f"{name} expects a CUDA bf16 [n, dim] tensor with unit inner stride")
    n, dim = rows.shape
    width = width(dim)
    dev = rows.device
    with torch.cuda.device(dev):
        st = stream if stream is not None else torch.cuda.current_stream(dev)
        with torch.cuda.stream(st):
            codes = torch.empty((n, width), dtype=dtype, device=dev)
            scales = torch.empty((n,), dtype=torch.float32, device=dev)
            rc = getattr(_native.load(), fn)(rows.data_ptr() if n else 0, n, dim, rows.stride(0) if n else dim,
                                             codes.data_ptr() if n else 0, width, scales.data_ptr() if n else 0,
                                             st.cuda_stream)
            _native.check(rc, fn)
    return codes, scales


def quantize_rows(rows: torch.Tensor, dim8: int, stream: Optional[torch.cuda.Stream] = None
                  ) -> Tuple[torch.Tensor, torch.Tensor]:
    """crag_quantize_rows_i8 of a device bf16 [n, dim] tensor (unit inner stride): (int8 [n, dim8], fp32 scales [n])."""
    return _encode_rows("quantize_rows", "crag_quantize_rows_i8", rows, lambda dim: dim8, torch.int8, stream)


def check_place(where: str, arg: str) -> None:
    """A snapshot's bf16 rows live on the "device" or in page-locked "host" memory; `arg` names the argument."""
    if where not in ("device", "host"):
        raise ValueError(f'{arg} must be "device" or "host"')


def place_rows(rows_bf16: torch.Tensor, where: str, device: torch.device) -> torch.Tensor:
    """The bf16 rows a snapshot keeps: `rows_bf16` itself (where="device") or a copy in page-locked host memory
    (where="host").  Synchronises `device`'s current stream, so the snapshot is complete when this returns."""
    if where == "host":
        host = torch.empty(tuple(rows_bf16.shape), dtype=torch.bfloat16, pin_memory=True)
        if rows_bf16.numel():
            host.copy_(rows_bf16)
        rows_bf16 = host
    with torch.cuda.device(device):
        torch.cuda.current_stream(device).synchronize()
    return rows_bf16


def rescored_candidates(k: int, candidates: Optional[int]) -> int:
    """Stage-1 candidates per query of a rescored search: default min(128, 4 k), and 1 <= k <= candidates <= 128."""
    if candidates is None:
        candidates = min(MAX_K, 4 * k)
    if not 1 <= k <= candidates <= MAX_K:
        raise ValueError(f"need 1 <= k <= candidates <= {MAX_K} (k={k}, candidates={candidates})")
    return candidates


class QuantizedIndex:
    """Frozen int8 snapshot of a DenseIndex's rows (rows added to the DenseIndex later are not seen).

    A subclass with another row code (binary.BinaryIndex) overrides _encode and _stage1; the snapshot, the query
    checks and the rescore are shared."""

    def __init__(self, rows_bf16: torch.Tensor, codes: torch.Tensor, scales: torch.Tensor, dim: int,
                 device: torch.device, row_offset: int):
        self._rows = rows_bf16          # [n, dim_pad] bf16, on the device or in page-locked host memory
        self._codes = codes             # [n, dim8] int8 (the subclass's code rows), device
        self._scales = scales           # [n] fp32, device
        self.dim = dim
        self.dim_pad = rows_bf16.shape[1]
        self.dim8 = _dim8(self.dim_pad)
        self.device = device
        self.row_offset = row_offset

    @staticmethod
    def _encode(rows: torch.Tensor, dim8: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """(code rows, per-row scales) of device bf16 rows."""
        return quantize_rows(rows, dim8)

    @staticmethod
    def _stage1(wide: bool) -> str:
        """The C entry of stage 1 over this class's codes: the top-k scan (<= 128 candidates) or, wide, the score-all
        pass and per-query select (<= 2048).  Both take the same arguments."""
        return "crag_knn_topk_i8" if wide else "crag_search_topk_i8"

    def _scan(self, q8: torch.Tensor, qs: torch.Tensor, candidates: int, c_ids: torch.Tensor, c_sc: torch.Tensor,
              ws: torch.Tensor, st: torch.cuda.Stream, wide: bool) -> None:
        """Stage 1: the top `candidates` rows of every query into (c_ids, c_sc)."""
        n, nq = self.n_rows, q8.shape[0]
        name = self._stage1(wide)
        rc = getattr(_native.load(), name)(self._codes.data_ptr() if n else 0, self._scales.data_ptr() if n else 0, n,
                                           self.dim8, self._codes.shape[1], self.row_offset, q8.data_ptr(),
                                           qs.data_ptr(), nq, candidates, c_ids.data_ptr(), c_sc.data_ptr(), 0,
                                           ws.data_ptr(), ws.numel(), st.cuda_stream)
        _native.check(rc, name)

    @classmethod
    def from_dense(cls, index: DenseIndex, rows: str = "device") -> "QuantizedIndex":
        """Quantise the rows `index` holds now.  rows="device" keeps a reference to the index's bf16 buffer;
        rows="host" copies the bf16 rows into page-locked host memory, so the DenseIndex may be dropped."""
        check_place(rows, "rows")
        buf, n = index._snapshot()
        dev = index.device
        bf16 = buf[:n]
        codes, scales = cls._encode(bf16 if n else torch.zeros((0, index.dim_pad), dtype=torch.bfloat16, device=dev),
                                    _dim8(index.dim_pad))
        return cls(place_rows(bf16, rows, dev), codes, scales, index.dim, dev, index.row_offset)

    @property
    def n_rows(self) -> int:
        return self._codes.shape[0]

    @property
    def rows_on_device(self) -> bool:
        return self._rows.is_cuda

    @property
    def device_bytes(self) -> int:
        """Bytes this index holds in device memory: code rows, scales and, with rows="device", the bf16 rows (shared
        with the DenseIndex it came from)."""
        b = self._codes.numel() + 4 * self._scales.numel()
        if self._rows.is_cuda:
            b += 2 * self._rows.shape[0] * self._rows.stride(0) if self._rows.shape[0] else 0
        return b

    # DenseIndex's conversion of host / device float queries to device bf16 [nq, dim_pad]
    prepare_queries = DenseIndex.prepare_queries

    def search_device(self, queries: torch.Tensor, k: int, candidates: Optional[int] = None,
                      stream: Optional[torch.cuda.Stream] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """Top k of a device bf16 [nq, dim_pad] query block: (ids int64 [nq, k], scores fp32 [nq, k]) on the device.
        Scores are the exact fp32 dots of the rescore (descending, ties by ascending id); -1 / -inf where fewer than
        k rows exist.  candidates (default min(128, 4 k)) rows per query come from the scan of the code rows."""
        return self._search_device(queries, k, rescored_candidates(k, candidates), stream, wide=False)

    def search_device_wide(self, queries: torch.Tensor, k: int, candidates: int,
                           stream: Optional[torch.cuda.Stream] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """search_device for up to 2048 candidates (1 <= k <= candidates <= 2048): at most 128 it is search_device;
        above, stage 1 is the exact top `candidates` of every row's code score (crag_knn_topk_i8 / _b1, per chunk of
        queries whose score rows fit index.knn_chunk's budget), and the rescore sorts them all."""
        if not 1 <= k <= candidates <= KNN_MAX_K:
            raise ValueError(f"need 1 <= k <= candidates <= {KNN_MAX_K} (k={k}, candidates={candidates})")
        if candidates <= MAX_K:
            return self.search_device(queries, k, candidates, stream)
        return self._search_device(queries, k, candidates, stream, wide=True)

    def _search_device(self, queries: torch.Tensor, k: int, candidates: int, stream: Optional[torch.cuda.Stream],
                       wide: bool) -> Tuple[torch.Tensor, torch.Tensor]:
        if queries.dtype != torch.bfloat16 or queries.dim() != 2 or queries.shape[1] != self.dim_pad or not queries.is_cuda:
            raise ValueError(f"queries must be device bf16 [nq, {self.dim_pad}]")
        queries = queries.contiguous()
        nq = queries.shape[0]
        n = self.n_rows
        lib = _native.load()
        dev = self.device
        with torch.cuda.device(dev):
            st = stream if stream is not None else torch.cuda.current_stream(dev)
            with torch.cuda.stream(st):
                q8, qs = quantize_rows(queries, self.dim8, st)
                c_ids = torch.empty((nq, candidates), dtype=torch.int64, device=dev)
                c_sc = torch.empty((nq, candidates), dtype=torch.float32, device=dev)
                if wide:
                    ws_bytes = lib.crag_knn_code_workspace_bytes(n, knn_chunk(nq, n))
                else:
                    ws_bytes = lib.crag_search_workspace_bytes(nq, candidates)
                ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
                self._scan(q8, qs, candidates, c_ids, c_sc, ws, st, wide)
                ids = torch.empty((nq, k), dtype=torch.int64, device=dev)
                scores = torch.empty((nq, k), dtype=torch.float32, device=dev)
                rc = lib.crag_rescore_topk(self._rows.data_ptr() if n else 0, n, self.dim_pad,
                                           self._rows.stride(0) if n else self.dim_pad, self.row_offset,
                                           queries.data_ptr(), nq, c_ids.data_ptr(), candidates, k, ids.data_ptr(),
                                           scores.data_ptr(), st.cuda_stream)
                _native.check(rc, "crag_rescore_topk")
        return ids, scores

    def search(self, queries, k: int, candidates: Optional[int] = None) -> Tuple[np.ndarray, np.ndarray]:
        """Host entry point: what DenseIndex.prepare_queries accepts in, numpy (ids int64 [nq, k], scores fp32
        [nq, k]) out."""
        ids, scores = self.search_device(self.prepare_queries(queries), k, candidates)
        return ids.cpu().numpy(), scores.cpu().numpy()

    def search_wide(self, queries, k: int, candidates: int) -> Tuple[np.ndarray, np.ndarray]:
        """search_device_wide's host twin, as search is search_device's."""
        if not 1 <= k <= candidates <= KNN_MAX_K:
            raise ValueError(f"need 1 <= k <= candidates <= {KNN_MAX_K} (k={k}, candidates={candidates})")
        ids, scores = self.search_device_wide(self.prepare_queries(queries), k, candidates)
        return ids.cpu().numpy(), scores.cpu().numpy()
