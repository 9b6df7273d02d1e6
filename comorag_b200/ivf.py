"""IVF residual inner-product index on one GPU (host side of crag_ivf_search; BASELINE config 4).

The reference has no IVF / ANN code (faiss-cpu is pinned at requirements.txt:34 and never imported; SURVEY.md
section 1) -- this module replaces nothing of the reference's.  Its semantic is the one oracle/ivf_oracle.py states:
rows belong to the centroid of largest inner product, a list stores bf16 residuals x - c_l, a query probes the
`nprobe` lists of largest q.c_l and a row scores q.c_l + q.r; the answer is the k best among the probed lists.

Layout in HBM (built once, `ivf_layout`): lists back to back in list order, ascending original id inside a list,
every list padded to whole 128-row tiles so that a tile belongs to exactly one list:

    centroids   DenseIndex bf16 [nlist, dim]            coarse pass = crag_search_topk(k = nprobe)
    residuals   bf16 [total_tiles * 128, dim]           zero rows as padding
    row_ids     int64 [total_tiles * 128]               original id of a stored row, -1 for padding
    list_tile_start int32 [nlist + 1], list_rows int32 [nlist]

Index BUILD: the assignment of rows to centroids (k-means iterations and the final pass) is crag_ivf_assign -- the scan
kernel with the rows as corpus and the centroid table as its query blocks; the centroid update and the counting sort
by list are torch index arithmetic (bookkeeping).  SEARCH is crag_ivf_search, or crag_ivf_search_i8 over an int8
snapshot of the residuals (QuantizedIVF).
"""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np
import torch

from . import _native
from .index import DenseIndex, KNN_MAX_K, MAX_K
from .quantized import _dim8, check_place, place_rows, quantize_rows, rescored_candidates

TILE_ROWS = 128


def ivf_layout(assignment: torch.Tensor, nlist: int) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """assignment int64 [n] (list of every row) -> (order, dest, list_tile_start, list_rows).

    `order[j]` = original id of the j-th row in (list, original id) order; `dest[j]` = its stored row in the padded
    layout; list_tile_start int32 [nlist + 1]; list_rows int32 [nlist].  Pure index arithmetic (CPU or CUDA)."""
    a = assignment.to(torch.int64)
    if a.numel() and (int(a.min()) < 0 or int(a.max()) >= nlist):
        raise ValueError("assignment out of range")
    order = torch.sort(a, stable=True).indices                     # list order; stable = ascending id inside a list
    counts = torch.bincount(a, minlength=nlist)
    tiles = (counts + TILE_ROWS - 1) // TILE_ROWS
    tile_start = torch.zeros(nlist + 1, dtype=torch.int64, device=a.device)
    tile_start[1:] = torch.cumsum(tiles, 0)
    first = torch.zeros(nlist + 1, dtype=torch.int64, device=a.device)
    first[1:] = torch.cumsum(counts, 0)
    lists_sorted = a[order]
    within = torch.arange(a.numel(), device=a.device) - first[lists_sorted]
    dest = tile_start[lists_sorted] * TILE_ROWS + within
    return order, dest, tile_start.to(torch.int32), counts.to(torch.int32)


def assign_device(rows_bf16: torch.Tensor, centroids_bf16: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """crag_ivf_assign: (list id int32 [n], best inner product fp32 [n]) of every bf16 row against the bf16 centroid
    table -- nlist / 32 passes of the scan kernel over the rows, no [rows, nlist] score matrix, no library GEMM."""
    lib = _native.load()
    n, dim = rows_bf16.shape
    dev = rows_bf16.device
    c = centroids_bf16.contiguous()
    with torch.cuda.device(dev):
        best = torch.empty(n, dtype=torch.float32, device=dev)
        ids = torch.empty(n, dtype=torch.int32, device=dev)
        ws_bytes = lib.crag_search_workspace_bytes(32, 1)
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
        rc = lib.crag_ivf_assign(rows_bf16.data_ptr(), n, dim, rows_bf16.stride(0), c.data_ptr(), c.shape[0],
                                 best.data_ptr(), ids.data_ptr(), ws.data_ptr(), ws_bytes,
                                 torch.cuda.current_stream(dev).cuda_stream)
        _native.check(rc, "crag_ivf_assign")
    return ids, best


def spherical_kmeans(x: torch.Tensor, nlist: int, iters: int = 10, seed: int = 0, block: int = 1 << 18) -> torch.Tensor:
    """Lloyd on the unit sphere, on x's device: assign by largest inner product (crag_ivf_assign over the bf16 sample
    and the current bf16 centroids), centroid = normalised mean of its rows (index_add: bookkeeping, not arithmetic
    worth a kernel); an empty list is re-seeded from the rows worst served by their centroid.  fp32 [nlist, dim]."""
    n, dim = x.shape
    if not 1 <= nlist <= n:
        raise ValueError("need 1 <= nlist <= rows")
    g = torch.Generator(device=x.device).manual_seed(seed)
    c = x[torch.randperm(n, generator=g, device=x.device)[:nlist]].float().clone()
    xb16 = x.to(torch.bfloat16).contiguous()
    for _ in range(iters):
        sums = torch.zeros((nlist, dim), dtype=torch.float32, device=x.device)
        counts = torch.zeros(nlist, dtype=torch.float32, device=x.device)
        a_all, best = assign_device(xb16, c.to(torch.bfloat16))
        a_all = a_all.to(torch.int64)
        for s in range(0, n, block):
            xb = x[s:s + block].float()
            a = a_all[s:s + block]
            sums.index_add_(0, a, xb)
            counts.index_add_(0, a, torch.ones_like(best[s:s + block]))
        empty = torch.nonzero(counts == 0).flatten()
        if empty.numel():
            worst = torch.topk(best, int(empty.numel()), largest=False).indices
            sums[empty], counts[empty] = x[worst].float(), 1.0
        c = torch.nn.functional.normalize(sums / counts[:, None].clamp_min(1.0), dim=1)
    return c


def assign_rows(x: torch.Tensor, centroids_bf16: torch.Tensor, block: int = 1 << 22) -> torch.Tensor:
    """argmax_l bf16(x) . bf16(c_l) with fp32 accumulation, ties to the smaller list id; int64 [n].  The rows go through
    crag_ivf_assign in blocks (the bf16 copy of a block is the only temporary)."""
    out = torch.empty(x.shape[0], dtype=torch.int64, device=x.device)
    for s in range(0, x.shape[0], block):
        ids, _ = assign_device(x[s:s + block].to(torch.bfloat16).contiguous(), centroids_bf16)
        out[s:s + block] = ids
    return out


class _IVFSearch:
    """The search plumbing IVFIndex and QuantizedIVF share; a subclass sets device, dim, nlist and centroids."""

    def _search(self, queries_bf16: torch.Tensor, nprobe: int, k: int, stream: Optional[torch.cuda.Stream],
                probed: Optional[Tuple[torch.Tensor, torch.Tensor]], ws_bytes: int, fine):
        """search_device's common part: the nprobe and query checks, the coarse pass or the check of the caller's
        `probed`, the outputs and the workspace.  fine(q, p_ids, p_scores, ids, scores, minmax, ws, st) runs the
        native fine pass on stream st."""
        if not 1 <= nprobe <= min(MAX_K, self.nlist):
            raise ValueError(f"nprobe must be in [1, {min(MAX_K, self.nlist)}]")
        if (queries_bf16.dtype != torch.bfloat16 or queries_bf16.dim() != 2 or queries_bf16.shape[1] != self.dim
                or queries_bf16.device != self.device):
            raise ValueError(f"queries must be bf16 [nq, {self.dim}] on {self.device}")
        q = queries_bf16.contiguous()
        nq, dev = q.shape[0], self.device
        with torch.cuda.device(dev):
            st = stream if stream is not None else torch.cuda.current_stream(dev)
            with torch.cuda.stream(st):
                if probed is None:
                    p_ids, p_scores, _ = self.centroids.search_device(q, nprobe, stream=st)
                else:
                    p_ids, p_scores = (t.contiguous() for t in probed)
                    if (p_ids.dtype != torch.int64 or p_scores.dtype != torch.float32 or
                            tuple(p_ids.shape) != (nq, nprobe) or tuple(p_scores.shape) != (nq, nprobe) or
                            p_ids.device != dev or p_scores.device != dev):
                        raise ValueError(f"probed must be (int64 [nq, {nprobe}], fp32 [nq, {nprobe}]) on {dev}")
                ids = torch.empty((nq, k), dtype=torch.int64, device=dev)
                scores = torch.empty((nq, k), dtype=torch.float32, device=dev)
                minmax = torch.empty((nq, 2), dtype=torch.float32, device=dev)
                ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
                fine(q, p_ids, p_scores, ids, scores, minmax, ws, st)
        return ids, scores, minmax, (p_ids, p_scores)

    def search(self, queries, nprobe: int, k: int, *args, **kw) -> Tuple[np.ndarray, np.ndarray]:
        """Host float [nq, dim] -> (ids int64 [nq, k], scores fp32 [nq, k]) as numpy; other arguments as search_device's."""
        q = torch.as_tensor(queries)
        if q.dim() == 1:
            q = q[None, :]
        q = q.to(self.device, non_blocking=True).to(torch.bfloat16)
        ids, scores, _, _ = self.search_device(q, nprobe, k, *args, **kw)
        return ids.cpu().numpy(), scores.cpu().numpy()


class IVFIndex(_IVFSearch):
    def __init__(self, centroids_bf16: torch.Tensor, residuals: torch.Tensor, row_ids: torch.Tensor,
                 list_tile_start: torch.Tensor, list_rows: torch.Tensor, n_rows: int):
        """row_ids carry GLOBAL ids: a rank of a row-sharded index builds with row_offset = its first global row."""
        self.device = residuals.device
        self.dim = residuals.shape[1]
        self.nlist = centroids_bf16.shape[0]
        self.n_rows = int(n_rows)
        self.centroids = DenseIndex.from_tensor(centroids_bf16.contiguous())
        self.residuals, self.row_ids = residuals, row_ids
        self.list_tile_start, self.list_rows = list_tile_start, list_rows
        self.total_tiles = residuals.shape[0] // TILE_ROWS
        self._lib = _native.load()

    @classmethod
    def build(cls, rows: torch.Tensor, nlist: int, iters: int = 10, seed: int = 0, centroids: Optional[torch.Tensor] = None,
              train_rows: int = 1 << 20, row_offset: int = 0) -> "IVFIndex":
        """rows: CUDA float [n, dim] (dim % 64 == 0), unit-norm.  Trains `nlist` centroids on a sample (unless
        given), assigns every row, and lays the residuals out by list.  `row_offset` = global id of rows[0]
        (row-sharded index: every rank passes the SAME centroids and its own offset)."""
        if not rows.is_cuda or rows.dim() != 2 or rows.shape[1] % 64 != 0 or rows.shape[1] > 1024:
            raise ValueError("IVFIndex.build expects a CUDA [n, dim] tensor with dim % 64 == 0 and dim <= 1024")
        n, dim = rows.shape
        dev = rows.device
        if centroids is None:
            g = torch.Generator(device=dev).manual_seed(seed + 1)
            sample = rows if n <= train_rows else rows[torch.randperm(n, generator=g, device=dev)[:train_rows]]
            centroids = spherical_kmeans(sample, nlist, iters=iters, seed=seed)
        c_bf16 = centroids.to(device=dev, dtype=torch.bfloat16).contiguous()
        assignment = assign_rows(rows, c_bf16)
        order, dest, tile_start, list_rows = ivf_layout(assignment, nlist)
        total = int(tile_start[-1]) * TILE_ROWS
        residuals = torch.zeros((max(total, TILE_ROWS), dim), dtype=torch.bfloat16, device=dev)
        row_ids = torch.full((max(total, TILE_ROWS),), -1, dtype=torch.int64, device=dev)
        cf = c_bf16.float()
        block = 1 << 18
        for s in range(0, n, block):
            o, d = order[s:s + block], dest[s:s + block]
            residuals[d] = (rows[o].float() - cf[assignment[o]]).to(torch.bfloat16)
            row_ids[d] = o + int(row_offset)
        self = cls(c_bf16, residuals[:total] if total else residuals[:0], row_ids[:total] if total else row_ids[:0],
                   tile_start.contiguous(), list_rows.contiguous(), n)
        self.assignment = assignment
        return self

    def search_device(self, queries_bf16: torch.Tensor, nprobe: int, k: int, stream: Optional[torch.cuda.Stream] = None,
                      probed: Optional[Tuple[torch.Tensor, torch.Tensor]] = None):
        """bf16 [nq, dim] on the device -> (ids int64 [nq, k], scores fp32 [nq, k], minmax fp32 [nq, 2],
        (probed list ids int64 [nq, nprobe], their coarse scores fp32)).  1 <= k <= 128, 1 <= nprobe <= min(128, nlist)."""
        if not 1 <= k <= MAX_K:
            raise ValueError(f"k must be in [1, {MAX_K}]")

        def fine(q, p_ids, p_scores, ids, scores, minmax, ws, st):
            _native.check(self._lib.crag_ivf_search(
                self.residuals.data_ptr(), self.residuals.shape[0], self.dim, self.residuals.stride(0),
                self.list_tile_start.data_ptr(), self.list_rows.data_ptr(), self.nlist, self.total_tiles,
                self.row_ids.data_ptr(), q.data_ptr(), q.shape[0], p_ids.data_ptr(), p_scores.data_ptr(), nprobe, k,
                ids.data_ptr(), scores.data_ptr(), minmax.data_ptr(), ws.data_ptr(), ws.numel(), st.cuda_stream), "crag_ivf_search")
        return self._search(queries_bf16, nprobe, k, stream, probed,
                            self._lib.crag_ivf_workspace_bytes(self.nlist, self.total_tiles, k), fine)


class _RescoredIVF(_IVFSearch):
    """A frozen snapshot of an IVFIndex whose fine pass scans a compressed copy of the stored residuals and rescores its
    candidates exactly from the bf16 residuals (QuantizedIVF, pq.PQIVF).  Shares the IVFIndex's centroid table, list
    layout and row ids; the bf16 residuals are read for the candidates only, so they may live in page-locked host
    memory."""

    def __init__(self, ivf: IVFIndex, residuals_bf16: torch.Tensor):
        self.device, self.dim, self.nlist, self.n_rows = ivf.device, ivf.dim, ivf.nlist, ivf.n_rows
        self.centroids = ivf.centroids
        self.row_ids, self.list_tile_start, self.list_rows = ivf.row_ids, ivf.list_tile_start, ivf.list_rows
        self.total_tiles = ivf.total_tiles
        self._rows = residuals_bf16     # bf16 [total_tiles * 128, dim], on the device or in page-locked host memory
        self._lib = _native.load()
        # list sizes, largest first, for probe_rows_bound (snapshots are built after place_rows has synchronised)
        self._rows_desc = np.sort(ivf.list_rows.cpu().numpy().astype(np.int64))[::-1]

    def probe_rows_bound(self, nprobe: int) -> int:
        """The most real rows a query probing `nprobe` distinct lists can see: the rows of the nprobe largest lists."""
        return int(self._rows_desc[:nprobe].sum())

    def _wide_fine(self, nprobe: int, candidates: int, k: int, max_probe_rows: int):
        """(workspace bytes, fine pass) of the subclass's wide C entry, as _IVFSearch._search takes them."""
        raise NotImplementedError

    def search_device_wide(self, queries_bf16: torch.Tensor, nprobe: int, k: int, candidates: int,
                           stream: Optional[torch.cuda.Stream] = None,
                           probed: Optional[Tuple[torch.Tensor, torch.Tensor]] = None):
        """search_device for up to 2048 candidates (1 <= k <= candidates <= 2048), with search_device's tuple.  At most
        128 it is search_device; above, stage 1 scores every probed row into a block of probe_rows_bound(nprobe)
        slots per query and keeps the exact top `candidates` by stage-1 score (crag_ivf_search_i8_wide /
        crag_ivf_search_pq_wide), and the rescore sorts them all."""
        if not 1 <= k <= candidates <= KNN_MAX_K:
            raise ValueError(f"need 1 <= k <= candidates <= {KNN_MAX_K} (k={k}, candidates={candidates})")
        if candidates <= MAX_K:
            return self.search_device(queries_bf16, nprobe, k, candidates, stream, probed)
        ws_bytes, fine = self._wide_fine(nprobe, candidates, k, max(1, self.probe_rows_bound(nprobe)))
        return self._search(queries_bf16, nprobe, k, stream, probed, ws_bytes, fine)

    def search_wide(self, queries, nprobe: int, k: int, candidates: int, *args, **kw) -> Tuple[np.ndarray, np.ndarray]:
        """search_device_wide's host twin, as search is search_device's."""
        if not 1 <= k <= candidates <= KNN_MAX_K:
            raise ValueError(f"need 1 <= k <= candidates <= {KNN_MAX_K} (k={k}, candidates={candidates})")
        q = torch.as_tensor(queries)
        if q.dim() == 1:
            q = q[None, :]
        q = q.to(self.device, non_blocking=True).to(torch.bfloat16)
        ids, scores, _, _ = self.search_device_wide(q, nprobe, k, candidates, *args, **kw)
        return ids.cpu().numpy(), scores.cpu().numpy()

    @property
    def residuals_on_device(self) -> bool:
        return self._rows.is_cuda

    def _code_bytes(self) -> int:
        """Device bytes of what the fine pass scans."""
        raise NotImplementedError

    @property
    def device_bytes(self) -> int:
        """Bytes of the fine index in device memory: what the fine pass scans and, with residuals="device", the bf16
        residuals (shared with the IVFIndex).  The centroid table, row_ids and list tables are not counted."""
        b = self._code_bytes()
        if self._rows.is_cuda:
            b += 2 * self._rows.shape[0] * self._rows.stride(0) if self._rows.shape[0] else 0
        return b


class QuantizedIVF(_RescoredIVF):
    """Frozen int8 snapshot of an IVFIndex (crag_ivf_search_i8; DESIGN.md section 7).  Every stored residual row is
    quantised to int8 with one fp32 scale; a search scans the probed tiles' int8 residuals for `candidates` positions
    per query (S1 = int8 dot * scales + coarse term) and rescores those exactly from their bf16 residuals
    (S2 = pinned-order fp32 dot + coarse term).  The fine pass reads dim8 + 4 bytes per probed stored row instead of
    2 dim."""

    def __init__(self, ivf: IVFIndex, residuals_bf16: torch.Tensor, residuals_i8: torch.Tensor, scales: torch.Tensor):
        super().__init__(ivf, residuals_bf16)
        self._i8 = residuals_i8         # int8 [total_tiles * 128, dim8], device
        self._scales = scales           # fp32 [total_tiles * 128], device; 0 on padding rows
        self.dim8 = residuals_i8.shape[1]

    @classmethod
    def from_ivf(cls, ivf: IVFIndex, residuals: str = "device") -> "QuantizedIVF":
        """Quantise `ivf`'s stored residuals.  residuals="device" shares the IVFIndex's bf16 residual buffer;
        residuals="host" copies it into page-locked host memory."""
        check_place(residuals, "residuals")
        i8, scales = quantize_rows(ivf.residuals, _dim8(ivf.dim))
        return cls(ivf, place_rows(ivf.residuals, residuals, ivf.device), i8, scales)

    def _code_bytes(self) -> int:
        return self._i8.numel() + 4 * self._scales.numel()

    def search_device(self, queries_bf16: torch.Tensor, nprobe: int, k: int, candidates: Optional[int] = None,
                      stream: Optional[torch.cuda.Stream] = None, probed: Optional[Tuple[torch.Tensor, torch.Tensor]] = None):
        """bf16 [nq, dim] on the device -> (ids int64 [nq, k], scores fp32 [nq, k], minmax fp32 [nq, 2],
        (probed list ids int64 [nq, nprobe], their coarse scores fp32)), as IVFIndex.search_device.  Scores are the
        exact S2 values; minmax is (min, max) of the int8 stage's S1 over the probed rows.  candidates (default
        min(128, 4 k)) positions per query come from the int8 scan; 1 <= k <= candidates <= 128."""
        candidates = rescored_candidates(k, candidates)

        def fine(q, p_ids, p_scores, ids, scores, minmax, ws, st):
            q8, qs = quantize_rows(q, self.dim8, st)
            _native.check(self._lib.crag_ivf_search_i8(
                self._i8.data_ptr(), self._scales.data_ptr(), self.dim8, self._i8.stride(0),
                self._rows.data_ptr(), self.dim, self._rows.stride(0), self._rows.shape[0],
                self.list_tile_start.data_ptr(), self.list_rows.data_ptr(), self.nlist, self.total_tiles,
                self.row_ids.data_ptr(), q8.data_ptr(), qs.data_ptr(), q.data_ptr(), q.shape[0],
                p_ids.data_ptr(), p_scores.data_ptr(), nprobe, candidates, k,
                ids.data_ptr(), scores.data_ptr(), minmax.data_ptr(), ws.data_ptr(), ws.numel(), st.cuda_stream),
                "crag_ivf_search_i8")
        return self._search(queries_bf16, nprobe, k, stream, probed,
                            self._lib.crag_ivf_i8_workspace_bytes(self.nlist, self.total_tiles, candidates), fine)

    def _wide_fine(self, nprobe: int, candidates: int, k: int, max_probe_rows: int):
        def fine(q, p_ids, p_scores, ids, scores, minmax, ws, st):
            q8, qs = quantize_rows(q, self.dim8, st)
            _native.check(self._lib.crag_ivf_search_i8_wide(
                self._i8.data_ptr(), self._scales.data_ptr(), self.dim8, self._i8.stride(0),
                self._rows.data_ptr(), self.dim, self._rows.stride(0), self._rows.shape[0],
                self.list_tile_start.data_ptr(), self.list_rows.data_ptr(), self.nlist, self.total_tiles,
                self.row_ids.data_ptr(), q8.data_ptr(), qs.data_ptr(), q.data_ptr(), q.shape[0],
                p_ids.data_ptr(), p_scores.data_ptr(), nprobe, candidates, k, max_probe_rows,
                ids.data_ptr(), scores.data_ptr(), minmax.data_ptr(), ws.data_ptr(), ws.numel(), st.cuda_stream),
                "crag_ivf_search_i8_wide")
        return self._lib.crag_ivf_i8_wide_workspace_bytes(self.nlist, self.total_tiles, candidates, max_probe_rows), fine


class ShardedIVF:
    """One rank's handle on a row-sharded IVF index (BASELINE config 4 on the GPUs of one box): every rank holds the
    SAME centroid table and the residual lists of its own rows, so all ranks probe the same lists; each searches its
    shard, ONE all-gather of the packed (ids, scores, min/max) records and the merge kernel give every rank the
    global answer -- the exchange step of the flat row-sharded index (dist.ShardedIndex).

    Two consequences of merging per-rank answers (DESIGN.md section 7):
    * exact ties break by (rank, position in the rank's answer), not by stored position as in one IVFIndex (list,
      then id): a tie between a lower rank's row in a higher list and a higher rank's row in a lower list goes to the
      lower rank here, to the lower list there.  The packed record carries no list id, and adding one would grow every
      exchange of the flat index too;
    * over a QuantizedIVF each rank keeps its own top `candidates` by S1 and rescores them, so up to world x
      candidates are rescored.  The answer can differ from one QuantizedIVF over all rows, and its S2 at every
      position is >= that index's: the global top `candidates` by S1 lie inside the union of the ranks'."""

    def __init__(self, local, group=None):
        """`local`: this rank's IVFIndex, QuantizedIVF or pq.PQIVF (a PQIVF rescores its own candidates, as a
        QuantizedIVF does)."""
        import torch.distributed as dist
        self.local, self.group = local, group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1

    def search_device(self, queries_bf16: torch.Tensor, nprobe: int, k: int):
        import torch.distributed as dist
        from .dist import pack_partial
        from .index import merge_topk_packed, packed_record_bytes
        ids, scores, minmax, _ = self.local.search_device(queries_bf16, nprobe, k)
        if self.world == 1:
            return ids, scores, minmax
        nq = queries_bf16.shape[0]
        mine = pack_partial(ids, scores, minmax)
        gathered = torch.empty(self.world * packed_record_bytes(nq, k), dtype=torch.uint8, device=mine.device)
        dist.all_gather_into_tensor(gathered, mine, group=self.group)
        return merge_topk_packed(gathered, self.world, nq, k)
