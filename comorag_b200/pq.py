"""IVF over product-quantized residual lists (host side of crag_ivf_search_pq; DESIGN.md section 7).

Every stored residual row of an IVFIndex is cut into `m` subspaces of dsub = dim / m columns and stored as m one-byte
codes, the index of the nearest of a subspace's 256 codewords.  A search scores the probed tiles' codes with one table
per query, S1 = sum_j LUT_q[j][code_j] + q.c_l, keeps `candidates` positions per query and rescores those exactly
from their bf16 residuals, as QuantizedIVF does.  The fine pass holds m bytes per stored row on the device (96 B at
m = 96 against 772 B in int8 and 1536 B in bf16); the bf16 residuals may live in page-locked host memory.

Codebook training is Lloyd k-means per subspace on a seeded sample of stored residuals: the assignment step is
crag_pq_encode, the update is torch index arithmetic (fp64 sums, so the result does not depend on the order of the
device's atomic adds).
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import _native
from .ivf import IVFIndex, _RescoredIVF
from .quantized import check_place, place_rows, rescored_candidates

CODEWORDS = 256
MAX_M = 192          # one query's table, m * 256 * 4 bytes, fits in shared memory
MAX_DSUB = 128       # one subspace's codebook and a block of its residuals fit in shared memory


def code_stride(m: int) -> int:
    """Bytes per stored code row: m rounded up to whole 16 bytes (the scan reads a row with 16-byte loads)."""
    return (m + 15) // 16 * 16


def check_shape(dim: int, m: int) -> None:
    if not (1 <= m <= MAX_M and dim % m == 0 and dim // m <= MAX_DSUB):
        raise ValueError(f"m must divide dim with 1 <= m <= {MAX_M} and dim / m <= {MAX_DSUB} (dim={dim}, m={m})")


def encode(rows_bf16: torch.Tensor, codebooks: torch.Tensor, out: Optional[torch.Tensor] = None,
           stream: Optional[torch.cuda.Stream] = None) -> torch.Tensor:
    """crag_pq_encode: bf16 [n, dim] rows (unit stride along dim) and fp32 [m, 256, dsub] codebooks on one device ->
    uint8 [n, code_stride(m)] codes (the padding bytes of a fresh output are 0; `out` may be given, n x >= m)."""
    n, dim = rows_bf16.shape
    m = codebooks.shape[0]
    check_shape(dim, m)
    if rows_bf16.dtype != torch.bfloat16 or rows_bf16.stride(1) != 1:
        raise ValueError("rows must be bf16 with unit stride along dim")
    if tuple(codebooks.shape) != (m, CODEWORDS, dim // m) or codebooks.dtype != torch.float32:
        raise ValueError(f"codebooks must be fp32 [m, {CODEWORDS}, dim / m]")
    cb = codebooks.contiguous()
    dev = rows_bf16.device
    if out is None:
        out = torch.zeros((n, code_stride(m)), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        st = stream if stream is not None else torch.cuda.current_stream(dev)
        _native.check(_native.load().crag_pq_encode(rows_bf16.data_ptr(), n, dim, rows_bf16.stride(0), cb.data_ptr(), m,
                                                    out.data_ptr(), out.stride(0), st.cuda_stream), "crag_pq_encode")
    return out


def train_codebooks(sample_bf16: torch.Tensor, m: int, iters: int = 10, seed: int = 0) -> torch.Tensor:
    """Lloyd k-means with 256 codewords in each of the m subspaces of a bf16 [n, dim] sample: fp32 [m, 256, dsub].
    The start is 256 seeded sample rows (drawn with replacement when n < 256); a codeword that loses all its rows
    keeps its place."""
    n, dim = sample_bf16.shape
    check_shape(dim, m)
    if n < 1:
        raise ValueError("need at least one training row")
    dsub, dev = dim // m, sample_bf16.device
    g = torch.Generator(device=dev).manual_seed(seed)
    start = (torch.randperm(n, generator=g, device=dev)[:CODEWORDS] if n >= CODEWORDS
             else torch.randint(0, n, (CODEWORDS,), generator=g, device=dev))
    x = sample_bf16.float().reshape(n, m, dsub)
    cb = x[start].permute(1, 0, 2).contiguous()                      # [m, 256, dsub]
    flat = x.reshape(n * m, dsub).double()
    base = torch.arange(m, device=dev) * CODEWORDS
    for _ in range(iters):
        codes = encode(sample_bf16, cb)[:, :m].long()
        idx = (codes + base).reshape(-1)                               # row-major [n, m] -> codeword of (row, j)
        sums = torch.zeros((m * CODEWORDS, dsub), dtype=torch.float64, device=dev).index_add_(0, idx, flat)
        counts = torch.bincount(idx, minlength=m * CODEWORDS).double()
        new = (sums / counts.clamp_min(1.0)[:, None]).float().reshape(m, CODEWORDS, dsub)
        cb = torch.where((counts > 0).reshape(m, CODEWORDS, 1), new, cb).contiguous()
    return cb


class PQIVF(_RescoredIVF):
    """Frozen product-quantized snapshot of an IVFIndex (crag_ivf_search_pq; DESIGN.md section 7).  Shares the
    IVFIndex's centroid table, list layout and row ids; holds the codes [n_rows_padded, code_stride(m)] and the
    codebooks [m, 256, dsub] on the device, and the bf16 residuals on the device or in page-locked host memory."""

    def __init__(self, ivf: IVFIndex, residuals_bf16: torch.Tensor, codes: torch.Tensor, codebooks: torch.Tensor):
        super().__init__(ivf, residuals_bf16)
        self.m = codebooks.shape[0]
        self.codebooks = codebooks      # fp32 [m, 256, dsub], device
        self.codes = codes              # uint8 [total_tiles * 128, code_stride(m)], device; 0 on padding rows

    @classmethod
    def from_ivf(cls, ivf: IVFIndex, m: int, codebooks: Optional[torch.Tensor] = None, train_rows: int = 1 << 20,
                 iters: int = 10, seed: int = 0, residuals: str = "device") -> "PQIVF":
        """Encode `ivf`'s stored residuals with m subspaces.  Without `codebooks`, trains them on up to `train_rows`
        stored rows drawn with `seed`; every rank of a row-sharded index passes the same codebooks.
        residuals="device" shares the IVFIndex's bf16 residual buffer; residuals="host" copies it into page-locked
        host memory."""
        check_place(residuals, "residuals")
        check_shape(ivf.dim, m)
        bf16, dev = ivf.residuals, ivf.device
        real = torch.nonzero(ivf.row_ids >= 0).flatten()
        if codebooks is None:
            g = torch.Generator(device=dev).manual_seed(seed + 1)
            pick = real[torch.randperm(real.numel(), generator=g, device=dev)[:train_rows]]
            codebooks = train_codebooks(bf16[pick].contiguous(), m, iters=iters, seed=seed)
        codebooks = codebooks.to(device=dev, dtype=torch.float32).contiguous()
        if tuple(codebooks.shape) != (m, CODEWORDS, ivf.dim // m):
            raise ValueError(f"codebooks must be [m, {CODEWORDS}, dim / m] = [{m}, {CODEWORDS}, {ivf.dim // m}]")
        codes = encode(bf16, codebooks)
        codes[ivf.row_ids < 0] = 0                                      # padding rows: code 0, never scored
        return cls(ivf, place_rows(bf16, residuals, dev), codes, codebooks)

    def _code_bytes(self) -> int:
        return self.codes.numel() + 4 * self.codebooks.numel()

    def search_device(self, queries_bf16: torch.Tensor, nprobe: int, k: int, candidates: Optional[int] = None,
                      stream: Optional[torch.cuda.Stream] = None, probed: Optional[Tuple[torch.Tensor, torch.Tensor]] = None):
        """bf16 [nq, dim] on the device -> (ids int64 [nq, k], scores fp32 [nq, k], minmax fp32 [nq, 2],
        (probed list ids int64 [nq, nprobe], their coarse scores fp32)), as IVFIndex.search_device.  Scores are the
        exact S2 values; minmax is (min, max) of the PQ stage's S1 over the probed rows.  candidates (default
        min(128, 4 k)) positions per query come from the PQ scan; 1 <= k <= candidates <= 128."""
        candidates = rescored_candidates(k, candidates)

        def fine(q, p_ids, p_scores, ids, scores, minmax, ws, st):
            _native.check(self._lib.crag_ivf_search_pq(
                self.codes.data_ptr(), self.m, self.codes.stride(0), self.codebooks.data_ptr(),
                self._rows.data_ptr(), self.dim, self._rows.stride(0), self._rows.shape[0],
                self.list_tile_start.data_ptr(), self.list_rows.data_ptr(), self.nlist, self.total_tiles,
                self.row_ids.data_ptr(), q.data_ptr(), q.shape[0], p_ids.data_ptr(), p_scores.data_ptr(), nprobe,
                candidates, k, ids.data_ptr(), scores.data_ptr(), minmax.data_ptr(), ws.data_ptr(), ws.numel(),
                st.cuda_stream), "crag_ivf_search_pq")
        return self._search(queries_bf16, nprobe, k, stream, probed,
                            self._lib.crag_ivf_pq_workspace_bytes(self.nlist, self.total_tiles, candidates, self.m), fine)

    def _wide_fine(self, nprobe: int, candidates: int, k: int, max_probe_rows: int):
        def fine(q, p_ids, p_scores, ids, scores, minmax, ws, st):
            _native.check(self._lib.crag_ivf_search_pq_wide(
                self.codes.data_ptr(), self.m, self.codes.stride(0), self.codebooks.data_ptr(),
                self._rows.data_ptr(), self.dim, self._rows.stride(0), self._rows.shape[0],
                self.list_tile_start.data_ptr(), self.list_rows.data_ptr(), self.nlist, self.total_tiles,
                self.row_ids.data_ptr(), q.data_ptr(), q.shape[0], p_ids.data_ptr(), p_scores.data_ptr(), nprobe,
                candidates, k, max_probe_rows, ids.data_ptr(), scores.data_ptr(), minmax.data_ptr(), ws.data_ptr(),
                ws.numel(), st.cuda_stream), "crag_ivf_search_pq_wide")
        return (self._lib.crag_ivf_pq_wide_workspace_bytes(self.nlist, self.total_tiles, candidates, max_probe_rows,
                                                           self.m), fine)
