"""Shared helpers for the search parity tests (test infrastructure)."""
from __future__ import annotations

import numpy as np
import torch


def make_unit_rows(n: int, dim: int, seed: int, device="cpu") -> torch.Tensor:
    """Seeded N(0,1) rows, L2-normalised in fp32, rounded to bf16 (SURVEY.md 8d synthetic corpus).  Generated in
    slabs of at most 2^28 fp32 values (1 GiB), so that a 10M x 1024 corpus fits on an 80 GB GPU; below one slab the
    rows are those of a single randn call."""
    g = torch.Generator(device=device).manual_seed(seed)
    out = torch.empty((n, dim), dtype=torch.bfloat16, device=device)
    slab = max(1, (1 << 28) // dim)
    for s0 in range(0, n, slab):
        x = torch.randn((min(slab, n - s0), dim), generator=g, device=device, dtype=torch.float32)
        out[s0:s0 + x.shape[0]] = torch.nn.functional.normalize(x, dim=1).to(torch.bfloat16)
    return out


def torch_reference_topk(corpus_bf16: torch.Tensor, queries_bf16: torch.Tensor, k: int, row_offset: int = 0,
                         chunk: int = 1 << 18):
    """fp64 ground truth on whatever device the tensors live on; same outputs as oracle.topk_exact."""
    n = corpus_bf16.shape[0]
    nq = queries_bf16.shape[0]
    dev = corpus_bf16.device
    q = queries_bf16.double()
    kk = min(k + 1, n)
    best_s = torch.empty((nq, 0), dtype=torch.float64, device=dev)
    best_i = torch.empty((nq, 0), dtype=torch.int64, device=dev)
    mn = torch.full((nq,), float("inf"), dtype=torch.float64, device=dev)
    mx = torch.full((nq,), float("-inf"), dtype=torch.float64, device=dev)
    for s0 in range(0, n, chunk):
        blk = corpus_bf16[s0:s0 + chunk].double()
        sc = q @ blk.T
        mn = torch.minimum(mn, sc.min(dim=1).values)
        mx = torch.maximum(mx, sc.max(dim=1).values)
        ids = torch.arange(s0, s0 + blk.shape[0], device=dev, dtype=torch.int64).expand(nq, -1)
        cs = torch.cat([best_s, sc], dim=1)
        ci = torch.cat([best_i, ids], dim=1)
        # sort by score desc then id asc: stable sort on ids first (already ascending within blocks,
        # but the carried-over best block comes first) then stable sort by -score
        o1 = torch.argsort(ci, dim=1, stable=True)
        cs, ci = torch.gather(cs, 1, o1), torch.gather(ci, 1, o1)
        o2 = torch.argsort(cs, dim=1, descending=True, stable=True)[:, :kk]
        best_s, best_i = torch.gather(cs, 1, o2), torch.gather(ci, 1, o2)
    out_i = np.full((nq, k), -1, dtype=np.int64)
    out_s = np.full((nq, k), -np.inf)
    gaps = np.full((nq, k), np.inf)
    m = min(k, n)
    bs, bi = best_s.cpu().numpy(), best_i.cpu().numpy()
    out_i[:, :m] = bi[:, :m] + row_offset
    out_s[:, :m] = bs[:, :m]
    if n > 0:
        d = bs[:, :-1] - bs[:, 1:]
        gaps[:, :d.shape[1]][:, :k] = d[:, :k]
    return out_i, out_s, np.stack([mn.cpu().numpy(), mx.cpu().numpy()], axis=1), gaps
