"""One-bit snapshot of a DenseIndex: a scan that reads dim8 / 8 + 4 bytes per row, then an exact bf16 rescore.

Every row is stored as its sign bits plus one fp32 scale, alpha = mean |x_i|: 132 bytes per row at dim 1024, against
2048 for bf16 and 1028 for int8.  A search quantises the queries to int8 (crag_quantize_rows_i8), runs
crag_search_topk_b1 (crag_knn_topk_b1 above 128 candidates, search_wide) over the codes for `candidates` rows per
query, then crag_rescore_topk recomputes each candidate's score from its bf16 row and the bf16 query and keeps the best
k, as QuantizedIndex does.  The returned scores are those
exact fp32 dots; only the choice of candidates comes from the one-bit scores.  The bf16 rows may live in page-locked
host memory (rows="host").  Semantics: DESIGN.md section 3f and tests/binary_oracle.py.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from .quantized import QuantizedIndex, _dim8, _encode_rows


def binarize_rows(rows: torch.Tensor, stream: Optional[torch.cuda.Stream] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """crag_binarize_rows of a device bf16 [n, dim] tensor (unit inner stride): (uint8 codes [n, dim8 / 8], fp32 alpha
    [n]), dim8 = dim rounded up to a multiple of 128."""
    return _encode_rows("binarize_rows", "crag_binarize_rows", rows, lambda dim: _dim8(dim) // 8, torch.uint8, stream)


class BinaryIndex(QuantizedIndex):
    """Frozen one-bit snapshot of a DenseIndex's rows (rows added to the DenseIndex later are not seen).  The surface
    is QuantizedIndex's: from_dense(index, rows="device" | "host"), search_device, search, search_device_wide,
    search_wide, prepare_queries, n_rows, rows_on_device and device_bytes."""

    @staticmethod
    def _encode(rows: torch.Tensor, dim8: int) -> Tuple[torch.Tensor, torch.Tensor]:
        return binarize_rows(rows)

    @staticmethod
    def _stage1(wide: bool) -> str:
        return "crag_knn_topk_b1" if wide else "crag_search_topk_b1"
