"""QuantizedIVF / crag_ivf_search_i8 on the GPU against tests/ivf_i8_oracle.py bit for bit (ids, S2 scores and the S1
(min, max)), with the device's own probed lists; device against page-locked host residuals, two streams, ids beyond
2^32, a -1 / -inf tail, ShardedIVF over a QuantizedIVF, recall, and argument errors that launch nothing."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import ivf_oracle as ivf

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ivf_i8_oracle as io  # noqa: E402
from test_oracle_ivf_i8 import RECALL_MIN, clustered  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _lib():
    assert torch.cuda.is_available()
    from comorag_b200 import _native
    _native.load()


def _bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape
    if a.dtype == np.float32:
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), np.argwhere(a.view(np.uint32) != b.view(np.uint32))[:5]
    else:
        assert np.array_equal(a, b), np.argwhere(a != b)[:5]


def _build(n, d, nlist, nq, seed=0, row_offset=0):
    from comorag_b200.ivf import IVFIndex
    x, q = clustered(n, d, nq, seed)
    idx = IVFIndex.build(torch.from_numpy(x).to(DEV), nlist, iters=4, seed=seed, row_offset=row_offset)
    return idx, torch.from_numpy(q).to(DEV).to(torch.bfloat16), x, q


def _oracle(idx, qb, probed, k, n_cand):
    return io.search_i8(idx.residuals.float().cpu().numpy(), idx.row_ids.cpu().numpy(), idx.list_tile_start.cpu().numpy(),
                        idx.list_rows.cpu().numpy(), qb.float().cpu().numpy(),
                        (probed[0].cpu().numpy(), probed[1].cpu().numpy()), k, n_cand)


def _check(qi, idx, qb, nprobe, k, candidates, **kw):
    ids, sc, mm, probed = qi.search_device(qb, nprobe, k, candidates, **kw)
    torch.cuda.synchronize()
    n_cand = min(128, 4 * k) if candidates is None else candidates
    w_ids, w_sc, w_mm, _ = _oracle(idx, qb, probed, k, n_cand)
    _bits(ids.cpu().numpy(), w_ids)
    _bits(sc.cpu().numpy(), w_sc)
    _bits(mm.cpu().numpy(), w_mm)
    return ids, sc, mm, probed


@pytest.mark.parametrize("n,d,nlist,nprobe,k,nq", [(20000, 128, 64, 8, 10, 8), (50000, 768, 128, 16, 100, 40),
                                                   (3000, 64, 16, 16, 10, 3), (700, 64, 32, 2, 64, 5),
                                                   (20000, 128, 64, 8, 10, 40), (20000, 128, 64, 8, 10, 70)])
def test_matches_oracle(n, d, nlist, nprobe, k, nq):
    from comorag_b200.ivf import QuantizedIVF
    idx, qb, _, _ = _build(n, d, nlist, nq)
    qi = QuantizedIVF.from_ivf(idx)
    for candidates in dict.fromkeys([k, None, 128]):
        ids, _, _, _ = _check(qi, idx, qb, nprobe, k, candidates)
    h_ids, _ = qi.search(qb.float().cpu().numpy(), nprobe, k, 128)   # host entry point: same answer
    _bits(h_ids, ids.cpu().numpy())


def test_host_and_device_residuals_and_two_streams_agree():
    from comorag_b200.ivf import QuantizedIVF
    idx, qb, _, _ = _build(20000, 256, 64, 37, seed=4)
    dq, hq = QuantizedIVF.from_ivf(idx, "device"), QuantizedIVF.from_ivf(idx, "host")
    assert dq.residuals_on_device and not hq.residuals_on_device
    assert hq._rows.is_pinned()
    assert dq.device_bytes == hq.device_bytes + 2 * idx.residuals.numel()
    want = _check(dq, idx, qb, 8, 20, None)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    a = hq.search_device(qb, 8, 20, stream=s1)
    b = dq.search_device(qb, 8, 20, stream=s2)
    torch.cuda.synchronize()
    for got in (a, b):
        for g, w in zip(got[:3], want[:3]):
            _bits(g.cpu().numpy(), w.cpu().numpy())


def test_row_offset_beyond_2_32_maps_through_row_ids():
    from comorag_b200.ivf import QuantizedIVF
    idx, qb, _, _ = _build(5000, 128, 16, 6, seed=2, row_offset=(1 << 33) + 7)
    ids, _, _, _ = _check(QuantizedIVF.from_ivf(idx), idx, qb, 4, 10, None)
    assert (ids >= (1 << 33) + 7).all()


def test_fewer_probed_rows_than_k_leave_a_tail():
    from comorag_b200.ivf import QuantizedIVF
    idx, qb, _, _ = _build(700, 64, 32, 4, seed=5)
    rows = idx.list_rows.cpu().numpy()
    l = int(np.argmin(np.where(rows > 0, rows, 1 << 30)))
    k = int(rows[l]) + 3
    probed = (torch.full((4, 1), l, dtype=torch.int64, device=DEV), torch.zeros((4, 1), device=DEV))
    ids, sc, _, _ = _check(QuantizedIVF.from_ivf(idx), idx, qb, 1, k, 128, probed=probed)
    assert (ids[:, -3:] == -1).all() and torch.isneginf(sc[:, -3:]).all() and (ids[:, :-3] >= 0).all()


def test_sharded_ivf_world_1_wraps_a_quantized_ivf():
    from comorag_b200.ivf import QuantizedIVF, ShardedIVF
    idx, qb, _, _ = _build(20000, 128, 64, 12, seed=6)
    qi = QuantizedIVF.from_ivf(idx)
    got = ShardedIVF(qi).search_device(qb, 8, 10)
    want = qi.search_device(qb, 8, 10)
    for g, w in zip(got, want[:3]):
        _bits(g.cpu().numpy(), w.cpu().numpy())


def test_recall_against_bf16_ivf_at_full_probe():
    from comorag_b200.ivf import QuantizedIVF
    idx, qb, _, _ = _build(20000, 128, 32, 40)
    bf_ids, _, _, probed = idx.search_device(qb, 32, 10)
    ids, _, _, _ = _check(QuantizedIVF.from_ivf(idx), idx, qb, 32, 10, None, probed=probed)
    assert ivf.recall_at_k(ids.cpu().numpy(), bf_ids.cpu().numpy()) >= RECALL_MIN


def _raw_call(qi, qb, rows, nprobe, k, n_cand, ids, sc, mm):
    from comorag_b200 import _native
    from comorag_b200.quantized import quantize_rows
    lib = _native.load()
    q8, qs = quantize_rows(qb, qi.dim8)
    p_ids, p_sc, _ = qi.centroids.search_device(qb, min(nprobe, qi.nlist))
    ws_bytes = lib.crag_ivf_i8_workspace_bytes(qi.nlist, qi.total_tiles, max(1, min(n_cand, 128)))
    ws = torch.empty(max(ws_bytes, 256), dtype=torch.uint8, device=DEV)
    torch.cuda.synchronize()
    return lib.crag_ivf_search_i8(qi._i8.data_ptr(), qi._scales.data_ptr(), qi.dim8, qi._i8.stride(0), rows.data_ptr(),
                                  qi.dim, rows.stride(0), rows.shape[0], qi.list_tile_start.data_ptr(),
                                  qi.list_rows.data_ptr(), qi.nlist, qi.total_tiles, qi.row_ids.data_ptr(),
                                  q8.data_ptr(), qs.data_ptr(), qb.data_ptr(), qb.shape[0], p_ids.data_ptr(),
                                  p_sc.data_ptr(), nprobe, n_cand, k, ids.data_ptr(), sc.data_ptr(), mm.data_ptr(),
                                  ws.data_ptr(), ws_bytes, torch.cuda.current_stream().cuda_stream)


def test_argument_errors_launch_nothing():
    from comorag_b200.ivf import QuantizedIVF
    idx, qb, _, _ = _build(2000, 64, 8, 3, seed=7)
    qi = QuantizedIVF.from_ivf(idx)
    with pytest.raises(ValueError):
        qi.search_device(qb, 9, 10)                      # nprobe > nlist
    with pytest.raises(ValueError):
        qi.search_device(qb, 2, 10, candidates=5)        # k > candidates
    with pytest.raises(ValueError):
        qi.search_device(qb, 2, 10, candidates=129)      # candidates > 128
    with pytest.raises(ValueError):
        qi.search_device(qb.float(), 2, 10)              # dtype
    with pytest.raises(ValueError):
        qi.search_device(qb[:, :32].contiguous(), 2, 10)  # width
    with pytest.raises(ValueError):
        QuantizedIVF.from_ivf(idx, "disk")
    # the C entry point: every rejected call returns an error and leaves the outputs untouched
    from comorag_b200 import _native
    lib = _native.load()
    pageable = idx.residuals.cpu()
    assert not pageable.is_pinned()
    cases = [(pageable, 2, 10, 40, "pageable"), (idx.residuals, 9, 10, 40, "nprobe"),
             (idx.residuals, 2, 10, 5, "n_cand"), (idx.residuals, 2, 10, 129, "n_cand")]
    for rows, nprobe, k, n_cand, what in cases:
        ids = torch.full((3, k), -7, dtype=torch.int64, device=DEV)
        sc = torch.full((3, k), -7.0, device=DEV)
        mm = torch.full((3, 2), -7.0, device=DEV)
        rc = _raw_call(qi, qb, rows, nprobe, k, n_cand, ids, sc, mm)
        torch.cuda.synchronize()
        assert rc != 0, what
        assert what in lib.crag_last_error().decode(), what
        assert (ids == -7).all() and (sc == -7).all() and (mm == -7).all(), what
