"""Self-tests of tests/ivf_i8_oracle.py, the numpy statement of the IVF search over int8 residuals.

With n_cand covering every probed row the int8 stage chooses nothing, so the answer must be the exact S2 ranking of the
probed rows.  With nprobe = nlist on clustered data its recall against oracle/ivf_oracle.search (bf16 IVF) must reach
RECALL_MIN, the threshold tests/test_ivf_i8_gpu.py applies to the device; the device equals this oracle bit for bit,
so the CPU run fixes the threshold."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import ivf_oracle as ivf
from oracle import quant_oracle as qo

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ivf_i8_oracle as io  # noqa: E402

# recall@10 of QuantizedIVF against bf16 IVF (nprobe = nlist, clustered data, default candidates = 40): 1.000 here
RECALL_MIN = 0.99


def clustered(n, d, nq, seed=0, n_dirs=60):
    g = torch.Generator().manual_seed(seed)
    dirs = torch.nn.functional.normalize(torch.randn(n_dirs, d, generator=g), dim=1)
    sigma = 0.5 / d ** 0.5
    x = torch.nn.functional.normalize(dirs[torch.randint(0, n_dirs, (n,), generator=g)] + sigma * torch.randn(n, d, generator=g), dim=1)
    q = torch.nn.functional.normalize(dirs[torch.randint(0, n_dirs, (nq,), generator=g)] + sigma * torch.randn(nq, d, generator=g), dim=1)
    return x.numpy(), q.numpy()


def _index(n, d, nlist, nq, seed=0):
    x, q = clustered(n, d, nq, seed)
    c = ivf.spherical_kmeans(x, nlist, iters=4, seed=seed)
    lists = ivf.IVFLists(x, c)
    return lists, ivf.bf16_round(q), q


def test_padded_layout_matches_lists():
    lists, _, _ = _index(1500, 64, 7, 1)
    res, row_ids, starts, list_rows = io.padded_layout(lists, row_offset=1 << 33)
    assert res.shape[0] == starts[-1] * 128
    for l in range(lists.nlist):
        p0, m = starts[l] * 128, list_rows[l]
        assert np.array_equal(row_ids[p0:p0 + m] - (1 << 33), lists.ids[lists.offsets[l]:lists.offsets[l + 1]])
        assert (row_ids[p0 + m:starts[l + 1] * 128] == -1).all() and not res[p0 + m:starts[l + 1] * 128].any()
        assert (io.list_of_positions(starts, np.arange(p0, p0 + m)) == l).all()


@pytest.mark.parametrize("nprobe,k", [(2, 10), (3, 1), (1, 50)])
def test_all_probed_rows_as_candidates_is_exact_s2_ranking(nprobe, k):
    lists, qv, q = _index(400, 128, 16, 6, seed=nprobe)
    res, row_ids, starts, list_rows = io.padded_layout(lists)
    probed = ivf.probe_lists(lists, q, nprobe)
    probed = (probed[0], probed[1].astype(np.float32))
    n_probed = max(int(list_rows[probed[0][i]].sum()) for i in range(len(q)))
    assert n_probed <= 128
    ids, sc, mm, (c_pos, _) = io.search_i8(res, row_ids, starts, list_rows, qv, probed, k, 128)
    for i in range(len(q)):
        pos = np.concatenate([starts[l] * 128 + np.arange(list_rows[l]) for l in probed[0][i]])
        assert set(c_pos[i][c_pos[i] >= 0].tolist()) == set(pos.tolist())
        cs = dict(zip(probed[0][i].tolist(), probed[1][i].tolist()))
        s2 = np.array([qo.s2_scores(res[p:p + 1], qv[i])[0] for p in pos], np.float32)
        s2 = (s2 + np.array([cs[int(l)] for l in io.list_of_positions(starts, pos)], np.float32)).astype(np.float32)
        want_pos, want_sc = qo.topk_keys(s2, pos, k)
        assert np.array_equal(ids[i], np.where(want_pos >= 0, row_ids[np.maximum(want_pos, 0)], -1))
        assert np.array_equal(sc[i].view(np.uint32), want_sc.view(np.uint32))
        assert mm[i, 0] <= mm[i, 1]


def test_recall_against_bf16_ivf_at_full_probe():
    lists, qv, q = _index(20000, 128, 32, 40)
    res, row_ids, starts, list_rows = io.padded_layout(lists)
    probed = ivf.probe_lists(lists, q, lists.nlist)
    probed = (probed[0], probed[1].astype(np.float32))
    ids, _, _, _ = io.search_i8(res, row_ids, starts, list_rows, qv, probed, 10, 40)
    want, _, _ = ivf.search(lists, q, lists.nlist, 10, probed=probed)
    assert ivf.recall_at_k(ids, want) >= RECALL_MIN


def test_fewer_probed_rows_than_k_leave_a_tail():
    lists, qv, q = _index(300, 64, 16, 3)
    res, row_ids, starts, list_rows = io.padded_layout(lists)
    l = int(np.argmin(np.where(list_rows > 0, list_rows, 1 << 30)))
    probed = (np.full((3, 1), l, np.int64), np.zeros((3, 1), np.float32))
    k = int(list_rows[l]) + 3
    ids, sc, _, _ = io.search_i8(res, row_ids, starts, list_rows, qv, probed, k, max(k, 40))
    assert (ids[:, -3:] == -1).all() and np.isneginf(sc[:, -3:]).all() and (ids[:, :-3] >= 0).all()
