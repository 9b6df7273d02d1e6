"""GPU parity of the IVF residual-IP search (crag_ivf_search, BASELINE config 4) against oracle/ivf_oracle.py.
The reference has no IVF code: the oracle is our own statement of the semantic (parity unpinned)."""
import numpy as np
import pytest
import torch

from oracle import ivf_oracle as ivf
from oracle import search_oracle as so

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from comorag_b200 import _native
    _native.load()
    return torch.device("cuda:0")


def _clustered(n, d, nq, seed=0, n_dirs=60):
    g = torch.Generator().manual_seed(seed)
    dirs = torch.nn.functional.normalize(torch.randn(n_dirs, d, generator=g), dim=1)
    sigma = 0.5 / d ** 0.5
    x = torch.nn.functional.normalize(dirs[torch.randint(0, n_dirs, (n,), generator=g)] + sigma * torch.randn(n, d, generator=g), dim=1)
    q = torch.nn.functional.normalize(dirs[torch.randint(0, n_dirs, (nq,), generator=g)] + sigma * torch.randn(nq, d, generator=g), dim=1)
    return x.numpy(), q.numpy()


@pytest.mark.parametrize("n,d,nlist,nprobe,k,nq", [(20000, 128, 64, 8, 10, 8), (50000, 768, 128, 16, 100, 40),
                                                   (3000, 64, 16, 16, 10, 3), (700, 64, 32, 2, 64, 5)])
def test_ivf_search_matches_oracle(dev, n, d, nlist, nprobe, k, nq):
    from comorag_b200.ivf import IVFIndex, TILE_ROWS
    x, q = _clustered(n, d, nq)
    idx = IVFIndex.build(torch.from_numpy(x).to(dev), nlist, iters=4, seed=0)
    c = idx.centroids.matrix().float().cpu().numpy()                 # bf16 centroid values
    a = idx.assignment.cpu().numpy()
    # assignment = float64 argmax over the same bf16 inputs, except rows on a near tie between two centroids
    a64 = ivf.assign(x, c)
    s64 = ivf.bf16_round(x).astype(np.float64) @ c.astype(np.float64).T
    off = np.nonzero(a != a64)[0]
    assert off.size <= max(3, n // 2000)
    assert np.all(np.abs(s64[off, a[off]] - s64[off, a64[off]]) < 1e-5)
    # layout: the oracle's grouping of the engine's own assignment, padded to tiles
    L = ivf.IVFLists(x, c, assignment=a)
    tile_start, list_rows = idx.list_tile_start.cpu().numpy(), idx.list_rows.cpu().numpy()
    np.testing.assert_array_equal(list_rows, np.diff(L.offsets))
    row_ids, res = idx.row_ids.cpu().numpy(), idx.residuals.float().cpu().numpy()
    for l in (0, nlist // 2, nlist - 1):
        s0, m = tile_start[l] * TILE_ROWS, list_rows[l]
        np.testing.assert_array_equal(row_ids[s0:s0 + m], L.ids[L.offsets[l]:L.offsets[l + 1]])
        np.testing.assert_array_equal(res[s0:s0 + m], L.residuals[L.offsets[l]:L.offsets[l + 1]])
        assert np.all(row_ids[s0 + m:tile_start[l + 1] * TILE_ROWS] == -1)
    # search
    qb = torch.from_numpy(q).to(dev).to(torch.bfloat16)
    ids, scores, mm, (p_ids, p_sc) = idx.search_device(qb, nprobe, k)
    torch.cuda.synchronize()
    p_ids, p_sc = p_ids.cpu().numpy(), p_sc.cpu().numpy()
    want_p, want_ps, _, gaps_p = so.topk_exact(c, ivf.bf16_round(q), nprobe)
    so.assert_topk_matches(p_ids, p_sc.astype(np.float64), want_p, want_ps, gaps_p)           # coarse pass
    w_ids, w_sc, gaps = ivf.search(L, q, nprobe, k, probed=(p_ids, p_sc))                      # fine pass, same lists
    got_i, got_s = ids.cpu().numpy(), scores.cpu().numpy().astype(np.float64)
    so.assert_topk_matches(got_i, got_s, w_ids, w_sc, gaps, score_tol=1e-3)
    has = w_ids[:, 0] >= 0
    np.testing.assert_allclose(mm.cpu().numpy()[has, 1], got_s[has, 0], atol=1e-6)            # max over probed rows = best score
    # end to end (own coarse pass in the oracle too): recall against exact search over the same bf16 rows
    exact, _, _, _ = so.topk_exact(ivf.bf16_round(x), ivf.bf16_round(q), min(k, 10))
    if nprobe == nlist:
        assert ivf.recall_at_k(got_i[:, :min(k, 10)], exact) > 0.9
    # host entry point returns the same thing
    h_ids, h_sc = idx.search(q, nprobe, k)
    np.testing.assert_array_equal(h_ids, got_i)


def test_ivf_argument_errors(dev):
    from comorag_b200.ivf import IVFIndex
    x, q = _clustered(2000, 64, 2)
    idx = IVFIndex.build(torch.from_numpy(x).to(dev), 8, iters=2)
    qb = torch.from_numpy(q).to(dev).to(torch.bfloat16)
    with pytest.raises(ValueError):
        idx.search_device(qb, 9, 10)                 # nprobe > nlist
    with pytest.raises(ValueError):
        idx.search_device(qb, 2, 129)
    with pytest.raises(ValueError):
        idx.search_device(qb.float(), 2, 10)
    with pytest.raises(ValueError):
        idx.search_device(qb.cpu(), 2, 10)           # queries on the host
    p_ids, p_sc, _ = idx.centroids.search_device(qb, 2)
    for probed in [(p_ids[:, :1], p_sc[:, :1]), (p_ids[:1], p_sc[:1]), (p_ids.to(torch.int32), p_sc)]:
        with pytest.raises(ValueError):               # mis-shaped or int32 probed lists
            idx.search_device(qb, 2, 10, probed=probed)
    with pytest.raises(ValueError):
        IVFIndex.build(torch.from_numpy(x), 8)       # host tensor: no CPU fallback
