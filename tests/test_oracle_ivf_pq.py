"""Self-tests of tests/ivf_pq_oracle.py, the numpy statement of the IVF search over product-quantized residuals.

The encode, table and stage-1 sums are checked against scalar loops that spell out the rounding of every operation.
The exactness invariant: when each subspace holds at most 256 distinct residual sub-vectors and the codebooks hold them
all, PQ is lossless; with values whose products and sums are exact in fp32, S1 then equals the bf16 IVF score of every
probed row, and the answer equals the exact ranking of the probed rows (oracle/ivf_oracle.py's rule)."""
import os
import sys

import numpy as np
import pytest

from oracle import ivf_oracle as ivf

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ivf_i8_oracle as io  # noqa: E402
import ivf_pq_oracle as po  # noqa: E402

F32 = np.float32


def test_encode_matches_a_scalar_loop():
    rng = np.random.default_rng(0)
    m, dsub = 3, 4
    cb = rng.standard_normal((m, 256, dsub)).astype(F32)
    cb[1, 7] = cb[1, 3]                                   # duplicate codewords: the smaller index wins
    x = ivf.bf16_round(rng.standard_normal((40, m * dsub)).astype(F32))
    x[5, dsub:2 * dsub] = cb[1, 3]
    got = po.encode(x, cb)
    for r in range(x.shape[0]):
        for j in range(m):
            best, bc = F32(np.inf), 0
            for c in range(256):
                d = None
                for t in range(dsub):
                    diff = F32(x[r, j * dsub + t] - cb[j, c, t])
                    d = F32(diff * diff) if d is None else F32(d + F32(diff * diff))
                if d < best:
                    best, bc = d, c
            assert got[r, j] == bc
    assert got[5, 1] == 3


def test_table_and_sums_match_scalar_loops():
    rng = np.random.default_rng(1)
    m, dsub, nq = 4, 3, 2
    cb = rng.standard_normal((m, 256, dsub)).astype(F32)
    q = ivf.bf16_round(rng.standard_normal((nq, m * dsub)).astype(F32))
    lut = po.table(q, cb)
    for i in range(nq):
        for j in range(m):
            for c in (0, 17, 255):
                acc = F32(q[i, j * dsub] * cb[j, c, 0])
                for t in range(1, dsub):
                    acc = F32(acc + F32(q[i, j * dsub + t] * cb[j, c, t]))
                assert lut[i, j, c].view(np.uint32) == acc.view(np.uint32)
    codes = rng.integers(0, 256, (10, m)).astype(np.uint8)
    s = po.pq_sums(lut[0], codes)
    for r in range(10):
        acc = lut[0, 0, codes[r, 0]]
        for j in range(1, m):
            acc = F32(acc + lut[0, j, codes[r, j]])
        assert s[r].view(np.uint32) == acc.view(np.uint32)


LIST_ROWS = [0, 1, 127, 128, 129, 0, 40]


def lossless_case(rng, dim, m, nq, values_per_sub=200):
    """A padded layout whose residual sub-vectors take at most `values_per_sub` distinct values per subspace, the
    codebooks that hold them (the rest of each codebook repeats its last entry), and exact-arithmetic values:
    residuals in multiples of 1/8 within [-1, 1], queries in multiples of 1/16, coarse scores in multiples of 1/4."""
    dsub = dim // m
    nlist = len(LIST_ROWS)
    tiles = [(r + 127) // 128 for r in LIST_ROWS]
    starts = np.concatenate([[0], np.cumsum(tiles)]).astype(np.int32)
    n = int(starts[-1]) * 128
    cb = np.empty((m, 256, dsub), F32)
    res = np.zeros((n, dim), F32)
    row_ids = np.full(n, -1, np.int64)
    for j in range(m):
        vals = rng.integers(-8, 9, (values_per_sub, dsub)).astype(F32) / 8
        cb[j, :values_per_sub] = vals
        cb[j, values_per_sub:] = vals[-1]
    nid = 0
    for l, r in enumerate(LIST_ROWS):
        p = starts[l] * 128 + np.arange(r)
        for j in range(m):
            res[p, j * dsub:(j + 1) * dsub] = cb[j, rng.integers(0, values_per_sub, r)]
        row_ids[p] = nid + np.arange(r)
        nid += r
    # identical rows in two lists, which get the same coarse scores below: the tie goes to the smaller position
    a, b = starts[3] * 128 + 5, starts[4] * 128 + 7
    res[b] = res[a]
    q = rng.integers(-16, 17, (nq, dim)).astype(F32) / 16
    probed = np.tile(np.arange(nlist, dtype=np.int64), (nq, 1))
    coarse = (rng.integers(-8, 9, (nq, nlist)).astype(F32) / 4)
    coarse[:, 4] = coarse[:, 3]
    return res, row_ids, starts, np.array(LIST_ROWS, np.int32), cb, q, (probed, coarse), (a, b)


@pytest.mark.parametrize("dim,m", [(64, 8), (192, 96), (192, 192)])
def test_lossless_codebooks_reproduce_the_bf16_ivf_answer(dim, m):
    rng = np.random.default_rng(dim + m)
    nq, k = 3, 20
    res, row_ids, starts, lrows, cb, q, probed, (a, b) = lossless_case(rng, dim, m, nq)
    codes = po.encode(res, cb)
    dsub = dim // m
    recon = cb[np.arange(m)[None, :], codes.astype(np.int64)].reshape(-1, dim)
    real = row_ids >= 0
    assert np.array_equal(recon[real], res[real])            # every stored residual is a codeword sequence
    ids, s2, mm, (c_pos, c_s1) = po.search_pq(res, codes, cb, row_ids, starts, lrows, q, probed, k, n_cand=k)
    for i in range(nq):
        pos = np.nonzero(real)[0]
        lists = io.list_of_positions(starts, pos)
        exact = res[pos].astype(np.float64) @ q[i].astype(np.float64) + probed[1][i][lists].astype(np.float64)
        order = np.lexsort((pos, -exact))[:k]
        assert np.array_equal(c_pos[i], pos[order])
        assert np.array_equal(c_s1[i].astype(np.float64), exact[order])     # S1 is the exact IVF score
        assert np.array_equal(ids[i], row_ids[pos[order]])
        assert np.array_equal(s2[i], c_s1[i])
        assert mm[i, 0] == exact.min() and mm[i, 1] == exact.max()
    assert dsub * m == dim


def test_ties_go_to_the_smaller_position():
    rng = np.random.default_rng(3)
    res, row_ids, starts, lrows, cb, q, probed, (a, b) = lossless_case(rng, 64, 8, 1)
    codes = po.encode(res, cb)
    _, _, _, (c_pos, c_s1) = po.search_pq(res, codes, cb, row_ids, starts, lrows, q, probed, 128, n_cand=128)
    s = (res[[a, b]] @ q[0] + probed[1][0][[3, 4]]).astype(F32)
    assert s[0] == s[1]
    pos = list(c_pos[0])
    if a in pos:
        assert b in pos and pos.index(b) == pos.index(a) + 1


def test_probes_absent_duplicated_and_empty():
    rng = np.random.default_rng(4)
    res, row_ids, starts, lrows, cb, q, probed, _ = lossless_case(rng, 64, 8, 2)
    codes = po.encode(res, cb)
    ids_p = np.array([[3, -1, 3, 99, 0], [5, 5, -7, 1, 1]], np.int64)   # list 0 and 5 are empty
    sc_p = np.take_along_axis(probed[1], np.clip(ids_p, 0, len(lrows) - 1), axis=1)
    sc_p[0, 2] = sc_p[0, 0]
    sc_p[1, 1], sc_p[1, 4] = sc_p[1, 0], sc_p[1, 3]
    ids, s2, mm, (c_pos, _) = po.search_pq(res, codes, cb, row_ids, starts, lrows, q, (ids_p, sc_p), 128, n_cand=128)
    assert (c_pos[0] >= 0).sum() == 128 and set(io.list_of_positions(starts, c_pos[0][c_pos[0] >= 0])) == {3}
    assert (c_pos[1] >= 0).sum() == 1 and (ids[1, 1:] == -1).all() and np.isneginf(s2[1, 1:]).all()
    only = po.search_pq(res, codes, cb, row_ids, starts, lrows, q[:1], (np.array([[0, 5]]), sc_p[:1, :2]), 4, 4)
    assert (only[0] == -1).all() and np.isposinf(only[2][0, 0]) and np.isneginf(only[2][0, 1])


def test_recall_of_trained_codebooks_against_bf16_ivf():
    """Lossy PQ on clustered data: the rescored answer finds most of the bf16 IVF answer (m = 16 at dim 64)."""
    from test_oracle_ivf_i8 import _index
    lists, qb, _ = _index(3000, 64, 8, 8, seed=5)
    res, row_ids, starts, lrows = io.padded_layout(lists)
    rng = np.random.default_rng(0)
    real = np.nonzero(row_ids >= 0)[0]
    m = 16
    cb = res[rng.choice(real, 256, replace=False)].reshape(256, m, 4).transpose(1, 0, 2).copy()
    for _ in range(4):                                       # a few Lloyd steps on the CPU
        codes = po.encode(res[real], cb)
        for j in range(m):
            for c in range(256):
                sel = codes[:, j] == c
                if sel.any():
                    cb[j, c] = res[real][sel, j * 4:(j + 1) * 4].mean(axis=0)
    codes = np.zeros((res.shape[0], m), np.uint8)
    codes[real] = po.encode(res[real], cb)
    probed = ivf.probe_lists(lists, qb, lists.nlist)
    probed = (probed[0], probed[1].astype(F32))
    want, _, _ = ivf.search(lists, qb, lists.nlist, 10, probed=probed)
    got, _, _, _ = po.search_pq(res, codes, cb, row_ids, starts, lrows, qb, probed, 10, n_cand=40)
    assert ivf.recall_at_k(got, want) >= 0.9
