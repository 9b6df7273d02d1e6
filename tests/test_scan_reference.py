"""CPU checks of tests/scan_reference.py, the exact reference the bf16 scan family is compared with on the GPU.

The helpers are checked against a brute-force restatement (plain Python sorts over (score, row) pairs) on hand-made
score matrices and IVF layouts; the comparator must reject five specific mutants of the IVF answer; and the score
bound (SCORE_BOUND) is calibrated on a torch model of the scan's fp32 accumulation, in the style of
test_kernel_error_bounds.py, whose input generator this file reuses."""
import math
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import scan_reference as sr  # noqa: E402
from ivf_i8_oracle import padded_layout  # noqa: E402
from oracle import ivf_oracle as ivf  # noqa: E402
from test_kernel_error_bounds import gemm_inputs  # noqa: E402

F32 = np.float32


def _f32(*v):
    return torch.tensor(v, dtype=torch.float32)


def _korder(s, row):
    """Sort key of the brute force: (orderable score descending, row ascending)."""
    return (-int(sr.orderable(_f32(s))[0]), row)


# ---------------------------------------------------------------------------------------------------------- keys
def test_keys_order_scores_then_rows():
    s = _f32(1.0, 1.0, 0.0, -0.0, float("inf"), float("-inf"), -1.0, 2.0 ** -149)
    rows = torch.tensor([5, 3, 0, 0, 9, 1, 2, 4])
    k = sr.keys(s, rows).numpy().view(np.uint64)
    assert k[1] > k[0]                                     # equal scores: the smaller row ranks higher
    assert k[2] > k[3]                                     # +0 above -0
    assert k[4] == k.max()                                 # +inf on top
    assert k[5] == k.min() and k[5] > 0                    # -inf at the bottom, still a valid (non-zero) key
    assert k[7] > k[2] > k[3] > k[6]                       # smallest denormal > +0 > -0 > -1
    assert np.array_equal(np.argsort(k[:4]), [3, 2, 0, 1])
    bits = 0x3F800000 << 32 | (0xFFFFFFFF - 5) | (1 << 63)    # orderable(1.0) = 0xBF800000
    assert int(k[0]) == bits


# ---------------------------------------------------------------------------------------------------------- flat
def _brute_flat(S, k, row_offset=0):
    nq, n = S.shape
    ids = np.full((nq, k), -1, np.int64)
    sc = np.full((nq, k), -np.inf, F32)
    for q in range(nq):
        order = sorted(range(n), key=lambda r: _korder(float(S[q, r]), r))[:k]
        ids[q, :len(order)] = np.array(order, np.int64) + row_offset
        sc[q, :len(order)] = S[q, order].numpy()
    return torch.from_numpy(ids), torch.from_numpy(sc)


def test_topk_from_scores_ties_zeros_infinities_and_tail():
    S = torch.stack([_f32(0.5, 0.5, -0.0, 0.0, 0.5, float("inf"), -1.0),
                     _f32(-3.0, -2.0, -2.0, -5.0, -2.0, -1.0, -4.0),
                     _f32(float("-inf"), 0.0, -0.0, 0.0, -0.0, 1.0, 1.0)])
    for k in (1, 3, 7, 10):
        ids, sc, mm, last = sr.topk_from_scores(S, k, row_offset=(1 << 33) + 7)
        w_ids, w_sc = _brute_flat(S, k, (1 << 33) + 7)
        sr.assert_bits(ids, w_ids, "ids")
        sr.assert_bits(sc, w_sc, "scores")
        if k > 7:
            assert (ids[:, 7:] == -1).all() and torch.isneginf(sc[:, 7:]).all() and (last == 0).all()
    sr.assert_bits(ids[0, :5], torch.tensor([5, 0, 1, 4, 3]) + (1 << 33) + 7)   # +inf, ties by row, +0 before -0
    sr.assert_bits(mm, torch.stack([_f32(-1.0, float("inf")), _f32(-5.0, -1.0), _f32(float("-inf"), 1.0)]))
    _, _, mm2, _ = sr.topk_from_scores(_f32(0.0, -0.0, 0.0)[None], 2)
    sr.assert_bits(mm2, _f32(-0.0, 0.0)[None])                # (min, max) order zeros as the keys do


def test_topk_from_scores_pages_continue_exactly():
    g = torch.Generator().manual_seed(1)
    S = (torch.randint(-4, 5, (3, 700), generator=g).float() / 8)      # dense in exact ties
    full_ids, full_sc, _, _ = sr.topk_from_scores(S, 650)
    after, got_i, got_s = None, [], []
    for p0 in range(0, 650, 128):
        kk = min(128, 650 - p0)
        i, s, _, after = sr.topk_from_scores(S, kk, after_keys=after)
        got_i.append(i), got_s.append(s)
        want_last = sr.keys(full_sc[:, p0 + kk - 1], full_ids[:, p0 + kk - 1])
        sr.assert_bits(after, want_last, "last key")
    sr.assert_bits(torch.cat(got_i, 1), full_ids)
    sr.assert_bits(torch.cat(got_s, 1), full_sc)
    i, s, _, last = sr.topk_from_scores(S, 128, after_keys=after)        # 700 - 650 = 50 rows left
    assert (i[:, :50] >= 0).all() and (i[:, 50:] == -1).all() and (last == 0).all()
    i, _, _, _ = sr.topk_from_scores(S, 4, after_keys=torch.zeros(3, dtype=torch.int64))
    assert (i == -1).all()                                                # key 0: nothing is below it


# ----------------------------------------------------------------------------------------------------------- IVF
def _layout(list_rows, row_offset=0, seed=0):
    """Hand-made padded layout: list_rows int [nlist] -> (tile_start, list_rows, row_ids, n_pos).  Original ids
    are dealt in reverse list order, so position order and id order disagree across lists."""
    rows = np.asarray(list_rows, np.int64)
    tiles = (rows + 127) // 128
    starts = np.concatenate([[0], np.cumsum(tiles)])
    n_pos = max(int(starts[-1]) * 128, 128)
    row_ids = np.full(n_pos, -1, np.int64)
    nxt = 0
    for l in reversed(range(rows.size)):
        p = starts[l] * 128 + np.arange(rows[l])
        row_ids[p] = nxt + np.arange(rows[l]) + row_offset
        nxt += rows[l]
    return (torch.from_numpy(starts.astype(np.int32)), torch.from_numpy(rows.astype(np.int32)),
            torch.from_numpy(row_ids), n_pos)


def _brute_ivf(S, p_ids, p_sc, starts, lrows, row_ids, k, bug=None):
    """Plain restatement of the IVF rule, and its mutants:
    id_ties  exact ties broken by original id instead of position;   pad   padding rows of probed lists compete;
    tail     rows past the first tile of a list are dropped;          mask  (min, max) over every query's probes."""
    nq, n_pos = S.shape
    ids = np.full((nq, k), -1, np.int64)
    sc = np.full((nq, k), -np.inf, F32)
    mm = np.tile(np.array([np.inf, -np.inf], F32), (nq, 1))
    probes = []
    for q in range(nq):
        d = {}
        for l, s in zip(p_ids[q].tolist(), p_sc[q].tolist()):
            if 0 <= l < lrows.numel() and l not in d:
                d[l] = F32(s)
        probes.append(d)
    for q in range(nq):
        cand = []
        mm_lists = {l for d in probes for l in d} if bug == "mask" else set(probes[q])
        for l in sorted(set(probes[q]) | mm_lists):
            n_real = int(lrows[l])
            n_tiles = int(starts[l + 1] - starts[l])
            span = n_tiles * 128 if bug == "pad" else n_real
            if bug == "tail":
                span = min(span, 128)
            c = probes[q].get(l, F32(0))
            for j in range(span):
                p = int(starts[l]) * 128 + j
                s = F32(F32(S[q, p]) + c)
                if l in probes[q]:
                    cand.append((s, p))
                if l in mm_lists and j < n_real:
                    o = int(sr.orderable(_f32(s))[0])
                    if o < int(sr.orderable(_f32(mm[q, 0]))[0]):
                        mm[q, 0] = s
                    if o > int(sr.orderable(_f32(mm[q, 1]))[0]):
                        mm[q, 1] = s
        tie = (lambda sp: _korder(sp[0], int(row_ids[sp[1]]))) if bug == "id_ties" else (lambda sp: _korder(*sp))
        cand.sort(key=tie)
        for j, (s, p) in enumerate(cand[:k]):
            ids[q, j], sc[q, j] = int(row_ids[p]), s
    return torch.from_numpy(ids), torch.from_numpy(sc), torch.from_numpy(mm)


def _ivf_case(seed=0):
    """nlist 6 with an empty list, 128- and 129-row lists, exact ties inside one list and across lists, an
    all-negative query, duplicate / -1 / out-of-range probes, and a query that probes only empty lists."""
    starts, lrows, row_ids, n_pos = _layout([5, 0, 128, 129, 3, 40], row_offset=(1 << 33) + 7)
    g = torch.Generator().manual_seed(seed)
    nq = 6
    S = torch.randn(nq, n_pos, generator=g)
    S[:, starts[4] * 128:starts[4] * 128 + 3] = S[:, 0:3]        # list 4 repeats list 0's first rows: cross-list ties
    S[:, starts[2] * 128 + 7] = S[:, starts[2] * 128 + 3]        # and a tie inside list 2
    S[:, starts[3] * 128 + 128] = 4.0                            # the 129th row of list 3 is every query's best there
    S[3] = -S[3].abs() - 1.0                                     # query 3: every score negative
    S[:, 0:1] = torch.where(torch.arange(nq)[:, None] == 2, 0.0, S[:, 0:1])
    S[2, starts[4] * 128] = -0.0                                 # +0 (list 0) against -0 (list 4)
    p_ids = torch.tensor([[0, 4, 2, 3], [3, 3, -1, 9], [0, 4, 6, -1], [5, 2, 0, 4], [1, 1, 1, 1], [2, 5, 3, 0]])
    p_sc = torch.tensor([[0.5, 0.5, 0.25, 0.0], [1.0, 1.0, 0.0, 2.0], [0.0, 0.0, 7.0, 0.0], [-0.5, -1.0, -2.0, -2.0],
                         [3.0, 3.0, 3.0, 3.0], [0.125, 0.25, 0.375, -0.125]])
    return S, p_ids, p_sc, starts, lrows, row_ids


@pytest.mark.parametrize("k", [1, 4, 10, 200, 400])
def test_ivf_from_scores_matches_the_brute_force(k):
    S, p_ids, p_sc, starts, lrows, row_ids = _ivf_case()
    got = sr.ivf_from_scores(S, p_ids, p_sc, starts, lrows, row_ids, k)
    want = _brute_ivf(S, p_ids, p_sc, starts, lrows, row_ids, k)
    for g, w, what in zip(got, want, ("ids", "scores", "minmax")):
        sr.assert_bits(g, w, what)
    ids, sc, mm = got
    assert (ids[4] == -1).all() and torch.isneginf(sc[4]).all()                      # only an empty list probed
    sr.assert_bits(mm[4], _f32(float("inf"), float("-inf")))
    if k >= 4:                                                                       # position order across lists
        sr.assert_bits(ids[0, :1], row_ids[starts[3] * 128 + 128:starts[3] * 128 + 129])
    if k >= 200:
        assert (ids[1] >= 0).sum() == 129 and (ids[3] >= 0).sum() == 5 + 128 + 3 + 40   # list 3 once; no padding


@pytest.mark.parametrize("bug", ["id_ties", "pad", "tail", "mask"])
def test_comparator_rejects_mutants(bug):
    S, p_ids, p_sc, starts, lrows, row_ids = _ivf_case()
    k = 200
    got = sr.ivf_from_scores(S, p_ids, p_sc, starts, lrows, row_ids, k)
    bad = _brute_ivf(S, p_ids, p_sc, starts, lrows, row_ids, k, bug=bug)
    with pytest.raises(AssertionError):
        for g, w in zip(got, bad):
            sr.assert_bits(g, w)


def test_comparator_rejects_one_ulp():
    S, p_ids, p_sc, starts, lrows, row_ids = _ivf_case()
    ids, sc, mm = sr.ivf_from_scores(S, p_ids, p_sc, starts, lrows, row_ids, 10)
    off = sc.clone()
    off[5, 3] = float(np.nextafter(F32(off[5, 3]), F32(np.inf)))
    with pytest.raises(AssertionError):
        sr.assert_bits(off, sc)
    with pytest.raises(AssertionError):
        sr.assert_bits(_f32(-0.0), _f32(0.0))


def test_ivf_oracle_breaks_exact_ties_by_stored_position():
    """oracle/ivf_oracle.search and ivf_from_scores rank an exact cross-list tie alike: the smaller list wins, though
    its rows carry the larger original ids.  Dyadic values make every sum exact in fp32 and float64."""
    g = torch.Generator().manual_seed(3)
    d = 64
    base = (torch.randint(-3, 4, (6, d), generator=g).float() / 8).numpy()
    x = np.concatenate([base, base, base[:2] + F32(0.125)])       # rows 0-5 = rows 6-11
    cent = np.zeros((2, d), F32)
    assignment = np.array([1] * 6 + [0] * 6 + [1, 0])             # ids 6-11 in list 0, their twins 0-5 in list 1
    L = ivf.IVFLists(x, cent, assignment=assignment)
    q = (torch.randint(-3, 4, (3, d), generator=g).float() / 8).numpy()
    probed = (np.array([[0, 1], [1, 0], [1, 1]]), np.array([[0.5, 0.5], [0.5, 0.5], [0.25, 0.25]], F32))
    o_ids, o_sc, _ = ivf.search(L, q, 2, 14, probed=probed)
    res, row_ids, starts, counts = padded_layout(L)
    S = torch.from_numpy((q.astype(np.float64) @ res.astype(np.float64).T).astype(F32))
    ids, sc, _ = sr.ivf_from_scores(S, torch.from_numpy(probed[0]), torch.from_numpy(probed[1]),
                                    torch.from_numpy(starts), torch.from_numpy(counts), torch.from_numpy(row_ids), 14)
    sr.assert_bits(ids[:2], torch.from_numpy(o_ids[:2]))
    assert np.array_equal(sc[:2].double().numpy(), o_sc[:2])
    for r in range(2):                                            # every twin pair: list 0's row (id + 6) first
        for i in range(6):
            a, b = np.flatnonzero(o_ids[r] == i + 6), np.flatnonzero(o_ids[r] == i)
            assert a.size == b.size == 1 and a[0] < b[0]
    assert set(o_ids[2][o_ids[2] >= 0].tolist()) == {0, 1, 2, 3, 4, 5, 12}    # list 1 probed twice counts once


# -------------------------------------------------------------------------------------------------------- assign
def test_assign_from_scores_first_argmax():
    S = torch.stack([_f32(1.0, -2.0, -0.0, 5.0), _f32(1.0, -1.0, 0.0, 5.0), _f32(0.5, -1.0, 0.0, 6.0)])
    ids, best = sr.assign_from_scores(S)
    sr.assert_bits(ids, torch.tensor([0, 1, 0, 2], dtype=torch.int32))
    sr.assert_bits(best, _f32(1.0, -1.0, -0.0, 6.0))        # +0 does not beat -0 (the kernel compares floats)


# ------------------------------------------------------------------------------------------- score bound calibration
def scan_model(q, x, bug=None):
    """The scan's arithmetic: fp32 accumulation over 64-wide K-blocks, no output rounding.
    bug="bf16_acc": the accumulator is rounded to bf16 after every K-block; bug="drop_last": the last K-block is
    skipped."""
    qf, xf = q.float(), x.float()
    K = q.shape[1]
    acc = torch.zeros(q.shape[0], x.shape[0])
    last = K - 64 if bug == "drop_last" else K
    for k0 in range(0, last, 64):
        acc = acc + qf[:, k0:k0 + 64] @ xf[:, k0:k0 + 64].T
        if bug == "bf16_acc":
            acc = acc.bfloat16().float()
    return acc


@pytest.mark.parametrize("K", [64, 128, 384, 1024])
@pytest.mark.parametrize("kind", ["random", "scaled"])
def test_score_bound_is_calibrated(K, kind):
    """fp32 accumulation stays well under 2^-16 sum |q_i x_i|; a bf16 accumulator or a dropped last K-block
    exceeds it several times over.  Rows are gemm_inputs' A (scaled: row r times 2^(r % 17 - 8)), queries its W."""
    x, q, _, _ = gemm_inputs(300, 40, K, kind, seed=K + (kind == "scaled"))
    ref, mag = sr.score_reference(q, x)
    good = sr.err_over_bound(scan_model(q, x), ref, mag)
    acc = sr.err_over_bound(scan_model(q, x, "bf16_acc"), ref, mag)
    drop = sr.err_over_bound(scan_model(q, x, "drop_last"), ref, mag)
    assert good < 0.1, good
    assert acc > 4, acc
    assert drop > 4, drop
    assert math.isfinite(good)
