"""CPU checks of tests/knn_cases.py, the case builders of tests/test_knn_exact_gpu.py.

An exact GPU comparison only proves what its cases reach.  So every integer case must really be exact (float64
scores equal to their fp32 values, sum |q_i x_i| below 2^24 at every query scale), must land in the regime of
csrc/knn_select.cuh it is named for (the radix pass that decides the k-th row, the tie quota, the gather iterations
the tie run spans), and the exact reference must give a different answer from the wrong selectors the case targets:
a gather that keeps the last ties, and a select that ignores the trailing rows of a partial float4."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import knn_cases as kc  # noqa: E402
import scan_reference as sr  # noqa: E402


@pytest.fixture(scope="module", params=sorted(kc.INT_CASES))
def case(request):
    name = request.param
    rows, q, S, k, s = kc.int_case(name)
    return name, rows, q, S, k, s


def test_integer_case_is_exact(case):
    name, rows, q, S, k, s = case
    ref, worst = kc.exactness(rows, q)
    assert worst < kc.EXACT_LIMIT, f"{name}: sum |q_i x_i| = {worst} reaches 2^24"
    assert torch.equal(ref, S), f"{name}: the rows do not encode the planned scores"
    assert torch.equal(S.float().double(), S), f"{name}: a score is not an fp32 value"
    assert torch.equal(S[0], s.double()), name
    assert not bool(torch.signbit(S[S == 0]).any()), f"{name}: an exact zero must be +0"


def test_integer_case_lands_in_its_regime(case):
    name, rows, q, S, k, s = case
    want, _ = kc.INT_CASES[name]
    for j in range(S.shape[0]):                # the query scales are powers of two: the regime is the same at each
        if kc.QUERY_SCALES[j] < 0:
            continue
        r = kc.regime(S[j].float(), k)
        assert r["take_all"] == want.get("take_all", False), (name, j)
        if r["take_all"]:
            continue
        for key in ("pass", "ordered_ties"):
            if key in want:
                assert r[key] == want[key], (name, j, key, r[key])
        assert 1 <= r["quota"] <= r["n_eq"] and r["quota"] <= k
        if want.get("long"):                   # a run of hundreds to thousands, the quota met mid-iteration
            assert r["n_eq"] >= 900 and r["quota"] < r["n_eq"] // 2, (name, r["quota"], r["n_eq"])
            assert r["iters_to_quota"] >= 3, (name, r["iters_to_quota"])
            assert 0 < r["quota_pos"] < kc.GATHER_ROWS - 1 and r["ties_after_in_iter"] >= 1, (name, r["quota_pos"])
            assert r["tie_iters"][-1] > r["quota_iter"]
        if want.get("all_negative"):
            assert bool((S[j] < 0).all())
        if "first_tie_row" in want:
            assert int(r["tie_rows"][0]) == 0 and r["quota_row"] < int(r["tie_rows"][-1])
        if "last_tie_row" in want:
            assert int(r["tie_rows"][-1]) == r["n"] - 1 and r["quota_row"] == r["n"] - 1 and r["n"] % 4 != 0
            assert r["T_score"] == 0.0        # the dead lanes of the last float4 read as 0.0 = T
        if want.get("n_eq") == "n":
            assert r["n_eq"] == r["n"] and r["quota"] == k
        if "dup_stride" in want:
            d = want["dup_stride"]
            assert torch.equal(rows[d:], rows[:-d]), name
            assert len(r["tie_iters"]) >= 3 and r["quota_iter"] > 0
    assert S.shape[1] % 4 != 0 or name == "take_all", "every case leaves a partial float4"


def _differs(a, b):
    return any(not torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x,
                               y.view(torch.int32) if y.dtype == torch.float32 else y) for x, y in zip(a, b))


def test_reference_rejects_the_wrong_selectors(case):
    name, rows, q, S, k, s = case
    _, catches = kc.INT_CASES[name]
    ids, sc, mm, _ = sr.topk_from_scores(S.float(), k, row_offset=(1 << 33) + 7)
    last = kc.topk_keep_last_ties(S.float(), k, row_offset=(1 << 33) + 7)
    trail = kc.topk_drop_trailing(S.float(), k, row_offset=(1 << 33) + 7)
    if "last_ties" in catches:
        assert _differs((ids[0], sc[0]), (last[0][0], last[1][0])), name
    else:                                      # no tie decision at the positive scales: the two gathers agree
        assert _differs((ids[:2], sc[:2]), (last[0][:2], last[1][:2])) is False, name
    if "trailing_row" in catches:
        assert _differs((ids[0], sc[0], mm[0]), (trail[0][0], trail[1][0], trail[2][0])), name


def test_wrong_selectors_are_only_wrong_where_they_claim():
    """On a shard with distinct scores and n % 4 == 0 both wrong selectors give the reference's answer."""
    g = torch.Generator().manual_seed(3)
    S = torch.randn(3, 4096, generator=g)
    ids, sc, mm, _ = sr.topk_from_scores(S, 129)
    last = kc.topk_keep_last_ties(S, 129)
    trail = kc.topk_drop_trailing(S, 129)
    assert torch.equal(last[0], ids) and torch.equal(last[1], sc)
    assert torch.equal(trail[0], ids) and torch.equal(trail[1], sc) and torch.equal(trail[2], mm)


def test_regime_digits_and_gather_iterations():
    """regime() on hand-made rows: the deciding digit of one-ulp, one-middle-digit and one-exponent gaps, and the
    iterations of a tie run planted at rows 10, 2 050, 4 100 and 6 200."""
    one = torch.tensor([1.0], dtype=torch.float32)
    up = torch.nextafter(one, torch.tensor([2.0]))
    assert kc.regime(torch.cat([up, one]), 1)["pass"] == 2
    assert kc.regime(torch.tensor([1.5, 1.0]), 1)["pass"] == 0          # mantissa bit 22 is in the top digit
    assert kc.regime(torch.tensor([1.0 + 2 ** -12, 1.0]), 1)["pass"] == 1
    assert kc.regime(torch.tensor([2.0, 1.0]), 1)["pass"] == 0
    s = torch.zeros(8000)
    s[[10, 2050, 4100, 6200]] = 1.0
    r = kc.regime(s, 3)
    assert r["pass"] == "tie" and r["quota"] == 3 and r["n_eq"] == 4 and r["ordered_ties"]
    assert r["tie_iters"] == [0, 1, 2, 3] and r["iters_to_quota"] == 3
    assert (r["quota_row"], r["quota_iter"], r["quota_pos"], r["ties_after_in_iter"]) == (4100, 2, 4, 0)
    assert kc.regime(s, 8000)["take_all"]
