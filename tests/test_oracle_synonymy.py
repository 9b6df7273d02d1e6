"""The numpy walk of tests/synonymy_oracle.py against the synonymy-edge loop run directly over a retrieve_knn-shaped
dict {key: (neighbour keys, scores as Python floats)} built from the same fp32 self-join scores: the walk with the fp32
threshold, self row and '' exclusion must produce exactly the loop's assignments, in order.  Adversarial score
matrices: ties straddling the threshold and the list's end, scores exactly at the threshold, self and excluded rows
before, at and after the cut, more rows above the threshold than the list holds, more candidates than the cap, and
+-0.0 at threshold 0."""
import os
import re
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import synonymy_oracle as so  # noqa: E402


def _knn_dict(S, keys, k):
    return {keys[q]: ([keys[r] for r in so.rank_order(S[q], k)], S[q, so.rank_order(S[q], k)].tolist())
            for q in range(S.shape[0])}


def _walk_edges(S, keys, contents, t, k, cap):
    eligible = [q for q, key in enumerate(keys) if len(re.sub('[^A-Za-z0-9]', '', contents[key])) > 2]
    empty = [r for r, key in enumerate(keys) if contents[key] == '']
    counts, ids, sc = so.walk_all(S[eligible], so.fp32_threshold(t), k, cap, self_rows=eligible, exclude_rows=empty)
    return [((keys[q], keys[int(ids[i, j])]), float(sc[i, j])) for i, q in enumerate(eligible) for j in range(counts[i])]


def _contents(n, rng, empty_row=None, short_rows=()):
    c = [f"entity number {i}" for i in range(n)]
    for r in short_rows:
        c[r] = ["ab", "a-b", "!!", "x"][r % 4]
    if empty_row is not None:
        c[empty_row] = ''
    keys = [f"entity-{i:06d}" for i in range(n)]
    return keys, dict(zip(keys, c))


def _levels(n, levels, rng):
    return np.asarray(levels, dtype=np.float32)[rng.integers(0, len(levels), size=(n, n))]


CASES = {
    "random": lambda n, rng: rng.uniform(-1, 1, size=(n, n)).astype(np.float32),
    "ties_at_threshold": lambda n, rng: _levels(n, [0.9, 0.8, 0.8, np.nextafter(np.float32(0.8), 0)], rng),
    "many_above": lambda n, rng: rng.uniform(0.8, 1.0, size=(n, n)).astype(np.float32),
    "exactly_threshold": lambda n, rng: _levels(n, [np.float32(0.8), np.float32(0.7), so.fp32_threshold(0.7)], rng),
}


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("k,cap", [(2047, 101), (5, 101), (300, 3), (40, 2000)])
def test_walk_equals_the_loop_over_knn_lists(case, k, cap):
    rng = np.random.default_rng(1000 * sorted(CASES).index(case) + k + cap)
    n = 257
    S = CASES[case](n, rng)
    np.fill_diagonal(S, 1.0)                  # the self row first, as in a self-join of unit rows
    S[3, :] = S[5, :]                         # a row whose self score sits mid-list
    keys, contents = _contents(n, rng, empty_row=7, short_rows=(1, 2, 11))
    S[:, 7] = 0.95                            # the '' entity above the threshold for every query
    for t in (0.8, 0.7):
        want = so.edges_from_knn(_knn_dict(S, keys, k), contents, t, cap)
        got = _walk_edges(S, keys, contents, t, k, cap)
        assert got == want, (case, t)
        if case == "many_above" and k == 2047:
            assert sum(1 for (a, _), _ in got if a == keys[0]) == min(cap, n - 2)


def test_self_and_excluded_rows_before_at_and_after_the_cut():
    s = np.array([0.99, 0.9, 0.85, 0.8, 0.8, 0.79, 0.5], dtype=np.float32)
    t = so.fp32_threshold(0.8)
    assert so.walk(s, t, 10, 10)[0] == 5                                     # 0.8 is accepted
    for skip, want in ((0, [1, 2, 3, 4]), (3, [0, 1, 2, 4]), (4, [0, 1, 2, 3]), (5, [0, 1, 2, 3, 4])):
        count, ids, _ = so.walk(s, t, 10, 10, self_row=skip)
        assert ids[:count].tolist() == want
        count, ids, _ = so.walk(s, t, 10, 10, exclude_rows=[skip, skip])
        assert ids[:count].tolist() == want
    assert so.walk(s, t, 10, 2, self_row=0)[1].tolist() == [1, 2]            # the cap counts accepted rows only
    assert so.walk(s, t, 3, 10, self_row=0)[0] == 2                          # the list ends at `limit`
    assert so.walk(s, t, 10, 10, self_row=0, exclude_rows=[1, 2, 3, 4])[0] == 0


def test_ties_straddling_the_list_end_resolve_by_row():
    s = np.array([0.5, 0.9, 0.9, 0.9, 0.9, 0.9], dtype=np.float32)
    count, ids, _ = so.walk(s, so.fp32_threshold(0.8), 3, 10)
    assert ids[:count].tolist() == [1, 2, 3]


def test_signed_zero_at_threshold_zero():
    s = np.array([-0.0, 0.0, -1e-42, 1e-42, -0.0], dtype=np.float32)
    count, ids, sc = so.walk(s, np.float32(0.0), 10, 10)
    assert ids[:count].tolist() == [3, 1, 0, 4]                              # +0 ranks above -0, both pass >= 0
    assert np.signbit(sc[2]) and not np.signbit(sc[1])
    assert so.rank_order(s, 10).tolist() == [3, 1, 0, 4, 2]


def test_fp32_rounding_of_the_threshold():
    for t in (0.8, 0.7, 0.5, 1.0 / 3.0):
        f = so.fp32_threshold(t)
        assert float(f) >= t and float(np.nextafter(f, np.float32(-np.inf))) < t
    assert so.fp32_threshold(0.8) == np.float32(0.8)                          # float32(0.8) rounds up
    assert float(np.float32(0.7)) < 0.7 and so.fp32_threshold(0.7) == np.nextafter(np.float32(0.7), np.float32(1))
    below = np.float32(0.7)                                                    # just below the double 0.7
    assert not (float(below) >= 0.7) and not (below >= so.fp32_threshold(0.7))
    assert below >= np.float32(0.7)                                            # the naive conversion would accept it
    from comorag_b200.index import fp32_threshold
    for t in (0.8, 0.7, 0.5, 1.0 / 3.0, 0.0, -0.25):
        assert fp32_threshold(t) == float(so.fp32_threshold(t))
