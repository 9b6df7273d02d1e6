"""The merge rule of the row-sharded search, on the CPU: shard_cases.merge_reference against a brute-force sort of
(score word, part, position) tuples on hand-made records, the mutants its comparator must reject, the statement in
comorag_b200.dist (what test_dist_gloo.py merges with), and the shard layouts and corpora of test_shard_exact_gpu.py."""
import os
import struct
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import knn_cases as kc  # noqa: E402
import scan_reference as sr  # noqa: E402
import shard_cases as sc  # noqa: E402

INF = float("inf")


def _word(x: float) -> int:
    """orderable_f32 of one fp32 value, from its bits (no torch)."""
    u = struct.unpack("<I", struct.pack("<f", x))[0]
    return (~u) & 0xFFFFFFFF if u & 0x80000000 else u | 0x80000000


def brute_merge(ids, scores, minmax, k):
    """Sort every valid candidate by (score word descending, part, position); minmax by the score word."""
    parts, nq, _ = scores.shape
    out_i = torch.full((nq, k), -1, dtype=torch.int64)
    out_s = torch.full((nq, k), -INF, dtype=torch.float32)
    mm = torch.tensor([[INF, -INF]] * nq, dtype=torch.float32)
    for q in range(nq):
        cand = [(-_word(float(scores[p, q, j])), p, j) for p in range(parts) for j in range(k) if int(ids[p, q, j]) >= 0]
        for t, (_, p, j) in enumerate(sorted(cand)[:k]):
            out_i[q, t], out_s[q, t] = ids[p, q, j], scores[p, q, j]
        if parts:
            mm[q, 0] = min((float(minmax[p, q, 0]) for p in range(parts)), key=_word)
            mm[q, 1] = max((float(minmax[p, q, 1]) for p in range(parts)), key=_word)
    return out_i, out_s, mm


def hand_records():
    """8 parts, 5 queries, k = 4.
      q0  all absent (scores that are not -inf under id -1), every part's (min, max) (+inf, -inf)
      q1  +0 and -0 in different parts, -0 in the lower part: +0 must come first; a valid id with -inf
      q2  a tie at the k-th entry spread over all 8 parts: the lower parts win; ids >= 2^40 and not ascending by part
      q3  parts unsorted, the best candidate last in its part, and the 4th entry of every part the winner
      q4  one part holds everything valid, the others are empty with (+inf, -inf)"""
    parts, nq, k = 8, 5, 4
    ids = torch.full((parts, nq, k), -1, dtype=torch.int64)
    s = torch.full((parts, nq, k), 0.25, dtype=torch.float32)
    mm = torch.tensor([-1.0, 1.0]).repeat(parts, nq, 1)
    mm[:, 0] = torch.tensor([INF, -INF])
    # q1
    s[:, 1] = -5.0
    ids[:, 1] = torch.arange(parts * k).view(parts, k) + (1 << 40)
    s[2, 1, 0], s[5, 1, 3] = -0.0, 0.0
    s[0, 1, 1] = -INF
    s[6, 1, 2] = 7.0
    mm[:, 1] = torch.tensor([0.0, 0.0])
    mm[4, 1] = torch.tensor([-0.0, -0.0])
    # q2: 2 clear winners, then a tie of value 1.0 in every part
    ids[:, 2] = ((1 << 41) - torch.arange(parts * k)).view(parts, k)
    s[:, 2] = torch.tensor([1.0, 0.5, 0.5, 0.5])
    s[6, 2, 0], s[3, 2, 0] = 9.0, 8.0
    # q3
    ids[:, 3] = torch.arange(parts * k).view(parts, k) * 3 + 11
    s[:, 3] = torch.tensor([0.1, 0.2, 0.3, 2.0])
    s[7, 3, 3] = 2.5
    ids[1, 3, 3] = -1                     # absent, whatever its score
    mm[:, 3] = torch.tensor([-0.0, 0.0])
    # q4
    ids[5, 4] = torch.tensor([4, 3, 2, 1]) + (1 << 40)
    s[5, 4] = torch.tensor([-INF, 0.0, -0.0, -INF])
    mm[:, 4] = torch.tensor([INF, -INF])
    mm[5, 4] = torch.tensor([-INF, 0.0])
    return ids, s, mm, k


def cases():
    yield "hand", hand_records()
    for parts, nq, k, seed in [(8, 6, 4, 1), (3, 5, 7, 2), (1, 4, 3, 3), (0, 3, 2, 4), (16, 4, 5, 5)]:
        i, s, mm = sc.adversarial_records(parts, nq, k, seed)
        yield f"adv{parts}x{nq}x{k}", (i, s, mm, k)


@pytest.mark.parametrize("name,case", list(cases()), ids=[n for n, _ in cases()])
def test_merge_reference_equals_brute_force(name, case):
    ids, s, mm, k = case
    want = brute_merge(ids, s, mm, k)
    sc.assert_merge(sc.merge_reference(ids, s, mm, k), want, name)
    from comorag_b200.dist import merge_partials_reference
    sc.assert_merge(merge_partials_reference(ids, s, mm, k), want, f"{name} dist")


def test_hand_records_pin_the_edges():
    ids, s, mm, k = hand_records()
    oi, os_, om = sc.merge_reference(ids, s, mm, k)
    assert (oi[0] == -1).all() and torch.isneginf(os_[0]).all() and om[0].tolist() == [INF, -INF]
    assert oi[1].tolist() == [ids[6, 1, 2], ids[5, 1, 3], ids[2, 1, 0], ids[0, 1, 0]]   # 7, +0, -0, then -5 (part 0)
    assert struct.pack("<ff", *om[1].tolist()) == struct.pack("<ff", -0.0, 0.0)
    assert oi[2].tolist() == [ids[6, 2, 0], ids[3, 2, 0], ids[0, 2, 0], ids[1, 2, 0]]
    assert oi[3].tolist() == [ids[7, 3, 3], ids[0, 3, 3], ids[2, 3, 3], ids[3, 3, 3]]
    assert oi[4].tolist() == [ids[5, 4, 1], ids[5, 4, 2], ids[5, 4, 0], ids[5, 4, 3]]   # -inf with a valid id stays
    assert om[4].tolist() == [-INF, 0.0]


MUTANTS = {
    "ties by rank descending": dict(tie="rank_desc"),
    "ties by id": dict(tie="id"),
    "+0 and -0 ranked equal": dict(zero_equal=True),
    "each part's last entry dropped": dict(drop_last=True),
    "an empty part's (min, max) is (0, 0)": dict(empty_minmax=(0.0, 0.0)),
}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_comparator_rejects_mutant(mutant):
    ids, s, mm, k = hand_records()
    want = sc.merge_reference(ids, s, mm, k)
    got = sc.merge_reference(ids, s, mm, k, **MUTANTS[mutant])
    with pytest.raises(AssertionError):
        sc.assert_merge(got, want, mutant)


def test_old_statement_of_the_rule_is_rejected():
    """The argsort statement dist.merge_partials_reference had: a stable sort of the scores ranks -0 level with +0 and
    turns a valid id with score -inf into -1.  The kernels' rule differs on the hand records."""
    ids, s, mm, k = hand_records()
    world, nq, kk = s.shape
    flat_s = s.permute(1, 0, 2).reshape(nq, world * kk).clone()
    flat_i = ids.permute(1, 0, 2).reshape(nq, world * kk)
    flat_s[flat_i < 0] = -INF
    order = torch.argsort(flat_s, dim=1, descending=True, stable=True)[:, :k]
    old_s, old_i = flat_s.gather(1, order), flat_i.gather(1, order)
    old_i = torch.where(torch.isneginf(old_s), torch.full_like(old_i, -1), old_i)
    want_i, want_s, _ = sc.merge_reference(ids, s, mm, k)
    assert not torch.equal(old_i, want_i)


def test_virtual_group_is_a_pure_python_barrier():
    g = sc.VirtualGroup(3)
    assert [g.rank(r).rank for r in range(3)] == [0, 1, 2] and g.barrier.parties == 3


@pytest.mark.parametrize("world,k", [(3, 10), (5, 33), (8, 128), (16, 1)])
def test_edge_bounds(world, k):
    n = 3000
    for kind in ("even", "ragged", "small"):
        offs = sc.edge_bounds(n, world, kind, k)
        assert offs[0] == 0 and offs[-1] == n and len(offs) == world + 1
        assert all(a <= b for a, b in zip(offs, offs[1:]))
    ragged = sc.edge_bounds(n, world, "ragged", k)
    assert all(o % 128 for o in ragged[1:-1])
    small = sc.edge_bounds(n, world, "small", k)
    w = [b - a for a, b in zip(small, small[1:])]
    assert w[0] == 0 and w[-1] == 0 and (world < 4 or w[world // 2] == 0)
    if world >= 5:
        assert 1 in w and any(0 < x < k for x in w) or k == 1


@pytest.mark.parametrize("kind", ["boundary", "all_equal", "mixed"])
def test_planned_corpora_are_exact(kind):
    n, k, world = 1500, 33, 5
    offs = sc.edge_bounds(n, world, "ragged", k)
    x, s = sc.planned_corpus(kind, n, k, offs, seed=3)
    ref, mag = kc.exactness(x, kc.int_queries())
    assert mag < kc.EXACT_LIMIT and torch.equal(ref[0], s.double())
    q = sc.exact_queries(9, seed=4)
    assert {tuple(r) for r in kc.int_queries().view(torch.int16).tolist()} <= {tuple(r) for r in q.view(torch.int16).tolist()}
    _, mag = sr.score_reference(q[3:], x)                   # dyadic queries: 1/8 steps
    assert float(mag.max()) * 8 < kc.EXACT_LIMIT
    if kind == "boundary":
        top = torch.topk(s * n - torch.arange(n), k).indices           # ties by ascending row
        cut = [o for o in offs[1:-1] if o > 0 and o < n]
        assert any(bool((top < c).any() and (top >= c).any() and (s[top[-1]] == s[c - 1]) and s[c] == s[c - 1])
                   for c in cut)
