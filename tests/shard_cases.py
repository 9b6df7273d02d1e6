"""Cases and references for the row-sharded search (test infrastructure: CPU or CUDA tensors, seeded).

A row-sharded search ends with a merge of the ranks' answers: crag_merge_topk / crag_merge_topk_packed (the all-gather
formulation, ShardedIVF) or the merge step of finalize_exchange_kernel (the peer formulation).  All three rank the
parts' candidates by the same 64-bit key as the scan (topk.cuh), with the candidate's position in place of the row:

  key       orderable(score) << 32 | (0xFFFFFFFF - c), c = p * k + j for candidate j of part p, compared unsigned:
            score descending with +0 above -0, then part (rank) ascending, then position in the part ascending.
            A candidate is absent iff its id < 0; a valid id keeps its key whatever its score, -inf included.
  output    the first k keys: their ids and scores, -1 / -inf past the valid candidates.
  minmax    fminf / fmaxf over the parts' (min, max): +0 and -0 ordered as the keys order them (measured on H100,
            test_shard_exact_gpu.py); no part gives (+inf, -inf).

merge_reference states that rule from scan_reference's key construction.  VirtualGroup gives each virtual rank of one
GPU an all-gather with the shape of dist.all_gather_into_tensor, so SearchSession(gather=...), ShardedIndex and
ShardedIVF run their exchange between threads of one process.  The corpus builders place exact ties where shards
meet: knn_cases.int_rows scores are exact in fp32 under any summation order, so a tie is a tie on every rank."""
from __future__ import annotations

import os
import sys
import threading

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import knn_cases as kc  # noqa: E402
import scan_reference as sr  # noqa: E402

BIG_BASE = (1 << 33) + 7          # a global row offset beyond 2^33


# ------------------------------------------------------------------------------------------------------- merge rule
def _flat(ids: torch.Tensor, scores: torch.Tensor):
    """[parts, nq, k] -> candidates [nq, parts * k] in position order c = p * k + j."""
    parts, nq, k = scores.shape
    return (ids.permute(1, 0, 2).reshape(nq, parts * k).to(torch.int64),
            scores.permute(1, 0, 2).reshape(nq, parts * k).to(torch.float32))


def merge_minmax(minmax: torch.Tensor) -> torch.Tensor:
    """(min, max) over parts of minmax fp32 [parts, nq, 2], ordered as the keys order scores; (+inf, -inf) when
    there is no part."""
    parts, nq, _ = minmax.shape
    if parts == 0:
        return torch.tensor([float("inf"), float("-inf")], device=minmax.device).repeat(nq, 1)
    lo = minmax[..., 0].T.contiguous()
    hi = minmax[..., 1].T.contiguous()
    mn = lo.gather(1, sr.orderable(lo).argmin(dim=1, keepdim=True))[:, 0]
    mx = hi.gather(1, sr.orderable(hi).argmax(dim=1, keepdim=True))[:, 0]
    return torch.stack([mn, mx], dim=1)


def merge_reference(ids: torch.Tensor, scores: torch.Tensor, minmax: torch.Tensor, k: int, *, tie="position",
                    zero_equal=False, drop_last=False, empty_minmax=None):
    """The kernels' merge of per-part answers ids int64 / scores fp32 [parts, nq, k], minmax fp32 [parts, nq, 2]:
    (ids int64 [nq, k], scores fp32 [nq, k], minmax fp32 [nq, 2]).

    The keyword arguments build deliberately wrong rules (mutants) that the comparator must reject: tie="rank_desc"
    breaks ties by part descending, tie="id" by id ascending; zero_equal ranks -0 level with +0; drop_last ignores
    each part's last entry; empty_minmax gives a part without a valid id that (min, max)."""
    parts, nq, kk = scores.shape
    assert kk == k, "every part holds k entries"
    dev = scores.device
    out_i = torch.full((nq, k), -1, dtype=torch.int64, device=dev)
    out_s = torch.full((nq, k), float("-inf"), dtype=torch.float32, device=dev)
    mm = minmax.to(torch.float32)
    if empty_minmax is not None:
        empty = (ids < 0).all(dim=2)
        mm = torch.where(empty[..., None], torch.tensor(empty_minmax, dtype=torch.float32, device=dev), mm)
    if parts == 0:
        return out_i, out_s, merge_minmax(mm)
    i, s = _flat(ids, scores)
    n = parts * k
    c = torch.arange(n, device=dev, dtype=torch.int64)
    if tie == "rank_desc":
        c = (parts - 1 - c // k) * k + c % k
    if tie == "id":
        c = i.argsort(dim=1, stable=True).argsort(dim=1)
    rank = sr._rank(torch.where((s == 0) & zero_equal, torch.zeros_like(s), s), c.expand(nq, n))
    valid = i >= 0
    if drop_last:
        valid &= (torch.arange(n, device=dev) % k != k - 1)[None, :]
    top, col, present = sr._select(rank, valid, k)
    colc = col.clamp(max=n - 1)
    out_i = torch.where(present, i.gather(1, colc), out_i)
    out_s = torch.where(present, s.gather(1, colc), out_s)
    return out_i, out_s, merge_minmax(mm)


def assert_merge(got, want, what=""):
    """ids, scores and (min, max) bit for bit."""
    for g, w, name in zip(got, want, ("ids", "scores", "minmax")):
        sr.assert_bits(g, w, f"{what} {name}")


# ------------------------------------------------------------------------------------------------ merge records
def adversarial_records(parts: int, nq: int, k: int, seed: int, device="cpu"):
    """(ids int64, scores fp32 [parts, nq, k], minmax fp32 [parts, nq, 2]) built to stress the merge:
      * scores from a small pool, so exact ties run across parts, with +0 / -0, +-inf and one-ulp neighbours;
      * valid ids whose score is -inf, absent entries (id -1, a score that is not -inf), ids up to 2^41;
      * query 0 all absent; query 1 one tie value everywhere (the answer is positions 0 .. k - 1); query 2 a tie run
        that the k-th answer cuts across parts; parts sorted or not (the merge ranks every candidate);
      * (min, max) records with +0 / -0 and empty parts' (+inf, -inf)."""
    g = torch.Generator().manual_seed(seed)
    one = torch.tensor(1.0)
    pool = torch.tensor([float("-inf"), -2.5, -1.0, -0.0, 0.0, 0.5, 1.0, float(torch.nextafter(one, 2 * one)),
                         3.0, float("inf")])
    sc = pool[torch.randint(len(pool), (parts, nq, k), generator=g)]
    sc = torch.where(torch.rand(parts, nq, k, generator=g) < 0.3, torch.randn(parts, nq, k, generator=g), sc)
    ids = torch.randint(0, 1 << 41, (parts, nq, k), generator=g)
    ids[torch.rand(parts, nq, k, generator=g) < 0.15] = -1
    if nq > 0:
        ids[:, 0] = -1
    if nq > 1:
        sc[:, 1] = 0.75
        ids[:, 1] = torch.randint(0, 1 << 41, (parts, k), generator=g)
    if nq > 2 and parts > 0:
        sc[:, 2] = torch.where(torch.arange(k) < k // 2, 2.0, 1.25).expand(parts, k)
        ids[:, 2] = torch.randint(0, 1 << 41, (parts, k), generator=g)
    srt = torch.rand(parts, nq, generator=g) < 0.5          # about half the parts arrive sorted by key
    order = sr._rank(sc.reshape(-1, k), torch.arange(k).expand(parts * nq, k)).argsort(dim=1, descending=True)
    sorted_sc = sc.reshape(-1, k).gather(1, order).reshape(parts, nq, k)
    sorted_ids = ids.reshape(-1, k).gather(1, order).reshape(parts, nq, k)
    sc = torch.where(srt[..., None], sorted_sc, sc)
    ids = torch.where(srt[..., None], sorted_ids, ids)
    zeros = torch.tensor([[0.0, 0.0], [-0.0, -0.0], [-0.0, 0.0], [float("inf"), float("-inf")]])
    mm = torch.randn(parts, nq, 2, generator=g).sort(dim=2).values
    pick = torch.randint(0, 8, (parts, nq), generator=g)
    mm = torch.where((pick < 4)[..., None], zeros[pick.clamp(max=3)], mm)
    return ids.to(device), sc.to(device), mm.to(device)


# ---------------------------------------------------------------------------------------------- virtual all-gather
class VirtualGroup:
    """`world` virtual ranks of one process, one thread each: the process-group stand-in of the exchange tests."""

    def __init__(self, world: int, timeout: float = 120.0):
        self.world = world
        self.barrier = threading.Barrier(world, timeout=timeout)
        self.sent = [None] * world

    def rank(self, r: int) -> "VirtualRank":
        return VirtualRank(self, r)


class VirtualRank:
    """Rank r's handle on a VirtualGroup: what ShardedIndex / ShardedIVF hold as `group`."""

    def __init__(self, group: VirtualGroup, rank: int):
        self.group, self.rank = group, rank

    def gather(self, out: torch.Tensor, mine: torch.Tensor) -> None:
        """all_gather_into_tensor(out, mine): every rank's `mine`, in rank order, into `out`."""
        g = self.group
        torch.cuda.current_stream(mine.device).synchronize()      # this rank's record is complete ...
        g.sent[self.rank] = mine
        g.barrier.wait()                                          # ... and so is every other rank's
        n = mine.numel()
        assert out.numel() == g.world * n, (out.numel(), g.world, n)
        for r, m in enumerate(g.sent):
            assert m.numel() == n
            out[r * n:(r + 1) * n].copy_(m)
        torch.cuda.current_stream(out.device).synchronize()
        g.barrier.wait()                 # no rank overwrites its record before every rank has copied it


def virtual_all_gather(out, mine, group=None, async_op=False):
    """dist.all_gather_into_tensor for a VirtualRank group (install with monkeypatch)."""
    assert isinstance(group, VirtualRank) and not async_op
    group.gather(out, mine)


def run_ranks(world: int, fn, device, timeout: float = 300.0):
    """fn(r) on `world` threads at once, each on its own stream of `device`; returns [fn(0), ..., fn(world - 1)] once
    every stream has drained."""
    results, errors = [None] * world, [None] * world
    streams = [torch.cuda.Stream(device) for _ in range(world)]
    torch.cuda.synchronize(device)          # inputs the caller made on its own stream are complete

    def body(r):
        try:
            with torch.cuda.device(device), torch.cuda.stream(streams[r]):
                results[r] = fn(r)
                streams[r].synchronize()
        except BaseException as e:          # noqa: BLE001 -- re-raised in the caller's thread
            errors[r] = e
    threads = [threading.Thread(target=body, args=(r,), daemon=True) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout)
    assert not any(t.is_alive() for t in threads), "a virtual rank did not finish"
    for e in errors:
        if e is not None and not isinstance(e, threading.BrokenBarrierError):
            raise e
    for e in errors:
        if e is not None:
            raise e
    return results


def virtual_sharded_index(local, rank: VirtualRank, peer=None):
    """The ShardedIndex of virtual rank `rank` over its DenseIndex `local`, with the attributes __init__ sets:
    "peer" formulation when `peer` (a PeerExchange.from_local_buffers) is given, else the all-gather one."""
    from comorag_b200.dist import ShardedIndex
    s = ShardedIndex.__new__(ShardedIndex)
    s.local, s.group = local, rank
    s.world, s.rank = rank.group.world, rank.rank
    s.peer = peer
    s.exchange_mode = "peer" if peer is not None else "nccl"
    s._sessions = {}
    s._lock = threading.RLock()
    return s


def virtual_sharded_ivf(local, rank: VirtualRank):
    """The ShardedIVF of virtual rank `rank` over its IVFIndex / QuantizedIVF `local`."""
    from comorag_b200.ivf import ShardedIVF
    s = ShardedIVF.__new__(ShardedIVF)
    s.local, s.group, s.world = local, rank, rank.group.world
    return s


# --------------------------------------------------------------------------------------------------- shard layouts
def edge_bounds(n: int, world: int, kind: str, k: int = 1):
    """Row bounds offs[0 .. world] of a contiguous split of n rows:
      even        dist.shard_bounds
      ragged      cuts away from multiples of 128 (n >= 2 world)
      small       shards of fewer than k rows, a 1-row shard, and empty shards first, in the middle and last
                  (world >= 3; the rest of the rows on the second rank)"""
    from comorag_b200.dist import shard_bounds
    if kind == "even":
        return shard_bounds(n, world)
    if kind == "ragged":
        offs = shard_bounds(n, world)
        for r in range(1, world):
            if offs[r] % 128 == 0 and offs[r] + 1 < offs[r + 1]:
                offs[r] += 1
        return offs
    assert kind == "small" and world >= 3
    sizes = [0] * world
    rest = n
    for r in range(2, world - 1):
        sizes[r] = 0 if r == world // 2 else min(rest, 1 if r % 2 else max(k - 1, 1))
        rest -= sizes[r]
    sizes[1] = rest
    offs = [0]
    for s in sizes:
        offs.append(offs[-1] + s)
    return offs


# -------------------------------------------------------------------------------------------------------- corpora
def planned_corpus(kind: str, n: int, k: int, offs, seed: int):
    """(rows bf16 [n, INT_DIM], planned int64 scores [n] against knn_cases.int_queries()[0]):
      boundary    a run of equal scores across the boundary of the largest shard, with k // 2 rows above it, so the
                  k-th answer cuts the run, part on one rank and part on the next; copies of one row on both sides
      all_equal   every row identical: the answer is global rows 0 .. k - 1, in rank order
      mixed       random integers from a small range: ties everywhere"""
    g = torch.Generator().manual_seed(seed)
    if kind == "all_equal":
        s = torch.full((n,), 12345, dtype=torch.int64)
        return kc.int_rows(s, seed, identical_noise=True), s
    s = torch.randint(-5000, 5000, (n,), generator=g)
    if kind == "mixed":
        s = torch.randint(-40, 41, (n,), generator=g) * 1000
        return kc.int_rows(s, seed), s
    assert kind == "boundary"
    widths = [offs[r + 1] - offs[r] for r in range(len(offs) - 1)]
    r = max(range(len(widths)), key=lambda i: widths[i])
    cut = offs[r + 1] if r + 1 < len(offs) - 1 else offs[r]        # a boundary with rows on both sides
    run = torch.arange(max(cut - max(k // 4, 1), 0), min(cut + k, n))
    s[run] = 700_000
    above = torch.randperm(n, generator=g)
    above = above[~torch.isin(above, run)][: k // 2]
    s[above] = 800_000 + torch.arange(above.numel())
    x = kc.int_rows(s, seed)
    if 0 < cut < n:
        x[cut] = x[cut - 1]                                          # one row copied across the boundary
        s[cut] = s[cut - 1]
    return x, s


def exact_queries(nq: int, seed: int) -> torch.Tensor:
    """bf16 [nq, INT_DIM]: knn_cases.int_queries (scales 1, 2^-12, -2^6) in a seeded order, then dyadic rows (entries
    in {-3/8 .. 3/8}).  Against int_rows corpora every score is exact in fp32 under any summation order."""
    g = torch.Generator().manual_seed(seed)
    base = kc.int_queries()
    base = base[torch.randperm(base.shape[0], generator=g)]
    dy = (torch.randint(-3, 4, (max(nq - base.shape[0], 0), kc.INT_DIM), generator=g).float() / 8).bfloat16()
    return torch.cat([base, dy])[:nq]
