"""Row-sharded index across the GPUs of one box: one process per GPU (torch.distributed), each rank scans
its own shard with the fused kernel; the per-rank (ids, scores, min/max) records then reach every rank either by
the fused finalize + exchange + merge kernel over NVLink peer memory (PeerExchange, the default under NCCL) or by ONE
all_gather_into_tensor of the packed records + a merge kernel (the formulation north_star names) -- either way every
rank ends with the global top-k (SURVEY.md section 8e).

Rank r owns global rows [offsets[r], offsets[r+1]); ids written by the shard kernel are already global.
The reference has no distributed code (SURVEY.md 2a) -- this is the exchange step the shard layout adds.
"""
from __future__ import annotations

import os
import threading
from typing import List, Optional, Tuple

import torch
import torch.distributed as dist


def shard_bounds(n_rows: int, world: int) -> List[int]:
    """Contiguous, near-equal row blocks: offsets[r] .. offsets[r+1] for rank r (first n % world ranks get one more)."""
    base, rem = divmod(int(n_rows), int(world))
    offs = [0]
    for r in range(world):
        offs.append(offs[-1] + base + (1 if r < rem else 0))
    return offs


def pack_partial(ids: torch.Tensor, scores: torch.Tensor, minmax: torch.Tensor) -> torch.Tensor:
    """(int64 [nq,k], fp32 [nq,k], fp32 [nq,2]) -> one contiguous uint8 buffer (a single collective payload)."""
    from .index import packed_record_bytes, packed_views
    nq, k = ids.shape
    buf = torch.zeros(packed_record_bytes(nq, k), dtype=torch.uint8, device=ids.device)
    v_ids, v_scores, v_mm = packed_views(buf, nq, k)
    v_ids.copy_(ids)
    v_scores.copy_(scores)
    v_mm.copy_(minmax)
    return buf


def unpack_partials(buf: torch.Tensor, world: int, nq: int, k: int) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """[world * bytes] uint8 -> ids int64 [world,nq,k], scores fp32 [world,nq,k], minmax fp32 [world,nq,2]."""
    from .index import packed_record_bytes
    per = packed_record_bytes(nq, k)
    b = buf.view(world, per)
    a, c = nq * k * 8, nq * k * 8 + nq * k * 4
    ids = b[:, :a].contiguous().view(torch.int64).view(world, nq, k)
    scores = b[:, a:c].contiguous().view(torch.float32).view(world, nq, k)
    minmax = b[:, c:c + nq * 8].contiguous().view(torch.float32).view(world, nq, 2)
    return ids, scores, minmax


def _orderable(x: torch.Tensor) -> torch.Tensor:
    """The kernels' orderable_f32 of fp32 values, as int64 in [0, 2^32): unsigned order = score order, +0 above -0."""
    u = x.contiguous().to(torch.float32).view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    return torch.where(u >= (1 << 31), (~u) & 0xFFFFFFFF, u | (1 << 31))


def merge_partials_reference(ids: torch.Tensor, scores: torch.Tensor, minmax: torch.Tensor, k: int):
    """Plain-torch statement of the merge rule of crag_merge_topk (used by the CPU/gloo tests of the exchange step;
    the product path runs the kernel on the device).  Candidate j of rank p sits at position c = p * k + j and ranks
    by the kernels' key orderable(score) << 32 | (0xFFFFFFFF - c): score descending with +0 above -0, then rank, then
    position.  A candidate is absent iff its id < 0; a valid id with score -inf is kept.  -1 / -inf past the valid
    candidates; (min, max) over the ranks in the same score order, (+inf, -inf) from no rank."""
    world, nq, kk = scores.shape
    n = world * kk
    s = scores.permute(1, 0, 2).reshape(nq, n).to(torch.float32)
    i = ids.permute(1, 0, 2).reshape(nq, n).to(torch.int64)
    c = torch.arange(n, device=s.device, dtype=torch.int64)
    key = (_orderable(s) - (1 << 31)) * (1 << 32) + (0xFFFFFFFF - c)      # the unsigned key, shifted into int64
    key = torch.where(i >= 0, key, torch.full_like(key, -(1 << 63)))
    top, col = torch.sort(key, dim=1, descending=True)
    top, col = top[:, :k], col[:, :k]
    present = top != -(1 << 63)
    out_i = torch.full((nq, k), -1, dtype=torch.int64, device=s.device)
    out_s = torch.full((nq, k), float("-inf"), dtype=torch.float32, device=s.device)
    m = col.shape[1]
    out_i[:, :m] = torch.where(present, i.gather(1, col), out_i[:, :m])
    out_s[:, :m] = torch.where(present, s.gather(1, col), out_s[:, :m])
    mm = torch.tensor([float("inf"), float("-inf")], device=s.device).repeat(nq, 1)
    if world:
        lo, hi = minmax[..., 0].to(torch.float32), minmax[..., 1].to(torch.float32)
        mm[:, 0] = lo.gather(0, _orderable(lo).argmin(dim=0, keepdim=True))[0]
        mm[:, 1] = hi.gather(0, _orderable(hi).argmax(dim=0, keepdim=True))[0]
    return out_i, out_s, mm


class PeerExchange:
    """Symmetric exchange buffers for crag_search_finalize_exchange: one buffer per rank, every buffer mapped into
    every process (torch.distributed._symmetric_memory: cuMem allocations whose handles are swapped through the
    process group's store), so a kernel on rank r can store straight into rank d's buffer over NVLink.

    `peer_ptrs` is the device address of the [world] pointer table.  `from_local_buffers` builds the same object
    out of ordinary tensors of ONE process (several "virtual ranks" on one GPU, used by the single-GPU protocol test)."""

    def __init__(self, group: Optional[dist.ProcessGroup], device: torch.device):
        import torch.distributed._symmetric_memory as symm
        from . import _native
        lib = _native.load()
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        nbytes = int(lib.crag_exchange_buffer_bytes(self.world))
        if nbytes == 0:
            raise ValueError(f"world size {self.world} is not supported by the peer exchange (max 16)")
        self.buf = symm.empty(nbytes, dtype=torch.uint8, device=device)
        self.buf.zero_()
        self.handle = symm.rendezvous(self.buf, group if group is not None else dist.group.WORLD)
        self.peer_ptrs = int(self.handle.buffer_ptrs_dev)
        self.epochs = torch.zeros(32, dtype=torch.int64, device=device)
        self.status = torch.zeros(1, dtype=torch.int32, device=device)
        torch.cuda.synchronize(device)
        dist.barrier(group)          # every buffer is zeroed before any rank pushes into it

    @classmethod
    def from_local_buffers(cls, bufs: List[torch.Tensor], rank: int) -> "PeerExchange":
        self = cls.__new__(cls)
        self.world, self.rank = len(bufs), rank
        self.buf = bufs[rank]
        self._table = torch.tensor([b.data_ptr() for b in bufs], dtype=torch.int64, device=bufs[0].device)
        self.peer_ptrs = self._table.data_ptr()
        self.epochs = torch.zeros(32, dtype=torch.int64, device=bufs[0].device)
        self.status = torch.zeros(1, dtype=torch.int32, device=bufs[0].device)
        return self

    def check(self) -> None:
        if int(self.status.item()) != 0:
            raise RuntimeError("peer exchange: a rank's record did not arrive within 4 s (see crag_search_finalize_exchange)")


class ShardedIndex:
    """One rank's handle on a row-sharded index (world size 1 degenerates to the local DenseIndex)."""

    def __init__(self, local_index, group: Optional[dist.ProcessGroup] = None, exchange: str = "auto"):
        """exchange: "peer" = fused finalize + exchange + merge kernel over symmetric memory, "nccl" = one
        all_gather_into_tensor + merge kernel (the formulation north_star names), "auto" = peer when the symmetric
        memory rendezvous works on this box, else nccl.  Both give every rank the same global answer."""
        self.local = local_index
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.peer: Optional[PeerExchange] = None
        self.exchange_mode = "none" if self.world == 1 else "nccl"
        mode = os.environ.get("CRAG_EXCHANGE", exchange)
        if self.world > 1 and mode in ("auto", "peer") and dist.get_backend(group) == "nccl":
            ok = torch.zeros(1, dtype=torch.int32, device=local_index.device)
            try:
                self.peer = PeerExchange(group, local_index.device)
                ok += 1
            except Exception as e:   # no P2P / fabric handles on this box: say so and use the NCCL formulation
                if mode == "peer":
                    raise
                import logging
                logging.getLogger(__name__).warning("peer exchange unavailable (%r); using the NCCL all-gather", e)
            dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)   # all ranks or none
            if int(ok.item()) == 1:
                self.exchange_mode = "peer"
            else:
                self.peer = None
        self._sessions = {}
        self._lock = threading.RLock()      # sessions own static buffers: one search at a time per ShardedIndex

    def session(self, nq: int, k: int, use_graph: bool = True):
        """Reusable CUDA-graph-captured step for (nq <= 32, k <= 128): scan + fused finalize/exchange/merge (peer
        mode) or scan + finalize + all-gather + merge (nccl mode).  A collective: build and run on all ranks alike."""
        from .index import SearchSession
        key = (nq, k, use_graph)
        s = self._sessions.get(key)
        if s is None or s.stale():
            if self.world == 1:
                s = SearchSession(self.local, nq, k, use_graph=use_graph)
            elif self.peer is not None:
                s = SearchSession(self.local, nq, k, exchange=self.peer, world=self.world, use_graph=use_graph)
            else:
                # NCCL formulation: launched kernel by kernel.  (Capturing the all-gather in a CUDA graph works, but
                # tearing the process group down while such graphs are alive hung until NCCL's watchdog fired --
                # measured in round 2 -- so the graph is reserved for the peer-memory formulation.)
                s = SearchSession(self.local, nq, k, world=self.world, use_graph=False,
                                  gather=lambda out, mine: dist.all_gather_into_tensor(out, mine, group=self.group))
            self._sessions[key] = s
        return s

    def search_device(self, queries_bf16: torch.Tensor, k: int, use_graph: bool = True):
        """Every rank passes the SAME query block; every rank returns the same global (ids, scores, minmax).

        Per block of 32 queries: scan kernel + fused finalize/exchange/merge kernel (peer mode), or scan + finalize +
        ONE all_gather_into_tensor + merge kernel (nccl mode); each block runs as a captured CUDA graph over the
        session's static buffers.  k <= 128 (the single-GPU rank continuation is shard-local)."""
        if self.world == 1:
            return self.local.search_device(queries_bf16, k)
        if k > 128:
            raise ValueError("ShardedIndex.search_device supports k <= 128 (rank continuation is per shard); "
                             "merge several shards' paged results on the host for larger k")
        nq = queries_bf16.shape[0]
        outs = []
        with self._lock:
            for q0 in range(0, nq, 32):
                blk = queries_bf16[q0:q0 + 32]
                sess = self.session(blk.shape[0], k, use_graph)
                res = sess.run(blk)
                outs.append(res if nq <= 32 else tuple(t.clone() for t in res))
        if len(outs) == 1:
            return outs[0]
        return tuple(torch.cat([o[i] for o in outs], 0) for i in range(3))

    def close(self) -> None:
        """Drop the captured sessions (call before dist.destroy_process_group())."""
        with self._lock:
            self._sessions.clear()

    def search(self, queries, k: int):
        """Host-buffer entry point on every rank: numpy / torch queries [nq, dim] in, numpy (ids, scores, minmax) out."""
        q = self.local.prepare_queries(queries)
        ids, scores, mm = self.search_device(q, k)
        ids_h = ids.cpu().numpy()
        if self.peer is not None and ids_h.size and (ids_h[:, 0] < 0).any():
            self.peer.check()        # the exchange kernel answers an all-empty row when a peer's record never arrived
        return ids_h, scores.cpu().numpy(), mm.cpu().numpy()


def pair_bounds(n_pairs: int, world: int) -> List[int]:
    """Rank r reranks pairs [b[r], b[r+1]): contiguous, near-equal (same rule as shard_bounds)."""
    return shard_bounds(n_pairs, world)


def sharded_rerank(score_fn, token_lists, group: Optional[dist.ProcessGroup] = None, device=None,
                   n_labels: Optional[int] = None) -> torch.Tensor:
    """BASELINE config 5 across the GPUs of one box: after the row-sharded search every rank holds the SAME global
    candidate list, so the (query, passage) pairs are split by rank (no data-path collective for the scoring),
    each rank runs its slice through `score_fn(list of token lists) -> float32 [m, n_labels]` (the cross-encoder,
    CrossEncoderReranker.score_token_lists) and ONE all-gather of the logits gives every rank all of them.

    Returns float32 [n_pairs, n_labels] on `device` (default: where the local logits live), pair order preserved."""
    n = len(token_lists)
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    b = pair_bounds(n, world)
    mine = torch.as_tensor(score_fn(token_lists[b[rank]:b[rank + 1]]), dtype=torch.float32)
    if mine.dim() == 1:
        mine = mine[:, None]
    if device is not None:
        mine = mine.to(device)
    if world == 1:
        return mine
    # a rank with an empty slice (fewer pairs than ranks) cannot know the label count from its own (0, ?) output:
    # agree on it (max over ranks) before sizing the collective
    lab = torch.tensor([n_labels if n_labels is not None else (mine.shape[1] if mine.shape[0] else 0)],
                       dtype=torch.int64, device=mine.device)
    dist.all_reduce(lab, op=dist.ReduceOp.MAX, group=group)
    labels = max(int(lab.item()), 1)
    if mine.shape[0] == 0:
        mine = mine.new_zeros((0, labels))
    per = b[1] - b[0]                      # the largest slice (the first n % world ranks hold one more pair)
    send = torch.zeros((per, labels), dtype=torch.float32, device=mine.device)
    send[: mine.shape[0]] = mine
    gathered = torch.empty((world * per, labels), dtype=torch.float32, device=mine.device)
    dist.all_gather_into_tensor(gathered, send, group=group)
    parts = [gathered[r * per: r * per + (b[r + 1] - b[r])] for r in range(world)]
    return torch.cat(parts, 0)
