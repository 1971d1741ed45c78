"""Row-sharded corpus across the GPUs of one box: one process per GPU, each scans its shard, then a
SINGLE all-gather of the per-shard hit lists (NCCL over NVLink) and a local merge on every rank.

The reference has no distributed path (SURVEY.md section 2.1); this is the H100-native equivalent of
"one big chunk_embedding table": chunks are partitioned into contiguous ranges (never splitting a
chunk's vectors), queries are replicated, and ``GROUP BY chunk / ORDER BY / LIMIT`` (_search.py:143-150)
runs over the gathered top-``num_hits`` vectors, which is exactly what a single table would produce.
"""

from __future__ import annotations

from typing import Any

import torch
import torch.distributed as dist

from ._index import CorpusIndex, ScanResult, limit_hits_to_nearest, merge_hits, merge_packed


def pack_hits(hit_sim: torch.Tensor, hit_chunk: torch.Tensor, hit_count: torch.Tensor,
              status: torch.Tensor | None = None) -> torch.Tensor:
    """One contiguous byte buffer per rank: chunk ids (int64) | sims (float32) | counts (int32) [| status (int32)].
    The status words ride along so that every rank learns of an overflow on any shard from the one
    collective of the path."""
    parts = [hit_chunk.contiguous().view(torch.uint8).reshape(-1), hit_sim.contiguous().view(torch.uint8).reshape(-1),
             hit_count.contiguous().view(torch.uint8).reshape(-1)]
    if status is not None:
        parts.append(status.to(torch.int32).contiguous().view(torch.uint8).reshape(-1))
    return torch.cat(parts)


def unpack_hits(buf: torch.Tensor, R: int, B: int, H: int, with_status: bool = False
                ) -> tuple[torch.Tensor, ...]:
    """Inverse of :func:`pack_hits` for ``R`` concatenated rank buffers -> ``[R, B, H]`` views."""
    per = B * H * 12 + B * 4 + (B * 4 if with_status else 0)
    buf = buf.reshape(R, per)
    n8, n4 = B * H * 8, B * H * 4
    chunk = buf[:, :n8].contiguous().view(torch.int64).reshape(R, B, H)
    sim = buf[:, n8:n8 + n4].contiguous().view(torch.float32).reshape(R, B, H)
    count = buf[:, n8 + n4:n8 + n4 + B * 4].contiguous().view(torch.int32).reshape(R, B)
    if not with_status:
        return sim, chunk, count
    status = buf[:, n8 + n4 + B * 4:].contiguous().view(torch.int32).reshape(R, B)
    return sim, chunk, count, status


def gather_hits(hit_sim: torch.Tensor, hit_chunk: torch.Tensor, hit_count: torch.Tensor, group: Any | None,
                status: torch.Tensor | None = None) -> tuple[torch.Tensor, ...]:
    """The single collective of the path: all-gather every rank's packed hit list (and status words)."""
    B, H = int(hit_sim.shape[0]), int(hit_sim.shape[1])
    if group is None or dist.get_world_size(group) == 1:
        out = (hit_sim[None], hit_chunk[None], hit_count[None])
        return out if status is None else (*out, status[None])
    R = dist.get_world_size(group)
    mine = pack_hits(hit_sim, hit_chunk, hit_count, status)
    out = torch.empty(R * mine.numel(), dtype=torch.uint8, device=mine.device)
    dist.all_gather_into_tensor(out, mine, group=group)
    return unpack_hits(out, R, B, H, with_status=status is not None)


def shard_ranges(chunk_off: Any, world: int) -> list[tuple[int, int]]:
    """Contiguous chunk ranges with (nearly) equal vector counts; a chunk is never split."""
    import numpy as np

    chunk_off = np.asarray(chunk_off, dtype=np.int64)
    n_chunks = len(chunk_off) - 1
    total = int(chunk_off[-1])
    cuts = [0]
    for r in range(1, world):
        target = total * r // world
        c = int(np.searchsorted(chunk_off, target, side="left"))
        cuts.append(min(max(c, cuts[-1]), n_chunks))
    cuts.append(n_chunks)
    return [(cuts[i], cuts[i + 1]) for i in range(world)]


CHUNK_STRIDE = 1 << 40   # default spacing of the shards' global chunk ranges (see ShardedIndex)


class ShardedIndex:
    """A ``CorpusIndex`` shard plus the process group it is one part of.

    Global chunk indices: shard ``r`` owns ``[chunk_base_r, chunk_base_r + n_chunks_r)``; the ranges of the
    shards must never overlap, because ``rl_topk_merge`` groups by that index.  A shard can therefore only
    grow (``CorpusIndex.append``, the flushes of ``insert_documents``) while it stays below the next
    shard's base: build the shards with spaced bases (``chunk_base = rank * CHUNK_STRIDE``, what
    ``shard_bases`` returns) if they are to follow inserts; contiguous bases (``rank * chunks_per_shard``)
    are fine for a static corpus and make ``append`` on any shard but the last raise."""

    def __init__(self, local: CorpusIndex, group: Any | None = None, chunk_ids: list[str] | None = None):
        self.local = local
        self.group = group
        self.world = dist.get_world_size(group) if group is not None else 1
        self.rank = dist.get_rank(group) if group is not None else 0
        self.global_chunk_ids = chunk_ids     # legacy: one list over a contiguous global numbering
        self.shard_chunk_ids: list[list[str] | None] | None = None
        self.last_status: torch.Tensor | None = None
        self.ranges: list[tuple[int, int]] = []
        if hasattr(local, "chunk_base"):
            self.refresh()
            local._shard_guard = self

    @staticmethod
    def shard_bases(world: int, stride: int = CHUNK_STRIDE) -> list[int]:
        """Spaced ``chunk_base`` values that let every shard grow independently."""
        return [r * stride for r in range(world)]

    def refresh(self, *, chunk_ids: bool = False) -> None:
        """(Collective) re-gather ``(chunk_base, n_chunks)`` of every shard -- after ``append`` / ``compact`` on
        any rank -- and check that the ranges are disjoint; ``chunk_ids=True`` also gathers each shard's
        chunk-id table so that ``chunk_id_of`` resolves hits owned by other ranks."""
        mine = (int(self.local.chunk_base), int(self.local.n_chunks))
        if self.group is not None and self.world > 1:
            got: list[Any] = [None] * self.world
            dist.all_gather_object(got, mine, group=self.group)
            self.ranges = [tuple(x) for x in got]
        else:
            self.ranges = [mine]
        order = sorted(range(len(self.ranges)), key=lambda r: self.ranges[r][0])
        for a, b in zip(order[:-1], order[1:], strict=True):
            if self.ranges[a][0] + self.ranges[a][1] > self.ranges[b][0]:
                raise ValueError(f"shards {a} and {b} overlap in the global chunk numbering: {self.ranges[a]} / {self.ranges[b]}")
        if chunk_ids:
            if self.group is not None and self.world > 1:
                tables: list[Any] = [None] * self.world
                dist.all_gather_object(tables, self.local.chunk_ids, group=self.group)
                self.shard_chunk_ids = tables
            else:
                self.shard_chunk_ids = [self.local.chunk_ids]
            self.global_chunk_ids = None

    def check_local_growth(self, new_n_chunks: int) -> None:
        """Called by ``CorpusIndex.append``: the shard must stay below the next shard's base."""
        base = int(self.local.chunk_base)
        nxt = min((b for b, _ in self.ranges if b > base), default=None)
        if nxt is not None and base + new_n_chunks > nxt:
            raise ValueError(
                f"appending to shard {self.rank} would run its global chunk indices [{base}, {base + new_n_chunks}) into "
                f"the next shard's range starting at {nxt}; build the shards with spaced bases (ShardedIndex.shard_bases) "
                "to let them follow inserts")
        self.shard_chunk_ids = None   # stale until the next refresh(chunk_ids=True)
        if self.global_chunk_ids is not None:
            raise ValueError("this ShardedIndex holds one global chunk-id list, which an append would invalidate; "
                             "use per-shard tables (refresh(chunk_ids=True)) for a corpus that grows")

    def search_pipeline(  # noqa: PLR0913
        self, Q: torch.Tensor, *, k: int, num_hits: int, metric: str = "cosine", algo: str = "auto",
        row_allowed: torch.Tensor | None = None, mask_has_tombstones: bool = False, flags: int = 0, cand_cap: int = 0,
        sample_stride: int = 0, rank_first_limit: int | None = None,
    ) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
        """Scan the local shard, all-gather (hits + status words), merge: everything is enqueued on the
        current stream, nothing synchronises.  Returns ``(sim [B, k], chunk [B, k], count [B],
        status [R, B])``; every rank holds the same four tensors."""
        res: ScanResult = self.local.scan(Q, k=k, num_hits=num_hits, metric=metric, algo=algo, row_allowed=row_allowed,
                                          mask_has_tombstones=mask_has_tombstones, flags=flags, cand_cap=cand_cap,
                                          sample_stride=sample_stride)
        B, H = int(res.hit_sim.shape[0]), int(res.hit_sim.shape[1])
        if res.packed is not None and rank_first_limit is None and Q.is_cuda:
            # The scan wrote its outputs into one packed buffer: all-gather it as is, merge the gathered
            # copies in place -- no pack / unpack kernels around the collective.
            R = self.world
            if self.group is not None and R > 1:
                allb = torch.empty(R * res.packed.numel(), dtype=torch.uint8, device=res.packed.device)
                dist.all_gather_into_tensor(allb, res.packed, group=self.group)
            else:
                allb = res.packed
            per = allb.numel() // R
            off = B * H * 12 + B * 4
            status = torch.as_strided(allb.view(torch.int32), (R, B), (per // 4, 1), off // 4)
            self.last_status = status
            out = merge_packed(allb, R, B, H, num_hits=num_hits, k=k)
            return (*out, status)
        sim, chunk, count, status = gather_hits(res.hit_sim, res.hit_chunk, res.hit_count, self.group, res.status)
        self.last_status = status
        if rank_first_limit is not None:
            count = limit_hits_to_nearest(self, Q, sim, count, k=k, num_hits=num_hits, metric=metric, algo=algo,
                                          limit=rank_first_limit)
        out = merge_hits(sim, chunk, count, num_hits=num_hits, k=k)
        return (*out, status)

    def search_device(self, Q: torch.Tensor, *, k: int, num_hits: int, metric: str = "cosine", algo: str = "auto",
                      row_allowed: torch.Tensor | None = None, checked: bool = True, flags: int = 0,
                      sample_stride: int = 0, rank_first_limit: int | None = None
                      ) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """``search_pipeline`` returning device tensors.  ``checked=True`` reads the gathered status words back
        and resolves overflows collectively (every rank sees every shard's status, so all ranks re-run
        together); ``checked=False`` never synchronises (``last_status`` holds the status words)."""
        from ._index import RL_STATUS_CAND_OVERFLOW, next_overflow_attempt

        kw = dict(k=k, num_hits=num_hits, metric=metric, algo=algo, row_allowed=row_allowed, sample_stride=sample_stride,
                  rank_first_limit=rank_first_limit)
        with self.local._lock:
            sim, chunk, count, status = self.search_pipeline(Q, flags=flags, **kw)
            cap = 0
            for attempt in range(1, 16):
                if not checked or not bool((status & RL_STATUS_CAND_OVERFLOW).any()):
                    return sim, chunk, count
                cap, fl = next_overflow_attempt(self.local, attempt, cap, flags)
                sim, chunk, count, status = self.search_pipeline(Q, flags=fl, cand_cap=cap, **kw)
        raise RuntimeError("candidate lists still overflow with a list as large as the shard")

    def sum_over_shards(self, x: torch.Tensor) -> torch.Tensor:
        """All-reduce (sum) of a small per-query tensor: row counts of the rank-then-filter probe."""
        if self.group is not None and self.world > 1:
            x = x.clone()
            dist.all_reduce(x, op=dist.ReduceOp.SUM, group=self.group)
        return x

    def max_over_shards(self, x: torch.Tensor) -> torch.Tensor:
        """All-reduce (max): e.g. the largest row norm of the whole corpus."""
        if self.group is not None and self.world > 1:
            x = x.clone()
            dist.all_reduce(x, op=dist.ReduceOp.MAX, group=self.group)
        return x

    def chunk_id_of(self, global_chunk: int) -> str:
        g = int(global_chunk)
        if self.global_chunk_ids is not None:
            return self.global_chunk_ids[g]
        if self.shard_chunk_ids is not None:
            for r, (base, n) in enumerate(self.ranges):
                table = self.shard_chunk_ids[r]
                if base <= g < base + n and table is not None:
                    return table[g - base]
        lo = self.local.chunk_base
        if self.local.chunk_ids is not None and lo <= g < lo + self.local.n_chunks:
            return self.local.chunk_ids[g - lo]
        return str(g)
