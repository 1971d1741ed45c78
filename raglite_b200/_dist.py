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

from ._index import CorpusIndex, run_until_no_overflow, scan_gather_merge


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

    def __init__(self, local: CorpusIndex, group: Any | None = None):
        self.local = local
        self.group = group
        self.world = dist.get_world_size(group) if group is not None else 1
        self.rank = dist.get_rank(group) if group is not None else 0
        self.shard_chunk_ids: list[list[str] | None] | None = None
        self._any_chunk_ids = False   # some shard held chunk ids at the last gather of the tables
        self.last_status: torch.Tensor | None = None
        self.ranges: list[tuple[int, int]] = []
        if hasattr(local, "chunk_base"):
            self.refresh(chunk_ids=True)   # hits owned by other ranks resolve to their ids from the first search on
            local._shard_guard = self

    @staticmethod
    def shard_bases(world: int, stride: int = CHUNK_STRIDE) -> list[int]:
        """Spaced ``chunk_base`` values that let every shard grow independently."""
        return [r * stride for r in range(world)]

    def refresh(self, *, chunk_ids: bool = False) -> None:
        """(Collective) re-gather ``(chunk_base, n_chunks)`` of every shard -- after ``append`` / ``compact`` on
        any rank -- and check that the ranges are disjoint; ``chunk_ids=True`` also gathers each shard's
        chunk-id table so that ``chunk_id_of`` resolves hits owned by other ranks.  The constructor gathers the
        tables; after ``append`` / ``compact`` on any rank call ``refresh(chunk_ids=True)`` on every rank."""
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
            self._any_chunk_ids = any(t is not None for t in self.shard_chunk_ids)

    def check_local_growth(self, new_n_chunks: int) -> None:
        """Called by ``CorpusIndex.append``: the shard must stay below the next shard's base."""
        base = int(self.local.chunk_base)
        nxt = min((b for b, _ in self.ranges if b > base), default=None)
        if nxt is not None and base + new_n_chunks > nxt:
            raise ValueError(
                f"appending to shard {self.rank} would run its global chunk indices [{base}, {base + new_n_chunks}) into "
                f"the next shard's range starting at {nxt}; build the shards with spaced bases (ShardedIndex.shard_bases) "
                "to let them follow inserts")

    def add_tsvector_rows(self, rows: Any) -> int:
        """``CorpusIndex.add_tsvector_rows`` for this rank's shard, not a collective: of the ``(chunk_id, text)`` rows it
        keeps those of the chunks this shard holds and ignores the rest, so every rank can be handed the whole result
        set of ``SELECT id, to_tsvector('simple', body)::text FROM chunk``.  Returns the number of rows kept."""
        return self.local._add_tsvector_rows(rows, others_ok=True)

    def search_pipeline(self, Q: torch.Tensor, **kw: Any) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
        """``scan_gather_merge`` over the shards of the group; ``last_status`` keeps the gathered status words."""
        out = scan_gather_merge(self, Q, **kw)
        self.last_status = out[3]
        return out

    def search_device(self, Q: torch.Tensor, *, k: int, num_hits: int, metric: str = "cosine", algo: str = "auto",
                      row_allowed: torch.Tensor | None = None, checked: bool = True, flags: int = 0,
                      sample_stride: int = 0, rank_first_limit: int | None = None
                      ) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """``search_pipeline`` returning device tensors.  ``checked=True`` reads the gathered status words back
        and resolves overflows collectively (``run_until_no_overflow``: every rank sees every shard's status, so
        all ranks re-run together); ``checked=False`` never synchronises (``last_status`` holds the status words)."""
        kw = dict(k=k, num_hits=num_hits, metric=metric, algo=algo, row_allowed=row_allowed, sample_stride=sample_stride,
                  rank_first_limit=rank_first_limit)
        out = None

        def run(flags: int, cand_cap: int) -> torch.Tensor:
            nonlocal out
            out = self.search_pipeline(Q, flags=flags, cand_cap=cand_cap, **kw)
            return out[3]

        with self.local._lock:
            if not checked:
                run(flags, 0)
            else:
                run_until_no_overflow(self.local, run, flags=flags)
        return out[:3]

    def sum_over_shards(self, x: torch.Tensor) -> torch.Tensor:
        """All-reduce (sum) of a small tensor: row counts of the rank-then-filter probe, the BM25 statistics of a
        keyword search."""
        if self.group is not None and self.world > 1:
            x = x.clone()
            dist.all_reduce(x, op=dist.ReduceOp.SUM, group=self.group)
        return x

    def gather_shards(self, x: torch.Tensor) -> torch.Tensor:
        """All-gather (into one tensor) of an equally sized per-rank buffer: ``[R * x.numel()]``, rank r's part at
        ``r * x.numel()``; ``x`` itself on a one-rank index."""
        if self.group is not None and self.world > 1:
            out = torch.empty(self.world * x.numel(), dtype=x.dtype, device=x.device)
            dist.all_gather_into_tensor(out, x, group=self.group)
            return out
        return x

    def max_over_shards(self, x: torch.Tensor) -> torch.Tensor:
        """All-reduce (max): e.g. the largest row norm of the whole corpus."""
        if self.group is not None and self.world > 1:
            x = x.clone()
            dist.all_reduce(x, op=dist.ReduceOp.MAX, group=self.group)
        return x

    def chunk_id_of(self, global_chunk: int) -> str:
        """The chunk id of a global chunk index: this rank's own chunks from the shard itself, the other ranks' from
        the tables the last ``refresh(chunk_ids=True)`` gathered.  An index whose shards hold no chunk ids names a
        chunk by its number (``str``, as ``CorpusIndex.chunk_id_of``).  A chunk outside every gathered table -- one
        that another rank appended after that refresh -- raises ``LookupError`` rather than pass a number off as an
        id: call ``refresh(chunk_ids=True)`` on every rank after ``append`` or ``compact``."""
        g = int(global_chunk)
        lo = self.local.chunk_base
        if self.local.chunk_ids is not None and lo <= g < lo + self.local.n_chunks:
            return self.local.chunk_ids[g - lo]
        if self.shard_chunk_ids is not None:
            for r, (base, n) in enumerate(self.ranges):
                table = self.shard_chunk_ids[r]
                if table is not None and base <= g < base + min(n, len(table)):
                    return table[g - base]
        if self._any_chunk_ids or self.local.chunk_ids is not None:
            raise LookupError(f"global chunk {g} is in no chunk-id table gathered by the last refresh: call "
                              "refresh(chunk_ids=True) on every rank after append or compact")
        return str(g)
