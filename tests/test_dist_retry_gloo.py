"""world_size-2 ``gloo`` test (CPU) of the candidate-overflow retry loop on shards of different sizes: every run
all-gathers the status words, as the sharded search does, and both ranks must leave the loop after the same number
of runs -- with the result, or with ``RagliteB200Error``.  A rank that left early would leave the other one waiting
in the next all-gather; the process group's short timeout turns such a hang into a failure."""

from __future__ import annotations

import os
import sys
from datetime import timedelta
from pathlib import Path
from types import SimpleNamespace

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = Path(__file__).resolve().parents[1]
SMALL, LARGE = 2_000, 1_000_000     # rows of shard 0 and shard 1


def _worker(rank: int, world: int, port: int, tmp: str) -> None:
    sys.path.insert(0, str(ROOT))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=timedelta(seconds=30))
    from raglite_b200._index import MAX_SCAN_RUNS, run_until_no_overflow
    from raglite_b200._lib import RL_FLAG_REUSE_THRESHOLDS, RagliteB200Error

    local = SimpleNamespace(n_rows=(SMALL, LARGE)[rank], scan_stats=lambda: {"cand_cap": 1000})

    def scripted(overflows):
        """A search whose shard overflows while ``overflows(cand_cap)``; returns the gathered status and the runs."""
        runs = []

        def run(flags, cand_cap):
            runs.append((flags, cand_cap))
            mine = torch.tensor([int(overflows(cand_cap))], dtype=torch.int32)
            status = torch.empty(world, dtype=torch.int32)
            dist.all_gather_into_tensor(status, mine)
            return status

        return run, runs

    # Only the large shard overflows, until its list holds 16000 entries -- four times more than the small shard's
    # list may grow to (SMALL + 1024).  The small shard clamps its list and keeps re-running with the large one.
    run, runs = scripted(lambda cap: rank == 1 and cap < 16_000)
    run_until_no_overflow(local, run)
    REUSE = RL_FLAG_REUSE_THRESHOLDS
    top = (SMALL + 1024, 16_000)[rank]
    assert runs == [(0, 0), (REUSE, 0), (0, min(4000, top)), (REUSE, min(4000, top)), (0, top)], runs
    counts = [None] * world
    dist.all_gather_object(counts, len(runs))
    assert counts == [5, 5]

    # An overflow that never clears: both ranks raise after the same number of runs, lists clamped at their shard.
    run, runs = scripted(lambda cap: rank == 1)
    with pytest.raises(RagliteB200Error):
        run_until_no_overflow(local, run)
    assert len(runs) == MAX_SCAN_RUNS and max(c for _, c in runs) == local.n_rows + 1024
    dist.all_gather_object(counts, len(runs))
    assert counts == [MAX_SCAN_RUNS] * world
    dist.barrier()
    dist.destroy_process_group()
    Path(tmp, f"ok{rank}").write_text("ok")


def test_two_rank_retry_stops_together(tmp_path):
    port = 25500 + (os.getpid() % 2000)
    mp.spawn(_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    assert (tmp_path / "ok0").exists() and (tmp_path / "ok1").exists()
