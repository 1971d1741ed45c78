"""An in-process R-rank collective for tests: R Python threads on one GPU stand in for the R processes of a sharded
search.  Each thread is one rank with its own ``CorpusIndex`` shard and, on a GPU, its own CUDA stream; the collectives
the library calls (``torch.distributed`` as ``raglite_b200._dist.dist`` / ``raglite_b200._index.dist``) are replaced by
``ThreadDist``, which hands tensors between the threads.  So the library's real host pipeline -- ``ShardedIndex``,
``scan_gather_merge``, ``search_to_host``, ``run_until_no_overflow``, ``limit_hits_to_nearest`` -- runs with R > 1 without
ports, child processes or NCCL.

A rank that raises aborts the shared barrier, so the other ranks leave their next collective with
``threading.BrokenBarrierError`` at once; a rank that stops calling collectives ends the others' wait after
``timeout`` seconds.  ``run_ranks`` re-raises the first real exception."""

from __future__ import annotations

import pickle
import threading
from collections.abc import Callable
from typing import Any

import torch
import torch.distributed as tdist

DEFAULT_TIMEOUT = 120.0


class _Shared:
    """State every rank of one group sees: the barrier and one deposit slot per rank."""

    def __init__(self, world: int, timeout: float):
        self.world = world
        self.barrier = threading.Barrier(world, timeout=timeout)
        self.slots: list[Any] = [None] * world

    def wait(self) -> None:
        self.barrier.wait()


class RankGroup:
    """The ``group=`` handle of one rank: the shared state plus the rank it stands for."""

    def __init__(self, shared: _Shared, rank: int):
        self.shared, self.rank = shared, rank

    def __repr__(self) -> str:
        return f"RankGroup(rank={self.rank}, world={self.shared.world})"


def make_groups(world: int, timeout: float = DEFAULT_TIMEOUT) -> list[RankGroup]:
    shared = _Shared(world, timeout)
    return [RankGroup(shared, r) for r in range(world)]


def _settle(t: torch.Tensor) -> None:
    """Wait until the work this thread's current stream has enqueued on ``t`` is done (no-op on the CPU)."""
    if t.is_cuda:
        torch.cuda.current_stream(t.device).synchronize()


class ThreadDist:
    """The part of ``torch.distributed`` the library calls, over ``RankGroup`` handles.  Tensor collectives: each rank
    settles its input on its current stream and deposits it; after a barrier each rank reads every deposit on its own
    current stream and settles that work; a second barrier keeps a rank from reusing (or writing) its input while
    another rank still reads it."""

    ReduceOp = tdist.ReduceOp

    def __init__(self) -> None:
        self.calls: dict[str, int] = {}

    def _count(self, name: str, group: RankGroup) -> None:
        if group.rank == 0:
            self.calls[name] = self.calls.get(name, 0) + 1

    @staticmethod
    def _group(group: RankGroup | None) -> RankGroup:
        if not isinstance(group, RankGroup):
            raise TypeError(f"ThreadDist needs the rank's RankGroup as group=, got {group!r}")
        return group

    def get_world_size(self, group: RankGroup | None = None) -> int:
        return self._group(group).shared.world

    def get_rank(self, group: RankGroup | None = None) -> int:
        return self._group(group).rank

    def barrier(self, group: RankGroup | None = None, **_: Any) -> None:
        self._group(group).shared.wait()

    def all_gather_into_tensor(self, output: torch.Tensor, input: torch.Tensor, group: RankGroup | None = None,  # noqa: A002
                               async_op: bool = False) -> None:
        g = self._group(group)
        sh = g.shared
        self._count("all_gather_into_tensor", g)
        if output.numel() != sh.world * input.numel():
            raise ValueError(f"all_gather_into_tensor: output holds {output.numel()} elements, {sh.world} x {input.numel()} needed")
        _settle(input)
        sh.slots[g.rank] = input
        sh.wait()
        parts = output.view(sh.world, -1)
        for r in range(sh.world):
            parts[r].copy_(sh.slots[r].reshape(-1))
        _settle(output)
        sh.wait()

    def all_reduce(self, tensor: torch.Tensor, op: Any = tdist.ReduceOp.SUM, group: RankGroup | None = None,
                   async_op: bool = False) -> None:
        g = self._group(group)
        sh = g.shared
        self._count("all_reduce", g)
        _settle(tensor)
        sh.slots[g.rank] = tensor
        sh.wait()
        stacked = torch.stack([sh.slots[r].to(tensor.device) for r in range(sh.world)])   # rank order on every rank
        if op == tdist.ReduceOp.SUM:
            out = stacked.sum(0, dtype=tensor.dtype)
        elif op == tdist.ReduceOp.MAX:
            out = stacked.amax(0)
        else:
            raise NotImplementedError(f"ThreadDist.all_reduce: {op}")
        _settle(out)
        sh.wait()                 # nobody reads the inputs any more: now each rank may overwrite its own
        tensor.copy_(out)
        _settle(tensor)

    def all_gather_object(self, object_list: list[Any], obj: Any, group: RankGroup | None = None) -> None:
        g = self._group(group)
        sh = g.shared
        self._count("all_gather_object", g)
        sh.slots[g.rank] = pickle.dumps(obj)      # the objects travel pickled, as torch.distributed sends them
        sh.wait()
        got = [pickle.loads(sh.slots[r]) for r in range(sh.world)]
        sh.wait()
        object_list[:] = got


def install(monkeypatch: Any) -> ThreadDist:
    """Route the library's collectives through a new ``ThreadDist`` for one test; ``torch.distributed`` itself is
    untouched."""
    import raglite_b200._dist as D
    import raglite_b200._index as I

    shim = ThreadDist()
    monkeypatch.setattr(D, "dist", shim)
    monkeypatch.setattr(I, "dist", shim)
    return shim


def run_ranks(world: int, fn: Callable[[int, RankGroup], Any], *, timeout: float = DEFAULT_TIMEOUT,
              streams: bool | None = None) -> list[Any]:
    """Run ``fn(rank, group)`` in ``world`` threads and return the per-rank results.  With ``streams`` (the default when
    CUDA is available) each rank runs on a CUDA stream of its own.  The first exception a rank raised is re-raised
    here (a ``BrokenBarrierError`` only when no rank raised anything else); every thread has ended by then."""
    groups = make_groups(world, timeout)
    use_streams = torch.cuda.is_available() if streams is None else streams
    results: list[Any] = [None] * world
    errors: list[BaseException | None] = [None] * world

    def body(r: int) -> None:
        try:
            if use_streams:
                with torch.cuda.stream(torch.cuda.Stream()):
                    results[r] = fn(r, groups[r])
                    torch.cuda.current_stream().synchronize()
            else:
                results[r] = fn(r, groups[r])
        except BaseException as e:  # noqa: BLE001  (reported by the caller)
            errors[r] = e
            groups[r].shared.barrier.abort()    # release the ranks waiting in a collective

    threads = [threading.Thread(target=body, args=(r,), name=f"rank{r}", daemon=True) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout + 60.0)
    if any(t.is_alive() for t in threads):
        groups[0].shared.barrier.abort()
        for t in threads:
            t.join(timeout)
        raise TimeoutError("a rank did not finish")
    real = [e for e in errors if e is not None and not isinstance(e, threading.BrokenBarrierError)]
    if real:
        raise real[0]
    broken = [e for e in errors if e is not None]
    if broken:
        raise broken[0]
    return results
