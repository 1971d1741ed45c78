"""CPU tests of the in-process R-rank collective (``thread_group``) and of ``ShardedIndex``'s host logic run through it:
the collectives mean what ``torch.distributed`` means where the library relies on it, a failing rank ends the run instead
of hanging it, and chunk ids resolve on every rank of a freshly built sharded index."""

from __future__ import annotations

import threading
import time

import numpy as np
import pytest
import torch
from thread_group import ThreadDist, install, run_ranks

import raglite_b200._dist as D

ReduceOp = torch.distributed.ReduceOp


@pytest.mark.parametrize("world", [1, 2, 3])
def test_collectives_match_torch_distributed(world):
    shim = ThreadDist()

    def rank_fn(r, g):
        assert shim.get_world_size(g) == world and shim.get_rank(g) == r
        # all_gather_into_tensor: rank r's input lands at rows [r * n, (r + 1) * n) of every rank's output
        inp = torch.arange(5, dtype=torch.uint8) + 10 * r
        out = torch.empty(world * 5, dtype=torch.uint8)
        shim.all_gather_into_tensor(out, inp, group=g)
        inp.fill_(255)      # the inputs may be reused once the collective has returned on this rank
        # all_reduce in place, SUM and MAX, int64 and float32
        s = torch.tensor([r + 1, -r, 7], dtype=torch.int64)
        shim.all_reduce(s, op=shim.ReduceOp.SUM, group=g)
        m = torch.tensor([float(r), -float(r), 0.5], dtype=torch.float32)
        shim.all_reduce(m, op=ReduceOp.MAX, group=g)
        # all_gather_object: rank-ordered copies, not the depositing rank's object
        mine = {"rank": r, "ids": [f"r{r}-{i}" for i in range(r + 1)]}
        objs = [None] * world
        shim.all_gather_object(objs, mine, group=g)
        mine["ids"].append("later")
        shim.barrier(group=g)
        return out, s, m, objs

    results = run_ranks(world, rank_fn, streams=False)
    want_gather = torch.cat([torch.arange(5, dtype=torch.uint8) + 10 * r for r in range(world)])
    want_sum = torch.tensor([sum(r + 1 for r in range(world)), -sum(range(world)), 7 * world])
    want_max = torch.tensor([world - 1.0, 0.0, 0.5])
    want_objs = [{"rank": r, "ids": [f"r{r}-{i}" for i in range(r + 1)]} for r in range(world)]
    for out, s, m, objs in results:
        assert torch.equal(out, want_gather)
        assert torch.equal(s, want_sum) and s.dtype == torch.int64
        assert torch.equal(m, want_max)
        assert objs == want_objs


def test_all_gather_into_tensor_refuses_a_wrong_output_size():
    shim = ThreadDist()

    def rank_fn(r, g):
        shim.all_gather_into_tensor(torch.empty(3, dtype=torch.uint8), torch.zeros(2, dtype=torch.uint8), group=g)

    with pytest.raises(ValueError, match="output holds"):
        run_ranks(2, rank_fn, streams=False)


@pytest.mark.parametrize("world", [2, 3])
def test_a_failing_rank_ends_the_run_instead_of_hanging(world):
    """The last rank raises before its first collective; the others sit in a barrier that would last 120 s.  The
    run must end at once with the rank's own error, and no rank thread may outlive it."""
    shim = ThreadDist()

    def rank_fn(r, g):
        if r == world - 1:
            time.sleep(0.2)
            raise RuntimeError("rank failed")
        x = torch.zeros(2, dtype=torch.int64)
        shim.all_reduce(x, group=g)
        return x

    before = {t.name for t in threading.enumerate()}
    t0 = time.monotonic()
    with pytest.raises(RuntimeError, match="rank failed"):
        run_ranks(world, rank_fn, streams=False)
    assert time.monotonic() - t0 < 30.0
    assert not [t for t in threading.enumerate() if t.name.startswith("rank") and t.name not in before]


def test_a_rank_that_stops_calling_collectives_times_out():
    shim = ThreadDist()

    def rank_fn(r, g):
        if r == 0:
            shim.barrier(group=g)     # rank 1 never arrives
        return r

    with pytest.raises(threading.BrokenBarrierError):
        run_ranks(2, rank_fn, streams=False, timeout=0.5)


class FakeLocal:
    """The attributes of a ``CorpusIndex`` shard ``ShardedIndex`` reads on the host, as ``test_dist_gloo`` builds them."""

    def __init__(self, rank, base, n, ids=True):
        self.chunk_base, self.n_chunks = base, n
        self.chunk_ids = [f"r{rank}-c{i}" for i in range(n)] if ids else None


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("spaced", [False, True])
def test_fresh_sharded_index_resolves_every_shards_ids(monkeypatch, world, spaced):
    """A ``ShardedIndex`` resolves the chunk ids of every shard from its first search on, without an explicit
    ``refresh(chunk_ids=True)``: a hit owned by another rank must never come back as the number of its chunk."""
    install(monkeypatch)
    sizes = [5 + 2 * r for r in range(world)]
    bases = D.ShardedIndex.shard_bases(world) if spaced else list(np.cumsum([0] + sizes[:-1]).tolist())

    def rank_fn(r, g):
        sh = D.ShardedIndex(FakeLocal(r, bases[r], sizes[r]), g)
        return {(o, i): sh.chunk_id_of(bases[o] + i) for o in range(world) for i in range(sizes[o])}

    for got in run_ranks(world, rank_fn, streams=False):
        assert got == {(o, i): f"r{o}-c{i}" for o in range(world) for i in range(sizes[o])}


def test_shards_without_ids_name_chunks_by_number(monkeypatch):
    install(monkeypatch)
    bases = D.ShardedIndex.shard_bases(2)

    def rank_fn(r, g):
        sh = D.ShardedIndex(FakeLocal(r, bases[r], 4, ids=False), g)
        return [sh.chunk_id_of(bases[o] + 1) for o in range(2)]

    for got in run_ranks(2, rank_fn, streams=False):
        assert got == [str(bases[0] + 1), str(bases[1] + 1)]


def test_chunk_appended_on_another_rank_raises_until_refresh(monkeypatch):
    """After rank 1 appends a chunk and before the next ``refresh(chunk_ids=True)``, rank 0 has no table entry for
    it: ``chunk_id_of`` raises ``LookupError`` (it cannot refresh on its own: that is a collective).  Rank 1 resolves
    its own new chunk from its shard at once; after the collective refresh every rank resolves it."""
    install(monkeypatch)
    bases = D.ShardedIndex.shard_bases(2)
    new = bases[1] + 6

    def rank_fn(r, g):
        local = FakeLocal(r, bases[r], 6)
        sh = D.ShardedIndex(local, g)
        if r == 1:   # CorpusIndex.append: the growth check, then the new chunk and its id
            sh.check_local_growth(7)
            local.chunk_ids = local.chunk_ids + ["r1-new"]
            local.n_chunks = 7
        D.dist.barrier(group=g)
        if r == 0:
            with pytest.raises(LookupError, match="refresh"):
                sh.chunk_id_of(new)
            before = None
        else:
            before = sh.chunk_id_of(new)
        others = [sh.chunk_id_of(bases[o] + 2) for o in range(2)]
        sh.refresh(chunk_ids=True)
        return before, others, sh.chunk_id_of(new)

    r0, r1 = run_ranks(2, rank_fn, streams=False)
    assert r0 == (None, ["r0-c2", "r1-c2"], "r1-new")
    assert r1 == ("r1-new", ["r0-c2", "r1-c2"], "r1-new")


def test_sharded_collectives_go_through_the_shim(monkeypatch):
    """``sum_over_shards`` / ``max_over_shards`` reduce over the thread ranks, and the overlap check of the gathered
    shard ranges raises on every rank."""
    shim = install(monkeypatch)

    def rank_fn(r, g):
        sh = D.ShardedIndex(FakeLocal(r, r * 10, 10), g)
        s = sh.sum_over_shards(torch.tensor([r, 1], dtype=torch.int64))
        m = sh.max_over_shards(torch.tensor([float(r)]))
        return s.tolist(), m.tolist()

    assert run_ranks(3, rank_fn, streams=False) == [([3, 3], [2.0])] * 3
    assert shim.calls["all_reduce"] == 2 and shim.calls["all_gather_object"] == 2   # ranges + id tables

    def overlapping(r, g):
        D.ShardedIndex(FakeLocal(r, 0 if r == 0 else 3, 5), g)

    with pytest.raises(ValueError, match="overlap"):
        run_ranks(2, overlapping, streams=False)
