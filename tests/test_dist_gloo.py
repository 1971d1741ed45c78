"""world_size-2 ``gloo`` test (CPU) of the N>1 host logic: shard ranges never split a chunk, the
single all-gather moves packed per-shard hit lists intact, and merging the gathered top-num_hits
vectors reproduces the single-table SQL semantics (what rl_topk_merge computes on the GPU)."""

from __future__ import annotations

import os
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = Path(__file__).resolve().parents[1]


def shard_hits_numpy(E, off, Q, lo, hi, num_hits, allowed_chunks=None):
    """Per-shard output of rl_maxsim_topk restated in NumPy: top-num_hits vectors (sim, global chunk);
    ``allowed_chunks`` (bool per global chunk) restates the ``row_allowed`` mask."""
    from oracle import vector_search as ovs

    r0, r1 = int(off[lo]), int(off[hi])
    Es = E[r0:r1]
    r2c = ovs.row_to_chunk(off[lo:hi + 1] - r0, r1 - r0) + lo
    B = len(Q)
    sim = np.full((B, num_hits), -np.inf, np.float32)
    chunk = np.full((B, num_hits), -1, np.int64)
    count = np.zeros(B, np.int32)
    for b, q in enumerate(Q):
        dist_ = ovs.vector_distances_f64(Es, q, "cosine")
        rows = np.arange(len(dist_)) if allowed_chunks is None else np.nonzero(np.asarray(allowed_chunks)[r2c])[0]
        order = rows[np.argsort(dist_[rows], kind="stable")][:num_hits]
        n = len(order)
        sim[b, :n] = (1.0 - dist_[order]).astype(np.float32)
        chunk[b, :n] = r2c[order]
        count[b] = n
    return sim, chunk, count


def merge_numpy(sim, chunk, count, num_hits, k):
    """rl_topk_merge restated: merge R sorted lists, keep num_hits, group by chunk (first = max), top-k."""
    R, B, H = sim.shape
    out = []
    for b in range(B):
        s = np.concatenate([sim[r, b, :count[r, b]] for r in range(R)])
        c = np.concatenate([chunk[r, b, :count[r, b]] for r in range(R)])
        o = np.argsort(-s.astype(np.float64), kind="stable")[:num_hits]
        s, c = s[o], c[o]
        uniq, first = np.unique(c, return_index=True)
        keep = np.sort(first)[:k]
        out.append((c[keep], s[keep]))
    return out


def _worker(rank: int, world: int, port: int, tmp: str) -> None:
    sys.path.insert(0, str(ROOT))
    sys.path.insert(0, str(ROOT / "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from synth import make_corpus, make_queries

    from oracle import vector_search as ovs
    from raglite_b200._dist import shard_ranges
    from raglite_b200._index import hits_views, new_scan_result

    E, off = make_corpus(600, (1, 9), 32, seed=3)
    Q = make_queries(E, 5, seed=4)
    k, num_hits = 20, 80
    ranges = shard_ranges(off, world)
    assert ranges[0][0] == 0 and ranges[-1][1] == len(off) - 1
    assert all(ranges[i][1] == ranges[i + 1][0] for i in range(world - 1))
    lo, hi = ranges[rank]

    def gather(sim, chunk, count, status=0):
        """The search's one collective: this rank's hits and status words in one packed list (as the scan writes
        it), all-gathered; returns the ``hits_views`` of the gathered buffer."""
        res = new_scan_result(len(Q), num_hits, num_hits, k, "cpu")
        res.hit_sim.copy_(torch.from_numpy(sim))
        res.hit_chunk.copy_(torch.from_numpy(chunk))
        res.hit_count.copy_(torch.from_numpy(count))
        res.status.fill_(status)
        allb = torch.empty(world * res.packed.numel(), dtype=torch.uint8)
        dist.all_gather_into_tensor(allb, res.packed)
        return hits_views(allb, world, len(Q), num_hits)

    # Every rank's list arrives intact, and the status words ride along in the same all-gather.
    g_chunk, g_sim, g_count, g_status = gather(*shard_hits_numpy(E, off, Q, lo, hi, num_hits), status=rank)
    assert g_sim.shape == (world, len(Q), num_hits) and g_status.shape == (world, len(Q))
    for r in range(world):
        sim, chunk, count = shard_hits_numpy(E, off, Q, *ranges[r], num_hits)
        assert torch.equal(g_sim[r], torch.from_numpy(sim)) and torch.equal(g_chunk[r], torch.from_numpy(chunk))
        assert torch.equal(g_count[r], torch.from_numpy(count)) and g_status[r].tolist() == [r] * len(Q)
    merged = merge_numpy(g_sim.numpy(), g_chunk.numpy(), g_count.numpy(), num_hits, k)
    for b, q in enumerate(Q):
        ref_ids, ref_sims, _ = ovs.vector_search_sql(E, off, q, num_results=k, f64=True)
        assert merged[b][0].tolist() == ref_ids.tolist()
        assert np.allclose(merged[b][1], ref_sims, atol=1e-6)
    # Rank-then-filter metadata branch on a sharded corpus (_search.py:122-143): the counts of the rank
    # probe are all-reduced, the cut is found by bisection, every rank truncates the gathered lists alike.
    from raglite_b200._dist import ShardedIndex
    from raglite_b200._index import limit_hits_to_nearest

    class FakeShard:   # the local CorpusIndex, restated on the host: exact float64 similarities
        storage, stats = "fp32", torch.tensor([1.0, 1.0, 1.0, 0.0])

        def count_at_least(self, Qd, floor, **_):
            r0, r1 = int(off[lo]), int(off[hi])
            sims = [1.0 - ovs.vector_distances_f64(E[r0:r1], q, "cosine") for q in Qd.numpy()]
            return torch.tensor([int((s >= float(f)).sum()) for s, f in zip(sims, floor)], dtype=torch.int32)

    limit = 300
    score0 = ovs.maxsim_scores(E, off, Q[0], "cosine", f64=True)
    order0 = np.argsort(-score0)
    tagged = np.zeros(len(off) - 1, dtype=bool)
    tagged[order0[len(order0) // 2:]] = True       # far from query 0 ...
    tagged[order0[[0, 3, 7]]] = True               # ... plus three near chunks
    g_chunk, g_sim, g_count, _ = gather(*shard_hits_numpy(E, off, Q, lo, hi, num_hits, allowed_chunks=tagged))
    sharded = ShardedIndex(FakeShard(), dist.group.WORLD)
    g_count.copy_(limit_hits_to_nearest(sharded, torch.from_numpy(Q), g_sim, g_count, k=k, num_hits=num_hits,
                                        metric="cosine", limit=limit))
    both = [torch.zeros_like(g_count) for _ in range(world)]
    dist.all_gather(both, g_count.contiguous())
    assert torch.equal(both[0], both[1]), "every rank must keep the same hits"
    merged = merge_numpy(g_sim.numpy(), g_chunk.numpy(), g_count.numpy(), num_hits, k)
    changed = 0
    for b, q in enumerate(Q):
        ref_ids, ref_sims, _ = ovs.vector_search_sql(E, off, q, num_results=k, allowed_chunks=tagged, f64=True,
                                                     filter_first_max=0, rank_first_limit=limit)
        assert merged[b][0].tolist() == ref_ids.tolist(), (b, merged[b][0], ref_ids)
        assert np.allclose(merged[b][1], ref_sims, atol=1e-6)
        first_ids, _, _ = ovs.vector_search_sql(E, off, q, num_results=k, allowed_chunks=tagged, f64=True)
        changed += ref_ids.tolist() != first_ids.tolist()
    assert changed >= 1, "the cut must change at least query 0's answer"

    # ADVICE r1: dot metric, shards whose largest row norms differ -- the bisection bracket must be the
    # same on every rank (max over shards), or the summed counts mix different thresholds.
    scale = np.where(np.arange(len(E)) >= int(off[ranges[1][0]]), 3.0, 1.0).astype(np.float32)[:, None]
    Ed = E * scale

    class FakeDotShard:
        storage = "fp32"
        stats = torch.tensor([float(np.linalg.norm(Ed[int(off[lo]):int(off[hi])], axis=1).max()), 1.0, 1.0, 0.0])

        def count_at_least(self, Qd, floor, **_):
            r0, r1 = int(off[lo]), int(off[hi])
            sims = [1.0 - ovs.vector_distances_f64(Ed[r0:r1], q, "dot") for q in Qd.numpy()]
            return torch.tensor([int((s >= float(f)).sum()) for s, f in zip(sims, floor)], dtype=torch.int32)

    def shard_hits_dot(allowed):
        r0, r1 = int(off[lo]), int(off[hi])
        r2c = ovs.row_to_chunk(off[lo:hi + 1] - r0, r1 - r0) + lo
        sim_ = np.full((len(Q), num_hits), -np.inf, np.float32); ch_ = np.full((len(Q), num_hits), -1, np.int64)
        cn_ = np.zeros(len(Q), np.int32)
        for b, q in enumerate(Q):
            d_ = ovs.vector_distances_f64(Ed[r0:r1], q, "dot")
            rows_ = np.nonzero(allowed[r2c])[0]
            o_ = rows_[np.argsort(d_[rows_], kind="stable")][:num_hits]
            sim_[b, :len(o_)] = (1.0 - d_[o_]).astype(np.float32); ch_[b, :len(o_)] = r2c[o_]; cn_[b] = len(o_)
        return sim_, ch_, cn_

    g_chunk, g_sim, g_count, _ = gather(*shard_hits_dot(tagged))
    sharded = ShardedIndex(FakeDotShard(), dist.group.WORLD)
    g_count.copy_(limit_hits_to_nearest(sharded, torch.from_numpy(Q), g_sim, g_count, k=k, num_hits=num_hits,
                                        metric="dot", limit=limit))
    both = [torch.zeros_like(g_count) for _ in range(world)]
    dist.all_gather(both, g_count.contiguous())
    assert torch.equal(both[0], both[1]), "every rank must keep the same hits"
    merged = merge_numpy(g_sim.numpy(), g_chunk.numpy(), g_count.numpy(), num_hits, k)
    for b, q in enumerate(Q):
        ref_ids, ref_sims, _ = ovs.vector_search_sql(Ed, off, q, num_results=k, metric="dot", allowed_chunks=tagged, f64=True,
                                                     filter_first_max=0, rank_first_limit=limit)
        assert merged[b][0].tolist() == ref_ids.tolist(), (b, merged[b][0], ref_ids)

    # ADVICE r1: shard ranges are gathered and checked; chunk ids resolve across ranks after refresh(chunk_ids=True).
    class FakeLocal:
        def __init__(self, base, n):
            self.chunk_base, self.n_chunks, self.chunk_ids = base, n, [f"r{rank}-c{i}" for i in range(n)]

    bases = ShardedIndex.shard_bases(world)
    sh = ShardedIndex(FakeLocal(bases[rank], 5 + rank), dist.group.WORLD)
    assert sh.ranges == [(bases[0], 5), (bases[1], 6)]
    sh.refresh(chunk_ids=True)
    assert sh.chunk_id_of(bases[1] + 3) == "r1-c3" and sh.chunk_id_of(2) == "r0-c2"
    sh.check_local_growth(1000)                       # spaced bases: room to grow
    with pytest.raises(ValueError, match="overlap"):
        ShardedIndex(FakeLocal(0 if rank == 0 else 3, 5), dist.group.WORLD)
    tight = ShardedIndex(FakeLocal(rank * 5, 5), dist.group.WORLD)
    if rank == 0:
        with pytest.raises(ValueError, match="next shard"):
            tight.check_local_growth(6)
    else:
        tight.check_local_growth(6)                   # the last shard may grow
    dist.barrier()
    dist.destroy_process_group()
    Path(tmp, f"ok{rank}").write_text("ok")


def test_two_rank_packed_gather_and_merge(tmp_path):
    port = 29500 + (os.getpid() % 2000)
    mp.spawn(_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    assert (tmp_path / "ok0").exists() and (tmp_path / "ok1").exists()


def test_shard_ranges_balance_and_edges():
    sys.path.insert(0, str(ROOT))
    from raglite_b200._dist import shard_ranges

    off = np.concatenate([[0], np.cumsum(np.random.default_rng(0).integers(1, 20, size=1000))])
    for world in (1, 2, 4, 8):
        rng = shard_ranges(off, world)
        rows = [off[b] - off[a] for a, b in rng]
        assert sum(rows) == off[-1] and max(rows) - min(rows) <= 2 * 19
    assert shard_ranges(np.array([0, 5]), 4) == [(0, 0), (0, 0), (0, 0), (0, 1)] or sum(b - a for a, b in shard_ranges(np.array([0, 5]), 4)) == 1


def test_hits_views_roundtrip():
    """Hit lists written through one scan result's views and laid end to end read back through ``hits_views``."""
    sys.path.insert(0, str(ROOT))
    from raglite_b200._index import hits_views, new_scan_result

    g = torch.Generator().manual_seed(0)
    B, H, R = 3, 7, 2
    bufs, want = [], []
    for _ in range(R):
        s = torch.randn((B, H), generator=g)
        c = torch.randint(0, 1 << 40, (B, H), generator=g)
        n = torch.randint(0, H, (B,), generator=g, dtype=torch.int32)
        st = torch.randint(0, 4, (B,), generator=g, dtype=torch.int32)
        res = new_scan_result(B, H, H, 1, "cpu")
        res.hit_sim.copy_(s); res.hit_chunk.copy_(c); res.hit_count.copy_(n); res.status.copy_(st)
        bufs.append(res.packed); want.append((s, c, n, st))
    chunk, sim, count, status = hits_views(torch.cat(bufs), R, B, H)
    for r in range(R):
        assert torch.equal(sim[r], want[r][0]) and torch.equal(chunk[r], want[r][1]) and torch.equal(count[r], want[r][2])
        assert torch.equal(status[r], want[r][3])
