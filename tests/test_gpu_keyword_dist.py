"""Two-GPU (NCCL) parity of the sharded BM25 keyword search: every rank builds its shard's postings, one all-reduce of
the query statistics, one all-gather of the packed per-shard top k, the merge on every rank -- bit-identical to one
``CorpusIndex`` over the whole corpus whose term ids follow sorted-stem order.  Skipped on a single-GPU box."""

from __future__ import annotations

import os
import sys
from pathlib import Path

import pytest

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]


def _worker(rank: int, world: int, port: int, tmp: str) -> None:
    sys.path.insert(0, str(ROOT))
    sys.path.insert(0, str(ROOT / "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import numpy as np
    import torch
    import torch.distributed as dist
    from synth import make_corpus
    from test_gpu_keyword import _queries
    from test_gpu_keyword_sharded import _sorted_stem_body, _to_single

    import keyword_oracle as ko
    import raglite_b200 as rl
    from raglite_b200._dist import ShardedIndex

    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    bodies = ko.make_bodies(8000, seed=51, vocab=2500)
    bodies[0] = _sorted_stem_body(bodies[1:])
    C = len(bodies)
    E, off = make_corpus(C, 1, 16, seed=1)
    docs = ["d-all"] + [f"d{c // 10}" for c in range(1, C)]
    chunks = [rl.Chunk(id=f"c{c}", document_id=docs[c], index=c % 10, body=bodies[c]) for c in range(C)]
    ranges = [(0, 3000), (3000, C)]
    bases = ShardedIndex.shard_bases(world)
    lo, hi = ranges[rank]
    local = rl.CorpusIndex(E[lo:hi], off[lo:hi + 1] - lo, chunk_base=bases[rank], chunk_ids=[f"c{c}" for c in range(lo, hi)],
                           chunks=chunks[lo:hi], device=f"cuda:{rank}")
    index = ShardedIndex(local, dist.group.WORLD)
    single = rl.CorpusIndex(E, off, chunk_ids=[f"c{c}" for c in range(C)], chunks=chunks, device=f"cuda:{rank}")
    single.delete_documents(["d-all"])
    if rank == 0:
        local.delete_documents(["d-all"])
    queries = _queries(53, 51, 2500, 100)
    for k in (1, 10, 4096):
        ids, sc, cnt = rl.keyword_search_batch(queries, num_results=k, index=index)
        w_ids, w_sc, w_cnt = rl.keyword_search_batch(queries, num_results=k, index=single)
        assert np.array_equal(cnt, w_cnt) and np.array_equal(_to_single(ids, ranges, bases), w_ids)
        assert np.array_equal(sc.view(np.int64), w_sc.view(np.int64))
        both = [None] * world
        dist.all_gather_object(both, ids.tolist())
        assert both[0] == both[1], "every rank must hold the same merged result"
    dist.barrier()
    dist.destroy_process_group()
    Path(tmp, f"ok{rank}").write_text("ok")


def test_two_gpu_sharded_keyword_search(tmp_path):
    import torch
    import torch.multiprocessing as mp

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    port = 29800 + (os.getpid() % 1000)
    mp.spawn(_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    assert (tmp_path / "ok0").exists() and (tmp_path / "ok1").exists()
