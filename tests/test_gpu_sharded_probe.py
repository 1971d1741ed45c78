"""The rank-then-filter branch (``_search.py:122-143``) with its explicit rank probe, searched through a registered
``ShardedIndex(local, group=None)``: one GPU, one shard, the same pipeline the multi-GPU path runs.  Its ids, sims and
counts must be those of the bare ``CorpusIndex``, and right against the oracle."""

from __future__ import annotations

import numpy as np
import pytest
from parity import check_sql_semantics
from synth import make_corpus, make_queries

from oracle import vector_search as ovs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rl():
    import torch

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import raglite_b200

    return raglite_b200


def _search_both(rl, E, off, meta, Q, monkeypatch, **kw):
    """``vector_search_batch`` through a registered ``ShardedIndex(group=None)`` and through the bare shard;
    returns both results and how many counting passes (the explicit rank probe) the sharded search ran."""
    from raglite_b200._dist import ShardedIndex

    calls = {"n": 0}
    orig = rl.CorpusIndex.count_at_least

    def counting(self, *a, **k):
        calls["n"] += 1
        return orig(self, *a, **k)

    monkeypatch.setattr(rl.CorpusIndex, "count_at_least", counting)
    cfg = rl.RAGLiteConfig(db_url="test://sharded-probe", reranker=None)
    rl.register_index(cfg, ShardedIndex(rl.CorpusIndex(E, off, chunk_metadata=meta), group=None))
    try:
        sharded = rl.vector_search_batch(Q, config=cfg, **kw)
    finally:
        rl.unregister_index(cfg)
    n_probe = calls["n"]
    bare = rl.vector_search_batch(Q, config=rl.RAGLiteConfig(reranker=None), index=rl.CorpusIndex(E, off, chunk_metadata=meta),
                                  **kw)
    for got, want in zip(sharded, bare, strict=True):
        assert np.array_equal(got, want), (got, want)
    return sharded, n_probe


def test_sharded_rank_probe_keeps_the_filter_first_answer(rl, monkeypatch):
    """The float32 scan keeps no counters for the fused bound, so the explicit probe runs; it proves that at most
    20_000 rows are as near as the worst filtered hit, and the filter-first answer stands."""
    import raglite_b200._search as S

    monkeypatch.setattr(S, "FILTER_FIRST_MAX_ROWS", 1_000)
    monkeypatch.setattr(S, "RANK_FIRST_LIMIT", 20_000)
    E, off = make_corpus(30_000, (1, 6), 64, seed=3, fp16_round=True)
    C = len(off) - 1
    tagged = np.arange(C) % 2 == 0
    Q = make_queries(E, 24, seed=4)
    (ids, sims, counts), n_probe = _search_both(rl, E, off, [{"half": int(t)} for t in tagged], Q, monkeypatch,
                                                num_results=10, metadata_filter={"half": 1}, algo="fp32")
    assert n_probe >= 1, "the explicit rank probe must run"
    for b in range(len(Q)):
        check_sql_semantics(E, off, Q[b], ids[b, :counts[b]], sims[b, :counts[b]], k=10, allowed_chunks=tagged)


def test_sharded_rank_probe_cuts_the_filtered_hits(rl, monkeypatch):
    """Query 0's filter keeps the far half of the corpus plus four chunks near it: the probe's cut at the 400 nearest
    rows leaves only the near ones, so the answer differs from the filter-first one (constants scaled: 100_000 -> 60
    matching rows, 1_000_000 -> 400 nearest vectors)."""
    import raglite_b200._search as S

    monkeypatch.setattr(S, "FILTER_FIRST_MAX_ROWS", 60)
    monkeypatch.setattr(S, "RANK_FIRST_LIMIT", 400)
    k = 10
    E, off = make_corpus(600, (1, 5), 64, seed=320, fp16_round=True)
    C = len(off) - 1
    Q = make_queries(E, 3, seed=321, frac_random=0.0)
    order = np.argsort(-ovs.maxsim_scores(E, off, Q[0], "cosine", f64=True))
    tagged = np.zeros(C, dtype=bool)
    tagged[order[C // 2:]] = True
    tagged[order[[0, 2, 5, 30]]] = True
    meta = [{"topic": ["keep"] if t else ["drop"]} for t in tagged]
    (chunk, sim, count), n_probe = _search_both(rl, E, off, meta, Q, monkeypatch, num_results=k,
                                                metadata_filter={"topic": "keep"})
    assert n_probe >= 1, "the explicit rank probe must run"
    took_rank_first = False
    for b in range(len(Q)):
        got = chunk[b, :count[b]].tolist()
        options = [ovs.vector_search_sql(E, off, Q[b], num_results=k, allowed_chunks=tagged, f64=True, filter_first_max=60,
                                         rank_first_limit=lim)[:2] for lim in (400, 399, 401)]   # the row at the cut may fall either way
        assert got in [o[0].tolist() for o in options], (b, got, options[0][0])
        ref_sims = options[[o[0].tolist() for o in options].index(got)][1]
        assert np.allclose(sim[b, :count[b]], ref_sims, atol=1e-4)
        first_ids, _, _ = ovs.vector_search_sql(E, off, Q[b], num_results=k, allowed_chunks=tagged, f64=True)
        took_rank_first |= got != first_ids.tolist()
    assert took_rank_first, "query 0 must differ from the filter-first answer"
