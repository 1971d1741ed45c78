"""Parity at scale (``-m gpu``): the BASELINE configs in full and corpora large enough that the scan's
sampling (S up to 256), periodic threshold refresh, multi-flush ranks, staged-list overflow and the
streaming survivor path all run under the oracle.

The corpus is generated ON the device (seeded) and the oracle reads that very tensor back block by block
(``oracle.vector_search.topn_rows_blocked``: float64 distances, rounded to the FLOAT DuckDB returns,
ties by row), so neither side ever holds a second copy.  Results are compared through the reference's own
``ORDER BY dist LIMIT num_hits -> GROUP BY chunk -> max -> LIMIT k`` (``_search.py:65-79,143-153``)."""

from __future__ import annotations

import json
import os
import tempfile
import threading
from pathlib import Path

import numpy as np
import pytest
from parity import check_sql_from_topn

from oracle import vector_search as ovs

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
N_CHECK = 32   # queries compared per configuration (VERDICT r1: >= 32)


@pytest.fixture(scope="module")
def rl():
    import torch

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import raglite_b200

    return raglite_b200


def _record(name: str, payload: dict) -> None:
    """Append a line (test name + scan statistics) to scale_parity.jsonl in the temporary directory."""
    with (Path(tempfile.gettempdir()) / "scale_parity.jsonl").open("a") as f:
        f.write(json.dumps({"test": name, **payload}) + "\n")


def _oracle_lists(E, Q, n_keep, metric="cosine", rows=None):
    from synth_torch import host_blocks

    q = Q[:N_CHECK].cpu().numpy() if rows is None else Q[rows].cpu().numpy()
    return ovs.topn_rows_blocked(host_blocks(E), q, n_keep, metric, f32_ties=True)


def _compare(lists, vecs, ids, sims, counts, k, num_hits, chunk_base=0, which=None):
    exact = 0
    which = range(len(lists)) if which is None else which
    for j, b in enumerate(which):
        rows, dist = lists[j]
        n = int(counts[b])
        exact += bool(check_sql_from_topn(rows, dist, lambda r: r // vecs, ids[b, :n] - chunk_base, sims[b, :n], k=k,
                                          num_hits=num_hits))
    return exact


def test_c2_full(rl):
    """BASELINE configs[1] in full: 100k chunks x 8 vecs x 384-d fp32, batch 256, top-20."""
    import torch
    from synth_torch import gaussian_corpus_torch, queries_near_rows

    vecs, d, B, k = 8, 384, 256, 20
    E = gaussian_corpus_torch(100_000 * vecs, d, seed=0, device="cuda")
    idx = rl.CorpusIndex(E, vecs_per_chunk=vecs)
    Q = queries_near_rows(E, B, seed=1)
    cfg = rl.RAGLiteConfig(reranker=None)
    ids, sims, counts = rl.vector_search_batch(Q, num_results=k, config=cfg, index=idx)
    num_hits = 80
    lists = _oracle_lists(E, Q, num_hits + 8)
    exact = _compare(lists, vecs, ids, sims, counts, k, num_hits)
    st = idx.scan_stats()
    _record("c2_full", {"checked": N_CHECK, "exact": exact, **st})
    assert exact >= N_CHECK - 1
    # exact-MaxSim mode on the same corpus: per-chunk max over every vector (float64), top-k chunks
    ids, sims, counts = rl.vector_search_batch(Q, num_results=k, config=cfg, index=idx, exact_maxsim=True)
    q64 = Q[:8].double()
    s = (E.double() @ q64.T) / (E.double().norm(dim=1, keepdim=True) * q64.norm(dim=1)[None, :])
    m = s.reshape(-1, vecs, 8).amax(dim=1)
    for b in range(8):
        top = torch.topk(m[:, b], k + 1)
        assert counts[b] == k
        if float(top.values[k - 1] - top.values[k]) > 5e-6:
            assert set(ids[b].tolist()) == set(top.indices[:k].tolist())
        assert np.allclose(sims[b], top.values[:k].cpu().numpy(), atol=1e-4)


BIG_ROWS = 213_340 * 12   # 2.56 M rows x 1024-d (10.5 GB fp32): 20 000 tiles, about 152 per CTA on 132 SMs


@pytest.fixture(scope="module")
def big_gaussian(rl):
    from synth_torch import gaussian_corpus_torch, queries_near_rows

    E = gaussian_corpus_torch(BIG_ROWS, 1024, seed=2, device="cuda")
    idx = rl.CorpusIndex(E, vecs_per_chunk=12)
    Q = queries_near_rows(E, 256, seed=3)
    lists = _oracle_lists(E, Q, 400 + 8)
    yield E, idx, Q, lists
    del idx, E


def test_large_gaussian_batch256(rl, big_gaussian):
    """>= 2.5 M rows x 1024-d, batch 256, top-100 (num_hits 400): the headline shape at 1/6 scale through
    the public batched call -- sampled thresholds, periodic refresh (135 tiles per CTA), multiple flushes."""
    E, idx, Q, lists = big_gaussian
    ids, sims, counts = rl.vector_search_batch(Q, num_results=100, config=rl.RAGLiteConfig(reranker=None), index=idx)
    st = idx.scan_stats()
    exact = _compare(lists, 12, ids, sims, counts, 100, 400)
    _record("large_gaussian_b256", {"checked": N_CHECK, "exact": exact, **st})
    assert st["algo"] == 2 and st["sample_stride"] >= 64
    assert exact >= N_CHECK - 1


@pytest.mark.parametrize("stride,cap", [(256, 0), (2048, 0), (256, 2048)])
def test_large_gaussian_forced_sampling(rl, big_gaussian, stride, cap):
    """The same corpus with the sample made sparser than the heuristic would: S = 256 (the headline shard's
    stride), S = 2048 (a 10-block sample: the first thresholds let most rows through, so the staged hit list
    overflows into direct emits and the online refinement has to rescue the candidate lists), and a tiny
    candidate list (overflow -> threshold-reuse retry -> larger list)."""
    import torch

    E, idx, Q, lists = big_gaussian
    Qs = Q[:N_CHECK].contiguous()
    res = idx.scan_checked(Qs, k=100, num_hits=400, sample_stride=stride, cand_cap=cap)
    st = idx.scan_stats()
    sim, chunk, count = rl.merge_hits(res.hit_sim, res.hit_chunk, res.hit_count, num_hits=400, k=100)
    torch.cuda.synchronize()
    exact = _compare(lists, 12, chunk.cpu().numpy(), sim.cpu().numpy(), count.cpu().numpy(), 100, 400)
    _record(f"large_gaussian_S{stride}_cap{cap}", {"checked": N_CHECK, "exact": exact, **st})
    assert int(res.status.max()) == 0
    assert exact >= N_CHECK - 1


def test_large_clustered(rl):
    """Clustered / anisotropic data (tight clusters of thousands of near-duplicates + a low-rank background,
    float16-rounded like RAGLite's stored embeddings): whole clusters sit inside the coarse key's error
    band of the cut, so the survivor window overflows and ``finalize`` must stream.  Both storages."""
    import torch
    from synth_torch import clustered_corpus_torch, queries_near_rows

    vecs, d, B, k, num_hits = 12, 1024, 256, 100, 400
    E, cl = clustered_corpus_torch(BIG_ROWS, d, seed=4, device="cuda", mean_cluster=1536, max_cluster=8192)
    sizes = np.bincount(cl[cl >= 0])
    big_tight = np.nonzero((sizes >= 4500) & (np.arange(len(sizes)) % 4 <= 1))[0]   # spreads 0.02 / 0.05
    assert len(big_tight) >= 4
    rng = np.random.default_rng(5)
    n_near = B - B // 4
    rows = rng.integers(0, BIG_ROWS, size=n_near)
    for i in range(0, n_near, 2):   # every other "near" query aims into a big tight cluster
        rows[i] = rng.choice(np.nonzero(cl == big_tight[(i // 2) % len(big_tight)])[0])
    Q = queries_near_rows(E, B, seed=6, rows=rows)
    check = list(range(0, 2 * N_CHECK, 2))[: N_CHECK // 2] + list(range(1, 2 * N_CHECK, 2))[: N_CHECK // 2]
    lists = _oracle_lists(E, Q, num_hits + 8, rows=check)
    cfg = rl.RAGLiteConfig(reranker=None)
    for storage in ("fp32", "fp16"):
        idx = rl.CorpusIndex(E, vecs_per_chunk=vecs, storage=storage)
        torch.cuda.synchronize()
        ids, sims, counts = rl.vector_search_batch(Q, num_results=k, config=cfg, index=idx)
        st = idx.scan_stats()
        exact = _compare(lists, vecs, ids, sims, counts, k, num_hits, which=check)
        _record(f"large_clustered_{storage}", {"checked": len(check), "exact": exact, "fp32_fallback_queries": 0, **st})
        assert st["survivors_max"] > 4096, "the generator must exercise the streaming survivor path"
        assert exact >= len(check) - 2
        del idx


@pytest.mark.parametrize("metric", ["cosine", "dot", "l2"])
def test_several_query_groups_per_tile(rl, metric):
    """B > 128 (BASELINE configs[2] runs B = 1024): the scan walks every corpus tile once per group of 128
    queries inside ONE launch; 600 queries = four full groups and a ragged fifth."""
    from synth_torch import gaussian_corpus_torch, host_blocks, queries_near_rows

    vecs, d, B, k = 4, 256, 600, 20
    E = gaussian_corpus_torch(60_000 * vecs, d, seed=7, device="cuda")
    if metric != "cosine":
        E *= 1.5
    idx = rl.CorpusIndex(E, vecs_per_chunk=vecs)
    Q = queries_near_rows(E, B, seed=8)
    cfg = rl.RAGLiteConfig(reranker=None, vector_search_distance_metric=metric)
    ids, sims, counts = rl.vector_search_batch(Q, num_results=k, config=cfg, index=idx)
    st = idx.scan_stats()
    check = list(range(0, B, 7))
    lists = ovs.topn_rows_blocked(host_blocks(E), Q[check].cpu().numpy(), 80 + 8, metric, f32_ties=True)
    exact = _compare(lists, vecs, ids, sims, counts, k, 80, which=check)
    _record(f"multi_group_{metric}", {"checked": len(check), "exact": exact, **st})
    assert st["algo"] == 2 and exact >= len(check) - 2
    ids2, sims2, counts2 = rl.vector_search_batch(Q[256:512], num_results=k, config=cfg, index=idx)   # one group, same queries
    assert np.array_equal(ids2, ids[256:512]) and np.array_equal(counts2, counts[256:512])
    assert np.allclose(sims2, sims[256:512], atol=0, equal_nan=True)


def test_concurrent_searches_from_threads(rl):
    """Four host threads search one index at once, each on its own CUDA stream (reference callers use
    thread pools, ``_rag.py:317``), with a candidate list small enough that every call overflows and
    retries: the retry must read its own thresholds, not another thread's."""
    import torch
    from synth import make_corpus, make_queries

    E, off = make_corpus(6000, 4, 64, seed=21)
    idx = rl.CorpusIndex(E, off)
    Qs = [make_queries(E, 24, seed=100 + t) for t in range(4)]
    want = []
    for Qt in Qs:
        r = idx.scan_checked(torch.from_numpy(Qt).cuda(), k=10, num_hits=40)
        want.append((r.hit_sim.cpu().numpy().copy(), r.hit_chunk.cpu().numpy().copy()))
    errors: list[BaseException] = []
    got: list = [None] * 4

    def work(t: int) -> None:
        try:
            with torch.cuda.stream(torch.cuda.Stream()):
                Qd = torch.from_numpy(Qs[t]).cuda()
                for _ in range(6):
                    r = idx.scan_checked(Qd, k=10, num_hits=40, sample_stride=32, cand_cap=256)
                    torch.cuda.current_stream().synchronize()
                    assert int(r.status.max()) == 0
                    got[t] = (r.hit_sim.cpu().numpy(), r.hit_chunk.cpu().numpy())
                    assert np.array_equal(got[t][1], want[t][1]) and np.allclose(got[t][0], want[t][0], atol=1e-6)
        except BaseException as e:  # noqa: BLE001
            errors.append(e)

    threads = [threading.Thread(target=work, args=(t,)) for t in range(4)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors[0]
    assert len(idx._ws) >= 2   # one workspace per stream


def test_filtered_search_uses_cached_device_mask(rl):
    """Metadata filters resolve through the inverted index + ``rl_row_mask``; a repeated filter costs no
    host pass over the chunk table; appends and deletes invalidate the cache."""
    from synth import make_corpus, make_queries

    E, off = make_corpus(4000, (1, 6), 64, seed=31, fp16_round=True)
    n_chunks = len(off) - 1
    meta = [{"lang": "en" if c % 2 else "nl", "tags": [f"t{c % 5}", f"u{c % 7}"]} for c in range(n_chunks)]
    idx = rl.CorpusIndex(E, off, chunk_ids=[str(c) for c in range(n_chunks)], chunk_metadata=meta)
    cfg = rl.RAGLiteConfig(reranker=None)
    Q = make_queries(E, 6, seed=32)
    flt = {"lang": "en", "tags": ["t3", "u2"]}
    allowed = np.array([c % 2 == 1 and c % 5 == 3 and c % 7 == 2 for c in range(n_chunks)])
    from parity import check_sql_semantics

    for _ in range(2):
        ids, sims, counts = rl.vector_search_batch(Q, num_results=5, metadata_filter=flt, config=cfg, index=idx)
        for b in range(len(Q)):
            check_sql_semantics(E, off, Q[b], ids[b, :counts[b]], sims[b, :counts[b]], k=5, allowed_chunks=allowed)
    assert len(idx._filter_cache) == 1
    gone = [str(c) for c in np.nonzero(allowed)[0][:3]]
    idx.delete_chunks(gone)
    assert len(idx._filter_cache) == 0
    allowed[[int(g) for g in gone]] = False
    ids, sims, counts = rl.vector_search_batch(Q, num_results=5, metadata_filter=flt, config=cfg, index=idx)
    for b in range(len(Q)):
        assert not set(ids[b, :counts[b]].tolist()) & {int(g) for g in gone}
        check_sql_semantics(E, off, Q[b], ids[b, :counts[b]], sims[b, :counts[b]], k=5, allowed_chunks=allowed)


def test_sharded_index_growth_is_guarded(rl):
    """ADVICE r1: a shard may only grow while it stays below the next shard's global chunk range."""
    from synth import make_corpus

    from raglite_b200._dist import ShardedIndex

    E, off = make_corpus(40, 2, 32, seed=41)
    a = rl.CorpusIndex(E[:40], vecs_per_chunk=2, chunk_base=0)
    sh = ShardedIndex(a, group=None)
    sh.ranges = [(0, 20), (20, 20)]            # as gathered from a second rank with a contiguous base
    with pytest.raises(ValueError, match="next shard"):
        a.append(E[40:44], vecs_per_chunk=2)
    sh.ranges = [(0, 20), (ShardedIndex.shard_bases(2)[1], 20)]   # spaced bases: room to grow
    a.append(E[40:44], vecs_per_chunk=2)
    assert a.n_chunks == 22
