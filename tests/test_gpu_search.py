"""GPU parity tests proper: the CUDA path (through the C-ABI) against the oracle on seeded inputs."""

from __future__ import annotations

import json

import numpy as np
import pytest
from fake_llama import FakeLlama
from parity import check_exact_maxsim, check_sql_semantics
from synth import make_corpus, make_queries, random_orthogonal

from oracle import pool as opool
from oracle import vector_search as ovs

pytestmark = pytest.mark.gpu

ALGOS = ["fp32", "tcgen05"]


@pytest.fixture(scope="module")
def rl():
    import torch

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import raglite_b200

    return raglite_b200


def _algo_ok(rl, algo, d, metric="cosine"):
    if algo == "tcgen05":
        from raglite_b200 import _lib
        import ctypes

        p = _lib.ScanParams()
        p.n_rows, p.d, p.ld, p.B, p.k, p.metric, p.max_vecs_per_chunk = 1024, d, d, 1, 1, _lib.RL_METRIC[metric], 1
        p.E = 256
        p.algo = 2
        if _lib.load().rl_maxsim_workspace_bytes(ctypes.byref(p)) == 0:
            pytest.skip("tcgen05 scan does not support this shape/metric")


def test_row_stats_and_chunk_map(rl):
    E, off = make_corpus(300, (1, 9), 100, seed=1, normalize=False)
    idx = rl.CorpusIndex(E, off)
    nrm = np.linalg.norm(E.astype(np.float64), axis=1)
    assert np.allclose(idx.inv_norm.cpu().numpy(), 1 / nrm, rtol=1e-6)
    assert np.allclose(idx.sq_norm.cpu().numpy(), nrm**2, rtol=1e-6)
    assert np.array_equal(idx.row_chunk.cpu().numpy(), ovs.row_to_chunk(off).astype(np.int32))
    st = idx.stats.cpu().numpy()
    assert np.isclose(st[0], nrm.max(), rtol=1e-6) and np.isclose(st[1], np.abs(E).max(), rtol=1e-6)


@pytest.mark.parametrize("dtype", [np.float16, np.float32])
def test_adapter_apply_matches_reference_expression(rl, dtype):
    import torch

    d = 96
    A = random_orthogonal(d, seed=5)
    Q = make_queries(np.zeros((0, d), np.float32), 37, seed=3).astype(dtype)
    idx = rl.CorpusIndex(np.eye(d, dtype=np.float32))
    idx.set_query_adapter(A)
    got = idx.apply_adapter(torch.from_numpy(Q.astype(np.float32)).cuda(), round_fp16=(dtype == np.float16)).cpu().numpy()
    want = np.stack([ovs.apply_query_adapter(A, q) for q in Q])      # (A @ q).astype(q.dtype), _search.py:62
    assert want.dtype == dtype
    mism = got != want.astype(np.float32)
    assert mism.mean() < 1e-3                                          # rounding-boundary cases only
    assert np.allclose(got, want.astype(np.float32), atol=2e-3 if dtype == np.float16 else 1e-6)


@pytest.mark.parametrize("name", ["pool_small", "pool_multi", "pool_nonorm", "pool_wide"])
def test_late_chunking_pool_matches_reference_golden(rl, golden_dir, name):
    from raglite_b200 import _embed

    z = np.load(golden_dir / f"{name}.npz")
    meta = json.loads(bytes(z["meta"]).decode())
    llm = FakeLlama(n_ctx=meta["n_ctx"], dim=meta["dim"], seed=meta["seed"])
    cfg = rl.RAGLiteConfig(embedder="llama-cpp-python/fake/fake.gguf@64", embedder_normalize=meta["normalize"], reranker=None)
    rl.register_token_embedder(cfg.embedder, llm)
    got = rl.embed_strings(meta["sentences"], config=cfg)
    want = z["late_chunking"]
    assert got.dtype == np.float16 and got.shape == want.shape            # tests/test_embed.py:24
    assert np.all(np.isfinite(got))
    ulp = np.abs(got.view(np.int16).astype(np.int32) - want.view(np.int16).astype(np.int32))
    assert ulp.max() <= 1 and (ulp > 0).mean() < 1e-3
    simple = _embed.embed_strings_without_late_chunking(meta["sentences"][:7], config=cfg)
    ulp = np.abs(simple.view(np.int16).astype(np.int32) - z["simple"].view(np.int16).astype(np.int32))
    assert ulp.max() <= 1 and (ulp > 0).mean() < 1e-3
    assert np.array_equal(opool.embed_with_llama(meta["sentences"], llm, normalize=meta["normalize"]).view(np.uint16),
                          want.view(np.uint16))


CASES = [
    # n_chunks, vecs, dim, B, k, seed
    (1000, 1, 384, 4, 5, 0),        # BASELINE configs[0]: 1k chunks x 1 vec x 384 (bge-small)
    (700, 8, 64, 9, 20, 1),
    (513, (1, 16), 128, 5, 10, 2),  # variable vectors per chunk (CSR coverage)
    (3000, 4, 32, 3, 3, 3),
    (40, 3, 16, 2, 8, 4),           # fewer chunks than some k * oversample
]


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("case", CASES)
def test_vector_search_batch_sql_semantics(rl, case, algo):
    n_chunks, vecs, dim, B, k, seed = case
    _algo_ok(rl, algo, dim)
    E, off = make_corpus(n_chunks, vecs, dim, seed=seed)
    Q = make_queries(E, B, seed=seed + 100)
    idx = rl.CorpusIndex(E, off)
    cfg = rl.RAGLiteConfig(reranker=None)
    ids, sims, counts = rl.vector_search_batch(Q, num_results=k, config=cfg, index=idx, algo=algo)
    for b in range(B):
        n = counts[b]
        check_sql_semantics(E, off, Q[b], ids[b, :n], sims[b, :n], k=k)
        assert np.all(ids[b, n:] == -1)


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("case", CASES)
def test_vector_search_batch_exact_maxsim(rl, case, algo):
    n_chunks, vecs, dim, B, k, seed = case
    _algo_ok(rl, algo, dim)
    E, off = make_corpus(n_chunks, vecs, dim, seed=seed)
    Q = make_queries(E, B, seed=seed + 200)
    idx = rl.CorpusIndex(E, off)
    ids, sims, counts = rl.vector_search_batch(Q, num_results=k, config=rl.RAGLiteConfig(reranker=None), index=idx,
                                               exact_maxsim=True, algo=algo)
    for b in range(B):
        n = counts[b]
        assert n == min(k, n_chunks)
        check_exact_maxsim(E, off, Q[b], ids[b, :n], sims[b, :n], k=k)


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("metric", ["cosine", "dot", "l2"])
def test_metrics(rl, metric, algo):
    _algo_ok(rl, algo, 48, metric)
    E, off = make_corpus(900, (1, 6), 48, seed=7, normalize=False)
    E *= np.random.default_rng(1).uniform(0.5, 2.0, size=(E.shape[0], 1)).astype(np.float32)
    Q = 1.7 * make_queries(E, 6, seed=8)
    idx = rl.CorpusIndex(E, off)
    cfg = rl.RAGLiteConfig(vector_search_distance_metric=metric, reranker=None)
    ids, sims, counts = rl.vector_search_batch(Q, num_results=7, config=cfg, index=idx, algo=algo)
    ids2, sims2, counts2 = rl.vector_search_batch(Q, num_results=7, config=cfg, index=idx, algo=algo, exact_maxsim=True)
    for b in range(len(Q)):
        check_sql_semantics(E, off, Q[b], ids[b, :counts[b]], sims[b, :counts[b]], k=7, metric=metric)
        check_exact_maxsim(E, off, Q[b], ids2[b, :counts2[b]], sims2[b, :counts2[b]], k=7, metric=metric)


@pytest.mark.parametrize("d", [3, 17, 50])
def test_odd_dimensions_take_the_fp32_scan(rl, d):
    E, off = make_corpus(400, 2, d, seed=d)
    Q = make_queries(E, 3, seed=d + 1)
    idx = rl.CorpusIndex(E, off)
    ids, sims, counts = rl.vector_search_batch(Q, num_results=5, config=rl.RAGLiteConfig(reranker=None), index=idx)
    for b in range(3):
        check_sql_semantics(E, off, Q[b], ids[b, :counts[b]], sims[b, :counts[b]], k=5)


@pytest.mark.parametrize("algo", ALGOS)
def test_sampled_two_pass_path_and_oversample_rule(rl, algo):
    """Corpus large enough that the scan samples (S > 1) and the emit pass runs; chunk_max_size and
    oversample change num_hits as in _search.py:66-67."""
    _algo_ok(rl, algo, 64)
    E, off = make_corpus(6000, 8, 64, seed=11)
    Q = make_queries(E, 16, seed=12)
    idx = rl.CorpusIndex(E, off)
    cfg = rl.RAGLiteConfig(chunk_max_size=1024, reranker=None)
    ids, sims, counts = rl.vector_search_batch(Q, num_results=20, oversample=6, config=cfg, index=idx, algo=algo)
    st = idx.scan_stats()
    assert st["sample_stride"] > 1 and st["launches"] >= 5
    for b in range(len(Q)):
        check_sql_semantics(E, off, Q[b], ids[b, :counts[b]], sims[b, :counts[b]], k=20, oversample=6, chunk_max_size=1024)
    ids, sims, counts = rl.vector_search_batch(Q, num_results=20, config=cfg, index=idx, algo=algo, exact_maxsim=True)
    for b in range(len(Q)):
        check_exact_maxsim(E, off, Q[b], ids[b, :counts[b]], sims[b, :counts[b]], k=20)


def test_candidate_overflow_retry(rl):
    """Adversarial order: rows sorted by similarity to the query, tiny candidate capacity."""
    import torch

    E, off = make_corpus(4000, 4, 32, seed=21)
    q = make_queries(E, 1, seed=22)
    order = np.argsort(E @ q[0])          # ascending similarity: every later block beats the sample
    E = np.ascontiguousarray(E[order])
    idx = rl.CorpusIndex(E, off)
    Q = torch.from_numpy(q).cuda()
    res = idx.scan(Q, k=10, num_hits=40, sample_stride=16, cand_cap=256, algo="fp32")
    assert int(res.status.cpu()[0]) & 1   # overflow reported
    res = idx.scan_checked(Q, k=10, num_hits=40, sample_stride=16, cand_cap=256, algo="fp32")
    assert int(res.status.cpu()[0]) == 0
    sim, chunk, count = rl.merge_hits(res.hit_sim, res.hit_chunk, res.hit_count, num_hits=40, k=10)
    n = int(count[0])
    check_sql_semantics(E, off, q[0], chunk[0, :n].cpu().numpy(), sim[0, :n].cpu().numpy(), k=10)


def test_duplicates_and_ties(rl):
    E, off = make_corpus(300, 4, 32, seed=31)
    E[400:440] = E[7]                      # 40 identical vectors spread over 10 chunks
    Q = E[[7]].copy()
    idx = rl.CorpusIndex(E, off)
    ids, sims, counts = rl.vector_search_batch(Q, num_results=5, config=rl.RAGLiteConfig(reranker=None), index=idx,
                                               exact_maxsim=True)
    assert counts[0] == 5 and np.allclose(sims[0], 1.0, atol=1e-6)
    s = ovs.maxsim_scores(E, off, Q[0])
    assert np.allclose(s[ids[0]], 1.0, atol=1e-9)


def test_empty_database_and_tiny_inputs(rl):
    cfg = rl.RAGLiteConfig(db_url="mem://empty", reranker=None)
    idx = rl.CorpusIndex(np.zeros((0, 16), np.float32))
    rl.register_index(cfg, idx)
    ids, scores = rl.vector_search(np.ones(16, np.float32), num_results=5, config=cfg)
    assert ids == [] and scores == []     # tests/test_search.py:76-85
    E, off = make_corpus(1, 1, 16, seed=1)
    idx = rl.CorpusIndex(E, off, chunk_ids=["only"])
    rl.register_index(cfg, idx)
    ids, scores = rl.vector_search(E[0].astype(np.float16), num_results=5, config=cfg)
    assert ids == ["only"] and isinstance(scores[0], float) and abs(scores[0] - 1.0) < 1e-3


def test_vector_search_dropin_with_adapter_and_metadata(rl):
    E, off = make_corpus(500, (1, 5), 64, seed=41, fp16_round=True)
    n_chunks = len(off) - 1
    meta = [{"topic": ["Physics"] if c % 3 == 0 else ["Math"], "type": ["Paper"]} for c in range(n_chunks)]
    cfg = rl.RAGLiteConfig(db_url="mem://dropin", reranker=None)
    idx = rl.CorpusIndex(E, off, chunk_ids=[f"chunk-{c}" for c in range(n_chunks)], chunk_metadata=meta)
    A = random_orthogonal(64, seed=9)
    idx.set_query_adapter(A)
    rl.register_index(cfg, idx)
    q = make_queries(E, 1, seed=42)[0].astype(np.float16)      # string queries arrive as fp16 (_embed.py:140)
    ids, scores = rl.vector_search(q, num_results=5, config=cfg)
    assert len(ids) == len(scores) == 5 and all(isinstance(i, str) for i in ids) and all(isinstance(s, float) for s in scores)
    got = [int(i.split("-")[1]) for i in ids]
    check_sql_semantics(E, off, q, got, scores, k=5, adapter=A)
    cfg_off = rl.RAGLiteConfig(db_url="mem://dropin", vector_search_query_adapter=False, reranker=None)
    _, scores_no = rl.vector_search(q, num_results=5, config=cfg_off)
    assert scores != scores_no                                  # tests/test_query_adapter.py:37-40
    allowed = np.array([c % 3 == 0 for c in range(n_chunks)])
    ids_f, sc_f = rl.vector_search(q, num_results=5, metadata_filter={"type": "Paper", "topic": "Physics"}, config=cfg)
    got = [int(i.split("-")[1]) for i in ids_f]
    assert 0 < len(got) <= 5 and all(g % 3 == 0 for g in got)    # tests/test_search.py:88-127
    check_sql_semantics(E, off, q, got, sc_f, k=5, adapter=A, allowed_chunks=allowed)
    ids_e, _ = rl.vector_search(q, num_results=5, metadata_filter={"type": "Paper", "topic": "Chemistry"}, config=cfg)
    assert ids_e == []


def test_two_shards_merge_equals_single_index(rl):
    import torch

    E, off = make_corpus(2000, (1, 8), 64, seed=51)
    Q = make_queries(E, 8, seed=52)
    cut_chunk = 900
    cut_row = int(off[cut_chunk])
    a = rl.CorpusIndex(E[:cut_row], off[: cut_chunk + 1])
    b = rl.CorpusIndex(E[cut_row:], off[cut_chunk:] - cut_row, chunk_base=cut_chunk)
    Qd = torch.from_numpy(Q).cuda()
    for num_hits in (80, 0):
        ra = a.scan_checked(Qd, k=20, num_hits=num_hits)
        rb = b.scan_checked(Qd, k=20, num_hits=num_hits)
        sim, chunk, count = rl.merge_hits(torch.stack([ra.hit_sim, rb.hit_sim]), torch.stack([ra.hit_chunk, rb.hit_chunk]),
                                          torch.stack([ra.hit_count, rb.hit_count]), num_hits=num_hits, k=20)
        sim, chunk, count = sim.cpu().numpy(), chunk.cpu().numpy(), count.cpu().numpy()
        for i in range(len(Q)):
            if num_hits:
                check_sql_semantics(E, off, Q[i], chunk[i, :count[i]], sim[i, :count[i]], k=20)
            else:
                check_exact_maxsim(E, off, Q[i], chunk[i, :count[i]], sim[i, :count[i]], k=20)


def test_update_query_adapter_matches_oracle_fit(rl):
    """Adapter fit (SURVEY 8f-4): GPU retrieval + MaxSim picks, then the reference's float64 algebra."""
    from oracle import adapter as oad

    E, off = make_corpus(400, (1, 6), 48, seed=61)
    rng = np.random.default_rng(62)
    cfg = rl.RAGLiteConfig(db_url="mem://fit", reranker=None)
    idx = rl.CorpusIndex(E, off)
    rl.register_index(cfg, idx)
    evals = []
    for _ in range(12):
        c = int(rng.integers(0, len(off) - 1))
        q = E[off[c]] + 0.4 * rng.standard_normal(48).astype(np.float32)
        evals.append((q / np.linalg.norm(q), [c, int(rng.integers(0, len(off) - 1))]))
    A = rl.update_query_adapter(evals, optimize_top_k=10, config=cfg)
    assert A.shape == (48, 48) and np.isfinite(A).all()                  # tests/test_query_adapter.py:24-27
    assert np.allclose(A @ A.T, np.eye(48), atol=1e-9)                    # orthogonal Procrustes
    assert np.array_equal(idx.query_adapter, A)
    # oracle: same triplets through the NumPy restatement
    Qs, Ts = [], []
    for q, rel in evals:
        ids, _ = ovs.maxsim_topk_exact(E, off, q, 10)
        sql_ids, _, _ = ovs.vector_search_sql(E, off, q, num_results=10, f64=True)
        is_rel = np.array([c in rel for c in sql_ids])
        if not is_rel.any() or is_rel.all():
            continue
        best = np.stack([E[off[c]:off[c + 1]][oad.maxsim_row(E[off[c]:off[c + 1]], q)] for c in sql_ids])
        Ts.append(oad.optimize_query_target(q, best[is_rel], best[~is_rel], alpha=0.05)); Qs.append(q)
    want = oad.fit_query_adapter(np.vstack(Qs), np.vstack(Ts), "cosine")
    assert np.allclose(A, want, atol=1e-8)
    _, s_on = rl.vector_search(evals[0][0], num_results=5, config=cfg)
    _, s_off = rl.vector_search(evals[0][0], num_results=5, config=rl.RAGLiteConfig(db_url="mem://fit", reranker=None, vector_search_query_adapter=False))
    assert s_on != s_off


def test_index_from_chunk_embedding_rows(rl):
    """The chunk_embedding table read in insertion order (SURVEY 8f-1)."""
    E, off = make_corpus(50, (1, 5), 32, seed=71)
    row_ids = [f"doc-{c // 7}-chunk-{c}" for c in ovs.row_to_chunk(off)]
    idx = rl.CorpusIndex.from_chunk_embedding_rows(row_ids, E)
    assert np.array_equal(idx.chunk_off, off) and idx.chunk_ids[3] == "doc-0-chunk-3"
    cfg = rl.RAGLiteConfig(db_url="mem://rows", reranker=None)
    rl.register_index(cfg, idx)
    q = make_queries(E, 1, seed=72)[0]
    ids, scores = rl.vector_search(q, num_results=4, config=cfg)
    ref_ids, ref_sims, _ = ovs.vector_search_sql(E, off, q, num_results=4, f64=True)
    assert ids == [f"doc-{c // 7}-chunk-{c}" for c in ref_ids] and np.allclose(scores, ref_sims, atol=1e-4)
    with pytest.raises(ValueError):
        rl.CorpusIndex.from_chunk_embedding_rows(["a", "b", "a"], E[:3])


@pytest.mark.parametrize("metric", ["cosine", "dot", "l2"])
def test_fp16_storage_matches_oracle(rl, metric):
    """Lossless float16 corpus layout (SURVEY 8f-1): RAGLite's embeddings are fp16-rounded (_embed.py:140)."""
    E, off = make_corpus(3000, (1, 9), 128, seed=81, fp16_round=True)
    Q = make_queries(E, 12, seed=82)
    idx16 = rl.CorpusIndex(E, off, storage="fp16")
    assert idx16.E.dtype.is_floating_point and idx16.E.element_size() == 2
    cfg = rl.RAGLiteConfig(vector_search_distance_metric=metric, reranker=None)
    ids, sims, counts = rl.vector_search_batch(Q, num_results=10, config=cfg, index=idx16)
    ids2, sims2, counts2 = rl.vector_search_batch(Q, num_results=10, config=cfg, index=idx16, exact_maxsim=True)
    for b in range(len(Q)):
        check_sql_semantics(E, off, Q[b], ids[b, :counts[b]], sims[b, :counts[b]], k=10, metric=metric)
        check_exact_maxsim(E, off, Q[b], ids2[b, :counts2[b]], sims2[b, :counts2[b]], k=10, metric=metric)
    st = idx16.scan_stats()
    assert st["algo"] == 2


@pytest.mark.parametrize("d,n_chunks,B", [(72, 700, 5), (96, 1500, 64), (104, 900, 7), (200, 2600, 256), (1024, 300, 33)])
def test_fp16_storage_tensor_map_edges(rl, d, n_chunks, B):
    """fp16 storage brings the corpus tiles through a TMA tensor map (box 64 halves x 128 rows): dimensions that
    end inside a box (72, 96, 104, 200: the tail reads as zeros), a last tile with fewer than 128 rows, an odd number
    of tiles (the second CTA of the last pair has none) and batches that leave the pair kernel (B < 64)."""
    E, off = make_corpus(n_chunks, (1, 7), d, seed=500 + d, fp16_round=True)
    Q = make_queries(E, B, seed=501 + d)
    idx16 = rl.CorpusIndex(E, off, storage="fp16")
    cfg = rl.RAGLiteConfig(reranker=None)
    ids, sims, counts = rl.vector_search_batch(Q, num_results=8, config=cfg, index=idx16)
    assert idx16.scan_stats()["algo"] == 2
    for b in range(0, B, max(1, B // 12)):
        check_sql_semantics(E, off, Q[b], ids[b, :counts[b]], sims[b, :counts[b]], k=8)


def test_fp16_storage_rejects_lossy_input(rl):
    E, off = make_corpus(100, 2, 64, seed=83)          # general float32 values: not representable
    with pytest.raises(ValueError):
        rl.CorpusIndex(E, off, storage="fp16")


@pytest.mark.parametrize("algo", ALGOS)
def test_block_boundaries_and_batch_groups(rl, algo):
    """Rows exactly on / one past a 128-row block edge; batches of 1, 257 (three query groups of 128) and 1025 (the
    tensor-core scan's second launch: more than 8 groups)."""
    _algo_ok(rl, algo, 64)
    for n_rows in (128, 129, 256 * 3):
        E, off = make_corpus(n_rows, 1, 64, seed=n_rows)
        idx = rl.CorpusIndex(E, off)
        for B in (1, 257, 1025):
            Q = make_queries(E, B, seed=B)
            ids, sims, counts = rl.vector_search_batch(Q, num_results=3, config=rl.RAGLiteConfig(reranker=None), index=idx, algo=algo)
            for b in (0, B - 1):
                check_sql_semantics(E, off, Q[b], ids[b, :counts[b]], sims[b, :counts[b]], k=3)


def test_zero_rows_and_k_larger_than_corpus(rl):
    E, off = make_corpus(30, 2, 32, seed=91)
    E[10] = 0.0                                            # an all-zero embedding row
    idx = rl.CorpusIndex(E, off)
    Q = make_queries(E, 3, seed=92)
    ids, sims, counts = rl.vector_search_batch(Q, num_results=50, config=rl.RAGLiteConfig(reranker=None), index=idx,
                                               exact_maxsim=True)
    assert np.all(counts == 30) and np.all(np.isfinite(sims[:, :30]))
    for b in range(3):
        assert sorted(ids[b, :30].tolist()) == list(range(30))
        assert np.all(np.diff(sims[b, :30]) <= 1e-6)


def test_selection_larger_than_finalize_window_is_rejected(rl):
    from raglite_b200._lib import RagliteB200Error

    E, off = make_corpus(200, 40, 32, seed=93)             # 40 vectors per chunk
    idx = rl.CorpusIndex(E, off)
    Q = make_queries(E, 1, seed=94)
    with pytest.raises((RagliteB200Error, ValueError)):   # (k - 1) * 40 + 1 = 4361 rows would have to be ranked exactly
        rl.vector_search_batch(Q, num_results=110, config=rl.RAGLiteConfig(reranker=None), index=idx, exact_maxsim=True)
    # ... 3961 fit the 4096-entry window
    ids, sims, counts = rl.vector_search_batch(Q, num_results=100, config=rl.RAGLiteConfig(reranker=None), index=idx, exact_maxsim=True)
    check_exact_maxsim(E, off, Q[0], ids[0, :counts[0]], sims[0, :counts[0]], k=100)


def test_search_and_rerank_chunk_spans_pipeline(rl):
    """vector_search -> rerank_chunks -> span collation over one registered index (the callers right
    after the hot path, reference _search.py:400-433)."""
    from raglite_b200._rerank import ScoreFnRanker

    E, off = make_corpus(60, (1, 4), 32, seed=95)
    n = len(off) - 1
    chunks = [rl.Chunk(id=f"c{c}", document_id=f"doc{c // 10}", index=c % 10, body=f"body {c} " * (1 + c % 5)) for c in range(n)]
    idx = rl.CorpusIndex(E, off, chunk_ids=[c.id for c in chunks], chunks=chunks)
    cfg = rl.RAGLiteConfig(db_url="mem://spans", reranker=ScoreFnRanker(lambda q, docs: [len(d) for d in docs]))
    rl.register_index(cfg, idx)
    rl.register_token_embedder(cfg.embedder, FakeLlama(n_ctx=64, dim=32, seed=3))
    spans = rl.search_and_rerank_chunk_spans("alpha beta gamma", num_results=4, oversample=2, config=cfg)
    assert 1 <= len(spans) <= 4 * 3 and all(isinstance(s, rl.ChunkSpan) for s in spans)
    for s in spans:                                        # contiguous runs of one document
        assert len({c.document_id for c in s.chunks}) == 1
        assert [c.index for c in s.chunks] == list(range(s.chunks[0].index, s.chunks[0].index + len(s.chunks)))
    top = rl.search_and_rerank_chunks("alpha beta gamma", num_results=4, oversample=2, config=cfg)
    assert len(top) == 4 and [len(str(c)) for c in top] == sorted((len(str(c)) for c in top), reverse=True)


def _by_id(idx, rl, Q, k):
    """Search ``idx`` and spell the hits as (chunk id, score) lists -- comparable across layouts."""
    chunk, sim, count = rl.vector_search_batch(Q, num_results=k, index=idx, config=rl.RAGLiteConfig(reranker=None))
    return [[(idx.chunk_id_of(int(c)), float(s)) for c, s in zip(chunk[b, :count[b]], sim[b, :count[b]])]
            for b in range(len(Q))]


@pytest.mark.parametrize("storage", ["fp32", "fp16"])
def test_index_follows_inserts_and_deletes(rl, storage):
    """SURVEY 8f-1: the index tracks the chunk_embedding table as ``insert_documents`` flushes rows
    (``_insert.py:247-255``) and ``delete_documents`` cascades (``_delete.py:146-152``).  After every
    mutation the search must equal a search over an index built from scratch on the surviving rows,
    and that one is checked against the oracle."""
    d, k = 64, 7
    parts = []
    for f, n in enumerate((700, 450, 300)):
        E, off = make_corpus(n, (1, 6), d, seed=90 + f, fp16_round=True)
        owner = ovs.row_to_chunk(off)
        parts.append((E, [f"f{f}-c{c}" for c in owner], [rl.Chunk(id=f"f{f}-c{c}", document_id=f"doc-{f}-{c // 9}", index=c % 9)
                                                         for c in range(n)]))
    idx = rl.CorpusIndex.from_chunk_embedding_rows(parts[0][1], parts[0][0], chunks=parts[0][2], storage=storage)
    for E, row_ids, chunks in parts[1:]:
        idx.append_chunk_embedding_rows(row_ids, E, chunks=chunks)
    E_all = np.vstack([p[0] for p in parts])
    ids_all = [i for p in parts for i in p[1]]
    chunks_all = [c for p in parts for c in p[2]]
    fresh = rl.CorpusIndex.from_chunk_embedding_rows(ids_all, E_all, storage=storage)
    assert idx.n_rows == fresh.n_rows and np.array_equal(idx.chunk_off, fresh.chunk_off) and idx.max_vecs == fresh.max_vecs
    Q = make_queries(E_all, 12, seed=95)
    assert _by_id(idx, rl, Q, k) == _by_id(fresh, rl, Q, k)
    with pytest.raises(ValueError):
        idx.append_chunk_embedding_rows(["f0-c1"], E_all[:1], chunks=[rl.Chunk(id="f0-c1")])   # already present
    with pytest.raises(ValueError):
        idx.append_chunk_embedding_rows(["new"], E_all[:1])                                    # chunks are tracked

    # deletes: by chunk id and by document (the nearest neighbours of the first queries go away)
    doomed = {hits[0][0] for hits in _by_id(idx, rl, Q[:6], k)} | {"f1-c3", "not-there"}
    n_del = idx.delete_chunks(sorted(doomed))
    assert n_del == len(doomed) - 1 and idx.delete_chunks(sorted(doomed)) == 0
    gone_docs = ["doc-2-0", "doc-0-5"]
    n_del += idx.delete_documents(gone_docs)
    dead = doomed | {c.id for c in chunks_all if c.document_id in gone_docs}
    assert idx.n_live_chunks == len(chunks_all) - len(dead - {"not-there"}) == len(chunks_all) - n_del
    keep_rows = np.array([i not in dead for i in ids_all])
    ids_kept = [i for i in ids_all if i not in dead]
    fresh2 = rl.CorpusIndex.from_chunk_embedding_rows(ids_kept, E_all[keep_rows], storage=storage)
    want = _by_id(fresh2, rl, Q, k)
    assert _by_id(idx, rl, Q, k) == want
    for b in (0, 7):   # the rebuilt index itself against the oracle
        ref_ids, ref_sims, _ = ovs.vector_search_sql(E_all[keep_rows], fresh2.chunk_off, Q[b], num_results=k, f64=True)
        assert [h[0] for h in want[b]] == [fresh2.chunk_ids[c] for c in ref_ids]
        assert np.allclose([h[1] for h in want[b]], ref_sims, atol=1e-4)
    assert {c.id for c in idx.live_chunks} == set(ids_kept)

    idx.compact(block_rows=257)   # odd block size: kept runs straddle the staging blocks
    assert idx.n_rows == fresh2.n_rows and np.array_equal(idx.chunk_off, fresh2.chunk_off) and idx.chunk_ids == fresh2.chunk_ids
    import torch
    assert torch.equal(idx.E, fresh2.E) and torch.equal(idx.row_chunk, fresh2.row_chunk) and torch.equal(idx.inv_norm, fresh2.inv_norm)
    assert _by_id(idx, rl, Q, k) == want

    # a deleted document comes back with the same chunk ids (re-insert after delete)
    back = [c for c in chunks_all if c.id in doomed]
    rows_back = [r for r, i in enumerate(ids_all) if i in doomed]
    idx.append_chunk_embedding_rows([ids_all[r] for r in rows_back], E_all[rows_back], chunks=back)
    again = _by_id(idx, rl, Q[:6], k)
    first = _by_id(fresh, rl, Q[:6], k)
    assert [h[0][0] for h in again] == [h[0][0] for h in first]


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("metric", ["cosine", "dot", "l2"])
def test_count_at_least_brackets_the_exact_rank(rl, metric, algo):
    """``rl_maxsim_count_at_least``: lower bound <= exact #rows with sim >= floor <= upper bound."""
    import torch

    d = 64
    _algo_ok(rl, algo, d, metric)
    E, off = make_corpus(900, (1, 4), d, seed=310, normalize=(metric == "cosine"))
    Q = make_queries(E, 5, seed=311)
    idx = rl.CorpusIndex(E, off)
    sims = np.stack([1.0 - ovs.vector_distances_f64(E, q, metric) for q in Q])
    floor = np.array([np.sort(s)[::-1][r] for s, r in zip(sims, (0, 9, 100, 700, len(E) - 1))], dtype=np.float32)
    exact = (sims >= floor[:, None].astype(np.float64)).sum(1)
    Qd, fd = torch.from_numpy(Q).cuda(), torch.from_numpy(floor).cuda()
    ub = idx.count_at_least(Qd, fd, k=5, num_hits=40, metric=metric, algo=algo, bound=1).cpu().numpy()
    lb = idx.count_at_least(Qd, fd, k=5, num_hits=40, metric=metric, algo=algo, bound=-1).cpu().numpy()
    raw = idx.count_at_least(Qd, fd, k=5, num_hits=40, metric=metric, algo=algo, bound=0).cpu().numpy()
    assert np.all(lb <= exact) and np.all(exact <= ub), (lb, exact, ub)
    assert np.all(lb <= raw) and np.all(raw <= ub)
    slack = 2 if algo == "fp32" else 60   # the fp16-input scan brackets within ~2.5e-3 cosine units
    assert np.all(ub - lb <= slack + 0.1 * exact), (lb, exact, ub)
    none = idx.count_at_least(Qd, torch.full((5,), 3.0e4 if metric == "dot" else 1.5).cuda(), k=5, num_hits=40, metric=metric, algo=algo)
    assert int(none.sum()) == 0
    # tombstoned rows do not count
    idx2 = rl.CorpusIndex(E, off, chunk_ids=[str(c) for c in range(len(off) - 1)])
    idx2.delete_chunks([str(c) for c in range(0, len(off) - 1, 2)])
    alive_rows = np.repeat(np.arange(len(off) - 1) % 2 == 1, np.diff(off))
    exact2 = ((sims >= floor[:, None].astype(np.float64)) & alive_rows[None]).sum(1)
    ub2 = idx2.count_at_least(Qd, fd, k=5, num_hits=40, metric=metric, algo=algo, bound=1).cpu().numpy()
    lb2 = idx2.count_at_least(Qd, fd, k=5, num_hits=40, metric=metric, algo=algo, bound=-1).cpu().numpy()
    assert np.all(lb2 <= exact2) and np.all(exact2 <= ub2)


def test_metadata_rank_then_filter_branch(rl, monkeypatch):
    """``_search.py:96-143`` with both constants scaled down (100_000 -> 60 matching rows, 1_000_000 -> the
    400 nearest vectors): query 0's filter keeps chunks far from it plus a few near ones, so only the
    near ones survive the rank-first cut; for the other queries the one counting pass proves that the
    filter-first answer stands."""
    import raglite_b200._search as S

    monkeypatch.setattr(S, "FILTER_FIRST_MAX_ROWS", 60)
    monkeypatch.setattr(S, "RANK_FIRST_LIMIT", 400)
    d, k = 64, 10
    E, off = make_corpus(600, (1, 5), d, seed=320, fp16_round=True)
    C = len(off) - 1
    Q = make_queries(E, 3, seed=321, frac_random=0.0)
    score0 = ovs.maxsim_scores(E, off, Q[0], "cosine", f64=True)
    order = np.argsort(-score0)
    tagged = np.zeros(C, dtype=bool)
    tagged[order[C // 2:]] = True          # the far half of the corpus ...
    tagged[order[[0, 2, 5, 30]]] = True    # ... and four chunks near query 0
    meta = [{"topic": ["keep"] if t else ["drop"]} for t in tagged]
    idx = rl.CorpusIndex(E, off, chunk_metadata=meta)
    cfg = rl.RAGLiteConfig(reranker=None)
    chunk, sim, count = rl.vector_search_batch(Q, num_results=k, metadata_filter={"topic": "keep"}, index=idx, config=cfg)
    took_rank_first = False
    for b in range(3):
        got = chunk[b, :count[b]].tolist()
        options = []
        for lim in (400, 399, 401):   # the row sitting exactly at the cut may fall on either side
            ids, sims, _ = ovs.vector_search_sql(E, off, Q[b], num_results=k, allowed_chunks=tagged, f64=True,
                                                 filter_first_max=60, rank_first_limit=lim)
            options.append((ids.tolist(), sims))
        assert got in [o[0] for o in options], (b, got, options[0][0])
        ref_sims = options[[o[0] for o in options].index(got)][1]
        assert np.allclose(sim[b, :count[b]], ref_sims, atol=1e-4)
        first_ids, _, _ = ovs.vector_search_sql(E, off, Q[b], num_results=k, allowed_chunks=tagged, f64=True)
        took_rank_first |= got != first_ids.tolist()
    assert took_rank_first, "query 0 must differ from the filter-first answer"
    # few matching rows -> filter-first, whatever the corpus size
    few = np.zeros(C, dtype=bool)
    few[order[[1, 3, 400, 401, 402]]] = True
    idx_few = rl.CorpusIndex(E, off, chunk_metadata=[{"topic": ["keep"] if t else ["drop"]} for t in few])
    chunk, sim, count = rl.vector_search_batch(Q[:1], num_results=k, metadata_filter={"topic": "keep"}, index=idx_few, config=cfg)
    ids, sims, _ = ovs.vector_search_sql(E, off, Q[0], num_results=k, allowed_chunks=few, f64=True, filter_first_max=60,
                                         rank_first_limit=400)
    assert chunk[0, :count[0]].tolist() == ids.tolist() and len(ids) == 5


def test_rank_then_filter_is_proven_without_a_second_pass(rl, monkeypatch):
    """The usual rank-then-filter case (many rows match, the filtered hits are nowhere near the 1M-th nearest
    row): counters the filtered scan keeps anyway (``rl_maxsim_unfiltered_bound``) prove that the filter-first
    answer stands, so no counting pass over the corpus runs.  Constants scaled: 100_000 -> 1_000 matching rows,
    1_000_000 -> 20_000 nearest vectors."""
    import raglite_b200._search as S
    from raglite_b200._index import CorpusIndex

    monkeypatch.setattr(S, "FILTER_FIRST_MAX_ROWS", 1_000)
    monkeypatch.setattr(S, "RANK_FIRST_LIMIT", 20_000)

    def no_probe(*a, **k):
        raise AssertionError("the explicit rank probe must not run here")

    monkeypatch.setattr(CorpusIndex, "count_at_least", no_probe)
    E, off = make_corpus(20_000, 3, 64, seed=330, fp16_round=True)
    C = len(off) - 1
    tagged = (np.arange(C) % 2 == 0)
    idx = rl.CorpusIndex(E, off, chunk_ids=[str(c) for c in range(C)], chunk_metadata=[{"half": int(t)} for t in tagged])
    idx.delete_chunks([str(c) for c in range(0, C, 10)])         # tombstones must not count as live rows
    alive = np.arange(C) % 10 != 0
    Q = make_queries(E, 12, seed=331)
    cfg = rl.RAGLiteConfig(reranker=None)
    chunk, sim, count = rl.vector_search_batch(Q, num_results=10, metadata_filter={"half": 1}, index=idx, config=cfg)
    ub = idx.unfiltered_bound().cpu().numpy()
    assert (ub > 0).all() and ub.max() <= 20_000
    for b in range(len(Q)):
        # the bound really is an upper bound of the live rows at least as near as the worst filtered hit
        d = ovs.vector_distances_f64(E, Q[b], "cosine")
        rows_ok = np.repeat(tagged & alive, np.diff(off))
        worst = np.sort(d[rows_ok])[79]
        assert ub[b] >= int((d[np.repeat(alive, np.diff(off))] <= worst).sum())
        check_sql_semantics(E, off, Q[b], chunk[b, :count[b]], sim[b, :count[b]], k=10, allowed_chunks=tagged & alive)


def test_merge_of_more_hits_than_the_window(rl):
    """R * H > 8192 gathered hits (many shards x a large num_hits): ``rl_topk_merge`` first selects the num_hits best
    straight from global memory, then sorts / groups those -- same answer as merging everything."""
    import torch

    rng = np.random.default_rng(5)
    R, B, H, k = 8, 3, 2000, 500
    sim = np.sort(rng.random((R, B, H)).astype(np.float32), axis=2)[:, :, ::-1].copy()
    sim[:, 1, :] = np.round(sim[:, 1, :], 2)                    # massive ties in query 1
    sim[:, 1, :] = np.sort(sim[:, 1, :], axis=1)[:, ::-1]
    chunk = rng.integers(0, 3000, size=(R, B, H)).astype(np.int64)
    count = rng.integers(H - 50, H + 1, size=(R, B)).astype(np.int32)
    out_sim, out_chunk, out_count = rl.merge_hits(torch.from_numpy(sim).cuda(), torch.from_numpy(chunk).cuda(),
                                                  torch.from_numpy(count).cuda(), num_hits=H, k=k)
    out_sim, out_chunk, out_count = out_sim.cpu().numpy(), out_chunk.cpu().numpy(), out_count.cpu().numpy()
    for b in range(B):
        s = np.concatenate([sim[r, b, :count[r, b]] for r in range(R)])
        c = np.concatenate([chunk[r, b, :count[r, b]] for r in range(R)])
        o = np.argsort(-s.astype(np.float64), kind="stable")[:H]    # ties: shard-major position, like the kernel
        s, c = s[o], c[o]
        _, first = np.unique(c, return_index=True)
        keep = np.sort(first)[:k]
        n = int(out_count[b])
        assert n == len(keep)
        assert np.array_equal(out_chunk[b, :n], c[keep]) and np.array_equal(out_sim[b, :n], s[keep])


def test_async_searches_in_flight_match_the_serial_call(rl):
    """vector_search_batch_async: several batches in flight on their own streams (uploads, kernels, pinned downloads
    overlapping) return exactly what the serial call returns, in any collection order, with and without the query
    adapter and a metadata filter; a slot is reusable once its result has been collected."""
    import torch

    E, off = make_corpus(6000, (1, 10), 128, seed=31)
    n_chunks = len(off) - 1
    idx = rl.CorpusIndex(E, off, chunk_metadata=[{"even": int(c % 2 == 0)} for c in range(n_chunks)])
    idx.set_query_adapter(random_orthogonal(128, seed=5))
    batches = [make_queries(E, 24, seed=100 + i) for i in range(7)]
    for adapter, flt in ((False, None), (True, None), (True, {"even": 1})):
        cfg = rl.RAGLiteConfig(reranker=None, vector_search_query_adapter=adapter)
        kw = dict(num_results=10, config=cfg, index=idx, metadata_filter=flt)
        want = [rl.vector_search_batch(Q, **kw) for Q in batches]
        pinned = [torch.from_numpy(Q).pin_memory() for Q in batches]
        pend = [rl.vector_search_batch_async(Q, **kw) for Q in pinned[:3]]      # three in flight
        got = {2: pend[2].result(), 0: pend[0].result()}                         # out of order
        pend += [rl.vector_search_batch_async(Q, **kw) for Q in pinned[3:5]]    # reuses the two freed slots
        for i in (1, 3, 4):
            got[i] = pend[i].result()
        pend += [rl.vector_search_batch_async(Q, **kw) for Q in pinned[5:]]
        for i in (5, 6):
            got[i] = pend[i].result()
        assert pend[0].done() and pend[0].result() is got[0]
        for i, (ids, sims, counts) in enumerate(want):
            assert np.array_equal(got[i][0], ids) and np.array_equal(got[i][2], counts), (adapter, flt, i)
            assert np.array_equal(got[i][1], sims), (adapter, flt, i)
        if flt is not None:
            assert all(int(c) % 2 == 0 for c in got[0][0][got[0][0] >= 0])
    assert len(idx._slots) == 3 and not any(sl.busy for sl in idx._slots)
    from raglite_b200._index import search_async

    held = [search_async(idx, pinned[0], k=10, num_hits=40, metric="cosine", max_in_flight=3) for _ in range(3)]
    with pytest.raises(RuntimeError, match="in flight"):   # a fourth search needs a result() first
        search_async(idx, pinned[0], k=10, num_hits=40, metric="cosine", max_in_flight=3)
    first = held[0].result()
    again = search_async(idx, pinned[0], k=10, num_hits=40, metric="cosine", max_in_flight=3).result()
    assert np.array_equal(first[0], again[0])
    for h in held[1:]:
        assert np.array_equal(h.result()[0], first[0])
