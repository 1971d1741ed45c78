"""The ``l1`` metric on the GPU (pgvector's ``<+>``, PostgreSQL only): the L1 scan's key contract, searches against the
float64 restatement in ``l1_oracle``, the PostgreSQL query path (halfvec rounding, range check) and the sharded path.

The largest ``|key error| / eps`` of every key case is appended to ``l1_key_bounds.jsonl`` in the temporary directory.
"""

from __future__ import annotations

import json
import tempfile
from pathlib import Path

import numpy as np
import pytest
from l1_oracle import halfvec_query, l1_distances_f64, l1_maxsim_topk, l1_search_sql
from rounding import check as rounding_check
from rounding import f32
from synth import make_corpus, make_queries

from oracle import vector_search as ovs

pytestmark = pytest.mark.gpu

PG_URL = "postgresql://localhost/raglite_l1_tests"


@pytest.fixture(scope="module")
def rl():
    import torch

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import raglite_b200

    return raglite_b200


def _cfg(rl, **kw):  # noqa: ANN001, ANN202
    return rl.RAGLiteConfig(db_url=PG_URL, vector_search_distance_metric="l1", reranker=None,
                            vector_search_query_adapter=False, **kw)


def _record(name: str, payload: dict) -> None:
    with (Path(tempfile.gettempdir()) / "l1_key_bounds.jsonl").open("a") as f:
        f.write(json.dumps({"test": name, **payload}) + "\n")


# ---- key contract -------------------------------------------------------------------------------------------------
N_KEYS = 128 * 9 + 5   # several blocks and a ragged last one


def _key_corpus(kind: str, n: int, d: int, Q, seed: int):  # noqa: ANN001, ANN202
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    E = torch.randn((n, d), generator=g, device="cuda")
    if kind == "unit":
        E /= E.norm(dim=1, keepdim=True)
    elif kind == "gauss":
        E *= 1.5
    elif kind == "subnormal":     # most elements below 2^-14: fp16 subnormals
        E *= torch.pow(10.0, -4.0 - 4.0 * torch.rand((n, d), generator=g, device="cuda"))
    elif kind == "outlier":       # one row 1000x the rest
        E[n // 2] *= 1000.0
    elif kind == "near_dup":      # rows that nearly duplicate the queries: keys near 0
        m = min(n, Q.shape[0])
        E[:m] = Q[:m] + 1e-3 * E[:m]
    else:
        raise AssertionError(kind)
    return E


def _check_keys(name, dump, eps, E_stored, Q, n):  # noqa: ANN001, ANN202
    import torch

    exact = -torch.cdist(Q.double(), E_stored.double(), p=1)              # [B, n]
    err = (dump[:, :n].double() - exact).abs()
    ratio = float((err / eps.double()[:, None]).max())
    _record(name, {"max_err_over_eps": ratio})
    assert bool((err <= eps.double()[:, None]).all()), f"{name}: key error {ratio:.3g} x eps"
    assert bool(torch.isinf(dump[:, n:]).all())


@pytest.mark.parametrize("B", [1, 8, 17, 129, 1100])
@pytest.mark.parametrize("d,storage", [(1, "fp32"), (3, "fp32"), (64, "fp32"), (383, "fp32"), (384, "fp32"),
                                       (1024, "fp32"), (64, "fp16"), (384, "fp16"), (1024, "fp16")])
def test_l1_keys_within_eps(rl, d, storage, B):
    import torch

    g = torch.Generator(device="cuda").manual_seed(d * 7 + B)
    Q = torch.randn((B, d), generator=g, device="cuda")
    for kind in ("unit", "gauss", "subnormal", "outlier", "near_dup"):
        E = _key_corpus(kind, N_KEYS, d, Q, seed=d + B)
        if storage == "fp16":
            E = E.half().float()
        idx = rl.CorpusIndex(E, vecs_per_chunk=1, storage=storage)
        idx.scan(Q, k=1, num_hits=1, metric="l1", sample_stride=1)
        dump, eps = idx.debug_dump(), idx.debug_eps()
        _check_keys(f"{storage}-d{d}-B{B}-{kind}", dump, eps, idx.E.float(), Q, N_KEYS)


@pytest.mark.parametrize("d,ld", [(3, 5), (383, 385), (64, 67)])
def test_l1_keys_misaligned_fp32_rows(rl, d, ld):
    """Rows ``ld`` floats apart and not 16-byte aligned: the scalar loader."""
    import ctypes

    import torch

    from raglite_b200 import _lib

    g = torch.Generator(device="cuda").manual_seed(ld)
    buf = torch.randn(N_KEYS * ld + 1, generator=g, device="cuda")
    E = buf[1:].view(N_KEYS, ld)[:, :d]                                 # 4-byte offset: misaligned
    Q = torch.randn((9, d), generator=g, device="cuda")
    idx = rl.CorpusIndex(E.contiguous(), vecs_per_chunk=1)            # statistics and row map of the same rows
    lib = _lib.load()
    p = idx._params(Q, 1, 1, "l1", "fp32", None, 0, 1, 0)
    p.E, p.ld = E.data_ptr(), ld
    need = lib.rl_maxsim_workspace_bytes(ctypes.byref(p))
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    res = rl._index.new_scan_result(9, 1, 1, 1, idx.device)
    stream = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.rl_maxsim_topk(ctypes.byref(p), res.hit_sim.data_ptr(), res.hit_chunk.data_ptr(), res.hit_count.data_ptr(),
                                  res.status.data_ptr(), ws.data_ptr(), need, stream), "rl_maxsim_topk")
    n = ctypes.c_int64(0)
    dump = torch.empty((9, (N_KEYS + 127) // 128 * 128), dtype=torch.float32, device="cuda")
    _lib.check(lib.rl_maxsim_copy_dump(ctypes.byref(p), ws.data_ptr(), dump.data_ptr(), ctypes.byref(n), stream), "dump")
    eps = torch.empty(9, dtype=torch.float32, device="cuda")
    _lib.check(lib.rl_maxsim_copy_eps(ctypes.byref(p), ws.data_ptr(), eps.data_ptr(), stream), "eps")
    _check_keys(f"fp32-misaligned-d{d}-ld{ld}", dump, eps, E, Q, N_KEYS)


# ---- search against the oracle --------------------------------------------------------------------------------------
def _check_sims(sims, ids, E, off, Qh, what):  # noqa: ANN001, ANN202
    """Each sim is 1 - float(dist) of the chunk's nearest row.  Rows and queries are float16 values here, so every
    difference and every partial sum of a few hundred of them is exact in float64, in any order: the kernel's float64
    sum is the exact distance (bound 0), and one rounding to float32 (nearest even, also at exact midpoints) follows."""
    v = np.array([[l1_distances_f64(E[off[c]:off[c + 1]], Qh[b]).min() for c in ids[b]] for b in range(len(ids))])
    rounding_check(sims, v, 0.0, lambda x: np.float32(1.0) - f32(x), what=what, max_two=0)


@pytest.fixture(scope="module")
def corpus_a():
    E, off = make_corpus(6000, (1, 4), 64, seed=71, fp16_round=True)
    Q = make_queries(E, 300, seed=72)
    return E, off, Q


@pytest.mark.parametrize("storage", ["fp32", "fp16"])
@pytest.mark.parametrize("B", [1, 7, 256, 300])
def test_l1_search_matches_oracle(rl, corpus_a, storage, B):
    E, off, Q = corpus_a
    Q = Q[:B]
    Qh = np.stack([halfvec_query(q) for q in Q])
    idx = rl.CorpusIndex(E, off, storage=storage)
    cfg = _cfg(rl)
    for k, exact in ((10, False), (1024, False), (10, True), (1024, True)):
        ids, sims, counts = rl.vector_search_batch(Q, num_results=k, config=cfg, index=idx, exact_maxsim=exact)
        for b in range(B):
            if exact:
                w_ids, w_sims = l1_maxsim_topk(E, off, Qh[b], k)
            else:
                w_ids, w_sims, _ = l1_search_sql(E, off, Qh[b], num_results=k)
            n = int(counts[b])
            np.testing.assert_array_equal(ids[b, :n], w_ids, err_msg=f"k={k} exact={exact} b={b}")
            np.testing.assert_array_equal(sims[b, :n], w_sims)
        if B <= 7:
            _check_sims(sims[:, :int(counts.min())], ids[:, :int(counts.min())], E, off, Qh, f"l1-{storage}-{k}-{exact}")


def test_l1_tombstones_append_compact(rl, corpus_a):
    E, off, Q = corpus_a
    Q = Q[:16]
    Qh = np.stack([halfvec_query(q) for q in Q])
    C = len(off) - 1
    idx = rl.CorpusIndex(E, off, chunk_ids=[f"c{i}" for i in range(C)])
    cfg = _cfg(rl)
    dead = np.arange(0, C, 3)
    idx.delete_chunks([f"c{i}" for i in dead])
    E2, off2 = make_corpus(500, (1, 4), 64, seed=73, fp16_round=True)
    idx.append_chunk_embedding_rows([f"n{c}" for c in np.repeat(np.arange(500), np.diff(off2))], E2)
    allE = np.concatenate([E, E2])
    allOff = np.concatenate([off, off2[1:] + off[-1]])
    alive = np.ones(C + 500, bool)
    alive[dead] = False

    def check():  # noqa: ANN202
        ids, sims, counts = rl.vector_search_batch(Q, num_results=20, config=cfg, index=idx)
        keep = np.nonzero(alive)[0]
        rows = np.concatenate([np.arange(allOff[c], allOff[c + 1]) for c in keep])
        Ek = allE[rows]
        offk = np.concatenate([[0], np.cumsum(np.diff(allOff)[keep])])
        for b in range(len(Q)):
            w_ids, w_sims, _ = l1_search_sql(Ek, offk, Qh[b], num_results=20)
            got = ids[b, : counts[b]]
            if idx.n_chunks == len(keep):          # compacted: indices are positions among the live chunks
                np.testing.assert_array_equal(got, w_ids)
            else:
                np.testing.assert_array_equal(got, keep[w_ids])
            np.testing.assert_array_equal(sims[b, : counts[b]], w_sims)

    check()
    idx.compact()
    check()


def test_l1_metadata_filter_first_and_forced_overflow(rl, corpus_a):
    import torch

    E, off, Q = corpus_a
    Q = Q[:8]
    Qh = np.stack([halfvec_query(q) for q in Q])
    C = len(off) - 1
    meta = [{"lang": "en" if c % 4 == 0 else "fr"} for c in range(C)]
    idx = rl.CorpusIndex(E, off, chunk_metadata=meta)
    ids, sims, counts = rl.vector_search_batch(Q, num_results=10, config=_cfg(rl), index=idx, metadata_filter={"lang": "en"})
    ok = np.array([m["lang"] == "en" for m in meta])
    for b in range(len(Q)):
        w_ids, w_sims, _ = l1_search_sql(E, off, Qh[b], num_results=10, allowed_chunks=ok)
        np.testing.assert_array_equal(ids[b, : counts[b]], w_ids)
        np.testing.assert_array_equal(sims[b, : counts[b]], w_sims)
    # a candidate list far too small: the overflow-retry loop must end on the same hits
    Qd = torch.from_numpy(Qh).cuda()
    want = idx.scan_checked(Qd, k=10, num_hits=40, metric="l1")
    first = idx.scan(Qd, k=10, num_hits=40, metric="l1", cand_cap=256, sample_stride=64)
    assert bool((first.status & rl._lib.RL_STATUS_CAND_OVERFLOW).any()), "the small list should overflow"
    got = idx.scan_checked(Qd, k=10, num_hits=40, metric="l1", cand_cap=256, sample_stride=64)
    assert torch.equal(got.hit_chunk, want.hit_chunk) and torch.equal(got.hit_sim, want.hit_sim)


def test_l1_more_survivors_than_the_window(rl):
    """6000 copies of one row near the query: every copy is inside the error band of the cut."""
    E, off = make_corpus(20000, 1, 32, seed=74, fp16_round=True)
    q = E[5] * 0.5
    E[100:6100] = (E[5] * 0.5 + np.float32(2.0 ** -10)).astype(np.float16).astype(np.float32)
    idx = rl.CorpusIndex(E, off)
    ids, sims, counts = rl.vector_search_batch(q[None], num_results=1000, config=_cfg(rl), index=idx)
    w_ids, w_sims, _ = l1_search_sql(E, off, halfvec_query(q), num_results=1000)
    np.testing.assert_array_equal(ids[0, : counts[0]], w_ids)
    np.testing.assert_array_equal(sims[0, : counts[0]], w_sims)
    assert idx.scan_stats()["survivors_max"] > 4096


def test_l1_rank_then_filter(rl, monkeypatch):
    """More than 100 000 matching rows in a corpus of more than 1 000 000: the fused bound of the filtered scan proves
    the filter-first answer without a counting pass.  With a limit of 30 rows -- far below the rank of the worst
    filtered hit (about the 200th nearest row here) -- nothing can prove it: the count_at_least(bound=+1) pass exceeds
    the limit, and the bisection over raw keys (bound=0, the fp32 storage's L1 kernel) locates the 30th nearest row,
    which leaves 4 to 6 results per query.  A non-finite query on this branch raises from the status of the filtered
    scan, before any counting pass."""
    import torch

    from raglite_b200 import _index

    rng = np.random.default_rng(75)
    n = 1_100_000
    E = rng.standard_normal((n, 16)).astype(np.float16).astype(np.float32)
    off = np.arange(0, n + 1, 4, dtype=np.int64)
    C = len(off) - 1
    meta = [{"g": c % 5} for c in range(C)]
    Q = rng.standard_normal((4, 16)).astype(np.float32)
    Qh = np.stack([halfvec_query(q) for q in Q])
    idx = rl.CorpusIndex(E, off, chunk_metadata=meta)
    calls = []
    orig = _index.CorpusIndex.count_at_least

    def counting(self, *a, **kw):  # noqa: ANN001, ANN002, ANN003, ANN202
        calls.append((kw.get("bound"), kw.get("algo")))
        return orig(self, *a, **kw)

    monkeypatch.setattr(_index.CorpusIndex, "count_at_least", counting)
    ids, sims, counts = rl.vector_search_batch(Q, num_results=10, config=_cfg(rl), index=idx, metadata_filter={"g": 0})
    assert not calls, "the fused bound should have proven the rank-then-filter case"
    ok = np.array([c % 5 == 0 for c in range(C)])
    for b in range(len(Q)):
        w_ids, w_sims, _ = l1_search_sql(E, off, Qh[b], num_results=10, allowed_chunks=ok)
        np.testing.assert_array_equal(ids[b, : counts[b]], w_ids)
        np.testing.assert_array_equal(sims[b, : counts[b]], w_sims)
    chunk_ok, _ = idx.filter_chunks({"g": [0]})
    Qd = torch.from_numpy(Qh).cuda()
    limit = 30
    ids, sims, counts = _index.search_to_host(idx, Qd, k=10, num_hits=40, metric="l1", chunk_ok=chunk_ok, rank_first_limit=limit)
    assert calls[0] == (1, "auto"), calls[:1]                             # the upper-bound pass
    assert calls.count((0, "fp32")) == 26, calls                          # every bisection step, on the L1 kernel
    for b in range(len(Q)):
        w_ids, w_sims, _ = l1_search_sql(E, off, Qh[b], num_results=10, allowed_chunks=ok, filter_first_max=0,
                                         rank_first_limit=limit)
        assert len(w_ids) < 10        # the limit cut the filter-first answer
        np.testing.assert_array_equal(ids[b, : counts[b]], w_ids)
        np.testing.assert_array_equal(sims[b, : counts[b]], w_sims)
    calls.clear()
    Qbad = Qd.clone()
    Qbad[2, 7] = 7e4                  # beyond binary16: infinite as a halfvec
    with pytest.raises(ValueError, match="float16"):
        rl.vector_search_batch(Qbad, num_results=10, config=_cfg(rl), index=idx, metadata_filter={"g": 0})
    assert not calls, "a non-finite query must not reach the counting passes"


# ---- the PostgreSQL query path --------------------------------------------------------------------------------------
def test_postgresql_rows_and_halfvec_query(rl):
    """A float32 query whose halfvec rounding changes the ranking: the results follow the rounded query."""
    from raglite_b200._rows import vector_to_halfvec_text

    d = 8
    a = np.zeros(d, np.float16)
    a[0] = 1.0
    b = np.zeros(d, np.float16)
    b[0], b[1] = 1 + 2.0 ** -10, 2.0 ** -20
    rng = np.random.default_rng(76)
    far = (rng.standard_normal((50, d)) + 5.0).astype(np.float16)
    rows = [("A", vector_to_halfvec_text(a)), ("B", vector_to_halfvec_text(b))]
    rows += [(f"x{i}", vector_to_halfvec_text(v)) for i, v in enumerate(far)]
    idx = rl.CorpusIndex.from_table_rows(rows, "postgresql")
    q = np.zeros(d, np.float32)
    q[0] = 1 + 2.0 ** -11 + 2.0 ** -22            # above the binary16 tie: rounds to 1 + 2^-10
    import torch

    raw = idx.scan_checked(torch.from_numpy(q[None]).cuda(), k=2, num_hits=0, metric="l1")
    assert raw.hit_chunk[0].tolist() == [0, 1]     # the unrounded query is nearer to A
    cfg = _cfg(rl)
    rl.register_index(cfg, idx)
    try:
        chunk_ids, sims = rl.vector_search(q, num_results=2, config=cfg)
        assert chunk_ids == ["B", "A"]
        assert sims[0] == np.float32(1.0) - np.float32(2.0 ** -20)
        with pytest.raises(ValueError, match="float16"):   # host query beyond the binary16 range
            rl.vector_search(np.full(d, 7e4, np.float32), config=cfg)
        Qd = torch.zeros((3, d), device="cuda")
        Qd[2, 5] = -7e4                                     # device query: reported through the result status
        with pytest.raises(ValueError, match="float16"):
            rl.vector_search_batch(Qd, config=cfg, index=idx)
        with pytest.raises(ValueError, match="float16"):
            rl.vector_search_batch_async(Qd, config=cfg, index=idx).result()
        ids, _, _ = rl.vector_search_batch(Qd[:2], config=cfg, index=idx)   # the index is still usable
        assert ids.shape == (2, 3)
    finally:
        rl.unregister_index(cfg)


# ---- sharded --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [1, 2, 3, 8])
def test_l1_sharded_threads_match_single(rl, monkeypatch, R):
    from thread_group import install, run_ranks

    from raglite_b200._dist import ShardedIndex

    install(monkeypatch)
    E, off = make_corpus(3000, (1, 5), 64, seed=77, fp16_round=True)
    Q = make_queries(E, 16, seed=78)
    C = len(off) - 1
    cuts = np.linspace(0, C, R).round().astype(int).tolist() if R > 1 else [0]
    ranges = [(0, C)] if R == 1 else [(0, 0)] + [(cuts[i], cuts[i + 1]) for i in range(R - 1)]   # shard 0 empty
    bases = ShardedIndex.shard_bases(R)
    shards = [rl.CorpusIndex(E[off[lo]:off[hi]], off[lo:hi + 1] - off[lo], chunk_base=base) for (lo, hi), base in
              zip(ranges, bases, strict=True)]
    single = rl.CorpusIndex(E, off)
    cfg = _cfg(rl)
    want = [rl.vector_search_batch(Q, num_results=10, config=cfg, index=single, exact_maxsim=ex) for ex in (False, True)]

    def rank_fn(r, g):  # noqa: ANN001, ANN202
        sh = ShardedIndex(shards[r], g)
        return [rl.vector_search_batch(Q, num_results=10, config=cfg, index=sh, exact_maxsim=ex) for ex in (False, True)]

    for got in run_ranks(R, rank_fn):
        for (g_ids, g_sims, g_cnt), (w_ids, w_sims, w_cnt) in zip(got, want, strict=True):
            glob = g_ids.copy()
            for (lo, hi), base in zip(ranges, bases, strict=True):
                sel = (g_ids >= base) & (g_ids < base + (hi - lo))
                glob[sel] = g_ids[sel] - base + lo
            np.testing.assert_array_equal(g_cnt, w_cnt)
            np.testing.assert_array_equal(glob, w_ids)
            np.testing.assert_array_equal(g_sims.view(np.uint32), w_sims.view(np.uint32))
