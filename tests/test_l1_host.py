"""CPU tests of the ``l1`` metric: the NumPy restatement (``l1_oracle``), the halfvec query rounding, where ``l1`` is
accepted, and the C-ABI's argument handling for metric 3 (no device calls)."""

from __future__ import annotations

import ctypes
from types import SimpleNamespace

import numpy as np
import pytest

from l1_oracle import halfvec_query, l1_distances, l1_distances_f64, l1_maxsim_topk, l1_search_sql, l1_topn_rows_blocked
from oracle import vector_search as ovs


def test_l1_distance_hand_computed():
    E = np.array([[1.0, -2.0, 0.5], [0.0, 0.0, 0.0], [1.0, -2.0, 0.5]], np.float32)
    q = np.array([0.5, 1.0, -0.5], np.float32)
    want = np.array([0.5 + 3.0 + 1.0, 0.5 + 1.0 + 0.5, 4.5])
    np.testing.assert_array_equal(l1_distances(E, q), want)
    np.testing.assert_array_equal(l1_distances_f64(E, q), want)


def test_l1_distance_float32_running_sum():
    """pgvector's loop rounds after every term: 2^24 + 1 + 1 stays 2^24 in float32, not in float64."""
    E = np.array([[2.0 ** 24, 1.0, 1.0]], np.float32)
    q = np.zeros(3, np.float32)
    assert l1_distances(E, q)[0] == 2.0 ** 24
    assert l1_distances_f64(E, q)[0] == 2.0 ** 24 + 2


def test_l1_search_matches_brute_force():
    rng = np.random.default_rng(0)
    off = np.concatenate([[0], np.cumsum(rng.integers(1, 5, 300))])
    E = rng.standard_normal((int(off[-1]), 24)).astype(np.float32)
    for q in rng.standard_normal((5, 24)).astype(np.float32):
        ids, sims, rows = l1_search_sql(E, off, q, num_results=7, oversample=2)
        dist = ovs.float_distance_of_f64(np.abs(E.astype(np.float64) - q).sum(1), "l1")
        order = np.lexsort((np.arange(len(dist)), dist))[:20]          # num_hits = 2 * max(7, 10)
        np.testing.assert_array_equal(rows, order)
        r2c = ovs.row_to_chunk(off)
        best: dict[int, np.float32] = {}
        for r in order:
            best.setdefault(int(r2c[r]), np.float32(1.0) - dist[r])
        ranked = sorted(best.items(), key=lambda kv: (-float(kv[1]), kv[0]))[:7]
        np.testing.assert_array_equal(ids, [c for c, _ in ranked])
        np.testing.assert_array_equal(sims, np.array([s for _, s in ranked], np.float32))
        mids, msims = l1_maxsim_topk(E, off, q, 7)
        sim = np.float32(1.0) - dist
        per_chunk = np.array([sim[off[c]:off[c + 1]].max() for c in range(len(off) - 1)])
        np.testing.assert_array_equal(mids, np.lexsort((np.arange(len(per_chunk)), -per_chunk.astype(np.float64)))[:7])
        np.testing.assert_array_equal(msims, per_chunk[mids])


def test_l1_blocked_equals_unblocked_with_ties():
    rng = np.random.default_rng(1)
    E = rng.integers(-3, 4, (1000, 16)).astype(np.float32)      # integer rows: many exact ties
    E[500:520] = E[10]
    Q = rng.integers(-3, 4, (4, 16)).astype(np.float32)
    Q[0] = E[10]
    blocks = [(r, E[r:r + 137]) for r in range(0, len(E), 137)]
    ok = (np.arange(len(E)) % 3) != 0
    for row_ok in (None, lambda r0, n: ok[r0:r0 + n]):
        got = l1_topn_rows_blocked(blocks, Q, 50, f32_ties=True, row_ok=row_ok)
        for b in range(len(Q)):
            d = ovs.float_distance_of_f64(l1_distances_f64(E, Q[b]), "l1")
            rows = np.arange(len(E)) if row_ok is None else np.nonzero(ok)[0]
            o = rows[np.lexsort((rows, d[rows]))][:50]
            np.testing.assert_array_equal(got[b][0], o)
            np.testing.assert_array_equal(got[b][1], d[o])


def test_halfvec_query_rounds_to_nearest_even():
    # 1 + 2^-11 lies halfway between 1 and 1 + 2^-10: ties go to the even significand (1); 1 + 3 * 2^-11 goes up
    q = np.array([1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, -(1 + 2.0 ** -11), 65504.0], np.float32)
    np.testing.assert_array_equal(halfvec_query(q), np.array([1.0, 1 + 2 * 2.0 ** -10, -1.0, 65504.0], np.float32))
    assert halfvec_query(q).dtype == np.float32


def test_halfvec_query_double_rounding_of_float64():
    """float64 -> float32 -> binary16 (str -> strtof -> halfvec) differs from a direct float64 -> binary16 rounding
    where the first rounding lands on a binary16 tie."""
    x = 1 + 2.0 ** -11 + 2.0 ** -40            # just above the tie between 1 and 1 + 2^-10
    assert np.float64(x).astype(np.float16) == np.float16(1 + 2.0 ** -10)      # one rounding: up
    assert np.float32(x) == np.float32(1 + 2.0 ** -11)                          # float32 drops the 2^-40
    assert halfvec_query(np.array([x]))[0] == 1.0                               # then the tie goes to even: down


def test_halfvec_query_overflow_raises():
    with pytest.raises(ValueError, match="infinite"):
        halfvec_query(np.array([0.0, 65520.0], np.float32))    # rounds to inf in binary16
    with pytest.raises(ValueError, match="infinite"):
        halfvec_query(np.array([np.nan], np.float32))
    assert halfvec_query(np.array([65519.0], np.float32))[0] == 65504.0


def test_torch_halfvec_round_matches_oracle():
    import torch

    from raglite_b200._search import halfvec_round

    rng = np.random.default_rng(2)
    q64 = rng.standard_normal(4096) * 10.0 ** rng.uniform(-9, 4, 4096)
    q64[:3] = [1 + 2.0 ** -11 + 2.0 ** -40, 1 + 2.0 ** -11, 65519.0]
    for q in (q64, q64.astype(np.float32)):
        np.testing.assert_array_equal(halfvec_round(torch.from_numpy(q)).numpy(), halfvec_query(q))


def test_l1_on_duckdb_raises_before_index_lookup(monkeypatch):
    import raglite_b200 as rl
    from raglite_b200 import _search

    def no_lookup(config):  # noqa: ANN001, ANN202
        raise AssertionError("index looked up")

    monkeypatch.setattr(_search, "get_index", no_lookup)
    cfg = rl.RAGLiteConfig(db_url="duckdb:///x.db", vector_search_distance_metric="l1", reranker=None)
    q = np.zeros((1, 8), np.float32)
    with pytest.raises(ValueError, match="PostgreSQL"):
        rl.vector_search(q[0], config=cfg)
    with pytest.raises(ValueError, match="PostgreSQL"):
        rl.vector_search_batch(q, config=cfg)
    with pytest.raises(ValueError, match="PostgreSQL"):
        rl.vector_search_batch_async(q, config=cfg)
    with pytest.raises(ValueError, match="PostgreSQL"):
        rl.vector_search_batch(q, config=cfg, index=SimpleNamespace())   # an explicit index: still refused first


def test_l1_host_query_out_of_halfvec_range_raises_before_upload():
    import raglite_b200 as rl

    fake = SimpleNamespace(query_adapter=None, n_live_chunks=1)      # no device: the check must come first
    cfg = rl.RAGLiteConfig(db_url="postgresql://h/db", vector_search_distance_metric="l1", reranker=None)
    q = np.zeros((2, 8), np.float32)
    q[1, 3] = 70000.0
    with pytest.raises(ValueError, match="float16"):
        rl.vector_search_batch(q, config=cfg, index=fake)


def test_update_query_adapter_refuses_l1():
    from raglite_b200 import RAGLiteConfig
    from raglite_b200._query_adapter import update_query_adapter

    cfg = RAGLiteConfig(db_url="postgresql://h/db", vector_search_distance_metric="l1", reranker=None)
    with pytest.raises(ValueError, match="Unsupported metric: l1"):
        update_query_adapter([(np.zeros(8, np.float32), [0])], config=cfg, index=SimpleNamespace(n_rows=10))


@pytest.mark.parametrize("e_dtype", [0, 1])
def test_workspace_query_accepts_l1_with_auto_and_fp32(e_dtype):
    from raglite_b200 import _lib

    lib = _lib.load()
    p = _lib.ScanParams()
    p.n_rows, p.d, p.ld, p.B, p.k, p.num_hits, p.max_vecs_per_chunk = 100_000, 384, 384, 256, 20, 80, 8
    p.metric, p.e_dtype = _lib.RL_METRIC["l1"], e_dtype
    for algo in ("auto", "fp32"):
        p.algo = _lib.RL_ALGO[algo]
        assert lib.rl_maxsim_workspace_bytes(ctypes.byref(p)) > 0, lib.rl_last_error()
    p.algo = _lib.RL_ALGO["tcgen05"]
    assert lib.rl_maxsim_workspace_bytes(ctypes.byref(p)) == 0
    assert b"l1" in lib.rl_last_error() and b"tensor-core" in lib.rl_last_error()
    p.algo, p.metric = _lib.RL_ALGO["auto"], 4
    assert lib.rl_maxsim_workspace_bytes(ctypes.byref(p)) == 0
    assert b"unknown metric 4" in lib.rl_last_error()


def test_workspace_query_l1_fp16_rules():
    from raglite_b200 import _lib

    lib = _lib.load()
    p = _lib.ScanParams()
    p.n_rows, p.d, p.ld, p.B, p.k, p.num_hits, p.max_vecs_per_chunk = 1000, 383, 383, 4, 5, 0, 1
    p.metric, p.algo = _lib.RL_METRIC["l1"], _lib.RL_ALGO["auto"]
    assert lib.rl_maxsim_workspace_bytes(ctypes.byref(p)) > 0         # float32: any d and ld
    p.ld = 390
    assert lib.rl_maxsim_workspace_bytes(ctypes.byref(p)) > 0
    p.e_dtype = 1
    assert lib.rl_maxsim_workspace_bytes(ctypes.byref(p)) == 0        # float16: d % 8, ld % 8
    assert b"float16 storage" in lib.rl_last_error()
    p.d, p.ld = 384, 392
    assert lib.rl_maxsim_workspace_bytes(ctypes.byref(p)) > 0
