"""Sharded BM25 keyword search, host side: the query plan every rank builds (``Analyzer.query_plan``), the packed
buffer's size, and the C-ABI refusals of the top-k and merge entry points (no GPU needed)."""

from __future__ import annotations

import ctypes

import numpy as np
import pytest

from keyword_oracle import make_bodies
from raglite_b200 import _fts


def test_plan_is_independent_of_the_dictionary_order():
    bodies = make_bodies(300, seed=5, vocab=200)
    a, b = _fts.Analyzer(), _fts.Analyzer()
    a.analyze(bodies)
    b.analyze(bodies[::-1])                      # the same stems, numbered in another order
    assert a.term_ids.keys() == b.term_ids.keys() and a.term_ids != b.term_ids
    queries = [bodies[3], "Cats cat CAT dogs", bodies[10] + " " + bodies[11], "zzyzx unknownword", "", "!!!", "the of"]
    off_a, stems_a, ids_a = a.query_plan(queries)
    off_b, stems_b, ids_b = b.query_plan(queries)
    assert np.array_equal(off_a, off_b) and stems_a == stems_b
    assert off_a.dtype == np.int32 and ids_a.dtype == np.int32 and off_a[0] == 0 and off_a[-1] == len(stems_a) == len(ids_a)
    for q, lo, hi in zip(queries, off_a[:-1], off_a[1:], strict=True):
        entries = stems_a[lo:hi]
        assert entries == sorted(set(_fts.query_terms(q)))             # distinct stems by code point
        assert all(t.isascii() for t in entries)
    for st, ia, ib in zip(stems_a, ids_a, ids_b, strict=True):         # the local ids translate back to the same stems
        assert ia == a.term_ids.get(st, -1) and ib == b.term_ids.get(st, -1)


def test_plan_unknown_stems_and_empty_queries():
    an = _fts.Analyzer()
    an.analyze(["cats and dogs", "zebra"])
    q_off, stems, ids = an.query_plan(["dogs zzyzx cats", "", "the", "qqq"])
    assert list(q_off) == [0, 3, 3, 4, 5]
    assert stems == ["cat", "dog", "zzyzx", "the", "qqq"]
    assert list(ids) == [an.term_ids["cat"], an.term_ids["dog"], -1, -1, -1]   # stop words are never in the dictionary
    q_off, stems, ids = an.query_plan([])
    assert list(q_off) == [0] and stems == [] and ids.shape == (0,)
    # query_ids (the single-index plan) is unchanged: known ids only, ascending
    assert list(an.query_ids("dogs zzyzx cats")) == sorted([an.term_ids["cat"], an.term_ids["dog"]])


@pytest.mark.parametrize("B,k", [(1, 1), (1, 3), (3, 1), (7, 10), (256, 64), (300, 4096), (4, 4096)])
def test_packed_bytes(B, k):
    from raglite_b200 import _lib

    lib = _lib.load()
    n = lib.rl_bm25_packed_bytes(B, k)
    raw = B * k * 16 + B * 4
    assert n % 16 == 0 and raw <= n < raw + 16


def test_packed_bytes_of_nothing():
    from raglite_b200 import _lib

    lib = _lib.load()
    assert lib.rl_bm25_packed_bytes(0, 10) == 0 and lib.rl_bm25_packed_bytes(10, 0) == 0 and lib.rl_bm25_packed_bytes(-1, 5) == 0


def test_topk_and_merge_abi_refusals_before_any_cuda_call():
    from raglite_b200 import _lib

    lib = _lib.load()
    d = ctypes.c_void_p(16)
    # rl_bm25_topk_global(term_off, doc, tf, doc_len, stats, n_terms, n_chunks, mask, q_off, q_terms, B, k, k1, b,
    #                     chunk_base, out_packed, workspace, workspace_bytes, stream)
    def topk(k=10, b=0.75, base=0, out=d, stats=d, ws=d, ws_bytes=1 << 20, B=4):
        return lib.rl_bm25_topk_global(d, d, d, d, stats, 10, 100, None, d, d, B, k, 1.2, b, base, out, ws, ws_bytes, None)

    assert topk(k=0) == -1 and topk(k=4097) == -1
    assert "outside [1, 4096]" in lib.rl_last_error().decode()
    assert topk(b=1.5) == -1 and topk(base=-1) == -1
    assert topk(stats=None) == -1 and topk(out=None) == -1 and topk(ws=None) == -1
    assert topk(out=ctypes.c_void_p(24)) == -1                                                 # not 16-byte aligned
    assert topk(ws_bytes=799) == -3                                                            # 100 chunks: 800 bytes a query
    assert "holds no query" in lib.rl_last_error().decode()
    assert topk(B=0, out=None, stats=None) == 0                                                # nothing to do

    # rl_bm25_merge_packed(gathered, R, B, k, out_chunk, out_score, out_count, stream)
    assert lib.rl_bm25_merge_packed(d, 0, 4, 10, d, d, d, None) == -1                          # R < 1
    assert lib.rl_bm25_merge_packed(d, 65, 4, 10, d, d, d, None) == -1                         # R above 64
    assert lib.rl_bm25_merge_packed(d, 2, 4, 0, d, d, d, None) == -1                           # k = 0
    assert lib.rl_bm25_merge_packed(d, 2, 4, 4097, d, d, d, None) == -1                        # k above the cap
    assert lib.rl_bm25_merge_packed(None, 2, 4, 10, d, d, d, None) == -1
    assert lib.rl_bm25_merge_packed(d, 2, 4, 10, d, None, d, None) == -1
    assert lib.rl_bm25_merge_packed(ctypes.c_void_p(8), 2, 4, 10, d, d, d, None) == -1         # not 16-byte aligned
    assert "rl_bm25_merge_packed" in lib.rl_last_error().decode()
    assert lib.rl_bm25_merge_packed(None, 2, 0, 10, None, None, None, None) == 0               # B = 0
