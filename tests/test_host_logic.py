"""CPU tests of the host-side logic and of the C-ABI surface (no compute calls without a GPU)."""

from __future__ import annotations

import ctypes
import json
import re
from dataclasses import fields
from pathlib import Path

import numpy as np
import pytest
from fake_llama import FakeLlama, make_sentences

from oracle import pool as opool
from oracle import vector_search as ovs

ROOT = Path(__file__).resolve().parents[1]


def test_library_builds_and_exports_every_declared_symbol():
    from raglite_b200 import _build, _lib

    path = _build.build()
    lib = ctypes.CDLL(str(path))
    header = (ROOT / "include" / "raglite_b200.h").read_text()
    declared = set(re.findall(r"\b(rl_[a-z0-9_]+)\s*\(", header))
    assert declared == set(_lib.EXPORTS), declared ^ set(_lib.EXPORTS)
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.rl_version() >= 100


def test_scan_params_struct_matches_header():
    from raglite_b200._lib import ScanParams, ScanStats

    header = (ROOT / "include" / "raglite_b200.h").read_text()
    body = header[header.index("typedef struct rl_scan_params {"):header.index("} rl_scan_params;")]
    names = re.findall(r"([a-z_A-Z]+);", body)
    assert names == [f[0] for f in ScanParams._fields_]
    body = header[header.index("typedef struct rl_scan_stats {"):header.index("} rl_scan_stats;")]
    assert re.findall(r"([a-z_A-Z]+);", body) == [f[0] for f in ScanStats._fields_]


def test_workspace_query_and_argument_validation_run_without_a_gpu():
    from raglite_b200 import _lib

    lib = _lib.load()
    p = _lib.ScanParams()
    p.n_rows, p.d, p.ld, p.B, p.k, p.num_hits, p.metric, p.max_vecs_per_chunk = 100_000, 384, 384, 256, 20, 80, 0, 8
    p.algo = _lib.RL_ALGO["fp32"]
    need = lib.rl_maxsim_workspace_bytes(ctypes.byref(p))
    assert need > 256 * 100_000 // 64 * 4
    p.k = 0
    assert lib.rl_maxsim_workspace_bytes(ctypes.byref(p)) == 0
    assert b"k must be positive" in lib.rl_last_error()
    p.k, p.metric = 20, 7
    assert lib.rl_maxsim_workspace_bytes(ctypes.byref(p)) == 0
    assert b"metric" in lib.rl_last_error()


def test_attention_hook_refuses_what_rl_xenc_score_refuses():
    """``rl_xenc_attention`` checks its arguments before any CUDA call (the pointers here are never dereferenced)."""
    from raglite_b200 import _lib

    lib = _lib.load()
    ptr, ws = 4096, 8192                                        # placeholders: every call below is refused first

    def call(*, qkv=ptr, P=4, T=100, max_len=64, hidden=384, heads=12, workspace=ws, ws_bytes=16):
        return lib.rl_xenc_attention(qkv, ptr, P, T, max_len, hidden, heads, ptr, workspace, ws_bytes, None)

    assert call(qkv=None) == -1
    assert call(hidden=48, heads=1) == -4                       # hidden % 32
    assert call(hidden=544, heads=17) == -4                     # hidden > 512
    assert call(hidden=384, heads=6) == -4                      # head_dim 64
    assert call(P=101) == -1                                    # more sequences than tokens
    assert call(max_len=0) == -1
    assert call(ws_bytes=15) == -3                              # 4 * P bytes
    assert call(workspace=ws + 4) == -3                         # 16-byte alignment
    assert call(workspace=None) == -3
    assert call(max_len=1281, T=2000) == -4                     # K / V of 1344 keys exceed the shared memory
    assert b"max_len=1281" in lib.rl_last_error()


def test_layernorm_and_head_hooks_refuse_bad_arguments():
    """``rl_xenc_embed_ln``, ``rl_xenc_add_ln`` and ``rl_xenc_cls_head`` check their arguments before any CUDA call (the
    pointers here are never dereferenced; a zero-sized call returns before any launch)."""
    from raglite_b200 import _lib

    lib = _lib.load()
    ptr = 4096                                                  # placeholder, 16-byte aligned

    def weights(hidden=384, vocab=100, max_pos=512, type_vocab=2, n_labels=1, tables=True, head=True):
        w = _lib.XencWeights()
        w.hidden, w.vocab, w.max_pos, w.type_vocab, w.n_labels, w.ln_eps = hidden, vocab, max_pos, type_vocab, n_labels, 1e-12
        if tables:
            w.word_emb = w.pos_emb = w.type_emb = w.emb_ln_g = w.emb_ln_b = ptr
        if head:
            w.pooler_w = w.pooler_b = w.cls_w = w.cls_b = ptr
        return ctypes.byref(w)

    def embed(w=None, ids=ptr, out=ptr, T=5):
        return lib.rl_xenc_embed_ln(weights() if w is None else w, ids, ptr, ptr, T, out, None)

    assert embed(ids=None) == -1
    assert embed(out=None) == -1
    assert embed(T=-1) == -1
    assert embed(w=weights(tables=False)) == -1
    assert embed(w=weights(hidden=48)) == -4                    # hidden % 32
    assert embed(w=weights(hidden=1056)) == -4                  # hidden > 1024
    assert embed(w=weights(hidden=0)) == -4
    assert embed(w=weights(vocab=0)) == -1
    assert embed(w=weights(type_vocab=0)) == -1
    assert embed(T=0) == 0

    def add_ln(x=ptr, res=ptr, gamma=ptr, beta=ptr, out=ptr, T=5, H=384, out_f32=0):
        return lib.rl_xenc_add_ln(x, res, gamma, beta, 1e-5, T, H, out_f32, out, None)

    assert add_ln(x=None) == -1
    assert add_ln(beta=None) == -1
    assert add_ln(T=-1) == -1
    assert add_ln(H=48) == -4
    assert add_ln(H=1056) == -4
    assert add_ln(H=0) == -4
    for name in ("x", "res", "gamma", "beta", "out"):          # the vectorised path's 8- / 16-byte pieces
        assert add_ln(**{name: ptr + 8}) == -1, name
        assert b"16-byte aligned" in lib.rl_last_error()
    assert add_ln(out_f32=1, out=ptr + 4) == -1
    assert add_ln(T=0) == 0
    assert add_ln(T=0, out=ptr, res=ptr) == 0                   # in place (out == res) is allowed

    def head(w=None, hidden=ptr, cu=ptr, P=3, logit=ptr, score=ptr):
        return lib.rl_xenc_cls_head(weights() if w is None else w, hidden, cu, P, logit, score, None)

    assert head(hidden=None) == -1
    assert head(cu=None) == -1
    assert head(score=None) == -1
    assert head(P=-1) == -1
    assert head(w=weights(head=False)) == -1
    assert head(w=weights(n_labels=3)) == -4
    assert b"n_labels=3" in lib.rl_last_error()
    assert head(w=weights(hidden=48)) == -4
    assert head(w=weights(hidden=1056)) == -4
    assert head(P=0) == 0
    assert head(P=0, w=weights(n_labels=0)) == 0                # 0 labels is read as 1
    assert head(P=0, w=weights(n_labels=2)) == 0


def test_config_mirrors_reference_fields():
    from raglite_b200 import RAGLiteConfig

    names = [f.name for f in fields(RAGLiteConfig)]
    assert names == ["db_url", "llm", "llm_max_tries", "embedder", "embedder_normalize", "chunk_max_size",
                     "vector_search_distance_metric", "vector_search_multivector", "vector_search_query_adapter",
                     "reranker", "search_method", "self_query"]  # reference _config.py:42-83
    cfg = RAGLiteConfig(reranker=None)
    assert cfg.chunk_max_size == 2048 and cfg.vector_search_distance_metric == "cosine"
    assert cfg.vector_search_multivector and cfg.vector_search_query_adapter and cfg.embedder_normalize
    assert cfg.llm_max_tries == 4 and not cfg.self_query
    assert hash(cfg) == hash(RAGLiteConfig(reranker=None))  # frozen + hashable (lru_cache key in the reference)
    with pytest.raises(Exception):  # noqa: B017, PT011
        cfg.chunk_max_size = 1  # type: ignore[misc]


def test_num_hits_rule_matches_oracle():
    from raglite_b200._search import num_hits_rule

    for k in (1, 3, 10, 20, 100):
        for over in (1, 2, 3, 4, 8):
            for size in (512, 1024, 2048, 3000, 4096):
                assert num_hits_rule(k, over, size) == ovs.num_hits_rule(k, over, size)


@pytest.mark.parametrize("seed", range(6))
def test_host_planning_matches_oracle(seed):
    from raglite_b200 import _embed

    llm = FakeLlama(n_ctx=64 + 16 * seed, dim=8, seed=seed)
    sentences = make_sentences(40 + 7 * seed, seed=seed)
    nt = _embed.count_tokens(sentences, llm)
    assert nt.tolist() == opool.count_tokens(sentences, llm).tolist()
    assert _embed.plan_segments(nt, llm.n_ctx(), llm.n_batch) == opool.plan_segments(nt, llm.n_ctx(), llm.n_batch)
    rng = np.random.default_rng(seed)
    for _ in range(50):
        toks = rng.integers(1, 30, size=int(rng.integers(1, 12)))
        rows = int(toks.sum() + rng.integers(0, 5))
        assert _embed.largest_remainder_sizes(rows, toks).tolist() == opool.largest_remainder_sizes(rows, toks).tolist()


def test_plan_segments_with_zero_token_sentences():
    from raglite_b200 import _embed

    nt = np.array([5, 0, 0, 9, 30, 0, 2, 40, 1, 0, 0, 3], dtype=np.intp)
    assert _embed.plan_segments(nt, 64, 64) == opool.plan_segments(nt, 64, 64)


def test_ranker_protocol():
    from raglite_b200._rerank import ScoreFnRanker

    r = ScoreFnRanker(lambda q, docs: [len(d) for d in docs])
    out = r.rank(query="q", docs=["a", "ccc", "bb"])
    assert [x.doc_id for x in out.results] == [1, 2, 0]
    assert [x.rank for x in out.results] == [1, 2, 3]


def test_rerank_chunks_contract():
    from raglite_b200 import Chunk, RAGLiteConfig, rerank_chunks
    from raglite_b200._rerank import ScoreFnRanker

    chunks = [Chunk(id=f"c{i}", body="x" * (i + 1)) for i in range(5)]
    cfg = RAGLiteConfig(reranker=None)
    assert rerank_chunks("q", chunks, config=cfg) == chunks       # no reranker -> identity (_search.py:376-377)
    cfg = RAGLiteConfig(reranker=ScoreFnRanker(lambda q, docs: [len(d) for d in docs]))
    assert [c.id for c in rerank_chunks("q", chunks, config=cfg)] == ["c4", "c3", "c2", "c1", "c0"]
    assert rerank_chunks("q", [], config=cfg) == []
    cfg = RAGLiteConfig(reranker={"other": ScoreFnRanker(lambda q, docs: [-len(d) for d in docs])})
    assert [c.id for c in rerank_chunks("q", chunks, config=cfg)][0] == "c0"


def test_chunk_str_matches_reference_layout():
    from raglite_b200 import Chunk

    c = Chunk(id="a", headings="# H1\n## H2", body=" body text ", metadata_={"filename": "f.pdf", "url": "u"})
    assert str(c) == "---\nfilename: f.pdf\nurl: u\n---\n\n# H1\n## H2\n\nbody text"
    assert str(Chunk(id="b", body="only")) == "only"


def test_golden_meta_is_readable(golden_dir):
    z = np.load(golden_dir / "pool_small.npz")
    meta = json.loads(bytes(z["meta"]).decode())
    assert len(meta["sentences"]) == z["late_chunking"].shape[0]


def test_reciprocal_rank_fusion_argument_handling():
    """(The fusion itself runs on the device: tests/test_fusion.py.)"""
    from raglite_b200 import reciprocal_rank_fusion

    assert reciprocal_rank_fusion([]) == ([], [])
    assert reciprocal_rank_fusion([[], []]) == ([], [])
    with pytest.raises(ValueError):
        reciprocal_rank_fusion([["a"]], weights=[1.0, 2.0])


def test_retrieve_chunk_spans_groups_and_ranks():
    """Span collation (reference _search.py:302-361) on Chunk objects: neighbours come from the
    registered table only when one exists, contiguous runs merge, order = summed reciprocal rank."""
    from raglite_b200 import Chunk, RAGLiteConfig, retrieve_chunk_spans

    mk = lambda d, i: Chunk(id=f"{d}-{i}", document_id=d, index=i, body=f"[{d}{i}]")  # noqa: E731
    ranked = [mk("A", 5), mk("B", 2), mk("A", 6), mk("A", 9)]
    spans = retrieve_chunk_spans(ranked, neighbors=None, config=RAGLiteConfig(db_url="mem://none", reranker=None))
    got = [[c.id for c in s.chunks] for s in spans]
    # A5+A6 merge (1 + 1/3), then B2 (1/2), then A9 (1/4)
    assert got == [["A-5", "A-6"], ["B-2"], ["A-9"]]
    assert str(spans[0]) == "[A5][A6]" and spans[0].document_id == "A"
    assert retrieve_chunk_spans([], config=RAGLiteConfig(reranker=None)) == []


def test_csr_from_row_chunk_ids_follows_the_table_layout():
    """One CSR segment per run of equal chunk ids (``_insert.py:247-251``); a re-appearing id is an error."""
    from raglite_b200._index import csr_from_row_chunk_ids

    off, ids = csr_from_row_chunk_ids(["a", "a", "b", "c", "c", "c"])
    assert off.tolist() == [0, 2, 3, 6] and ids == ["a", "b", "c"]
    off, ids = csr_from_row_chunk_ids([])
    assert off.tolist() == [0] and ids == []
    with pytest.raises(ValueError):
        csr_from_row_chunk_ids(["a", "b", "a"])
    with pytest.raises(ValueError):
        csr_from_row_chunk_ids(["x", "y"], known={"y"})


def test_scan_checked_resolves_or_raises():
    """Host control flow around the status bits: a candidate overflow is retried first with the
    thresholds the failed pass wrote, then with a four times larger list, until the list is as large as
    the shard; the index lock is held throughout."""
    import threading

    import torch

    from raglite_b200 import _lib
    from raglite_b200._index import CorpusIndex, ScanResult

    def fake_index(script, n_rows=100_000):
        idx = object.__new__(CorpusIndex)
        idx.storage, idx.device, idx.calls, idx.n_rows = "fp32", torch.device("cpu"), [], n_rows
        idx._lock = threading.RLock()
        idx.scan_stats = lambda: {"cand_cap": 1000}

        def scan(Q, *, out=None, **kw):
            assert idx._lock._is_owned()   # retries run under the index lock
            idx.calls.append((kw.get("flags", 0), kw.get("cand_cap", 0)))
            status = torch.tensor(script(len(idx.calls), int(Q.shape[0]), kw), dtype=torch.int32)
            B = int(Q.shape[0])
            tag = float(len(idx.calls))
            return ScanResult(torch.full((B, 2), tag), torch.full((B, 2), int(tag), dtype=torch.int64),
                              torch.full((B,), 2, dtype=torch.int32), status, 2, 1)

        idx.scan = scan
        return idx

    Q = torch.zeros((3, 4))
    REUSE = _lib.RL_FLAG_REUSE_THRESHOLDS
    # clean first pass
    idx = fake_index(lambda n, B, kw: [0] * B)
    assert idx.scan_checked(Q, k=1, num_hits=2).hit_sim[0, 0] == 1.0 and len(idx.calls) == 1
    # overflow, cleared by the threshold-reuse retry
    idx = fake_index(lambda n, B, kw: [1, 0, 0] if n < 2 else [0] * B)
    idx.scan_checked(Q, k=1, num_hits=2)
    assert idx.calls == [(0, 0), (REUSE, 0)]
    # overflow that needs a larger list: reuse -> 4x list (fresh thresholds) -> reuse -> 16x ...
    idx = fake_index(lambda n, B, kw: [1, 0, 0] if n < 5 else [0] * B)
    idx.scan_checked(Q, k=1, num_hits=2)
    assert idx.calls == [(0, 0), (REUSE, 0), (0, 4000), (REUSE, 4000), (0, 16000)]
    # overflow that never clears: the list grows up to the shard size, then a loud failure
    idx = fake_index(lambda n, B, kw: [1] * B, n_rows=10_000)
    with pytest.raises(_lib.RagliteB200Error):
        idx.scan_checked(Q, k=1, num_hits=2)
    assert max(c[1] for c in idx.calls) == 10_000 + 1024
    # ... and the last run's status is read: a list that clears on the last allowed run is a result, not an error
    from raglite_b200._index import MAX_SCAN_RUNS

    idx = fake_index(lambda n, B, kw: [1] * B if n < MAX_SCAN_RUNS else [0] * B, n_rows=10_000)
    assert idx.scan_checked(Q, k=1, num_hits=2).hit_sim[0, 0] == MAX_SCAN_RUNS and len(idx.calls) == MAX_SCAN_RUNS


