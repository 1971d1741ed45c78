"""``insert_documents`` / ``delete_documents`` / ``delete_documents_by_metadata`` on the GPU through the public path, with
a seeded SaT and a bge-m3-shaped token embedder: records and rows against ``insert_oracle`` over ``split_documents``,
search results against an index built from the same rows and records by ``from_chunk_embedding_rows``, the
``standard`` embedding type's blend bit for bit, ``rl_chunk_embedding_blend`` at the C-ABI, incremental and failed
inserts, deletes, and ``ts_rank`` on a ``postgresql`` config."""

from __future__ import annotations

import itertools
import re

import insert_oracle as io
import numpy as np
import pytest
import torch
import tsrank_oracle as to

import raglite_b200 as rl
from raglite_b200 import _insert as I  # noqa: N812

pytestmark = pytest.mark.gpu
_urls = itertools.count()


@pytest.fixture(scope="module")
def engine():
    """A seeded 1-layer SaT and a 2-layer bge-m3-shaped token embedder (n_ctx = 64), the splitter registered for the
    module."""
    from transformers import XLMRobertaConfig, XLMRobertaForTokenClassification

    from oracle import embed as oe
    from raglite_b200 import _sentences

    tok = oe.unigram_tokenizer()
    torch.manual_seed(0)
    sat_cfg = XLMRobertaConfig(vocab_size=1000, hidden_size=128, num_hidden_layers=1, num_attention_heads=2,
                               intermediate_size=256, max_position_embeddings=514, type_vocab_size=1, pad_token_id=1,
                               layer_norm_eps=1e-5, num_labels=1)
    sat = rl.SaTEngine.from_hf(XLMRobertaForTokenClassification(sat_cfg).eval(), tok)
    model = oe.seeded_model(oe.bge_m3_config(num_hidden_layers=2, vocab_size=1000, max_position_embeddings=514), seed=5)
    eng = rl.TokenEmbedderEngine.from_hf(model, tokenizer=tok, n_ctx=64)
    saved = list(_sentences._SPLITTER)
    rl.register_sentence_splitter(sat)
    yield eng
    _sentences._SPLITTER[:] = saved


def _config(engine, request, **kw) -> rl.RAGLiteConfig:
    """A config with its own db_url and the engine registered for its embedder; unregistered in teardown."""
    from raglite_b200 import _embed

    cfg = rl.RAGLiteConfig(db_url=kw.pop("db_url", f"insert-test://{next(_urls)}"), reranker=None, chunk_max_size=400, **kw)
    saved = _embed._TOKEN_EMBEDDERS.get(cfg.embedder)
    rl.register_token_embedder(cfg.embedder, engine)

    def undo() -> None:
        rl.unregister_index(cfg)
        if saved is None:
            _embed._TOKEN_EMBEDDERS.pop(cfg.embedder, None)
        else:
            rl.register_token_embedder(cfg.embedder, saved)

    request.addfinalizer(undo)
    return cfg


def _documents(n: int, seed: int) -> list[rl.Document]:
    rng = np.random.default_rng(seed)
    words = "alpha beta gamma delta light clock rod frame event time of the observer velocity".split()
    docs = []
    for i in range(n):
        parts = []
        for _ in range(int(rng.integers(1, 8))):
            if rng.random() < 0.4:
                parts.append("#" * int(rng.integers(1, 4)) + " " + " ".join(rng.choice(words, size=3)) + "\n\n")
            sent = [" ".join(rng.choice(words, size=int(rng.integers(3, 20)))).capitalize() + "."
                    for _ in range(int(rng.integers(1, 12)))]
            parts.append(" ".join(sent) + "\n\n")
        docs.append(rl.Document.from_text("".join(parts), topic=f"t{i % 3}", tags=["all", f"s{seed}"]))
    return docs


def _oracle(docs, cfg):
    """(records, fp16 rows, rows per chunk) of the documents as ``_create_chunk_records`` makes them from
    ``split_documents``, late chunking."""
    recs, rows, counts = [], [], []
    for doc, (chunks, embs) in zip(docs, rl.split_documents([d.content for d in docs], config=cfg), strict=True):
        recs += io.records(doc.id, doc.filename, doc.url, doc.metadata_, chunks)
        rows += embs
        counts += [len(e) for e in embs]
    return recs, np.concatenate(rows), np.asarray(counts)


def _rows(idx) -> np.ndarray:
    return idx.E[: idx.n_rows].to(torch.float16).cpu().numpy()


def _table_index(recs, rows, counts, storage):
    row_ids = [c.id for c, n in zip(recs, counts, strict=True) for _ in range(n)]
    return rl.CorpusIndex.from_chunk_embedding_rows(row_ids, rows, chunks=recs, chunk_metadata=[c.metadata_ for c in recs],
                                                   storage=storage)


QUERIES = ["alpha beta observer", "light clock", "the frame of time", "velocity event delta"]


def _results(idx, cfg, *, metadata_filter=None):
    """Vector, keyword and span results of the index, as comparable host values (chunk ids, not indices)."""
    Q = rl.embed_queries(QUERIES, config=cfg)
    ids, sims, counts = rl.vector_search_batch(Q, num_results=8, config=cfg, index=idx, metadata_filter=metadata_filter)
    vec = [([idx.chunk_ids[i] for i in ids[b, : counts[b]]], sims[b, : counts[b]].tolist()) for b in range(len(Q))]
    kids, ksc, kc = rl.keyword_search_batch(QUERIES, num_results=8, index=idx, metadata_filter=metadata_filter)
    kw = [([idx.chunk_ids[i] for i in kids[b, : kc[b]]], ksc[b, : kc[b]].tolist()) for b in range(len(QUERIES))]
    return vec, kw


def _spans(cfg, chunk_ids):
    return [[c.id for c in s.chunks] for s in rl.retrieve_chunk_spans(chunk_ids, config=cfg)]


# 1 + 2 ---------------------------------------------------------------------------------------------------------------------
def test_late_chunking_records_rows_and_search(engine, request):
    cfg = _config(engine, request)
    docs = _documents(14, 1)
    rl.insert_documents(docs, config=cfg)
    idx = rl.get_index(cfg)
    recs, rows, counts = _oracle(docs, cfg)
    assert idx.chunks == recs and idx.chunk_ids == [c.id for c in recs]
    assert idx.chunk_metadata == [c.metadata_ for c in recs]
    assert idx.storage == rl.CorpusIndex._pick_storage(rows, "auto")[1]
    np.testing.assert_array_equal(_rows(idx).view(np.uint16), rows.view(np.uint16))
    np.testing.assert_array_equal(np.diff(idx.chunk_off), counts)
    assert (counts > 1).sum() >= 5 and sum(1 for c in recs if c.headings) >= 3
    assert idx.documents == {d.id: d for d in docs}
    # the same search results as the table path over the oracle's rows and records
    ref = _table_index(recs, rows, counts, idx.storage)
    ref_cfg = _config(engine, request)
    rl.register_index(ref_cfg, ref)
    for flt in (None, {"topic": "t1"}, {"tags": ["all", "s1"]}):
        assert _results(idx, cfg, metadata_filter=flt) == _results(ref, ref_cfg, metadata_filter=flt)
    picks = [recs[i].id for i in (0, 3, 7, len(recs) - 1)]
    assert _spans(cfg, picks) == _spans(ref_cfg, picks)


# 3 -------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("multivector", [True, False])
def test_standard_blend_bit_for_bit(engine, request, multivector):
    cfg = _config(engine, request, embedder="test-standard/bge-m3-shaped", vector_search_multivector=multivector)
    assert rl._embed.embedding_type(config=cfg) == "standard"
    docs = _documents(10, 2)
    rl.insert_documents(docs, config=cfg)
    idx = rl.get_index(cfg)
    recs, want_rows, counts = [], [], []
    for doc in docs:
        chunklets = rl.split_chunklets(rl.split_sentences(doc.content, max_len=400), max_size=400)
        e = rl.embed_strings(chunklets, config=cfg)
        chunks, embs = rl.split_chunks(chunklets, e, max_size=400)
        doc_recs = io.records(doc.id, doc.filename, doc.url, doc.metadata_, chunks)
        f = rl.embed_strings([c.content for c in doc_recs], config=cfg)
        recs += doc_recs
        for chunk_e, chunk_f in zip(embs, f, strict=True):
            want_rows.append(io.blend_numpy(chunk_e, chunk_f[None, :]) if multivector else chunk_f[None, :])
            counts.append(len(want_rows[-1]))
    want = np.concatenate(want_rows)
    assert want.dtype == np.float16 and idx.chunks == recs
    np.testing.assert_array_equal(_rows(idx).view(np.uint16), want.view(np.uint16))
    np.testing.assert_array_equal(np.diff(idx.chunk_off), counts)
    if multivector:
        assert max(counts) > 1
    else:
        assert set(counts) == {1}


# 4 -------------------------------------------------------------------------------------------------------------------------
def _ties(v32: np.ndarray) -> np.ndarray:
    """float32 values exactly halfway between two neighbouring float16 values."""
    with np.errstate(over="ignore", invalid="ignore"):
        h = v32.astype(np.float16)
        v, hv = v32.astype(np.float64), h.astype(np.float64)
        other = np.nextafter(h, np.where(v > hv, np.float16(np.inf), np.float16(-np.inf))).astype(np.float64)
        return np.isfinite(v) & np.isfinite(other) & (v != hv) & (np.abs(v - hv) == np.abs(other - v))


def test_blend_kernel_edges():
    rng = np.random.default_rng(4)
    d, ld, N, C = 64, 72, 20000, 3001                       # N > 132 * 16 * 8 rows: the grid-stride loop wraps
    every = np.arange(1 << 16, dtype=np.uint16).reshape(-1, d)
    xb = rng.integers(0, 1 << 16, size=(N, ld), dtype=np.uint16)
    xb[: len(every), :d] = every
    xb[len(every): 2 * len(every), :d] = every[::-1]
    edges = np.float16([0.0, -0.0, 6e-8, -6e-8, 6.1e-5, 65504, -65504, 65000, np.inf, -np.inf, np.nan, 1.0]).view(np.uint16)
    xb[-64:, :d] = np.resize(edges, (64, d))
    fb = rng.integers(0, 1 << 16, size=(C, d), dtype=np.uint16)
    fb[: len(every)] = every[rng.permutation(len(every))]
    fb[-64:] = np.resize(edges[::-1], (64, d))
    xb[-1, :d] = fb[-1] = np.where(np.arange(d) % 2, 0x7BFF, 0xFBFF)      # +-65504 in the one-row last chunk
    xb[-2, :d] = fb[-2] = 0x8000                                              # -0 + -0 = -0
    # C chunks of random sizes; the last holds one row
    off = np.r_[0, np.sort(rng.choice(np.arange(1, N - 1), size=C - 2, replace=False)), N - 1, N]
    chunk = np.searchsorted(off, np.arange(N), side="right") - 1
    x16, f16 = xb.view(np.float16), fb.view(np.float16)
    want = io.blend_f32(x16[:, :d], f16[chunk])
    X = torch.from_numpy(xb.view(np.int16)).cuda().view(torch.float16)[:, :d]
    got = I.chunk_embedding_blend(X, torch.from_numpy(fb.view(np.int16)).cuda().view(torch.float16), off)
    got = got.cpu().numpy()
    nan = np.isnan(want)
    np.testing.assert_array_equal(np.isnan(got), nan)
    np.testing.assert_array_equal(got.view(np.uint16)[~nan], want.view(np.uint16)[~nan])
    # the planted cases are there
    a, b = np.float32(np.float16(I.ALPHA)), np.float32(np.float16(1 - I.ALPHA))
    with np.errstate(over="ignore", invalid="ignore"):
        p32, q32 = a * x16[:, :d].astype(np.float32), b * f16[chunk].astype(np.float32)
        s32 = p32.astype(np.float16).astype(np.float32) + q32.astype(np.float16).astype(np.float32)
    finite_in = np.isfinite(x16[:, :d]) & np.isfinite(f16[chunk])
    assert _ties(p32).sum() > 20 and _ties(q32).sum() > 20 and _ties(s32).sum() > 20   # half-ulp ties, each step
    # |fp16(a x)| + |fp16(b f)| <= 9824 + 55680 = 65504 for finite halves: the sum reaches 65504 and never overflows
    assert not (np.isinf(want) & finite_in).any() and (np.abs(want[-1]) == 65504).all()
    assert (np.isinf(want) & ~finite_in).any()
    assert ((want.view(np.uint16) & 0x7C00) == 0)[want != 0].sum() > 100   # subnormal results
    assert (want.view(np.uint16) == 0x8000).sum() > 0 and (want.view(np.uint16) == 0).sum() > 0
    assert np.diff(off).min() == 1 and np.diff(off)[-1] == 1 and np.diff(off).max() > 4


# 5 -------------------------------------------------------------------------------------------------------------------------
def test_incremental_skip_and_atomic_failure(engine, request):
    A, B = _documents(14, 1)[:6], _documents(14, 1)[6:11]
    both = _config(engine, request)
    rl.insert_documents(A + B, config=both)
    inc = _config(engine, request)
    rl.insert_documents(A, config=inc)
    rl.insert_documents(B + A[:2], config=inc)                 # A's documents are present: skipped
    i1, i2 = rl.get_index(both), rl.get_index(inc)
    assert i1.chunks == i2.chunks and np.array_equal(i1.chunk_off, i2.chunk_off)
    np.testing.assert_array_equal(_rows(i1).view(np.uint16), _rows(i2).view(np.uint16))
    assert _results(i1, both) == _results(i2, inc)
    n_rows = i2.n_rows
    rl.insert_documents(A + [A[0]], config=inc)
    assert i2.n_rows == n_rows
    before = (_rows(i2).copy(), list(i2.chunk_ids), _results(i2, inc))
    bad = rl.Document.from_text("A sentence with the sentinel ⊕ inside.\n\nMore text here.")
    with pytest.raises(ValueError, match="Error processing document: ") as e:
        rl.insert_documents([*_documents(12, 8)[:3], bad], config=inc)
    assert isinstance(e.value.__cause__, AssertionError) and "Sentinel" in str(e.value.__cause__)
    assert rl.get_index(inc) is i2 and i2.n_rows == n_rows
    np.testing.assert_array_equal(_rows(i2).view(np.uint16), before[0].view(np.uint16))
    assert i2.chunk_ids == before[1] and _results(i2, inc) == before[2]


# 6 -------------------------------------------------------------------------------------------------------------------------
def test_delete_reinsert_metadata_and_compact(engine, request):
    cfg = _config(engine, request)
    docs = _documents(12, 8)
    rl.insert_documents(docs, config=cfg)
    idx = rl.get_index(cfg)
    full = _results(idx, cfg)
    gone = [docs[1].id, docs[4].id, docs[9].id]
    gone_chunks = {c.id for c in idx.chunks if c.document_id in gone}
    assert rl.delete_documents([*gone, "no-such-document", docs[1].id], config=cfg) == 3
    assert rl.delete_documents(gone, config=cfg) == 0
    vec, kw = _results(idx, cfg)
    assert all(not (set(ids) & gone_chunks) for ids, _ in vec + kw) and any(set(ids) & gone_chunks for ids, _ in full[0])
    spans = _spans(cfg, [c.id for c in idx.live_chunks][:6])
    assert all(not (set(s) & gone_chunks) for s in spans)
    # the live chunks alone, as a fresh table index holds them
    live = [c for c in idx.chunks if c.document_id not in gone]
    recs, rows, counts = _oracle([d for d in docs if d.id not in gone], cfg)
    assert live == recs
    ref_cfg = _config(engine, request)
    rl.register_index(ref_cfg, _table_index(recs, rows, counts, idx.storage))
    assert (vec, kw) == _results(rl.get_index(ref_cfg), ref_cfg)
    # re-inserting restores the results exactly
    rl.insert_documents([docs[i] for i in (1, 4, 9)], config=cfg)
    assert _results(idx, cfg) == full
    # the query adapter
    idx.set_query_adapter(np.eye(idx.d))
    assert rl.delete_documents([docs[0].id], config=cfg, invalidate_query_adapter=False) == 1
    assert idx.query_adapter is not None
    assert rl.delete_documents([docs[2].id], config=cfg, invalidate_query_adapter=True) == 1
    assert idx.query_adapter is None
    # by metadata: what the oracle's containment selects among the documents still present
    for flt in ({"topic": "t1"}, {"tags": ["all", "s8"], "topic": ["t2"]}):
        present = {c.document_id for c in idx.live_chunks}
        want = {d.id for d in docs if d.id in present and io.contains(d.metadata_, flt)}
        assert want and rl.delete_documents_by_metadata(flt, config=cfg) == len(want)
        assert {c.document_id for c in idx.live_chunks} == present - want
    assert rl.delete_documents_by_metadata({"topic": "t1"}, config=cfg) == 0
    # compact keeps every result
    before = _results(idx, cfg)
    idx.compact()
    assert _results(idx, cfg) == before and idx.n_chunks == idx.n_live_chunks


# 7 -------------------------------------------------------------------------------------------------------------------------
def _tsvector(body: str) -> tuple[str, dict[str, int]]:
    held: dict[str, list[int]] = {}
    for pos, w in enumerate(re.findall(r"[a-z]+", body.lower()), start=1):
        held.setdefault(w, []).append(pos)
    return to.tsvector_text(held), {w: len(p) for w, p in held.items()}


def test_postgresql_ts_rank_needs_the_inserted_tsvectors(engine, request):
    from raglite_b200 import _pgfts

    cfg = _config(engine, request, db_url=f"postgresql://insert-test/{next(_urls)}")
    A, B = _documents(5, 9), _documents(4, 10)
    rl.insert_documents(A, config=cfg)
    idx = rl.get_index(cfg)
    idx.add_tsvector_rows([(c.id, _tsvector(c.body)[0]) for c in idx.chunks])
    n_a = idx.n_chunks
    rl.insert_documents(B, config=cfg)
    with pytest.raises(ValueError, match=f"{idx.n_chunks - n_a} live chunks have no tsvector"):
        rl.keyword_search_batch(QUERIES, num_results=10, config=cfg)
    idx.add_tsvector_rows([(c.id, _tsvector(c.body)[0]) for c in idx.chunks[n_a:]])
    ids, scores, counts = rl.keyword_search_batch(QUERIES, num_results=10, config=cfg)
    table = {i: _tsvector(c.body)[1] for i, c in enumerate(idx.chunks)}
    for b, q in enumerate(QUERIES):
        want = to.ts_rank_table(table, _pgfts.query_lexemes(q))
        w_ids = sorted(want, key=lambda c: (-float(want[c]), c))[:10]
        assert ids[b, : counts[b]].tolist() == w_ids
        assert scores[b, : counts[b]].tolist() == [float(want[c]) for c in w_ids]
    assert any(i >= n_a for b in range(len(QUERIES)) for i in ids[b, : counts[b]])
