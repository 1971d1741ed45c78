"""A ``CorpusIndex`` changed many times, step by step against a fresh build and the float64 oracle.

Seeded random programs interleave ``insert_documents`` (new, duplicate-id, already present, blank, re-inserted and failing
documents), ``delete_documents``, ``delete_documents_by_metadata``, ``append`` (chunks without a ``Document`` record,
re-appended dead ids, rows planted at the fp16 gate), ``delete_chunks``, ``compact`` (block_rows 1, 257 and the
default), ``add_tsvector_rows`` and the query adapter, on fp32 and fp16 storage and on a ``postgresql`` config.  After
every step (``lifecycle_oracle.Model`` states what the index must hold):

- the device state: chunk table, CSR, row owners, tombstones, stored rows, norms and statistics within the kernel's
  rounding bound, the ``rows_unit_scale`` decision, live counts, BM25 statistics;
- vector search (cosine, dot, l2, and l1 on postgresql; fp32, tcgen05 and auto; with and without a metadata filter;
  1, 10 and more results than live chunks): chunk ids and sims bit-identical to a fresh ``from_chunk_embedding_rows``
  index over the live chunks in the same order and storage, and sims within the last rounding of float64;
- BM25 against ``keyword_oracle`` over the live chunks in the index's own term order, ``ts_rank`` against
  ``tsrank_oracle`` (or the missing-tsvector error), spans against the host collation, ``retrieve_chunks``.

Also the storage gate's edges (fp16 indices that receive rows failing the gate keep answering cosine searches) and
insert groups (any grouping of the documents gives the same records and rows)."""

from __future__ import annotations

import itertools
import re

import insert_oracle as io
import keyword_oracle as ko
import lifecycle_oracle as lo
import numpy as np
import pytest
import rounding as rd
import torch
import tsrank_oracle as to
from synth import make_corpus, make_queries, random_orthogonal

import raglite_b200 as rl
from raglite_b200 import _insert as I  # noqa: N812

pytestmark = pytest.mark.gpu
_urls = itertools.count()
WORDS = "alpha beta gamma delta light clock rod frame event time of the observer velocity zebra quokka".split()
QUERIES = ["alpha beta observer", "light clock", "the frame of time", "velocity event delta", "zebra quokka", "nothing"]


@pytest.fixture(scope="module")
def engine():
    """A seeded 1-layer SaT and a 2-layer bge-m3-shaped token embedder (n_ctx = 64), the splitter registered for the
    module (as ``test_gpu_insert.py`` builds them)."""
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


def _config(engine, request, scheme="insert-test", **kw) -> rl.RAGLiteConfig:
    from raglite_b200 import _embed

    cfg = rl.RAGLiteConfig(db_url=f"{scheme}://lifecycle/{next(_urls)}", reranker=None, chunk_max_size=400, **kw)
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
    docs = []
    for i in range(n):
        parts = []
        for _ in range(int(rng.integers(1, 5))):
            if rng.random() < 0.4:
                parts.append("#" * int(rng.integers(1, 4)) + " " + " ".join(rng.choice(WORDS, size=3)) + "\n\n")
            sent = [" ".join(rng.choice(WORDS, size=int(rng.integers(3, 14)))).capitalize() + "."
                    for _ in range(int(rng.integers(1, 8)))]
            parts.append(" ".join(sent) + "\n\n")
        docs.append(rl.Document.from_text("".join(parts), topic=f"t{i % 3}", tags=["all", f"s{seed}"]))
    return docs


def _oracle_records(docs, cfg) -> dict[tuple[str, str], list[lo.Record]]:
    """Per document, the records and rows ``_create_chunk_records`` makes from ``split_documents`` (late chunking)."""
    out = {}
    for doc, (chunks, embs) in zip(docs, rl.split_documents([d.content for d in docs], config=cfg), strict=True):
        recs = io.records(doc.id, doc.filename, doc.url, doc.metadata_, chunks)
        out[(doc.id, doc.content)] = [lo.Record(c.id, c.document_id, c.index, c.body, c.metadata_,
                                                np.asarray(e, np.float16).astype(np.float32), chunk=c)
                                      for c, e in zip(recs, embs, strict=True)]
    return out


@pytest.fixture(scope="module")
def pool(engine):
    """Documents for the programs and their oracle records: eight documents, a second version of the first under its
    id, a blank document; the failing document of ``test_gpu_insert``."""
    from raglite_b200 import _embed

    cfg = rl.RAGLiteConfig(db_url="pool://lifecycle", reranker=None, chunk_max_size=400)
    saved = _embed._TOKEN_EMBEDDERS.get(cfg.embedder)
    rl.register_token_embedder(cfg.embedder, engine)
    docs = _documents(8, 31)
    docs.append(rl.Document.from_text("# Other\n\nA second text under the first id. Light clock.", id=docs[0].id,
                                      topic="t9", tags=["all"]))
    recs = _oracle_records(docs, cfg)
    docs.append(rl.Document.from_text("  \n\n  ", id="blank-document"))
    if saved is not None:
        rl.register_token_embedder(cfg.embedder, saved)
    bad = rl.Document.from_text("A sentence with the sentinel ⊕ inside.\n\nMore text here.")
    return docs, recs, bad


# ---- checks ----------------------------------------------------------------------------------------------------------
ONE = np.float32(1.0)
CHAINS = {   # the float32 roundings between the float64 value and the returned sim (test_gpu_rescoring.py)
    "cosine": lambda x: ONE - (ONE - rd.f32(np.clip(x, -1.0, 1.0))),
    "dot": lambda x: ONE - rd.f32(-x),
    "l2": lambda x: ONE - rd.f32(np.sqrt(np.maximum(x, 0.0))),
}


def _row_sims(E: np.ndarray, q: np.ndarray, metric: str) -> tuple[np.ndarray, np.ndarray]:
    """(float64 value, bound) of each row's similarity before the float32 roundings (test_gpu_rescoring.oracle)."""
    d = E.shape[1]
    E64, q64 = E.astype(np.float64), q.astype(np.float64)
    if metric == "l2":
        t = E64 - q64
        v = np.einsum("ij,ij->i", t, t)
        return v, 2 * rd.gamma(d) * v
    dot = E64 @ q64
    a = np.abs(E64) @ np.abs(q64)
    if metric == "dot":
        return dot, 2 * rd.gamma(d) * a
    den = np.sqrt(np.einsum("ij,ij->i", E64, E64) * (q64 @ q64))
    with np.errstate(divide="ignore", invalid="ignore"):
        s = dot / den
        return s, 2 * rd.gamma(d + 3) * (a / den + np.abs(s))


def _sim_in_bracket(rows: np.ndarray, q: np.ndarray, metric: str, sim: np.float32) -> bool:
    """Some row of the chunk gives ``sim`` through the kernel's roundings (zero rows have no cosine: left out)."""
    v, b = _row_sims(rows, q, metric)
    if metric == "cosine":                     # a zero row: 0 / 0 = NaN, which the kernel's clamp to [-1, 1] makes -1
        zero = np.abs(rows).max(axis=1) == 0
        v, b = np.where(zero, -1.0, v), np.where(zero, 0.0, b)
    lo_, hi_ = rd.bracket(v, b, CHAINS[metric])
    s = np.float64(sim)
    return bool(np.any((lo_ == s) | (hi_ == s) | ((s >= np.minimum(lo_, hi_)) & (s <= np.maximum(lo_, hi_)))))


def _fresh(model: lo.Model, storage: str, adapter) -> rl.CorpusIndex:
    live = model.live()
    row_ids = [r.id for r in live for _ in range(len(r.rows))]
    rows = np.concatenate([r.rows for r in live]) if live else np.zeros((0, model.d), np.float32)
    idx = rl.CorpusIndex.from_chunk_embedding_rows(row_ids, rows, storage=storage, chunks=[r.chunk for r in live],
                                                   chunk_metadata=[r.metadata for r in live])
    idx.set_query_adapter(adapter)
    return idx


def _check_state(idx: rl.CorpusIndex, model: lo.Model, tag: str) -> None:
    assert idx.storage == model.storage, (idx.storage, model.storage)
    recs = model.records
    assert idx.chunk_ids == [r.id for r in recs]
    assert idx.chunks == [r.chunk for r in recs]
    assert idx.chunk_metadata == [r.metadata for r in recs]
    np.testing.assert_array_equal(idx.chunk_off, model.chunk_off())
    np.testing.assert_array_equal(idx._chunk_alive, model.chunk_alive())
    assert idx.n_chunks == len(recs) and idx.n_rows == int(model.chunk_off()[-1])
    assert idx.n_live_chunks == len(model.live()) and idx.n_live_rows == model.n_live_rows()
    assert set(idx.documents) == set(model.documents)
    np.testing.assert_array_equal(idx.row_chunk.cpu().numpy(), model.row_chunk())
    alive = np.ones(idx.n_rows, bool) if idx._alive is None else idx._alive[: idx.n_rows].cpu().numpy() != 0
    np.testing.assert_array_equal(alive, model.row_alive())
    if recs:                                                             # a chunk filter that passes dead chunks too
        ok = np.arange(len(recs)) % 3 != 1
        got = idx.row_mask(torch.from_numpy(ok.astype(np.uint8)).cuda())
        np.testing.assert_array_equal(got.cpu().numpy() != 0, ok[model.row_chunk()] & model.row_alive())
    X = model.resident_rows()
    np.testing.assert_array_equal(idx.E[: idx.n_rows].float().cpu().numpy(), X)
    lo.check_row_stats(X, idx.inv_norm[: idx.n_rows].cpu().numpy(), idx.sq_norm[: idx.n_rows].cpu().numpy(),
                       idx.stats.cpu().numpy(), tag)
    assert idx.rows_unit_scale == model.rows_unit_scale()


def _check_vector(idx, model: lo.Model, cfgs: dict[str, rl.RAGLiteConfig], seed: int) -> None:
    live = model.live()
    if not live:
        return
    fresh = _fresh(model, idx.storage, idx.query_adapter)
    X = np.concatenate([r.rows for r in live])
    Q = make_queries(X, 4, seed=seed)
    Q[-1] *= np.float32(3.0)                                            # a query that is not unit norm
    big = len(live) + 5
    for metric, cfg in cfgs.items():
        Qa = Q
        if idx.query_adapter is not None and metric != "l1":
            Qa = idx.apply_adapter(torch.from_numpy(Q).cuda(), round_fp16=False).cpu().numpy()
        for algo, k, flt in itertools.product(("fp32", "tcgen05", "auto"), (1, 10, big), (None, {"topic": "t1"})):
            # fp16 rows have the tensor-core scan only, l1 has none: those pairs are refused by design
            if (flt is not None and k != 10) or (algo == "fp32" and idx.storage == "fp16") or (algo, metric) == ("tcgen05", "l1"):
                continue
            got = rl.vector_search_batch(Q, num_results=k, config=cfg, index=idx, algo=algo, metadata_filter=flt)
            want = rl.vector_search_batch(Q, num_results=k, config=cfg, index=fresh, algo=algo, metadata_filter=flt)
            what = (metric, algo, k, flt)
            np.testing.assert_array_equal(got[2], want[2], err_msg=str(what))
            for b in range(len(Q)):
                n = int(got[2][b])
                ids = [idx.chunk_ids[i] for i in got[0][b, :n]]
                assert ids == [fresh.chunk_ids[i] for i in want[0][b, :n]], what
                assert np.array_equal(got[1][b, :n].view(np.uint32), want[1][b, :n].view(np.uint32)), what
                assert all(idx._chunk_alive[i] for i in got[0][b, :n]), what
                if metric != "l1":
                    for i, s in zip(got[0][b, :n], got[1][b, :n], strict=True):
                        assert _sim_in_bracket(model.records[i].rows, Qa[b], metric, s), (what, b, i, s)
    fresh.close()


def _check_bm25(idx, model: lo.Model) -> None:
    from test_gpu_keyword import _check as check_bm25

    if not model.live():
        return
    kw = idx.keyword_index()
    order = kw.analyzer.term_ids
    ix = ko.create_fts_index([r.body for r in model.records], live=model.chunk_alive())
    st = kw.stats()
    assert st["N"] == ix.num_docs and st["avgdl"] == ix.avgdl
    assert all(st["df"][t] == ix.df[i] for t, i in ix.dict.items())
    for k in (1, 10, len(model.records) + 3):
        ids, scores, counts = rl.keyword_search_batch(QUERIES, num_results=k, index=idx)
        for b, q in enumerate(QUERIES):
            all_scores = ko.match_bm25(ix, q, term_order=order)
            want_ids, want_scores = ko.keyword_search(ix, q, num_results=k, term_order=order)
            check_bm25(ids[b], scores[b], counts[b], want_ids, want_scores, all_scores)


def _tsvector(body: str) -> tuple[str, dict[str, int]]:
    held: dict[str, list[int]] = {}
    for pos, w in enumerate(re.findall(r"[a-z]+", body.lower()), start=1):
        held.setdefault(w, []).append(pos)
    return to.tsvector_text(held), {w: len(p) for w, p in held.items()}


def _check_tsrank(idx, model: lo.Model, cfg) -> None:
    from raglite_b200 import _pgfts

    live = model.live()
    missing = sum(1 for r in live if not r.tsvector)
    if not model.has_tsrank:
        with pytest.raises(NotImplementedError, match="no tsvectors"):
            rl.keyword_search_batch(QUERIES, num_results=5, config=cfg, index=idx)
        return
    if missing:
        with pytest.raises(ValueError, match=f"{missing} live chunks have no tsvector"):
            rl.keyword_search_batch(QUERIES, num_results=5, config=cfg, index=idx)
        return
    table = {i: _tsvector(r.body)[1] for i, r in enumerate(model.records) if r.alive}
    ids, scores, counts = rl.keyword_search_batch(QUERIES, num_results=10, config=cfg, index=idx)
    for b, q in enumerate(QUERIES):
        want = to.ts_rank_table(table, _pgfts.query_lexemes(q))
        w_ids = sorted(want, key=lambda c: (-float(want[c]), c))[:10]
        assert ids[b, : counts[b]].tolist() == w_ids, q
        assert scores[b, : counts[b]].tolist() == [float(want[c]) for c in w_ids], q


def _check_spans(idx, model: lo.Model, cfg, rng) -> None:
    from raglite_b200._search import _retrieve_chunk_spans_host

    live = model.live()
    if not live:
        return
    dup = {r.id for r in model.records if not r.alive}
    ids = [r.id for r in live if r.id in dup][:3]                      # re-inserted ids first
    ids += [live[int(i)].id for i in rng.permutation(len(live))[:5] if live[int(i)].id not in ids]
    got = rl.retrieve_chunk_spans(ids, config=cfg)
    want = _retrieve_chunk_spans_host(ids, config=cfg)
    assert [[c.id for c in s.chunks] for s in got] == [[c.id for c in s.chunks] for s in want]
    assert {c.id for s in got for c in s.chunks} <= {r.id for r in live}
    assert rl.retrieve_chunks(ids, config=cfg) == [next(r.chunk for r in live if r.id == i) for i in ids]


# ---- programs ----------------------------------------------------------------------------------------------------------
STEPS = {"insert": 3.0, "insert_fail": 0.4, "delete_documents": 2.0, "delete_metadata": 0.8, "append": 3.5,
         "append_planted": 0.4, "delete_chunks": 2.0, "compact": 1.5, "tsvector": 2.0, "adapter": 0.7}
PROGRAMS = [("duckdb", "fp32"), ("duckdb", "fp16"), ("postgresql", "fp16")]
N_STEPS = 30


class _Synth:
    """Synthetic chunks appended without ``Document`` records: seeded bodies and rows, ids that come back after
    deletes."""

    def __init__(self, storage: str, d: int, seed: int):
        self.storage, self.d, self.seed, self.n, self.docs = storage, d, seed, 0, 0

    def rows(self, n_chunks: int, rng) -> tuple[list[np.ndarray], np.ndarray]:
        E, off = make_corpus(n_chunks, (1, 3), self.d, seed=int(rng.integers(1 << 30)), fp16_round=self.storage == "fp16")
        return [E[off[c]:off[c + 1]] for c in range(n_chunks)], off

    def record(self, cid: str, doc: str, index: int, rows: np.ndarray, rng) -> lo.Record:
        body = " ".join(rng.choice(WORDS, size=int(rng.integers(0, 12))))
        meta = {"topic": [f"t{int(rng.integers(0, 3))}"], "src": ["synth"]}
        chunk = rl.Chunk(id=cid, document_id=doc, index=index, body=body, metadata_=meta)
        return lo.Record(cid, doc, index, body, meta, np.ascontiguousarray(rows, np.float32), chunk=chunk)

    def fresh_records(self, n_chunks: int, rng) -> list[lo.Record]:
        rows, _ = self.rows(n_chunks, rng)
        out = []
        for c in range(n_chunks):
            if c == 0 or rng.random() < 0.3:
                self.docs += 1
                i = 0
            out.append(self.record(f"s{self.seed}-{self.n}", f"sd{self.seed}-{self.docs}", i, rows[c], rng))
            self.n, i = self.n + 1, i + 1
        return out


def _append(idx, recs: list[lo.Record]) -> None:
    rows = np.concatenate([r.rows for r in recs])
    off = np.concatenate([[0], np.cumsum([len(r.rows) for r in recs])])
    idx.append(rows, off, chunk_ids=[r.id for r in recs], chunks=[r.chunk for r in recs],
               chunk_metadata=[r.metadata for r in recs])


def _step(kind, idx, model, synth, pool, cfg, rng, log) -> None:  # noqa: PLR0912, PLR0915
    docs, orc, bad = pool
    copy_recs = lambda doc: [lo.Record(r.id, r.document_id, r.index, r.body, r.metadata, r.rows, chunk=r.chunk)  # noqa: E731
                             for r in orc[(doc.id, doc.content)]]
    if kind == "insert":
        pick = [docs[int(i)] for i in rng.choice(len(docs), size=int(rng.integers(1, 4)))]
        log.append(f"insert {[(d.id, len(d.content)) for d in pick]}")
        want = model.insert(pick, copy_recs)
        rl.insert_documents(pick, config=cfg)
        log[-1] += f" -> inserted {[d.id for d in want]}"
    elif kind == "insert_fail":
        pick = [docs[int(i)] for i in rng.choice(len(docs) - 1, size=2)] + [bad]
        log.append(f"insert (failing) {[d.id for d in pick]}")
        with pytest.raises(ValueError, match="Error processing document: "):
            rl.insert_documents(pick, config=cfg)
        model.insert(pick, copy_recs, fail=True)
    elif kind == "delete_documents":
        present = sorted(model.live_document_ids())
        pick = [present[int(i)] for i in rng.choice(len(present), size=min(len(present), int(rng.integers(1, 4))),
                                                    replace=False)] if present else []
        pick += ["no-such-document"] + pick[:1]
        inv = bool(rng.random() < 0.3)
        log.append(f"delete_documents {pick} invalidate_query_adapter={inv}")
        n = model.delete_documents(pick)
        assert rl.delete_documents(pick, config=cfg, invalidate_query_adapter=inv) == n
    elif kind == "delete_metadata":
        flt = {"topic": f"t{int(rng.integers(0, 3))}"} if rng.random() < 0.7 else {"tags": ["all"], "topic": ["t9"]}
        log.append(f"delete_documents_by_metadata {flt}")
        assert rl.delete_documents_by_metadata(flt, config=cfg) == model.delete_by_metadata(flt)
    elif kind in ("append", "append_planted"):
        dead = {r.id: r for r in model.records if not r.alive and r.id.startswith("s")}
        live_ids = {r.id for r in model.records if r.alive}
        back = [dead[i] for i in sorted(dead) if i not in live_ids][: int(rng.integers(0, 3))]
        recs = synth.fresh_records(int(rng.integers(1, 7)), rng)
        for r in back:                                                    # the same id, document and index again
            rows, _ = synth.rows(1, rng)
            recs.insert(int(rng.integers(0, len(recs) + 1)), synth.record(r.id, r.document_id, r.index, rows[0], rng))
        if kind == "append_planted":
            planted = lo.planted_gate_rows(model.d)
            names = list(planted)
            pick = [names[int(i)] for i in rng.choice(len(names), size=2, replace=False)]
            rows = np.stack([planted[n] for n in pick]).astype(np.float32)
            recs.append(synth.record(f"s{synth.seed}-{synth.n}", f"sd{synth.seed}-planted", synth.n, rows, rng))
            synth.n += 1
            log.append(f"append planted {pick} + {[r.id for r in recs[:-1]]}")
        else:
            log.append(f"append {[r.id for r in recs]}")
        model.append(recs)
        _append(idx, recs)
    elif kind == "delete_chunks":
        live = [r.id for r in model.records if r.alive]
        pick = [live[int(i)] for i in rng.choice(len(live), size=min(len(live), int(rng.integers(1, 5))), replace=False)]
        pick += ["no-such-chunk"]
        log.append(f"delete_chunks {pick}")
        assert idx.delete_chunks(pick) == model.delete_chunks(pick)
    elif kind == "compact":
        block = [1, 257, 1 << 20][int(rng.integers(0, 3))]
        log.append(f"compact block_rows={block}")
        idx.compact(block_rows=block)
        model.compact()
    elif kind == "tsvector":
        last = {r.id: r for r in model.records}
        todo = [r.id for r in last.values() if not r.tsvector]
        pick = [todo[int(i)] for i in rng.permutation(len(todo))[: max(1, len(todo) * 2 // 3)]] if todo else []
        log.append(f"add_tsvector_rows {pick}")
        assert idx.add_tsvector_rows([(i, _tsvector(last[i].body)[0]) for i in pick]) == len(pick)
        model.add_tsvectors(pick)
    elif kind == "adapter":
        if idx.query_adapter is None or rng.random() < 0.5:
            log.append("set_query_adapter")
            idx.set_query_adapter(random_orthogonal(model.d, seed=int(rng.integers(1 << 30))))
        else:
            present = sorted(model.live_document_ids())
            log.append(f"delete_documents {present[:1]} invalidate_query_adapter=True")
            n = model.delete_documents(present[:1])
            assert rl.delete_documents(present[:1], config=cfg, invalidate_query_adapter=True) == n
            assert (idx.query_adapter is None) == bool(n)


def _run_program(engine, pool, request, backend: str, storage: str, seed: int, kinds: list[str] | None = None) -> None:
    rng = np.random.default_rng(seed)
    cfg = _config(engine, request, scheme="postgresql" if backend == "postgresql" else "insert-test")
    metrics = ["cosine", "dot", "l2"] + (["l1"] if backend == "postgresql" else [])
    cfgs = {m: rl.RAGLiteConfig(db_url=cfg.db_url, reranker=None, chunk_max_size=400, vector_search_distance_metric=m)
            for m in metrics}
    d = next(iter(pool[1].values()))[0].rows.shape[1]
    synth = _Synth(storage, d, seed)
    model = lo.Model(storage, d)
    first = synth.fresh_records(int(rng.integers(20, 40)), rng)
    model.append(first)
    rows = np.concatenate([r.rows for r in first])
    off = np.concatenate([[0], np.cumsum([len(r.rows) for r in first])])
    idx = rl.CorpusIndex(rows, off, chunk_ids=[r.id for r in first], chunks=[r.chunk for r in first],
                         chunk_metadata=[r.metadata for r in first], storage=storage)
    rl.register_index(cfg, idx)
    names, weights = list(STEPS), np.asarray(list(STEPS.values()))
    if backend != "postgresql":
        weights[names.index("tsvector")] = 0.0
    log = [f"seed {seed}, {backend}, {storage}: build {len(first)} synthetic chunks"]
    plan = kinds if kinds is not None else [names[int(i)] for i in rng.choice(len(names), size=N_STEPS,
                                                                              p=weights / weights.sum())]
    for step, kind in enumerate([None, *plan]):
        try:
            if kind is not None:
                _step(kind, idx, model, synth, pool, cfg, rng, log)
            assert rl.get_index(cfg) is idx
            _check_state(idx, model, f"step {step}")
            _check_vector(idx, model, cfgs, seed * 1000 + step)
            if backend == "postgresql":
                _check_tsrank(idx, model, cfg)
            else:
                _check_bm25(idx, model)
            _check_spans(idx, model, cfg, rng)
        except Exception as e:
            raise AssertionError(f"seed {seed} step {step} ({backend}, {storage}) failed; the program so far:\n  "
                                 + "\n  ".join(log)) from e


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("backend,storage", PROGRAMS)
def test_random_program(engine, pool, request, backend, storage, seed):
    _run_program(engine, pool, request, backend, storage, 100 + seed)


@pytest.mark.parametrize("backend,storage", PROGRAMS)
def test_reinsert_twice_then_compact(engine, pool, request, backend, storage):
    """A document deleted and re-inserted twice (dead duplicates of its ids and (document, index) keys), a synthetic id
    re-appended, each compact block size, tsvectors for the re-inserted chunks."""
    kinds = ["insert", "insert", "tsvector", "delete_documents", "insert", "append", "delete_chunks", "append",
             "delete_documents", "insert", "tsvector", "compact", "insert", "delete_metadata", "append", "compact",
             "adapter", "delete_documents", "insert", "tsvector", "compact"]
    _run_program(engine, pool, request, backend, storage, 7, kinds)


# ---- the storage gate ------------------------------------------------------------------------------------------------
def test_host_and_device_gates_agree_on_the_planted_rows():
    from raglite_b200._index import fp16_rows_unit_scale, fp16_rows_unit_scale_device

    planted = lo.planted_gate_rows(1024)
    for name, row in planted.items():
        dev = fp16_rows_unit_scale_device(torch.from_numpy(row[None].view(np.int16)).cuda().view(torch.float16))
        assert dev == fp16_rows_unit_scale(row[None]) == lo.unit_scale(row[None].astype(np.float32)), name
        assert rl.CorpusIndex._pick_storage(row[None].astype(np.float32), "auto")[1] == ("fp16" if dev else "fp32"), name
    assert {fp16_rows_unit_scale(r[None]) for r in planted.values()} == {True, False}


def _cosine_matches_oracle(idx, Q: np.ndarray, model: lo.Model) -> None:
    cfg = rl.RAGLiteConfig(db_url="gate://lifecycle", reranker=None, chunk_max_size=400)
    for algo in ("fp32", "tcgen05", "auto") if idx.storage == "fp32" else ("tcgen05", "auto"):
        ids, sims, counts = rl.vector_search_batch(Q, num_results=len(model.records) + 2, config=cfg, index=idx, algo=algo)
        for b in range(len(Q)):
            assert 0 < counts[b] <= len(model.live())        # the nearest num_hits rows may cover fewer chunks
            for i, s in zip(ids[b, : counts[b]], sims[b, : counts[b]], strict=True):
                assert _sim_in_bracket(model.records[i].rows, Q[b], "cosine", s), (algo, b, i, s)


@pytest.mark.parametrize("name", list(lo.planted_gate_rows(64)))
@pytest.mark.parametrize("build", ["insert", "table_rows"])
def test_fp16_index_keeps_cosine_after_rows_that_fail_the_gate(engine, pool, request, build, name):
    docs, orc, _ = pool
    cfg = _config(engine, request)
    if build == "insert":
        rl.insert_documents(docs[:3], config=cfg)
        idx = rl.get_index(cfg)
        recs = [r for doc in docs[:3] for r in orc[(doc.id, doc.content)]]
        documents = {doc.id: doc for doc in docs[:3]}
    else:
        recs = [r for doc in docs[:3] for r in orc[(doc.id, doc.content)]]
        table = [(r.id, r.rows[j].tolist()) for r in recs for j in range(len(r.rows))]
        idx = rl.CorpusIndex.from_table_rows(table, "duckdb", chunks=[r.chunk for r in recs],
                                             chunk_metadata=[r.metadata for r in recs])
        rl.register_index(cfg, idx)
        documents = {}
    assert idx.storage == "fp16" and idx.rows_unit_scale
    model = lo.Model("fp16", idx.d)
    model.documents = documents
    model.append([lo.Record(r.id, r.document_id, r.index, r.body, r.metadata, r.rows, chunk=r.chunk) for r in recs])
    row = lo.planted_gate_rows(idx.d)[name].astype(np.float32)
    rec = lo.Record("planted", "planted-doc", 0, "planted", {}, np.stack([row, recs[0].rows[0]]),
                    chunk=rl.Chunk(id="planted", document_id="planted-doc", body="planted"))
    model.append([rec])
    _append(idx, [rec])
    Q = make_queries(model.resident_rows(), 3, seed=5)
    _cosine_matches_oracle(idx, Q, model)
    _check_state(idx, model, name)
    assert idx.storage == ("fp16" if lo.unit_scale(row[None]) else "fp32")
    # deleting the planted chunk changes nothing about that: the search goes on working
    idx.delete_chunks(["planted"])
    model.delete_chunks(["planted"])
    _cosine_matches_oracle(idx, Q, model)
    idx.compact()
    model.compact()
    _check_state(idx, model, name + " compact")
    _cosine_matches_oracle(idx, Q, model)


def test_unnormalised_insert_into_an_fp16_index(engine, pool, request):
    """``embedder_normalize=False`` rows (norms far from 1) inserted into an index built from normalised rows: the index
    widens only when a row fails the gate, and cosine search answers as the oracle says either way."""
    docs, orc, _ = pool
    cfg = _config(engine, request)
    rl.insert_documents(docs[:3], config=cfg)
    idx = rl.get_index(cfg)
    assert idx.storage == "fp16"
    raw = _config(engine, request, embedder_normalize=False)
    rl.register_index(raw, idx)
    rl.insert_documents(docs[3:6], config=raw)
    X = idx.E[: idx.n_rows].float().cpu().numpy()
    assert idx.storage == ("fp16" if lo.unit_scale(X) else "fp32")
    ids, sims, counts = rl.vector_search_batch(make_queries(X, 3, seed=9), num_results=5, config=cfg, index=idx)
    assert (counts > 0).all()
    for b, q in enumerate(make_queries(X, 3, seed=9)):
        for i, s in zip(ids[b], sims[b], strict=True):
            rows = X[idx.chunk_off[i]: idx.chunk_off[i + 1]]
            assert _sim_in_bracket(rows, q, "cosine", s)


# ---- insert groups -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("group_bytes", ["one", "split"])
def test_insert_groups_give_the_same_records_and_rows(engine, pool, request, monkeypatch, group_bytes):
    docs = pool[0][:8]
    whole = _config(engine, request)
    rl.insert_documents(docs, config=whole)
    width = int(I._token_embedder(whole).n_embd()) if hasattr(I._token_embedder(whole), "n_embd") else 1024
    need = [int((len(d.content) / 0.618 + 64) * 4 * width) for d in docs]
    limit = 1 if group_bytes == "one" else sum(need[:3])                  # every document alone / groups of about three
    monkeypatch.setattr(I, "_GROUP_TOKEN_BYTES", limit)
    groups = I._document_groups(docs, whole)
    assert len(groups) == len(docs) if group_bytes == "one" else 1 < len(groups) < len(docs)
    split = _config(engine, request)
    rl.insert_documents(docs, config=split)
    a, b = rl.get_index(whole), rl.get_index(split)
    assert a.chunks == b.chunks and a.chunk_ids == b.chunk_ids and a.chunk_metadata == b.chunk_metadata
    np.testing.assert_array_equal(a.chunk_off, b.chunk_off)
    assert a.storage == b.storage
    np.testing.assert_array_equal(a.E[: a.n_rows].cpu().numpy().view(np.uint16 if a.storage == "fp16" else np.uint32),
                                  b.E[: b.n_rows].cpu().numpy().view(np.uint16 if b.storage == "fp16" else np.uint32))
