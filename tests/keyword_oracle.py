"""BM25 oracle: DuckDB's FTS index tables and the ``match_bm25`` macro restated step by step in NumPy float64, as the
reference's ``keyword_search`` runs them (``_search.py:203-225``; index built by ``create_fts_index('chunk', 'id',
'body')``, ``_database.py:618``).  The text analysis is ``raglite_b200._fts`` (tokenizer, stop list, stemmer), pinned by
its own tests; this module restates only the tables and the arithmetic.  Test infrastructure (kept beside the tests so
that ``oracle/`` stays as it is).

    dict   (termid, term)              distinct stems of the indexed documents
    docs   (docid, len)                len = terms left after stop-word removal
    terms  (docid, termid)             one row per kept token
    stats  (num_docs, avgdl)
    match_bm25: tokens -> qtermids -> term_tf (tf per docid, termid) -> subscores -> sum per docid

``live`` is the set of chunks the index is built over (deleted chunks excluded, as the reference rebuilds the index
after deletes); ``allowed`` is the metadata filter, a ``WHERE`` around the macro that changes no statistic.
"""

from __future__ import annotations

from collections.abc import Sequence
from dataclasses import dataclass

import numpy as np

from raglite_b200 import _fts


@dataclass
class FTSIndex:
    dict: dict[str, int]          # term -> termid
    doc_len: np.ndarray           # int64 [n_docs] (0 for documents outside the index)
    live: np.ndarray              # bool [n_docs]
    term_doc: np.ndarray          # int64 [T]: the terms table
    term_id: np.ndarray           # int64 [T]
    num_docs: float
    avgdl: float
    df: np.ndarray                # int64 [V]


def create_fts_index(bodies: Sequence[str], live: Sequence[bool] | None = None) -> FTSIndex:
    live_arr = np.ones(len(bodies), bool) if live is None else np.asarray(live, bool)
    terms: dict[str, int] = {}
    doc_len = np.zeros(len(bodies), np.int64)
    rows_doc: list[int] = []
    rows_term: list[int] = []
    for d, body in enumerate(bodies):
        if not live_arr[d]:
            continue
        toks = _fts.document_terms(body)
        doc_len[d] = len(toks)
        for t in toks:
            rows_doc.append(d)
            rows_term.append(terms.setdefault(t, len(terms)))
    term_doc, term_id = np.asarray(rows_doc, np.int64), np.asarray(rows_term, np.int64)
    num_docs = float(live_arr.sum())
    avgdl = float(doc_len[live_arr].sum()) / num_docs if num_docs else float("nan")   # AVG(len)
    pairs = np.unique((term_id << 32) | term_doc)
    df = np.bincount(pairs >> 32, minlength=len(terms)).astype(np.int64)
    return FTSIndex(terms, doc_len, live_arr, term_doc, term_id, num_docs, avgdl, df)


def match_bm25(ix: FTSIndex, query: str, *, k1: float = 1.2, b: float = 0.75,
               term_order: dict[str, int] | None = None) -> dict[int, float]:
    """``fts_main_chunk.match_bm25(docid, query)`` for every document it is not NULL for.  The per-document sum runs over
    the query terms in ascending ``term_order`` id (default: the index's own termids)."""
    docs, scores = match_bm25_arrays(ix, query, k1=k1, b=b, term_order=term_order)
    return dict(zip(docs.tolist(), scores.tolist(), strict=True))


def match_bm25_arrays(ix: FTSIndex, query: str, *, k1: float = 1.2, b: float = 0.75,
                      term_order: dict[str, int] | None = None) -> tuple[np.ndarray, np.ndarray]:
    """``match_bm25`` as ``(docid int64 [M] ascending, score float64 [M])``."""
    tokens = {_fts.stem(w) for w in _fts.tokenize(query)}                          # DISTINCT stem(unnest(tokenize(q)))
    qterms = [t for t in tokens if t in ix.dict]                                    # qtermids: dict JOIN tokens
    if not qterms:
        return np.zeros(0, np.int64), np.zeros(0, np.float64)
    order = term_order if term_order is not None else ix.dict
    qterms.sort(key=lambda t: order[t])
    qids = np.asarray([ix.dict[t] for t in qterms], np.int64)
    sel = np.isin(ix.term_id, qids)                                                  # qterms
    pairs, tf = np.unique((ix.term_id[sel] << 32) | ix.term_doc[sel], return_counts=True)   # term_tf
    tid, doc = pairs >> 32, pairs & 0xFFFFFFFF
    df = ix.df[tid].astype(np.float64)
    tf = tf.astype(np.float64)
    length = ix.doc_len[doc].astype(np.float64)
    idf = np.log10(((ix.num_docs - df) + 0.5) / (df + 0.5) + 1.0)
    sub = idf * ((tf * (k1 + 1.0)) / (tf + k1 * ((1.0 - b) + b * (length / ix.avgdl))))   # subscores
    acc = np.zeros(len(ix.doc_len), np.float64)                                      # SUM(subscore) GROUP BY docid,
    for t in qids:                                                                   # term by term in term_order
        sel = tid == t
        acc[doc[sel]] += sub[sel]                                                    # (a term meets a doc once)
    docs = np.unique(doc)
    return docs, acc[docs]


def keyword_search(ix: FTSIndex, query: str, *, num_results: int, allowed: Sequence[bool] | None = None,
                   term_order: dict[str, int] | None = None) -> tuple[list[int], list[float]]:
    """``SELECT id, score ... WHERE score IS NOT NULL ORDER BY score DESC LIMIT k`` (ties: ascending docid)."""
    docs, scores = match_bm25_arrays(ix, query, term_order=term_order)
    if allowed is not None:
        keep = np.asarray(allowed, bool)[docs]
        docs, scores = docs[keep], scores[keep]
    top = np.lexsort((docs, -scores))[:num_results]
    return docs[top].tolist(), scores[top].tolist()


# ---- the device kernels' arithmetic over the postings CSR ------------------------------------------------------------
# ``rl_bm25_topk_global`` restated on the arrays it reads (include/raglite_b200.h): term_off int64 [V + 1], doc / tf
# int32 [P] sorted by chunk within each term, doc_len int32 [C], stats int64 [2 + J] = {N, sum of doc_len, df of each
# entry}, q_off int32 [B + 1], q_terms int32 [J] (-1: an entry this index does not hold).
def bm25_csr_scores(term_off, doc, tf, doc_len, stats, q_off, q_terms, k1, b, idf=None):
    """Per query, a dense float64 score per chunk and the mask of chunks holding one of its entries' terms: ``(score
    [B, C], matched bool [B, C])``.  Every step is the kernel's expression in its order (that of ``match_bm25_arrays``):
    avgdl = sum / N; idf = log10(((N - df) + 0.5) / (df + 0.5) + 1); norm = (1 - b) + b * (len / avgdl); sub = idf *
    ((f * (k1 + 1)) / (f + k1 * norm)); each chunk's sum runs in entry order.  ``idf`` (float64 [J]) replaces NumPy's
    log10 per entry, so that a device's own log10 can be fed in."""
    term_off, q_off, q_terms = np.asarray(term_off, np.int64), np.asarray(q_off, np.int64), np.asarray(q_terms, np.int64)
    doc, tf, doc_len, stats = np.asarray(doc), np.asarray(tf), np.asarray(doc_len), np.asarray(stats, np.int64)
    V, B, C = len(term_off) - 1, len(q_off) - 1, len(doc_len)
    N = np.float64(stats[0])
    with np.errstate(invalid="ignore", divide="ignore"):
        avgdl = np.float64(stats[1]) / N
        if idf is None:
            df = stats[2:].astype(np.float64)
            idf = np.log10(((N - df) + 0.5) / (df + 0.5) + 1.0)
    idf = np.asarray(idf, np.float64)
    scores = np.zeros((B, C), np.float64)
    matched = np.zeros((B, C), bool)
    for q in range(B):
        for j in range(q_off[q], q_off[q + 1]):
            t = q_terms[j]
            if t < 0 or t >= V:
                continue
            p0, p1 = term_off[t], term_off[t + 1]
            d = doc[p0:p1].astype(np.int64)
            f = tf[p0:p1].astype(np.float64)
            length = doc_len[d].astype(np.float64)
            sub = idf[j] * ((f * (k1 + 1.0)) / (f + k1 * ((1.0 - b) + b * (length / avgdl))))
            scores[q, d] += sub                  # a term holds a chunk at most once: no repeated index
            matched[q, d] = True
    return scores, matched


def bm25_topk(scores, matched, mask, k, chunk_base=0):
    """The exact top k of each query by (score desc, chunk asc) over the matched chunks that ``mask`` (bool [C] or None)
    allows, laid out as ``rl_bm25_packed_bytes`` describes: ``(chunk int64 [B, k] (-1 padded, chunk_base added), score
    float64 [B, k] (-inf padded), count int32 [B])``."""
    B = len(scores)
    ids = np.full((B, k), -1, np.int64)
    out = np.full((B, k), -np.inf, np.float64)
    count = np.zeros(B, np.int32)
    for q in range(B):
        keep = matched[q] if mask is None else matched[q] & np.asarray(mask, bool)
        cand = np.flatnonzero(keep)
        top = cand[np.lexsort((cand, -scores[q][cand]))[:k]]
        n = len(top)
        ids[q, :n], out[q, :n], count[q] = top + chunk_base, scores[q][top], n
    return ids, out, count


def csr_from_postings(postings, doc_len):
    """The CSR of ``postings`` (per term, ``(chunks, tfs)``; chunks distinct) sorted by chunk within each term:
    ``(term_off int64 [V + 1], doc int32 [P], tf int32 [P], doc_len int32 [C])``.  No text analysis: any tf, doc_len
    and corpus size can be built directly."""
    docs, tfs, counts = [], [], []
    for chunks, tf in postings:
        chunks = np.asarray(chunks, np.int64)
        tf = np.broadcast_to(np.asarray(tf, np.int64), chunks.shape)
        order = np.argsort(chunks, kind="stable")
        assert len(np.unique(chunks)) == len(chunks), "a term holds a chunk at most once"
        docs.append(chunks[order])
        tfs.append(tf[order])
        counts.append(len(chunks))
    term_off = np.concatenate([[0], np.cumsum(counts, dtype=np.int64)]).astype(np.int64)
    doc = np.concatenate([np.zeros(0, np.int64), *docs]).astype(np.int32)
    tf = np.concatenate([np.zeros(0, np.int64), *tfs]).astype(np.int32)
    doc_len = np.asarray(doc_len, np.int32)
    assert doc.size == 0 or (doc.min() >= 0 and doc.max() < len(doc_len))
    return term_off, doc, tf, doc_len


def csr_from_fts(ix: FTSIndex):
    """The postings CSR of an ``FTSIndex``'s terms table (term ids = the index's own termids)."""
    pairs, tf = np.unique((ix.term_id << 32) | ix.term_doc, return_counts=True)
    term = pairs >> 32
    term_off = np.concatenate([[0], np.cumsum(np.bincount(term, minlength=len(ix.dict)))]).astype(np.int64)
    return term_off, (pairs & 0xFFFFFFFF).astype(np.int32), tf.astype(np.int32), ix.doc_len.astype(np.int32)


# ---- seeded corpora ---------------------------------------------------------------------------------------------------
EVERYWHERE = "omnia"   # a word every non-empty synthetic body holds


def make_vocab(n: int, seed: int) -> list[str]:
    rng = np.random.default_rng(seed)
    letters = np.array(list("abcdefghijklmnopqrstuvwxyz"))
    words = {"".join(rng.choice(letters, size=int(rng.integers(3, 11)))) for _ in range(2 * n)}
    words = sorted(words)[:n]
    return [words[i] for i in rng.permutation(len(words))]


def make_bodies(n: int, seed: int, *, vocab: int = 4000, words: tuple[int, int] = (0, 60), empty: float = 0.02,
                dup: float = 0.02) -> list[str]:
    """Zipf-distributed words of a generated vocabulary, with stop words, upper case, punctuation, accents and
    digits mixed in; a fraction of empty bodies and of exact duplicates of earlier bodies."""
    rng = np.random.default_rng(seed)
    vocab_words = make_vocab(vocab, seed + 1) + ["The", "and", "of", "Café", "résumé", "COVID-19", "don't", "e.g.",
                                                 "connection", "connected", "running", "ponies", "\\alpha", "naïve"]
    p = 1.0 / np.arange(1, len(vocab_words) + 1) ** 1.07
    p /= p.sum()
    seps = np.array([" ", " ", " ", ", ", ". ", " - ", "\n"])
    bodies: list[str] = []
    for c in range(n):
        u = rng.random()
        if u < empty:
            bodies.append("")
            continue
        if u < empty + dup and bodies:
            bodies.append(bodies[int(rng.integers(0, len(bodies)))])
            continue
        m = int(rng.integers(max(words[0], 1), words[1] + 1))
        ids = rng.choice(len(vocab_words), size=m, p=p)
        parts = [vocab_words[i] for i in ids] + [EVERYWHERE]
        sep = seps[rng.integers(0, len(seps), size=len(parts))]
        bodies.append("".join(w + s for w, s in zip(parts, sep, strict=True)))
    return bodies


def make_queries(n: int, seed: int, *, corpus_seed: int, vocab: int = 4000, words: tuple[int, int] = (1, 12)) -> list[str]:
    """Queries over the vocabulary of ``make_bodies(..., seed=corpus_seed, vocab=vocab)``."""
    rng = np.random.default_rng(seed)
    vocab_words = make_vocab(vocab, corpus_seed + 1)
    out = []
    for _ in range(n):
        m = int(rng.integers(words[0], words[1] + 1))
        out.append(" ".join(vocab_words[int(i)] for i in rng.zipf(1.3, size=m) % len(vocab_words)))
    return out
