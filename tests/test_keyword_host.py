"""BM25 keyword search, host side: DuckDB fts's text analysis (``raglite_b200._fts``), the oracle's arithmetic on a
hand-written example, and the C-ABI's refusals (no GPU needed)."""

from __future__ import annotations

import ctypes
import math

import numpy as np
import pytest

from keyword_oracle import create_fts_index, keyword_search, make_bodies, match_bm25
from raglite_b200 import _fts

PORTER_PAIRS = {
    "caresses": "caress", "ponies": "poni", "ties": "ti", "cats": "cat", "feed": "feed", "agreed": "agre",
    "plastered": "plaster", "motoring": "motor", "sing": "sing", "conflated": "conflat", "troubled": "troubl",
    "sized": "size", "hopping": "hop", "tanned": "tan", "falling": "fall", "hissing": "hiss", "fizzed": "fizz",
    "failing": "fail", "filing": "file", "happy": "happi", "sky": "sky", "relational": "relat", "generalizations": "gener",
    "oscillators": "oscil", "connect": "connect", "connected": "connect", "connecting": "connect", "connection": "connect",
    "connections": "connect",
}


@pytest.mark.parametrize("word", sorted(PORTER_PAIRS))
def test_porter_published_pairs(word):
    assert _fts.stem(word) == PORTER_PAIRS[word]


def test_porter_more_steps():
    # Step 1b's e-restoring rules, step 2-4 suffixes, the 'ion' rule, 5a/5b, and the y -> Y consonant marking
    cases = {"hoping": "hope", "controlling": "control", "rolling": "roll", "probate": "probat", "rate": "rate",
             "cease": "ceas", "effective": "effect", "adjustment": "adjust", "adoption": "adopt", "onion": "onion",
             "says": "sai", "yelling": "yell", "played": "plai", "electricity": "electr", "hopefulness": "hope",
             "dependent": "depend", "a": "a", "is": "i"}
    assert {w: _fts.stem(w) for w in cases} == cases


def test_tokenizer():
    assert _fts.tokenize("Café Résumé") == ["cafe", "resume"]
    assert _fts.tokenize("COVID-19 cases") == ["covid", "cases"]
    assert _fts.tokenize("e.g. this") == ["e", "g", "this"]
    assert _fts.tokenize("don't") == ["don", "t"]
    assert _fts.tokenize(r"\alpha and \beta") == ["lpha", "and", "eta"]   # a backslash takes the next character along
    assert _fts.tokenize(r"a\\b") == ["a", "b"]
    assert _fts.tokenize("Привет мир 你好世界") == []                         # non-Latin letters are separators
    assert _fts.tokenize("UPPER Case MiXeD") == ["upper", "case", "mixed"]
    assert _fts.tokenize("") == [] and _fts.tokenize(" \t\n ") == []
    assert _fts.tokenize("naïve façade") == ["naive", "facade"]


def test_stop_list():
    assert len(_fts.STOPWORD_ENTRIES) == 571
    assert len(_fts.STOPWORDS) == 570 and _fts.STOPWORD_ENTRIES.count("would") == 2
    for w in ("the", "a", "and", "of", "would", "zero", "awfully", "c'mon"):
        assert w in _fts.STOPWORDS


def test_stop_words_document_side_only():
    # "alls" is not a stop word but stems to "all", which is; a query holding "all" (kept on the query side) matches it
    assert "alls" not in _fts.STOPWORDS and _fts.stem("alls") == "all" and "all" in _fts.STOPWORDS
    ix = create_fts_index(["alls quiet", "all quiet", "the end"])
    assert _fts.document_terms("all quiet") == ["quiet"]
    assert _fts.query_terms("all the") == ["all", "the"]
    assert set(match_bm25(ix, "all")) == {0}
    assert match_bm25(ix, "the") == {}


def test_query_terms_distinct():
    assert _fts.query_terms("Cats cat CAT dogs") == ["cat", "dog"]


def test_analyzer_matches_document_terms():
    bodies = make_bodies(400, seed=11, vocab=300) + ["Café \\alpha COVID-19 e.g. don't", "", "ÅNGSTRÖM Ünïcödé"]
    an = _fts.Analyzer()
    terms, owners, lens = an.analyze(bodies, batch=64)
    inv = {i: t for t, i in an.term_ids.items()}
    for c, body in enumerate(bodies):
        want = _fts.document_terms(body)
        assert [inv[int(t)] for t in terms[owners == c]] == want
        assert lens[c] == len(want)
    # growing the dictionary: known stems keep their ids, new ones are appended
    before = dict(an.term_ids)
    an.analyze(["zzyzx quiet", "cats"])
    assert all(an.term_ids[t] == i for t, i in before.items()) and an.term_ids["zzyzx"] == len(before)
    assert list(an.query_ids("zzyzx cats unknownword zzyzx")) == sorted({an.term_ids["zzyzx"], an.term_ids["cat"]})


def test_oracle_hand_computed_example():
    bodies = ["The cat sat on the mat.", "Cats and dogs. Cat!", "", "A dog."]
    ix = create_fts_index(bodies)
    # kept terms: [cat, sat, mat], [cat, dog, cat], [], [dog]
    assert list(ix.doc_len) == [3, 3, 0, 1] and ix.num_docs == 4.0 and ix.avgdl == 7 / 4
    k1, b, avgdl = 1.2, 0.75, 1.75
    idf = math.log10((4 - 2 + 0.5) / (2 + 0.5) + 1)            # cat and dog: df = 2 of N = 4

    def part(tf, dl):
        return idf * (tf * (k1 + 1) / (tf + k1 * (1 - b + b * (dl / avgdl))))

    want = {1: part(2, 3) + part(1, 3), 3: part(1, 1), 0: part(1, 3)}
    got = match_bm25(ix, "cat CAT dog cats")                     # repeated words count once
    assert got.keys() == want.keys()
    for d in want:
        assert got[d] == pytest.approx(want[d], rel=1e-15)
    ids, scores = keyword_search(ix, "cat dog", num_results=2)
    assert ids == [1, 3] and scores[0] > scores[1]
    # a filter is a WHERE around the macro: it removes results, not statistics
    ids, scores = keyword_search(ix, "cat dog", num_results=3, allowed=[True, False, True, True])
    assert ids == [3, 0] and scores == [got[3], got[0]]
    # a term in more than half of the chunks still scores above zero (the + 1 inside the log)
    ix2 = create_fts_index(["mat", "mat", "mat", "dog"])
    assert match_bm25(ix2, "mat")[0] == pytest.approx(math.log10(1.5 / 3.5 + 1) * 2.2 / (1 + 1.2 * (0.25 + 0.75 * 1)), rel=1e-15)
    # deleted chunks leave the statistics
    ix3 = create_fts_index(bodies, live=[True, True, False, False])
    assert ix3.num_docs == 2.0 and ix3.avgdl == 3.0 and match_bm25(ix3, "dog").keys() == {1}


def test_csr_restatement_matches_the_fts_oracle_bit_for_bit():
    """``bm25_csr_scores`` over the CSR of ``create_fts_index``'s tables (what the device kernels read) equals
    ``match_bm25_arrays`` bit for bit, and ``bm25_topk`` equals ``keyword_search``, with and without a filter."""
    import keyword_oracle as ko

    bodies = make_bodies(3000, seed=5, vocab=600, empty=0.03, dup=0.05)
    live = np.random.default_rng(5).random(len(bodies)) > 0.1
    ix = create_fts_index(bodies, live=live)
    term_off, doc, tf, doc_len = ko.csr_from_fts(ix)
    allowed = np.arange(len(bodies)) % 3 != 1
    queries = ko.make_queries(60, 6, corpus_seed=5, vocab=600) + [ko.EVERYWHERE, "qqqzzzx", bodies[7], bodies[8]]
    compared = 0
    for q in queries:
        qids = sorted({ix.dict[t] for t in _fts.query_terms(q) if t in ix.dict})
        stats = np.concatenate([[ix.num_docs, ix.doc_len.sum()], ix.df[qids]]).astype(np.int64)
        scores, matched = ko.bm25_csr_scores(term_off, doc, tf, doc_len, stats, [0, len(qids)], qids, 1.2, 0.75)
        docs, want = ko.match_bm25_arrays(ix, q)
        assert np.array_equal(np.flatnonzero(matched[0]), docs)
        assert np.array_equal(scores[0][docs].view(np.int64), want.view(np.int64))
        assert (scores[0][~matched[0]] == 0).all()
        for k, mask in ((1, None), (17, None), (4096, None), (50, allowed)):
            ids, sc, cnt = ko.bm25_topk(scores, matched, mask, k)
            w_ids, w_sc = keyword_search(ix, q, num_results=k, allowed=mask)
            assert cnt[0] == len(w_ids) and ids[0, :cnt[0]].tolist() == w_ids
            assert np.array_equal(sc[0, :cnt[0]].view(np.int64), np.asarray(w_sc, np.float64).view(np.int64))
            assert (ids[0, cnt[0]:] == -1).all() and np.isneginf(sc[0, cnt[0]:]).all()
        compared += len(docs)
    assert compared > 10_000
    # k1 = 0: every posting of a term scores its idf exactly, so the top k is the term's chunks in ascending order
    stats = np.array([ix.num_docs, ix.doc_len.sum(), ix.df[0]], np.int64)
    scores, matched = ko.bm25_csr_scores(term_off, doc, tf, doc_len, stats, [0, 1], [0], 0.0, 0.75)
    ids, sc, cnt = ko.bm25_topk(scores, matched, None, 4096, chunk_base=1 << 40)
    n = min(int(ix.df[0]), 4096)
    assert cnt[0] == n and np.array_equal(ids[0, :n], (1 << 40) + doc[term_off[0]:term_off[1]][:n].astype(np.int64))
    assert (sc[0, :n] == sc[0, 0]).all()
    assert sc[0, 0] == pytest.approx(math.log10((ix.num_docs - ix.df[0] + 0.5) / (ix.df[0] + 0.5) + 1), rel=1e-15)


def test_stats_abi_refusals_before_any_cuda_call():
    from raglite_b200 import _lib

    lib = _lib.load()
    dummy = ctypes.c_void_p(16)
    assert lib.rl_bm25_workspace_bytes(100, 3) == 2400 and lib.rl_bm25_workspace_bytes(0, 3) == 0
    # rl_bm25_stats(term_off, doc, doc_len, alive, n_terms, n_chunks, df, corpus, stream)
    assert lib.rl_bm25_stats(None, None, None, None, 1, 1, None, None, None) == -1
    assert lib.rl_bm25_stats(dummy, dummy, dummy, None, 10, 100, None, dummy, None) == -1      # df
    assert lib.rl_bm25_stats(dummy, dummy, dummy, None, 10, 100, dummy, None, None) == -1      # corpus
    assert lib.rl_bm25_stats(dummy, dummy, dummy, None, -1, 100, dummy, dummy, None) == -1     # n_terms < 0
    assert "rl_bm25_stats" in lib.rl_last_error().decode()


def test_keyword_search_refusals_without_a_device():
    import raglite_b200 as rl

    with pytest.raises(NotImplementedError, match="ts_rank"):
        rl.keyword_search("x", config=rl.RAGLiteConfig(db_url="postgresql://u@h/db"))
    with pytest.raises(ValueError, match="No index registered"):
        rl.keyword_search("x", config=rl.RAGLiteConfig(db_url="mem://keyword-none"))
    with pytest.raises(NotImplementedError, match="self_query"):
        rl.keyword_search("x", config=rl.RAGLiteConfig(db_url="mem://keyword-none", self_query=True))


def test_stopword_file_has_no_duplicates_besides_would():
    entries = np.asarray(_fts.STOPWORD_ENTRIES)
    vals, counts = np.unique(entries, return_counts=True)
    assert list(vals[counts > 1]) == ["would"]
