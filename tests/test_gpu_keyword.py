"""BM25 keyword search on a ``CorpusIndex`` (``rl_bm25_stats`` / ``rl_bm25_topk_global`` behind ``keyword_search`` and
``hybrid_search``, one shard: no collective, no merge) against the NumPy oracle of DuckDB's FTS tables and
``match_bm25`` (``tests/keyword_oracle.py``)."""

from __future__ import annotations

import threading

import numpy as np
import pytest

import keyword_oracle as ko

pytestmark = pytest.mark.gpu

REL = 1e-12


def _index(bodies, *, seed=0, metadata=None, ids=None):
    from synth import make_corpus

    import raglite_b200 as rl

    n = len(bodies)
    E, off = make_corpus(n, 1, 16, seed=seed)
    ids = ids or [f"c{c}" for c in range(n)]
    chunks = [rl.Chunk(id=ids[c], document_id=f"d{c // 10}", index=c % 10, body=bodies[c]) for c in range(n)]
    meta = metadata if metadata is not None else [{"bucket": c % 5} for c in range(n)]
    return rl.CorpusIndex(E, off, chunk_ids=ids, chunks=chunks, chunk_metadata=meta), E


def _check(got_ids, got_scores, count, want_ids, want_scores, all_scores, *, allowed=None):
    """Scores within REL of the oracle; ids identical wherever the oracle's neighbouring scores are more than REL apart
    (and otherwise every returned chunk carries the oracle score it is listed with).  Exactly, whatever the ties: the ids
    are distinct and in (score desc, chunk asc) order by the returned scores, and a full list (count = k) leaves out no
    chunk whose oracle score is more than 2 REL above that of its last entry."""
    k = len(got_ids)
    n = int(count)
    assert n == len(want_ids), (n, len(want_ids))
    got_ids, got_scores = [int(x) for x in got_ids[:n]], [float(x) for x in got_scores[:n]]
    np.testing.assert_allclose(got_scores, want_scores, rtol=REL, atol=0)
    ref = np.asarray(sorted((s for d, s in all_scores.items() if allowed is None or allowed[d]), reverse=True))
    close = np.abs(np.diff(ref[: n + 1])) <= REL * ref[: n + 1][1:] if len(ref) > 1 else np.zeros(0, bool)
    if not close.any():
        assert got_ids == want_ids
    for d, s in zip(got_ids, got_scores, strict=True):
        assert d in all_scores and abs(all_scores[d] - s) <= REL * abs(s)
        assert allowed is None or allowed[d]
    assert len(set(got_ids)) == n, "ids must be distinct"
    for i in range(n - 1):
        s0, s1 = got_scores[i], got_scores[i + 1]
        assert s1 < s0 or (s1 == s0 and got_ids[i + 1] > got_ids[i]), ("order", i, got_ids[i: i + 2], s0, s1)
    if n == k and n:
        last = all_scores[got_ids[-1]]
        kept = set(got_ids)
        missed = [d for d, s in all_scores.items() if s > last * (1 + 2 * REL) and (allowed is None or allowed[d])
                  and d not in kept]
        assert not missed, ("left out above the cut", missed[:5])


def _queries(seed, corpus_seed, vocab, n):
    rng = np.random.default_rng(seed)
    qs = ko.make_queries(n, seed, corpus_seed=corpus_seed, vocab=vocab)
    vocab_words = ko.make_vocab(vocab, corpus_seed + 1)
    specials = ["qqqzzzx unknownish", "the of and would", ko.EVERYWHERE, f"{ko.EVERYWHERE} {ko.EVERYWHERE} OMNIA",
                " ".join(vocab_words[:300]), " ".join(rng.permutation(vocab_words[:1000])[:200]), "Café résumé naïve",
                "connecting connections ponies \\alpha", "", "!!!"]
    return specials + qs


@pytest.fixture(scope="module")
def corpus():
    bodies = ko.make_bodies(30_000, seed=7, vocab=4000, empty=0.03, dup=0.03)
    idx, E = _index(bodies)
    return bodies, idx, ko.create_fts_index(bodies)


@pytest.mark.parametrize("B,k", [(1, 1), (7, 10), (256, 64), (300, 4096)])
def test_parity_with_oracle(corpus, B, k):
    import raglite_b200 as rl

    bodies, idx, ix = corpus
    queries = _queries(B, 7, 4000, B)
    queries = queries[-1:] if B == 1 else queries[:B]
    ids, scores, counts = rl.keyword_search_batch(queries, num_results=k, index=idx, config=rl.RAGLiteConfig(db_url="mem://kw"))
    assert ids.shape == (B, k) and scores.dtype == np.float64
    order = idx.keyword_index().analyzer.term_ids
    for b, q in enumerate(queries):
        all_scores = ko.match_bm25(ix, q, term_order=order)
        want_ids, want_scores = ko.keyword_search(ix, q, num_results=k, term_order=order)
        _check(ids[b], scores[b], counts[b], want_ids, want_scores, all_scores)
        assert (ids[b, counts[b]:] == -1).all() and np.isneginf(scores[b, counts[b]:]).all()
    if B >= 7:
        assert counts[0] == 0 and counts[1] == 0           # unknown-only and stop-word-only queries
        assert counts[2] == min(k, sum(1 for x in bodies if x))   # the word in every non-empty body


def test_statistics_and_duplicates(corpus):
    import raglite_b200 as rl

    bodies, idx, ix = corpus
    st = idx.keyword_index().stats()
    assert st["N"] == ix.num_docs and st["avgdl"] == ix.avgdl
    assert all(st["df"][t] == ix.df[i] for t, i in ix.dict.items())
    # exact duplicates score the same and come out by ascending chunk index
    first = {}
    for c, body in enumerate(bodies):
        if body and body in first:
            dup = (first[body], c)
            break
        first.setdefault(body, c)
    q = bodies[dup[0]]
    ids, scores, counts = rl.keyword_search_batch([q], num_results=4096, index=idx)
    row = list(ids[0, : counts[0]])
    i, j = row.index(dup[0]), row.index(dup[1])
    assert scores[0, i] == scores[0, j] and i < j


def test_metadata_filter_changes_results_not_statistics(corpus):
    import raglite_b200 as rl

    bodies, idx, ix = corpus
    before = idx.keyword_index().stats()
    cfg = rl.RAGLiteConfig(db_url="mem://kw-filter")
    queries = _queries(3, 7, 4000, 40)
    order = idx.keyword_index().analyzer.term_ids
    allowed = np.asarray([c % 5 == 2 for c in range(len(bodies))])
    ids, scores, counts = rl.keyword_search_batch(queries, num_results=50, metadata_filter={"bucket": 2}, index=idx, config=cfg)
    for b, q in enumerate(queries):
        all_scores = ko.match_bm25(ix, q, term_order=order)
        want_ids, want_scores = ko.keyword_search(ix, q, num_results=50, allowed=allowed, term_order=order)
        _check(ids[b], scores[b], counts[b], want_ids, want_scores, all_scores, allowed=allowed)
    assert idx.keyword_index().stats() == before
    _, _, counts = rl.keyword_search_batch(queries, num_results=50, metadata_filter={"bucket": 99}, index=idx, config=cfg)
    assert (counts == 0).all()


def test_index_follows_deletes_appends_and_compact():
    import raglite_b200 as rl
    from synth import make_corpus

    bodies = ko.make_bodies(20_000, seed=21, vocab=3000)
    idx, _ = _index(bodies, seed=3)
    queries = _queries(5, 21, 3000, 60) + ["zebraword quokkaword", "zebraword"]
    rl.keyword_search_batch(queries[:2], num_results=5, index=idx)          # build the postings before the changes

    def compare(all_bodies, live):
        order = idx.keyword_index().analyzer.term_ids
        ix = ko.create_fts_index(all_bodies, live=live)
        ids, scores, counts = rl.keyword_search_batch(queries, num_results=64, index=idx)
        for b, q in enumerate(queries):
            all_scores = ko.match_bm25(ix, q, term_order=order)
            want_ids, want_scores = ko.keyword_search(ix, q, num_results=64, term_order=order)
            _check(ids[b], scores[b], counts[b], want_ids, want_scores, all_scores)
        st = idx.keyword_index().stats()
        assert st["N"] == ix.num_docs and st["avgdl"] == ix.avgdl

    gone = [f"d{i}" for i in range(0, 2000, 7)]
    assert idx.delete_documents(gone) > 0
    live = np.asarray([c.document_id not in set(gone) for c in idx.chunks])
    compare(bodies, live)
    # append: new chunks with new terms
    extra = [f"zebraword quokkaword {b}" for b in ko.make_bodies(500, seed=22, vocab=3000)] + ["", "zebraword"]
    E, off = make_corpus(len(extra), 1, 16, seed=9)
    n0 = idx.n_chunks
    new = [rl.Chunk(id=f"x{c}", document_id=f"x{c // 10}", index=c % 10, body=extra[c]) for c in range(len(extra))]
    idx.append(E, off, chunk_ids=[c.id for c in new], chunks=new, chunk_metadata=[{"bucket": 0}] * len(new))
    assert idx.n_chunks == n0 + len(extra)
    all_bodies = bodies + extra
    live = np.concatenate([live, np.ones(len(extra), bool)])
    compare(all_bodies, live)
    # compact: chunk indices are renumbered
    idx.compact()
    kept = [b for b, ok in zip(all_bodies, live, strict=True) if ok]
    assert idx.n_chunks == len(kept)
    compare(kept, None)


def test_scale_across_query_groups():
    import raglite_b200 as rl

    bodies = ko.make_bodies(200_000, seed=31, vocab=20_000, words=(0, 24))
    idx, _ = _index(bodies, seed=4)
    queries = _queries(8, 31, 20_000, 40)
    ids, scores, counts = rl.keyword_search_batch(queries, num_results=100, index=idx)
    kw = idx.keyword_index()
    g_ids, g_scores, g_counts = kw.topk_to_host(queries, k=100, chunk_mask=kw.alive, max_group=16)   # 4 groups
    assert np.array_equal(ids, g_ids) and np.array_equal(scores, g_scores) and np.array_equal(counts, g_counts)
    ix = ko.create_fts_index(bodies)
    order = kw.analyzer.term_ids
    for b, q in enumerate(queries):
        want_ids, want_scores = ko.keyword_search(ix, q, num_results=100, term_order=order)
        _check(ids[b], scores[b], counts[b], want_ids, want_scores, ko.match_bm25(ix, q, term_order=order))


def test_two_threads_on_two_streams(corpus):
    import torch

    import raglite_b200 as rl

    bodies, idx, _ = corpus
    sets = [_queries(40 + i, 7, 4000, 64) for i in range(2)]
    want = [rl.keyword_search_batch(qs, num_results=64, index=idx) for qs in sets]
    got: list = [None, None]

    def worker(i):
        with torch.cuda.stream(torch.cuda.Stream()):
            for _ in range(3):
                got[i] = rl.keyword_search_batch(sets[i], num_results=64, index=idx)

    threads = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for w, g in zip(want, got, strict=True):
        assert all(np.array_equal(a, c) for a, c in zip(w, g, strict=True))


def test_reference_test_analogues():
    """tests/test_search.py:36-127 of the reference, for keyword_search."""
    import raglite_b200 as rl

    bodies = ["Einstein's theory of special relativity.", "The speed of light is constant.", "Photons have no mass.",
              "Relativity changed physics.", "", "Cats sleep a lot."]
    idx, _ = _index(bodies, metadata=[{"type": "physics"}] * 4 + [{"type": "other"}] * 2)
    cfg = rl.RAGLiteConfig(db_url="mem://kw-analogues")
    rl.register_index(cfg, idx)
    try:
        ids, scores = rl.keyword_search("What does Einstein's relativity say?", num_results=3, config=cfg)
        assert ids and all(isinstance(c, str) for c in ids) and all(isinstance(s, float) for s in scores)
        assert ids[0] in ("c0", "c3") and scores == sorted(scores, reverse=True)
        assert rl.keyword_search("qwertyuiop asdfghjkl", config=cfg) == ([], [])
        ids, _ = rl.keyword_search("relativity cats", num_results=5, metadata_filter={"type": "other"}, config=cfg)
        assert ids == ["c5"]
        with pytest.raises(ValueError, match="outside"):
            rl.keyword_search("light", num_results=5000, config=cfg)
    finally:
        rl.unregister_index(cfg)
    empty, _ = _index([])
    cfg2 = rl.RAGLiteConfig(db_url="mem://kw-empty")
    rl.register_index(cfg2, empty)
    try:
        assert rl.keyword_search("anything", config=cfg2) == ([], [])
    finally:
        rl.unregister_index(cfg2)
    from synth import make_corpus

    E, off = make_corpus(10, 1, 16)
    cfg3 = rl.RAGLiteConfig(db_url="mem://kw-nochunks")
    rl.register_index(cfg3, rl.CorpusIndex(E, off))
    try:
        with pytest.raises(ValueError, match="chunk texts"):
            rl.keyword_search("anything", config=cfg3)
    finally:
        rl.unregister_index(cfg3)


def test_hybrid_search_uses_the_device_keyword_search():
    from synth import make_queries

    import raglite_b200 as rl
    import raglite_b200._search as S
    from oracle import fusion as ofu

    bodies = ko.make_bodies(3000, seed=41, vocab=500)
    idx, E = _index(bodies, seed=6)
    cfg = rl.RAGLiteConfig(db_url="mem://kw-hybrid", reranker=None)
    rl.register_index(cfg, idx)
    q_text = " ".join(ko.make_vocab(500, 42)[:3])
    q_vec = make_queries(E, 1, seed=6)[0]
    orig_vs = S.vector_search
    S.vector_search = lambda query, **kw: orig_vs(q_vec, **kw)       # no text embedder here: route the string to a vector
    try:
        ids, scores = rl.hybrid_search(q_text, num_results=5, config=cfg)
    finally:
        S.vector_search = orig_vs
        rl.unregister_index(cfg)
    rl.register_index(cfg, idx)
    try:
        vs_ids, _ = rl.vector_search(q_vec, num_results=10, config=cfg)
    finally:
        rl.unregister_index(cfg)
    ix = ko.create_fts_index(bodies)
    kw_ids, _ = ko.keyword_search(ix, q_text, num_results=10, term_order=idx.keyword_index().analyzer.term_ids)
    assert kw_ids
    want_ids, want_scores = ofu.reciprocal_rank_fusion([vs_ids, [f"c{c}" for c in kw_ids]], weights=[0.75, 0.25])
    assert ids == want_ids[:5] and scores == want_scores[:5]
