"""BM25 keyword search on a ``ShardedIndex``: R thread ranks on one GPU (``thread_group``) run the real host pipeline --
``Analyzer.query_plan`` and the entries' statistics, one all-reduce, ``rl_bm25_topk_global``, one all-gather and
``rl_bm25_merge_packed`` (R = 1: neither collective nor the merge) -- against the bare ``CorpusIndex`` and the NumPy
oracle of ``match_bm25``.

* The merge kernel, bit for bit against a NumPy restatement, on synthetic packed buffers.
* Exactness: on a corpus whose single-index term ids follow sorted-stem order (chunk 0 holds every word, one per stem,
  ordered by stem, and is then deleted so that it counts for nothing) every R and shard layout returns the single
  index's ids, scores and counts bit for bit.
* On an ordinary corpus: the oracle bar of ``test_gpu_keyword._check`` (the sum over sorted stems), bit-identity across R.
* The index changing on one rank (delete, append, compact) and a metadata filter, against a single index put through the
  same changes; id resolution, ``hybrid_search``, and one all-reduce plus one all-gather per batch."""

from __future__ import annotations

import numpy as np
import pytest
from test_gpu_keyword import REL, _check, _queries
from thread_group import install, run_ranks

import keyword_oracle as ko
from raglite_b200 import _fts
from raglite_b200._dist import ShardedIndex

pytestmark = pytest.mark.gpu

STRIDE = 1 << 40


@pytest.fixture(scope="module")
def rl():
    import torch

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import raglite_b200

    return raglite_b200


# ---- a. the merge kernel against NumPy -------------------------------------------------------------------------------
def _sorted_list(rng, n, base, tie_values):
    """n entries of one shard: unique global chunks above ``base``, scores drawn from a few values (ties across shards),
    sorted by (score desc, chunk asc)."""
    chunk = base + rng.choice(max(4 * n, 1), size=n, replace=False).astype(np.int64)
    score = rng.choice(tie_values, size=n)
    order = np.lexsort((chunk, -score))
    return chunk[order], score[order]


def _packed(rng, R, B, k, counts, bases, tie_values):
    """R per-rank buffers of rl_bm25_packed_bytes(B, k) bytes, end to end, plus the lists they hold."""
    lists, parts = [], []
    for r in range(R):
        chunk = np.full((B, k), -1, np.int64)
        score = np.full((B, k), -np.inf, np.float64)
        for b in range(B):
            n = int(counts[r, b])
            chunk[b, :n], score[b, :n] = _sorted_list(rng, n, bases[r], tie_values)
        raw = chunk.tobytes() + score.tobytes() + counts[r].astype(np.int32).tobytes()
        parts.append(raw + b"\0" * ((-len(raw)) % 16))
        lists.append((chunk, score))
    return b"".join(parts), lists


def _merge_numpy(lists, counts, k):
    B = counts.shape[1]
    ids = np.full((B, k), -1, np.int64)
    sc = np.full((B, k), -np.inf, np.float64)
    cnt = np.zeros(B, np.int32)
    for b in range(B):
        c = np.concatenate([lists[r][0][b, :counts[r, b]] for r in range(len(lists))])
        s = np.concatenate([lists[r][1][b, :counts[r, b]] for r in range(len(lists))])
        top = np.lexsort((c, -s))[:k]
        ids[b, :len(top)], sc[b, :len(top)], cnt[b] = c[top], s[top], len(top)
    return ids, sc, cnt


def _merge_device(raw, R, B, k):
    import torch

    from raglite_b200 import _lib

    lib = _lib.load()
    assert len(raw) == R * lib.rl_bm25_packed_bytes(B, k)
    g = torch.frombuffer(bytearray(raw), dtype=torch.uint8).cuda()
    oc = torch.empty((B, k), dtype=torch.int64, device="cuda")
    os_ = torch.empty((B, k), dtype=torch.float64, device="cuda")
    on = torch.empty(B, dtype=torch.int32, device="cuda")
    _lib.check(lib.rl_bm25_merge_packed(g.data_ptr(), R, B, k, oc.data_ptr(), os_.data_ptr(), on.data_ptr(),
                                        torch.cuda.current_stream().cuda_stream), "rl_bm25_merge_packed")
    return oc.cpu().numpy(), os_.cpu().numpy(), on.cpu().numpy()


@pytest.mark.parametrize("k", [1, 64, 4096])
@pytest.mark.parametrize("R", [1, 2, 3, 8, 64])
def test_merge_kernel_matches_numpy(rl, R, k):
    rng = np.random.default_rng(R * 7919 + k)
    B = 6 if R * k < 64 * 4096 else 4
    bases = [r * STRIDE for r in range(R)] if R % 2 == 0 else list(range(0, R * 4 * k, 4 * k))   # spaced / contiguous
    counts = np.zeros((R, B), np.int64)
    counts[:, 1] = k                                                   # every list full
    counts[:, 2] = rng.integers(0, k + 1, size=R)                      # mixed
    counts[:, 3] = np.where(rng.random(R) < 0.5, 0, rng.integers(1, k + 1, size=R))
    if B > 4:
        counts[:, 4] = rng.integers(0, 2, size=R)                      # zeros and ones
        counts[R // 2, 5] = k                                          # one list holds everything
    # query 0: all lists empty
    tie_values = np.array([2.5, 1.0, 1.0 + 2**-52, 0.125, 7.75])      # few values: ties across ranks everywhere
    worst = 0
    for ties in (tie_values, rng.random(64) * 20):
        raw, lists = _packed(rng, R, B, k, counts, bases, ties)
        got = _merge_device(raw, R, B, k)
        want = _merge_numpy(lists, counts, k)
        for g, w in zip(got, want, strict=True):
            assert np.array_equal(g, w), (R, k)
        worst = max(worst, int(got[2].max()))
    assert got[2][0] == 0 and (got[0][0] == -1).all()
    print(f"merge R={R} k={k}: bit-identical to NumPy, up to {worst} entries per query")


def test_merge_ties_come_out_by_ascending_global_chunk(rl):
    """Every entry of every shard has the same score: the merge is then the ascending order of the global chunks,
    interleaving the shards (spaced bases above 2^40 and contiguous bases both)."""
    R, B, k = 4, 2, 64
    for bases in ([r * STRIDE + 5 for r in range(R)], [0, 1, 2, 3]):
        counts = np.full((R, B), 20, np.int64)
        parts, lists = [], []
        for r in range(R):
            chunk = np.full((B, k), -1, np.int64)
            score = np.full((B, k), -np.inf)
            chunk[:, :20] = bases[r] + np.arange(20) * (R if bases[1] == 1 else 1)
            score[:, :20] = 3.25
            raw = chunk.tobytes() + score.tobytes() + counts[r].astype(np.int32).tobytes()
            parts.append(raw + b"\0" * ((-len(raw)) % 16))
            lists.append((chunk, score))
        ids, sc, cnt = _merge_device(b"".join(parts), R, B, k)
        assert (cnt == k).all() and (sc == 3.25).all()
        want = np.sort(np.concatenate([lists[r][0][0, :20] for r in range(R)]))[:k]
        assert np.array_equal(ids[0], want) and np.array_equal(ids[1], want)


# ---- corpora and shards ---------------------------------------------------------------------------------------------
def _chunks(rl, bodies, lo, hi, *, ids=None, docs=None):
    ids = ids or [f"c{c}" for c in range(len(bodies))]
    docs = docs or [f"d{c // 10}" for c in range(len(bodies))]
    return [rl.Chunk(id=ids[c], document_id=docs[c], index=c % 10, body=bodies[c]) for c in range(lo, hi)]


def _build(rl, bodies, ranges, bases, *, docs=None, seed=0):
    """The single index over every body and one shard per range (chunk ids ``c<position>``, metadata bucket = position
    % 5, one embedding row per chunk)."""
    from synth import make_corpus

    n = len(bodies)
    E, off = make_corpus(n, 1, 16, seed=seed)
    meta = [{"bucket": c % 5} for c in range(n)]
    single = rl.CorpusIndex(E, off, chunk_ids=[f"c{c}" for c in range(n)], chunks=_chunks(rl, bodies, 0, n, docs=docs),
                            chunk_metadata=meta)
    shards = [rl.CorpusIndex(E[lo:hi], off[lo:hi + 1] - lo, chunk_base=base, chunk_ids=[f"c{c}" for c in range(lo, hi)],
                             chunks=_chunks(rl, bodies, lo, hi, docs=docs), chunk_metadata=meta[lo:hi])
              for (lo, hi), base in zip(ranges, bases, strict=True)]
    return single, shards, E


def _sorted_stem_body(bodies):
    """One word per stem of the corpus, ordered by stem: a chunk 0 with this body makes the single index's term ids
    follow sorted-stem order."""
    word_of: dict[str, str] = {}
    for body in bodies:
        for w in _fts.tokenize(body):
            if w not in _fts.STOPWORDS:
                word_of.setdefault(_fts.stem(w), w)
    return " ".join(word_of[s] for s in sorted(word_of))


def _layout(C, R, kind):
    """R contiguous chunk ranges over [0, C): for R >= 3 an empty shard and a one-chunk shard; for R >= 4 a shard of
    stop-word-only bodies (``STOP_RANGE``), which holds none of any query's terms."""
    if R == 1:
        return [(0, C)]
    if R == 2:
        return [(0, C // 3), (C // 3, C)]
    cuts = [0, 1, 1]   # shard 0: chunk 0 alone, shard 1: empty
    if R >= 4:
        cuts.append(STOP_RANGE[1])   # shard 2: the stop-word bodies STOP_RANGE
    rest = R + 1 - len(cuts)
    lo = cuts[-1]
    cuts += [lo + (C - lo) * i // rest for i in range(1, rest + 1)]
    assert len(cuts) == R + 1 and cuts[-1] == C
    if kind == "reverse":   # the empty and one-chunk shards last
        sizes = np.diff(cuts)[::-1]
        cuts = [0, *np.cumsum(sizes).tolist()]
    return [(int(a), int(b)) for a, b in zip(cuts[:-1], cuts[1:], strict=True)]


STOP_RANGE = (1, 40)   # chunks whose bodies hold stop words only (see exact_corpus)
N_EXACT = 12_000
PLANTED = [3720, 5000, 6600, 9240, 11160]   # identical bodies, in different shards of every layout with R >= 2


@pytest.fixture(scope="module")
def exact_corpus():
    bodies = ko.make_bodies(N_EXACT, seed=17, vocab=3000, empty=0.03, dup=0.03)
    for c in range(*STOP_RANGE):
        bodies[c] = "the of and would, which THE."
    planted = "xylophonia " + next(b for b in bodies[5000:] if len(b.split()) >= 8)   # a word only these chunks hold
    for c in PLANTED:
        bodies[c] = planted
    bodies[0] = _sorted_stem_body(bodies[1:])
    queries = [planted] + _queries(11, 17, 3000, 300)
    return bodies, queries


def _to_single(ids, ranges, bases):
    out = ids.copy()
    for (lo, hi), base in zip(ranges, bases, strict=True):
        sel = (ids >= base) & (ids < base + (hi - lo))
        out[sel] = ids[sel] - base + lo
    return out


BK = [(1, 1), (7, 10), (256, 64), (300, 4096)]


@pytest.mark.parametrize("R,kind,spaced", [(1, "", False), (2, "", True), (3, "", False), (3, "reverse", True),
                                           (4, "", True), (8, "", False), (8, "reverse", True)])
def test_bit_identical_to_the_single_index(rl, exact_corpus, monkeypatch, R, kind, spaced):
    install(monkeypatch)
    bodies, queries = exact_corpus
    ranges = _layout(len(bodies), R, kind)
    bases = ShardedIndex.shard_bases(R) if spaced else [lo for lo, _ in ranges]
    single, shards, _ = _build(rl, bodies, ranges, bases, docs=["d-all"] + [f"d{c // 10}" for c in range(1, len(bodies))])
    single.delete_documents(["d-all"])
    single_order = single.keyword_index().analyzer.term_ids
    stems = list(single_order)
    assert stems == sorted(stems), "chunk 0 must number the stems in sorted order"
    owner0 = next(r for r, (lo, hi) in enumerate(ranges) if lo <= 0 < hi)

    def rank_fn(r, g):
        sh = ShardedIndex(shards[r], g if R > 1 else None)   # R = 1: the one-rank index without a group
        if r == owner0:
            assert shards[r].delete_documents(["d-all"]) == 1
        out = []
        for B, k in BK:
            qs = queries[:1] if B == 1 else queries[:B]
            out.append(rl.keyword_search_batch(qs, num_results=k, index=sh))
        return out

    results = run_ranks(R, rank_fn)
    compared = 0
    for i, (B, k) in enumerate(BK):
        qs = queries[:1] if B == 1 else queries[:B]
        w_ids, w_sc, w_cnt = rl.keyword_search_batch(qs, num_results=k, index=single)
        for r in range(R):
            ids, sc, cnt = results[r][i]
            assert np.array_equal(cnt, w_cnt), (R, B, k, r)
            assert np.array_equal(_to_single(ids, ranges, bases), w_ids), (R, B, k, r)
            assert np.array_equal(sc.view(np.int64), w_sc.view(np.int64)), (R, B, k, r)
            assert r == 0 or all(np.array_equal(a, b) for a, b in zip(results[r][i], results[0][i], strict=True))
        compared += int(w_cnt.sum())
        if B >= 7:
            assert w_cnt[0] >= 5 and w_cnt[1] == 0      # the planted body; unknown-only query
    # the planted duplicates tie at the top (k = 1 cuts among them) and come out in ascending chunk order
    ids, sc, _ = results[0][2]
    assert list(_to_single(ids[0, :5], ranges, bases)) == PLANTED and (sc[0, :5] == sc[0, 0]).all() and sc[0, 5] < sc[0, 0]
    assert list(_to_single(results[0][0][0][0], ranges, bases)) == PLANTED[:1]
    print(f"R={R} {kind or 'forward'} {'spaced' if spaced else 'contiguous'}: {compared} scores bit-identical (0 ulp)")


# ---- b. an ordinary corpus against the oracle --------------------------------------------------------------------------
@pytest.fixture(scope="module")
def plain_corpus():
    bodies = ko.make_bodies(15_000, seed=23, vocab=4000)
    ix = ko.create_fts_index(bodies)
    order = {t: i for i, t in enumerate(sorted(ix.dict))}
    return bodies, ix, order, _queries(29, 23, 4000, 120)


def _oracle_check(ids, scores, counts, queries, ix, order, k, *, allowed=None, live=None):
    worst = 0.0
    for b, q in enumerate(queries):
        all_scores = ko.match_bm25(ix, q, term_order=order)
        want_ids, want_scores = ko.keyword_search(ix, q, num_results=k, term_order=order, allowed=allowed)
        _check(ids[b], scores[b], counts[b], want_ids, want_scores, all_scores, allowed=allowed)
        n = int(counts[b])
        if n:
            worst = max(worst, float(np.max(np.abs(scores[b, :n] - want_scores) / np.abs(want_scores))))
    return worst


def test_plain_corpus_against_the_oracle_and_across_r(rl, plain_corpus, monkeypatch):
    install(monkeypatch)
    bodies, ix, order, queries = plain_corpus
    C = len(bodies)
    first = None
    worst = 0.0
    for R, ranges in [(1, [(0, C)]), (2, [(0, 6000), (6000, C)]), (4, [(0, 100), (100, 100), (100, 9000), (9000, C)])]:
        bases = ShardedIndex.shard_bases(R)
        _, shards, _ = _build(rl, bodies, ranges, bases)
        got = run_ranks(R, lambda r, g, shards=shards: rl.keyword_search_batch(queries, num_results=64,
                                                                               index=ShardedIndex(shards[r], g)))
        ids, sc, cnt = got[0]
        for r in range(1, R):
            assert all(np.array_equal(a, b) for a, b in zip(got[r], got[0], strict=True))
        ids = _to_single(ids, ranges, bases)
        worst = max(worst, _oracle_check(ids, sc, cnt, queries, ix, order, 64))
        if first is None:
            first = (ids, sc, cnt)
        else:
            assert all(np.array_equal(a, b) for a, b in zip((ids, sc, cnt), first, strict=True)), R
    assert worst <= REL
    print(f"plain corpus: worst relative score error against the oracle {worst:.3e}; R = 1, 2, 4 bit-identical")


# ---- c. the index changing under the search ---------------------------------------------------------------------------
def _as_ids(resolve, result):
    """(chunk ids [B] lists, scores, counts) of a search result, resolved right after it (numbering changes at compact)."""
    ids, sc, cnt = result
    return [[resolve(int(c)) for c in ids[b, :cnt[b]]] for b in range(len(cnt))], sc, cnt


def test_changes_on_one_rank(rl, monkeypatch):
    from synth import make_corpus

    install(monkeypatch)
    bodies = ko.make_bodies(9000, seed=31, vocab=2500)
    R, C = 3, len(bodies)
    ranges = [(0, 2500), (2500, 6000), (6000, C)]
    single, shards, _ = _build(rl, bodies, ranges, ShardedIndex.shard_bases(R), seed=2)
    queries = _queries(37, 31, 2500, 50) + ["zebraword quokkaword", "zebraword"]
    extra = [f"zebraword quokkaword {b}" for b in ko.make_bodies(300, seed=32, vocab=2500)] + ["", "zebraword"]
    E2, off2 = make_corpus(len(extra), 1, 16, seed=9)
    new = [rl.Chunk(id=f"x{c}", document_id=f"x{c // 10}", index=c % 10, body=extra[c]) for c in range(len(extra))]
    meta_new = [{"bucket": 0}] * len(new)
    gone = [f"d{i}" for i in range(250, 600, 3)]           # documents of shard 1
    gone0 = ["d3", "d7"]                                    # documents of shard 0, deleted and compacted away
    k = 40

    def changes(idx, r, sh):
        """The searches and changes of one rank (``sh`` the ShardedIndex) or of the single index (``r`` None)."""
        resolve = sh.chunk_id_of if sh is not None else idx.chunk_id_of
        target = sh if sh is not None else idx
        out = [_as_ids(resolve, rl.keyword_search_batch(queries, num_results=k, index=target))]
        if r in (None, 1):
            assert idx.delete_documents(gone) > 0
        out.append(_as_ids(resolve, rl.keyword_search_batch(queries, num_results=k, index=target)))
        if r in (None, 2):
            idx.append(E2, off2, chunk_ids=[c.id for c in new], chunks=new, chunk_metadata=meta_new)
        if sh is not None:
            sh.refresh(chunk_ids=True)
        out.append(_as_ids(resolve, rl.keyword_search_batch(queries, num_results=k, index=target)))
        if r in (None, 0):
            assert idx.delete_documents(gone0) > 0
            idx.compact()
        if sh is not None:
            sh.refresh(chunk_ids=True)
        out.append(_as_ids(resolve, rl.keyword_search_batch(queries, num_results=k, index=target)))
        out.append(_as_ids(resolve, rl.keyword_search_batch(queries, num_results=k, index=target,
                                                            metadata_filter={"bucket": 2})))
        return out

    got = run_ranks(R, lambda r, g: changes(shards[r], r, ShardedIndex(shards[r], g)))
    want = changes(single, None, None)
    # the oracle over every body ever indexed, numbered by position; each step's live set and filter
    all_bodies = bodies + extra
    pos = {f"c{c}": c for c in range(C)} | {f"x{c}": C + c for c in range(len(extra))}
    doc_of = [f"d{c // 10}" for c in range(C)] + [c.document_id for c in new]
    present = np.arange(len(all_bodies)) < C
    after1 = present & ~np.isin(doc_of, gone)
    after2 = after1 | (np.arange(len(all_bodies)) >= C)
    after3 = after2 & ~np.isin(doc_of, gone0)
    bucket = np.asarray([c % 5 == 2 for c in range(C)] + [False] * len(extra))
    steps = [("built", present, None), ("delete on rank 1", after1, None), ("append on rank 2", after2, None),
             ("compact on rank 0", after3, None), ("filter", after3, bucket)]
    worst = 0.0
    for s, (name, live, allowed) in enumerate(steps):
        ix = ko.create_fts_index(all_bodies, live=live)
        order = {t: i for i, t in enumerate(sorted(ix.dict))}
        for r in range(R):
            assert got[r][s][0] == got[0][s][0] and np.array_equal(got[r][s][1], got[0][s][1]), (name, r)
        g_ids, g_sc, g_cnt = got[0][s]
        w_ids, w_sc, w_cnt = want[s]
        assert np.array_equal(g_cnt, w_cnt), name
        np.testing.assert_allclose(g_sc, w_sc, rtol=REL, atol=0, err_msg=name)      # the single index, same changes
        as_pos = np.full((len(queries), k), -1, np.int64)
        for b, row in enumerate(g_ids):
            as_pos[b, :len(row)] = [pos[c] for c in row]
        worst = max(worst, _oracle_check(as_pos, g_sc, g_cnt, queries, ix, order, k,
                                         allowed=None if allowed is None else allowed & live))
    print(f"changes on one rank: every step within {REL:g} of the single index; worst against the oracle {worst:.3e}")


# ---- d. ids, hybrid search, collectives -----------------------------------------------------------------------------
def test_keyword_and_hybrid_search_on_a_registered_sharded_index(rl, exact_corpus, monkeypatch):
    from synth import make_queries

    import raglite_b200._search as S

    shim = install(monkeypatch)
    bodies, queries = exact_corpus
    R = 3
    ranges = [(0, 3000), (3000, 7000), (7000, len(bodies))]
    single, shards, E = _build(rl, bodies, ranges, ShardedIndex.shard_bases(R), seed=5)
    q_text = queries[0]
    q_vec = make_queries(E, 1, seed=6)[0]
    cfg1 = rl.RAGLiteConfig(db_url="kw-threads://single", reranker=None)
    rl.register_index(cfg1, single)
    try:
        want_kw = rl.keyword_search(q_text, num_results=30, config=cfg1)
    finally:
        rl.unregister_index(cfg1)
    orig_vs = S.vector_search
    monkeypatch.setattr(S, "vector_search", lambda query, **kw: orig_vs(q_vec if isinstance(query, str) else query, **kw))
    calls = {}

    def rank_fn(r, g):
        cfg = rl.RAGLiteConfig(db_url=f"kw-threads://rank{r}", reranker=None)
        sh = ShardedIndex(shards[r], g)
        rl.register_index(cfg, sh)
        try:
            g.shared.wait()
            if r == 0:
                shim.calls.clear()
            g.shared.wait()
            rl.keyword_search_batch(queries[:40], num_results=20, index=sh)
            g.shared.wait()
            if r == 0:
                calls.update(shim.calls)
            kw_ids, kw_sc = rl.keyword_search(q_text, num_results=30, config=cfg)
            vs_ids, _ = rl.vector_search(q_vec, num_results=10, config=cfg)
            ks_ids, _ = rl.keyword_search(q_text, num_results=10, config=cfg)
            hy = rl.hybrid_search(q_text, num_results=5, config=cfg)
            return (kw_ids, kw_sc), vs_ids, ks_ids, hy
        finally:
            rl.unregister_index(cfg)

    got = run_ranks(R, rank_fn)
    assert calls == {"all_reduce": 1, "all_gather_into_tensor": 1}, calls
    owned = {f"c{c}" for c in range(ranges[0][1], len(bodies))}
    for r in range(R):
        (kw_ids, kw_sc), vs_ids, ks_ids, (h_ids, h_sc) = got[r]
        assert (kw_ids, kw_sc) == want_kw              # the chunk ids of every rank, the single index's scores
        assert set(kw_ids) & owned, "some keyword hits must be owned by ranks > 0"
        f_ids, f_sc = rl.reciprocal_rank_fusion([vs_ids, ks_ids], weights=[0.75, 0.25])
        assert h_ids == f_ids[:5] and h_sc == f_sc[:5]
        assert got[r][1:] == got[0][1:]
