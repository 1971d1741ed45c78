"""ts_rank keyword search on the GPU (``rl_tsrank_topk_global`` behind the PostgreSQL branch of ``keyword_search``)
against the bit-exact NumPy restatement of ``calc_rank_or`` in ``tsrank_oracle``: float32 scores bitwise equal and ids
equal, at the C-ABI, through the public path of a ``CorpusIndex`` built from PostgreSQL rows, and on a ``ShardedIndex``
of R thread ranks on one GPU (``thread_group``)."""

from __future__ import annotations

import numpy as np
import pytest
from thread_group import install, run_ranks

import keyword_oracle as ko
import tsrank_oracle as to
from raglite_b200 import _pgfts
from raglite_b200._dist import ShardedIndex

pytestmark = pytest.mark.gpu

PG = "postgresql://localhost/raglite_tsrank_tests"


@pytest.fixture(scope="module")
def rl():
    import torch

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import raglite_b200

    return raglite_b200


# ---- a. the kernels at the C-ABI ----------------------------------------------------------------------------------------
def _up(a, dtype):
    import torch

    a = np.concatenate([np.asarray(a, dtype).ravel(), np.zeros(1, dtype)])
    return torch.from_numpy(a).cuda()


def _device_topk(csr, C, q_off, q_terms, k, *, mask=None, chunk_base=0, group=None):
    """``rl_tsrank_topk_global`` on host arrays; the packed buffer starts filled with 0xA5 (pad bytes checked zeroed)."""
    import torch

    from raglite_b200 import _lib as L

    lib = L.load()
    term_off, doc, npos = csr
    B, V = len(q_off) - 1, len(term_off) - 1
    keep = [_up(term_off, np.int64), _up(doc, np.int32), _up(npos, np.int32), None if mask is None else _up(mask, np.uint8),
            _up(q_off, np.int32), _up(q_terms, np.int32)]
    ptr = [None if t is None else t.data_ptr() for t in keep]
    need = int(lib.rl_bm25_workspace_bytes(C, B if group is None else group))
    ws = torch.empty(need, dtype=torch.uint8, device="cuda") if need else None
    nbytes = int(lib.rl_bm25_packed_bytes(B, k))
    packed = torch.full((max(nbytes, 16),), 0xA5, dtype=torch.uint8, device="cuda")
    L.check(lib.rl_tsrank_topk_global(ptr[0], ptr[1], ptr[2], V, C, ptr[3], ptr[4], ptr[5], B, k, chunk_base,
                                      packed.data_ptr(), None if ws is None else ws.data_ptr(), need,
                                      torch.cuda.current_stream().cuda_stream), "rl_tsrank_topk_global")
    raw = packed.cpu().numpy()[:nbytes]
    used = B * k * 16 + B * 4
    assert (raw[used:] == 0).all(), "the packed buffer's pad bytes must be zeroed"
    return (raw[: B * k * 8].view(np.int64).reshape(B, k), raw[B * k * 8: B * k * 16].view(np.float64).reshape(B, k),
            raw[B * k * 16: used].view(np.int32))


def _assert_same(got, want, what):
    for g, w, name in zip(got, want, ("ids", "scores", "counts"), strict=True):
        if name == "scores":
            assert np.array_equal(g.view(np.int64), w.view(np.int64)), (what, name)
            fin = np.isfinite(g)
            assert np.array_equal(g[fin], g[fin].astype(np.float32).astype(np.float64)), "scores are widened float32"
        else:
            assert np.array_equal(g, w), (what, name)


def _random_csr(rng, V, C, *, max_npos=256, density=0.05):
    postings = []
    for _ in range(V):
        n = int(rng.integers(0, int(C * density) + 2))
        chunks = np.sort(rng.choice(C, size=min(n, C), replace=False))
        npos = np.where(rng.random(len(chunks)) < 0.7, 1 + rng.geometric(0.5, len(chunks)),
                        rng.integers(1, max_npos + 1, len(chunks)))
        postings.append((chunks, np.minimum(npos, max_npos)))
    term_off = np.concatenate([[0], np.cumsum([len(c) for c, _ in postings])]).astype(np.int64)
    doc = np.concatenate([c for c, _ in postings]).astype(np.int32)
    npos = np.concatenate([n for _, n in postings]).astype(np.int32)
    return term_off, doc, npos


def _random_plan(rng, V, B, *, max_entries=16, unknown=0.2):
    q_off, terms = [0], []
    for _ in range(B):
        m = int(rng.integers(1, max_entries + 1))
        ids = list(rng.choice(V, size=min(m, V), replace=False))
        ids = [-1 if rng.random() < unknown else int(t) for t in ids]
        terms += ids
        q_off.append(len(terms))
    return np.asarray(q_off, np.int32), np.asarray(terms, np.int32)


def test_every_npos_and_clamping(rl):
    """Lexeme 0 held by chunk c with npos c + 1 for c < 256: one query reaches every contribution.  Lexeme 1 holds
    npos values outside [1, 256] (clamped, never read out of bounds)."""
    C = 300
    bad = np.array([0, -7, 257, 1 << 20, 256, 1], np.int32)
    term_off = np.array([0, 256, 256 + len(bad)], np.int64)
    doc = np.concatenate([np.arange(256), np.arange(256, 256 + len(bad))]).astype(np.int32)
    npos = np.concatenate([np.arange(1, 257), bad]).astype(np.int32)
    q_off, q_terms = np.array([0, 1, 2, 4], np.int32), np.array([0, 1, 0, -1], np.int32)
    scores, matched = to.tsrank_csr_scores(term_off, doc, npos, q_off, q_terms, C)
    got = _device_topk((term_off, doc, npos), C, q_off, q_terms, 4096)
    _assert_same(got, to.tsrank_topk(scores, matched, None, 4096), "every npos")
    ids, sc, cnt = got
    assert cnt.tolist() == [256, len(bad), 256]
    by_chunk = dict(zip(ids[0, :256].tolist(), sc[0, :256].tolist(), strict=True))
    assert [by_chunk[c] for c in range(256)] == [float(to.rank([n], 1)) for n in range(1, 257)]
    assert str(np.float32(by_chunk[0])) == "0.06079271" and str(np.float32(by_chunk[1])) == "0.075990885"
    halved = dict(zip(ids[2, :256].tolist(), sc[2, :256].tolist(), strict=True))   # one unknown entry: size 2
    assert [halved[c] for c in range(256)] == [float(to.rank([n], 2)) for n in range(1, 257)]


@pytest.mark.parametrize("k", [1, 64, 4096])
def test_random_postings_against_the_oracle(rl, k):
    rng = np.random.default_rng(k)
    V, C, B = 60, 11_000, 40   # three score tiles, the last one partial
    csr = _random_csr(rng, V, C)
    q_off, q_terms = _random_plan(rng, V, B)
    q_terms[q_off[3]:q_off[4]] = -1                    # a query of unknown entries only
    scores, matched = to.tsrank_csr_scores(*csr, q_off, q_terms, C)
    mask = rng.random(C) < 0.8
    for m, base, group in ((None, 0, None), (mask, 0, 3), (mask, (1 << 40) + 17, 7), (None, 5, 1)):
        got = _device_topk(csr, C, q_off, q_terms, k, mask=m, chunk_base=base, group=group)
        _assert_same(got, to.tsrank_topk(scores, matched, m, k, chunk_base=base), (k, group))
        assert got[2][3] == 0
    assert int(matched.sum()) > 20_000


def test_massive_ties_at_the_cut(rl):
    """Every chunk holds lexeme 0 with npos 1: one score for all; the cut at k falls among equal scores and the chunks
    come out in ascending order.  A second query's lexeme is held by every other chunk, with npos 3."""
    C = 9000
    term_off = np.array([0, C, C + C // 2], np.int64)
    doc = np.concatenate([np.arange(C), np.arange(0, C, 2)]).astype(np.int32)
    npos = np.concatenate([np.ones(C), np.full(C // 2, 3)]).astype(np.int32)
    q_off, q_terms = np.array([0, 1, 2], np.int32), np.array([0, 1], np.int32)
    scores, matched = to.tsrank_csr_scores(term_off, doc, npos, q_off, q_terms, C)
    mask = (np.arange(C) % 7) != 3
    for k in (1, 2, 63, 64, 4095, 4096):
        for m in (None, mask):
            got = _device_topk((term_off, doc, npos), C, q_off, q_terms, k, mask=m, group=1)
            _assert_same(got, to.tsrank_topk(scores, matched, m, k), ("ties", k))
            allowed = np.flatnonzero(np.ones(C, bool) if m is None else m)
            assert got[0][0, :k].tolist() == allowed[:k].tolist()


def test_empty_shard_and_empty_batch(rl):
    csr = (np.zeros(3, np.int64), np.zeros(0, np.int32), np.zeros(0, np.int32))
    ids, sc, cnt = _device_topk(csr, 0, np.array([0, 2, 2], np.int32), np.array([0, -1], np.int32), 64, chunk_base=9)
    assert (cnt == 0).all() and (ids == -1).all() and np.isneginf(sc).all()
    ids, sc, cnt = _device_topk(csr, 0, np.array([0], np.int32), np.zeros(0, np.int32), 5)
    assert ids.shape == (0, 5) and cnt.shape == (0,)
    rng = np.random.default_rng(1)
    csr = _random_csr(rng, 10, 500)
    ids, _, cnt = _device_topk(csr, 500, np.array([0], np.int32), np.zeros(0, np.int32), 5)
    assert ids.shape == (0, 5)
    ids, sc, cnt = _device_topk(csr, 500, np.array([0, 0], np.int32), np.zeros(0, np.int32), 5)   # no entries: nothing
    assert cnt[0] == 0 and (ids == -1).all()


def test_identical_run_to_run(rl):
    rng = np.random.default_rng(9)
    csr = _random_csr(rng, 80, 20_000)
    q_off, q_terms = _random_plan(rng, 80, 64)
    a = _device_topk(csr, 20_000, q_off, q_terms, 256, group=5)
    b = _device_topk(csr, 20_000, q_off, q_terms, 256)
    _assert_same(a, b, "run to run")


# ---- b. the public path on a CorpusIndex built from PostgreSQL rows -------------------------------------------------------
def _corpus(n, seed, *, vocab_n=500):
    """Bodies of lowercase words and their ``to_tsvector('simple', body)::text`` (positions = word order, at most 256 per
    lexeme); ``table`` = chunk -> {lexeme: npos}.  Lexeme ids in order of first appearance differ from byte order."""
    rng = np.random.default_rng(seed)
    vocab = ko.make_vocab(vocab_n, seed)
    p = 1.0 / np.arange(1, len(vocab) + 1) ** 1.07
    p /= p.sum()
    bodies, texts, table = [], [], {}
    for c in range(n):
        m = int(rng.integers(0, 80)) if rng.random() > 0.03 else 0
        words = [vocab[i] for i in rng.choice(len(vocab), size=m, p=p)]
        if m and rng.random() < 0.05:
            words += [words[-1]] * int(rng.integers(1, 300))
        held: dict[str, list[int]] = {}
        for i, w in enumerate(words):
            held.setdefault(w, []).append(i + 1)
        held = {w: ps[:256] for w, ps in held.items()}
        bodies.append(" ".join(words))
        texts.append(to.tsvector_text(held))
        table[c] = {w: len(ps) for w, ps in held.items()}
    return vocab, bodies, texts, table


def _queries(vocab, seed, n):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        m = int(rng.integers(1, 14))
        ws = [vocab[int(i) % len(vocab)] for i in rng.zipf(1.3, size=m)]
        if rng.random() < 0.3:
            ws.append("qqzzunknown")
        out.append(", ".join(w.upper() if rng.random() < 0.2 else w for w in ws) + "?")
    return out + ["qqzzunknown", "!!!", vocab[0], f"{vocab[0]} {vocab[1]} {vocab[2]} {vocab[0]}"]


def _build(rl, n, seed, lo=0, hi=None, *, base=0, ids=None):
    from synth import make_corpus

    from raglite_b200._rows import vector_to_halfvec_text

    hi = n if hi is None else hi
    vocab, bodies, texts, table = _corpus(n, seed)
    E, _ = make_corpus(n, 1, 16, seed=seed, fp16_round=True)
    ids = ids or [f"c{c}" for c in range(n)]
    rows = [(ids[c], vector_to_halfvec_text(E[c])) for c in range(lo, hi)]
    chunks = [rl.Chunk(id=ids[c], document_id=f"d{c // 10}", index=c % 10, body=bodies[c]) for c in range(lo, hi)]
    meta = [{"bucket": c % 5} for c in range(lo, hi)]
    if hi > lo:
        idx = rl.CorpusIndex.from_table_rows(rows, "postgresql", chunks=chunks, chunk_metadata=meta, chunk_base=base)
    else:   # an empty shard
        idx = rl.CorpusIndex(E[:0], np.zeros(1, np.int64), chunk_ids=[], chunks=[], chunk_metadata=[], chunk_base=base)
    return idx, E, vocab, bodies, [(ids[c], texts[c]) for c in range(n)], table


def _oracle(table, live, queries, k):
    """(ids [B][<=k], float32 scores [B][<=k]) by (score desc, chunk asc) over the chunks ``live`` allows."""
    out = []
    for q in queries:
        s = to.ts_rank_table({c: h for c, h in table.items() if live[c]}, _pgfts.query_lexemes(q))
        order = sorted(s, key=lambda c: (-float(s[c]), c))[:k]
        out.append((order, [s[c] for c in order]))
    return out


def _check(result, want):
    ids, sc, cnt = result
    for b, (w_ids, w_sc) in enumerate(want):
        n = int(cnt[b])
        assert ids[b, :n].tolist() == w_ids, b
        assert np.array_equal(sc[b, :n], np.asarray(w_sc, np.float32).astype(np.float64)), b
        assert (ids[b, n:] == -1).all() and np.isneginf(sc[b, n:]).all()


def test_public_path_against_the_oracle(rl):
    n = 6000
    idx, E, vocab, bodies, tsv, table = _build(rl, n, 3)
    lex_first = list(dict.fromkeys(x for _, t in tsv for x in _pgfts.parse_tsvector(t)[0]))
    assert lex_first != sorted(lex_first, key=str.encode)
    cfg = rl.RAGLiteConfig(db_url=PG, reranker=None)
    with pytest.raises(NotImplementedError, match="add_tsvector_rows"):
        rl.keyword_search_batch(["x"], config=cfg, index=idx)
    rng = np.random.default_rng(0)
    order = rng.permutation(n)
    assert idx.add_tsvector_rows([tsv[i] for i in order]) == n          # any order
    with pytest.raises(ValueError, match="already has a tsvector"):
        idx.add_tsvector_rows([tsv[5]])
    with pytest.raises(ValueError, match="not in the index"):
        idx.add_tsvector_rows([("nope", "'a':1")])
    queries = _queries(vocab, 3, 60)
    live = np.ones(n, bool)
    for k in (1, 64, 4096):
        got = rl.keyword_search_batch(queries, num_results=k, config=cfg, index=idx)
        _check(got, _oracle(table, live, queries, k))
    # keyword_search: chunk ids and pg8000's float4 values
    rl.register_index(cfg, idx)
    try:
        w_ids, w_sc = _oracle(table, live, [queries[0]], 10)[0]
        got_ids, got_sc = rl.keyword_search(queries[0], num_results=10, config=cfg)
        assert got_ids == [f"c{c}" for c in w_ids]
        assert got_sc == [float(str(np.float32(s))) for s in w_sc] and all(isinstance(s, float) for s in got_sc)
        with pytest.raises(NotImplementedError, match="phrase"):
            rl.keyword_search("what’s new", config=cfg)
        with pytest.raises(ValueError, match="outside"):
            rl.keyword_search("x", num_results=4097, config=cfg)
        # metadata filter: a WHERE around the ranking
        allowed = np.arange(n) % 5 == 2
        got = rl.keyword_search_batch(queries, num_results=50, config=cfg, index=idx, metadata_filter={"bucket": 2})
        _check(got, _oracle(table, allowed, queries, 50))
        # hybrid_search = vector search + ts_rank + RRF composed on the host side
        from synth import make_queries

        import raglite_b200._search as S

        q_vec = make_queries(E, 1, seed=4)[0]
        orig = S.vector_search
        S.vector_search = lambda query, **kw: orig(q_vec if isinstance(query, str) else query, **kw)
        try:
            h_ids, h_sc = rl.hybrid_search(queries[1], num_results=5, config=cfg)
            vs_ids, _ = rl.vector_search(q_vec, num_results=10, config=cfg)
        finally:
            S.vector_search = orig
        ks_ids = [f"c{c}" for c in _oracle(table, live, [queries[1]], 10)[0][0]]
        f_ids, f_sc = rl.reciprocal_rank_fusion([vs_ids, ks_ids], weights=[0.75, 0.25])
        assert (h_ids, h_sc) == (f_ids[:5], f_sc[:5])
    finally:
        rl.unregister_index(cfg)
    # a DuckDB config on the same index still ranks by BM25
    duck = rl.keyword_search_batch(queries[:20], num_results=20, index=idx, config=rl.RAGLiteConfig(db_url="mem://duck"))
    ix = ko.create_fts_index(bodies)
    term_order = idx.keyword_index().analyzer.term_ids
    for b, q in enumerate(queries[:20]):
        w_ids, w_sc = ko.keyword_search(ix, q, num_results=20, term_order=term_order)
        assert duck[0][b, : duck[2][b]].tolist() == w_ids
        np.testing.assert_allclose(duck[1][b, : duck[2][b]], w_sc, rtol=1e-12)


def test_delete_compact_append_and_missing_tsvectors(rl):
    from synth import make_corpus

    from raglite_b200._rows import vector_to_halfvec_text

    n = 3000
    idx, _, vocab, _, tsv, table = _build(rl, n, 5)
    idx.add_tsvector_rows(tsv)
    cfg = rl.RAGLiteConfig(db_url=PG)
    queries = _queries(vocab, 5, 40)
    live = np.ones(n, bool)
    gone = [f"d{i}" for i in range(0, 300, 4)]
    assert idx.delete_documents(gone) > 0
    live &= ~np.isin([f"d{c // 10}" for c in range(n)], gone)
    _check(rl.keyword_search_batch(queries, num_results=64, config=cfg, index=idx), _oracle(table, live, queries, 64))
    idx.compact()
    kept = np.flatnonzero(live)
    got = rl.keyword_search_batch(queries, num_results=64, config=cfg, index=idx)
    want = _oracle(table, live, queries, 64)
    _check((np.where(got[0] >= 0, kept[np.maximum(got[0], 0)], -1), got[1], got[2]), want)
    # append 200 chunks: searching before their tsvectors arrive is refused, afterwards they rank
    _, _, e_texts, e_table = _corpus(200, 77)
    E2, off2 = make_corpus(200, 1, 16, seed=8, fp16_round=True)
    new = [rl.Chunk(id=f"x{c}", document_id=f"x{c // 10}", index=c % 10, body="") for c in range(200)]
    idx.append_table_rows([(f"x{c}", vector_to_halfvec_text(E2[c])) for c in range(200)], "postgresql", chunks=new,
                          chunk_metadata=[{"bucket": 0}] * 200)
    with pytest.raises(ValueError, match="200 live chunks have no tsvector"):
        rl.keyword_search_batch(queries, num_results=5, config=cfg, index=idx)
    idx.add_tsvector_rows([(f"x{c}", e_texts[c]) for c in range(200)])
    all_table = {i: table[int(c)] for i, c in enumerate(kept)} | {len(kept) + c: e_table[c] for c in range(200)}
    got = rl.keyword_search_batch(queries, num_results=64, config=cfg, index=idx)
    _check(got, _oracle(all_table, np.ones(len(all_table), bool), queries, 64))
    # a deleted chunk needs no tsvector
    idx2, _, _, _, tsv2, _ = _build(rl, 100, 6)
    idx2.add_tsvector_rows(tsv2[1:])
    with pytest.raises(ValueError, match="1 live chunks have no tsvector"):
        rl.keyword_search_batch(["x"], config=cfg, index=idx2)
    idx2.delete_chunks(["c0"])
    assert rl.keyword_search_batch(["x"], config=cfg, index=idx2)[2].shape == (1,)


# ---- c. a ShardedIndex of R thread ranks ---------------------------------------------------------------------------------
def _layout(n, R):
    if R == 1:
        return [(0, n)]
    cuts = [0, 1, 1] if R >= 3 else [0]   # R >= 3: a one-chunk shard and an empty shard
    rest = R + 1 - len(cuts)
    lo = cuts[-1]
    cuts += [lo + (n - lo) * i // rest for i in range(1, rest + 1)]
    return [(cuts[i], cuts[i + 1]) for i in range(R)]


@pytest.mark.parametrize("R", [1, 2, 3, 8])
def test_sharded_bit_identical_to_the_single_index(rl, monkeypatch, R):
    install(monkeypatch)
    n = 5000
    single, _, vocab, _, tsv, table = _build(rl, n, 11)
    single.add_tsvector_rows(tsv)
    ranges = _layout(n, R)
    bases = ShardedIndex.shard_bases(R) if R % 2 == 0 else [lo for lo, _ in ranges]
    shards = [_build(rl, n, 11, lo, hi, base=b)[0] for (lo, hi), b in zip(ranges, bases, strict=True)]
    cfg = rl.RAGLiteConfig(db_url=PG)
    queries = _queries(vocab, 11, 50)

    def rank_fn(r, g):
        sh = ShardedIndex(shards[r], g if R > 1 else None)
        assert sh.add_tsvector_rows(tsv) == ranges[r][1] - ranges[r][0]   # every rank gets the whole result set
        return [rl.keyword_search_batch(queries, num_results=k, config=cfg, index=sh) for k in (1, 64, 4096)] + [
            rl.keyword_search_batch(queries, num_results=30, config=cfg, index=sh, metadata_filter={"bucket": 1})]

    got = run_ranks(R, rank_fn)
    want = [rl.keyword_search_batch(queries, num_results=k, config=cfg, index=single) for k in (1, 64, 4096)] + [
        rl.keyword_search_batch(queries, num_results=30, config=cfg, index=single, metadata_filter={"bucket": 1})]
    for r in range(R):
        for (ids, sc, cnt), (w_ids, w_sc, w_cnt) in zip(got[r], want, strict=True):
            local = ids.copy()
            for (lo, hi), b in zip(ranges, bases, strict=True):
                sel = (ids >= b) & (ids < b + hi - lo)
                local[sel] = ids[sel] - b + lo
            assert np.array_equal(cnt, w_cnt) and np.array_equal(local, w_ids)
            assert np.array_equal(sc.view(np.int64), w_sc.view(np.int64))
    _check(want[1], _oracle(table, np.ones(n, bool), queries, 64))


def test_sharded_missing_tsvectors_raise_on_every_rank(rl, monkeypatch):
    install(monkeypatch)
    n, R = 2000, 3
    ranges = _layout(n, R)
    shards = [_build(rl, n, 13, lo, hi, base=lo)[0] for lo, hi in ranges]
    tsv = [(f"c{c}", t) for c, t in enumerate(_corpus(n, 13)[2])]
    cfg = rl.RAGLiteConfig(db_url=PG)

    def attempt(r, g, rows):
        sh = ShardedIndex(shards[r], g)
        if rows is not None:
            sh.add_tsvector_rows(rows)
        try:
            rl.keyword_search_batch(["a b c"], num_results=5, config=cfg, index=sh)
        except (ValueError, NotImplementedError) as e:
            return type(e).__name__, str(e)
        return "ok", ""

    # nobody has tsvectors: NotImplementedError everywhere
    got = run_ranks(R, lambda r, g: attempt(r, g, None), timeout=60)
    assert [x[0] for x in got] == ["NotImplementedError"] * R
    # the last shard misses one chunk's tsvector: every rank raises the same ValueError, none waits in the all-gather
    rows = [t for t in tsv if t[0] != f"c{n - 1}"]
    got = run_ranks(R, lambda r, g: attempt(r, g, rows), timeout=60)
    assert [x[0] for x in got] == ["ValueError"] * R and len({x[1] for x in got}) == 1
    assert "1 live chunks have no tsvector" in got[0][1]
