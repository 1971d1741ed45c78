"""SURVEY 8f-3: Reciprocal Rank Fusion / hybrid_search and the span collation of retrieve_chunk_spans, batched on
device chunk indices (``rl_rrf_fuse``, ``rl_span_collate``) against the oracle -- the RRF oracle itself is pinned
to outputs of the reference's own function (``tests/golden/rrf.npz``)."""

from __future__ import annotations

import json

import numpy as np
import pytest

from oracle import fusion as ofu


@pytest.fixture(scope="module")
def rrf_cases(golden_dir):
    return json.loads(bytes(np.load(golden_dir / "rrf.npz")["cases"]).decode())


def test_oracle_rrf_is_the_reference_function(rrf_cases):
    for c in rrf_cases:
        ids, scores = ofu.reciprocal_rank_fusion(c["rankings"], k=c["k"], weights=c["weights"])
        assert ids == c["ids"] and scores == c["scores"]          # same floats, bit for bit


def test_oracle_span_collation_example():
    table = {("A", i) for i in range(12)} | {("B", i) for i in range(5)}
    spans = ofu.collate_chunk_spans([("A", 5), ("B", 2), ("A", 6), ("A", 9)], table, neighbors=None)
    assert [s for s, _ in spans] == [[("A", 5), ("A", 6)], [("B", 2)], [("A", 9)]]
    spans = ofu.collate_chunk_spans([("A", 5), ("B", 2), ("A", 9)], table, neighbors=(-1, 1))
    assert [s for s, _ in spans][0] == [("A", 4), ("A", 5), ("A", 6)] and len(spans) == 3


@pytest.mark.gpu
def test_rrf_kernel_matches_the_reference_bit_for_bit(rrf_cases):
    import torch

    import raglite_b200 as rl

    for c in rrf_cases:
        R = len(c["rankings"])
        L = max(1, max(len(r) for r in c["rankings"]))
        t = np.full((1, R, L), -1, np.int64)
        for r, ranking in enumerate(c["rankings"]):
            t[0, r, : len(ranking)] = ranking
        ids, score, count = rl.rrf_fuse_device(torch.from_numpy(t).cuda(), c["weights"], k=c["k"])
        n = int(count[0])
        assert ids[0, :n].tolist() == c["ids"] and score[0, :n].tolist() == c["scores"]
        assert (ids[0, n:] == -1).all()
        got_ids, got_scores = rl.reciprocal_rank_fusion([[str(x) for x in r] for r in c["rankings"]], k=c["k"], weights=c["weights"])
        assert got_ids == [str(x) for x in c["ids"]] and got_scores == c["scores"]
    # a batch: many queries in one launch, with ties (equal weights, disjoint rankings)
    rng = np.random.default_rng(0)
    B, R, L = 64, 2, 40
    t = np.stack([np.stack([rng.permutation(200)[:L] for _ in range(R)]) for _ in range(B)]).astype(np.int64)
    t[:, 1, 30:] = -1
    ids, score, count = rl.rrf_fuse_device(torch.from_numpy(t).cuda(), [0.75, 0.25], num_results=25)
    for b in range(B):
        want_ids, want_scores = ofu.reciprocal_rank_fusion([t[b, 0].tolist(), t[b, 1, :30].tolist()], weights=[0.75, 0.25])
        assert ids[b].tolist() == want_ids[:25] and score[b].tolist() == want_scores[:25] and int(count[b]) == 25


@pytest.mark.gpu
def test_hybrid_search_and_device_span_collation():
    import torch
    from synth import make_corpus, make_queries

    import raglite_b200 as rl

    rng = np.random.default_rng(3)
    E, off = make_corpus(300, (1, 4), 32, seed=5, fp16_round=True)
    C = len(off) - 1
    docs = [f"doc-{c // 9:02d}" for c in range(C)]                      # 9 chunks per document, positions 0..8
    chunks = [rl.Chunk(id=f"c{c}", document_id=docs[c], index=c % 9, body=f"[{c}]") for c in range(C)]
    perm = rng.permutation(C)                                            # the table is not stored in document order
    inv = np.argsort(perm)
    rows = np.concatenate([np.arange(off[c], off[c + 1]) for c in perm])
    off_p = np.concatenate([[0], np.cumsum(np.diff(off)[perm])])
    idx = rl.CorpusIndex(E[rows], off_p, chunk_ids=[chunks[c].id for c in perm], chunks=[chunks[c] for c in perm])
    cfg = rl.RAGLiteConfig(db_url="mem://fusion", reranker=None)
    rl.register_index(cfg, idx)
    q = make_queries(E, 1, seed=6)[0]
    # hybrid_search: vector ranking from the device index, keyword ranking from a registered callable, RRF on the device
    kw = [f"c{c}" for c in rng.permutation(C)[:12]]
    rl.register_keyword_search(cfg, lambda query, *, num_results, metadata_filter=None, config=None: (kw[:num_results], [1.0] * num_results))
    import raglite_b200._search as S

    orig_vs = S.vector_search
    S.vector_search = lambda query, **k2: orig_vs(q, **k2)              # (no text embedder here: route the string to the vector)
    try:
        ids, scores = rl.hybrid_search("what?", num_results=5, config=cfg)
    finally:
        S.vector_search = orig_vs
    vs_ids, _ = rl.vector_search(q, num_results=10, config=cfg)
    want_ids, want_scores = ofu.reciprocal_rank_fusion([vs_ids, kw[:10]], weights=[0.75, 0.25])
    assert ids == want_ids[:5] and scores == want_scores[:5]
    # span collation on the device, through the drop-in and batched
    table = {(docs[c], c % 9) for c in range(C)}
    for trial in range(6):
        picked = [int(c) for c in rng.permutation(C)[: int(rng.integers(1, 14))]]
        nbrs = [(-1, 1), None, (-2, -1, 1), (1,)][trial % 4]
        spans = rl.retrieve_chunk_spans([f"c{c}" for c in picked], neighbors=nbrs, config=cfg)
        want = ofu.collate_chunk_spans([(docs[c], c % 9) for c in picked], table, neighbors=nbrs)
        assert [[(ch.document_id, ch.index) for ch in s.chunks] for s in spans] == [s for s, _ in want]
    ranked = torch.full((4, 10), -1, dtype=torch.int64)
    lists = [[int(inv[c]) for c in rng.permutation(C)[:n]] for n in (10, 3, 7, 1)]   # LOCAL indices of the permuted table
    for b, lst in enumerate(lists):
        ranked[b, : len(lst)] = torch.tensor(lst)
    out = rl.collate_spans_device(idx, ranked.cuda(), neighbors=(-1, 1))
    for b, lst in enumerate(lists):
        want = ofu.collate_chunk_spans([(docs[perm[i]], perm[i] % 9) for i in lst], table, neighbors=(-1, 1))
        ns = int(out["n_span"][b])
        assert ns == len(want)
        member = out["member"][b].tolist()
        for s, (span, score) in enumerate(want):
            st, ln = int(out["span_start"][b, s]), int(out["span_len"][b, s])
            got = [(docs[perm[member[st + j]]], int(perm[member[st + j]]) % 9) for j in range(ln)]
            assert got == span and float(out["span_score"][b, s]) == score
    # a deleted chunk is no neighbour
    idx.delete_chunks(["c4"])
    spans = rl.retrieve_chunk_spans(["c3"], neighbors=(-1, 1), config=cfg)
    assert [[ch.id for ch in s.chunks] for s in spans] == [["c2", "c3"]]


def _rrf_rankings(rng, B, R, L, b_mode):
    """``[B, R, L]`` int64 rankings, -1 padded at the tails.  Modes by query: 0 heavy overlap (R samples of one pool
    barely larger than L), 1 duplicates inside a ranking (drawn with replacement), 2 exact ties (disjoint rankings:
    ranking r holds r * L + i at position i, so with equal weights position i scores the same in every ranking),
    3 a mix of the three with ragged lengths."""
    t = np.full((B, R, L), -1, np.int64)
    for b in range(B):
        mode = b_mode(b)
        pool = rng.permutation(10 * R * L)[: L + L // 8 + 1]
        for r in range(R):
            m = mode if mode != 3 else int(rng.integers(0, 3))
            if m == 0:
                row = rng.permutation(pool)[:L]
            elif m == 1:
                row = rng.choice(pool[: max(1, L // 3)], size=L)
            else:
                row = r * L + np.arange(L)
            n = L if mode != 3 and rng.random() < 0.7 else int(rng.integers(0, L + 1))
            t[b, r, :n] = row[:n]
    return t


@pytest.mark.gpu
@pytest.mark.parametrize(("B", "R", "L", "weights", "k", "K"), [
    (3, 1, 4096, [1.0], 60, None),                              # R * L = 4096: one ranking
    (300, 4, 1024, [0.0, 0.75, -0.5, 0.25], 60, None),          # 4096, 300 queries, zero / unequal / negative weights
    (40, 3, 1365, [1.0, 1.0, 1.0], 1, 100),                     # 4095, equal weights (exact ties), k = 1
    (20, 4, 1024, [1.0, 1.0, 1.0, 1.0], 60, 1),                 # K = 1
    (20, 2, 2048, [0.5, 2.0], 1, 5000),                         # K larger than the number of unique ids
])
def test_rrf_kernel_at_its_size_limits(B, R, L, weights, k, K):
    """``rl_rrf_fuse`` at R * L = 4095 and 4096 (bitonic sorts over 4096 entries), bit for bit against the pinned
    oracle: ids, order (ties in first-appearance order) and float64 scores."""
    import torch

    import raglite_b200 as rl

    rng = np.random.default_rng(B * 7 + R)
    t = _rrf_rankings(rng, B, R, L, lambda b: b % 4)
    ids, score, count = rl.rrf_fuse_device(torch.from_numpy(t).cuda(), weights, k=k, num_results=K)
    ids, score, count = ids.cpu().numpy(), score.cpu().numpy(), count.cpu().numpy()
    K = R * L if K is None else K
    for b in range(B):
        want_ids, want_scores = ofu.reciprocal_rank_fusion([[int(x) for x in row if x >= 0] for row in t[b]], k=k,
                                                           weights=weights)
        n = min(len(want_ids), K)
        assert int(count[b]) == n, b
        assert ids[b, :n].tolist() == want_ids[:n], b
        assert score[b, :n].tolist() == want_scores[:n], b                 # same floats, bit for bit
        assert (ids[b, n:] == -1).all() and (score[b, n:] == 0.0).all(), b


@pytest.mark.gpu
def test_rrf_kernel_refuses_more_than_4096_entries():
    import torch

    import raglite_b200 as rl
    from raglite_b200._lib import RagliteB200Error

    t = torch.zeros((1, 1, 4097), dtype=torch.int64, device="cuda")
    with pytest.raises(RagliteB200Error, match=r"\(-4\).*4097"):
        rl.rrf_fuse_device(t, [1.0])
    t = torch.zeros((2, 17, 241), dtype=torch.int64, device="cuda")    # 4097 again, as R x L
    with pytest.raises(RagliteB200Error, match=r"\(-4\)"):
        rl.rrf_fuse_device(t, [1.0] * 17)


def _span_index(rng):
    """A registered index of ~7600 one-vector chunks in 28 documents of 1 to 600 chunks (stored in shuffled order,
    document ids not in creation order), with 3% of the chunks deleted."""
    import raglite_b200 as rl

    sizes = [1, 1, 2, 3, 600, 599, *rng.integers(1, 601, size=22).tolist()]
    names = [f"doc-{x:03d}" for x in rng.permutation(len(sizes))]
    keys = [(names[d], p) for d, n in enumerate(sizes) for p in range(n)]
    perm = rng.permutation(len(keys))
    keys = [keys[i] for i in perm]
    chunks = [rl.Chunk(id=f"c{i}", document_id=d, index=p, body="") for i, (d, p) in enumerate(keys)]
    E = rng.standard_normal((len(keys), 8)).astype(np.float32)
    idx = rl.CorpusIndex(E, vecs_per_chunk=1, chunk_ids=[c.id for c in chunks], chunks=chunks)
    dead = rng.choice(len(keys), size=len(keys) * 3 // 100, replace=False)
    idx.delete_chunks([chunks[i].id for i in dead])
    alive = np.setdiff1d(np.arange(len(keys)), dead)
    return idx, keys, alive, {keys[i] for i in alive}


def _check_collation(out, ranked, keys, table, neighbors):
    out = {name: v.cpu().numpy() for name, v in out.items()}
    for b in range(ranked.shape[0]):
        want = ofu.collate_chunk_spans([keys[int(c)] for c in ranked[b] if c >= 0], table, neighbors=neighbors)
        nm, ns = int(out["n_member"][b]), int(out["n_span"][b])
        member = out["member"][b]
        assert [keys[int(m)] for m in member[:nm]] == sorted({c for span, _ in want for c in span}), b   # document order
        assert (member[nm:] == -1).all(), b
        assert ns == len(want), b
        for s, (span, score) in enumerate(want):
            st, ln = int(out["span_start"][b, s]), int(out["span_len"][b, s])
            assert [keys[int(m)] for m in member[st:st + ln]] == span, (b, s)
            assert float(out["span_score"][b, s]) == score, (b, s)            # bit for bit


@pytest.mark.gpu
def test_span_collation_at_its_size_limits():
    """``rl_span_collate`` against the oracle at cap = M (1 + neighbours) of 1, 2, 4095 and 4096, on documents of 1
    to 600 chunks: offsets that step past both ends of a document, duplicate ids in one ranked list, deleted chunks
    as would-be neighbours, rows of different length padded with -1, and runs that would continue across a
    document boundary if the document were ignored."""
    import torch

    import raglite_b200 as rl

    rng = np.random.default_rng(11)
    idx, keys, alive, table = _span_index(rng)
    cfg = rl.RAGLiteConfig(db_url="mem://span-limits", reranker=None)
    rl.register_index(cfg, idx)

    def rows(M, lens, dup_row=None):
        r = np.full((len(lens), M), -1, np.int64)
        for b, n in enumerate(lens):
            r[b, :n] = rng.choice(alive, size=n, replace=b == dup_row)
        return r

    # cap = 1 (one chunk, no neighbours) and cap = 2, through the drop-in
    single = [i for i in alive if keys[i][0] in {d for d, p in keys if p == 0} - {d for d, p in keys if p == 1}]
    # (alive[-1]: a chunk index past the number of live chunks)
    for ids, nbrs in [([f"c{single[0]}"], None), ([f"c{alive[-1]}"], None), ([f"c{alive[7]}"], (1,)),
                      ([f"c{alive[8]}", f"c{alive[9]}"], None)]:
        spans = rl.retrieve_chunk_spans(ids, neighbors=nbrs, config=cfg)
        want = ofu.collate_chunk_spans([keys[int(c[1:])] for c in ids], table, neighbors=nbrs)
        assert [[(ch.document_id, ch.index) for ch in s.chunks] for s in spans] == [s for s, _ in want]
    # a few thousand members through the drop-in: cap = 800 x 5 = 4000
    picked = rng.choice(alive, size=800, replace=False)
    spans = rl.retrieve_chunk_spans([f"c{c}" for c in picked], neighbors=(-2, -1, 1, 2), config=cfg)
    want = ofu.collate_chunk_spans([keys[c] for c in picked], table, neighbors=(-2, -1, 1, 2))
    assert [[(ch.document_id, ch.index) for ch in s.chunks] for s in spans] == [s for s, _ in want]
    # runs that touch across a document boundary: (doc d, last position p) then (doc d + 1, position p + 1)
    by_doc = sorted({d for d, _ in keys})
    n_of = {d: sum(1 for k in keys if k[0] == d) for d in by_doc}
    pos_of = {k: i for i, k in enumerate(keys)}
    touch = []
    for a, b in zip(by_doc, by_doc[1:]):
        ka, kb = (a, n_of[a] - 1), (b, n_of[a])
        if ka in pos_of and kb in pos_of and ka in table and kb in table:
            touch += [pos_of[ka], pos_of[kb]]
    assert len(touch) >= 4
    batches = [
        (np.asarray(touch, np.int64)[None, :], None),
        (rows(1, [1, 1, 1, 1, 1]), None),                                # cap = 1
        (rows(2, [2, 1, 2]), None),                                      # cap = 2
        (rows(1, [1, 1, 1]), (1,)),                                      # cap = 2
        (rows(819, [819, 819, 500, 1], dup_row=1), (-2, -1, 1, 2)),      # cap = 4095
        (rows(4096, [4096, 4096, 1000], dup_row=1), None),               # cap = 4096
        (rows(1024, [1024, 1024, 300], dup_row=2), (-1, 1, 5)),          # cap = 4096
        (rows(2000, [2000, 1999], dup_row=0), (5,)),
    ]
    for ranked, nbrs in batches:
        out = rl.collate_spans_device(idx, torch.from_numpy(ranked).cuda(), neighbors=nbrs)
        _check_collation(out, ranked, keys, table, nbrs)
