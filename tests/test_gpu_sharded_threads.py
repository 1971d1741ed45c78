"""The sharded search with R > 1 shards on one GPU, checked against one ``CorpusIndex`` over the same rows and against
the float64 oracle.

* Kernel level: R real shard scans, their packed hit lists laid end to end and merged by ``rl_topk_merge_packed`` --
  against the single index's scan merged at R = 1.  Shard layouts include an empty shard, a one-chunk shard and a
  shard with fewer rows than num_hits; chunk bases are contiguous or spaced (``shard_bases``).
* Merge edges on synthetic packed buffers against a NumPy restatement of the merge, bit for bit.
* The whole host pipeline through R thread ranks (``thread_group``): ``ShardedIndex``, ``scan_gather_merge``,
  ``search_to_host``, ``run_until_no_overflow``, ``limit_hits_to_nearest`` and ``search_async``.
* The fused rank-then-filter bound of an empty shard (0, whatever its workspace holds).

The bar against the single index is bit-identity of ids, sims and counts.  The one exception is two entries whose
float32 sims are equal while their float64 values differ: the two configurations rescore different survivor sets and
may then order them differently.  ``_compare`` counts such cases; on these random corpora there are none.  Identical
rows planted in different shards have identical float64 values, so they must come out in global row order, as in the
single index."""

from __future__ import annotations

import threading

import numpy as np
import pytest
from parity import check_exact_maxsim, check_sql_semantics
from synth import make_corpus, make_queries
from thread_group import install, run_ranks

from raglite_b200._dist import ShardedIndex

from oracle import vector_search as ovs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rl():
    import torch

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import raglite_b200

    return raglite_b200


# ---- corpora and shards ------------------------------------------------------------------------------------------
def _edge_ranges(off, R, small_rows):
    """R contiguous chunk ranges: for R >= 3 a one-chunk shard, an empty shard and (R >= 4) a shard with fewer than
    ``small_rows`` rows, the rest of the corpus cut by ``shard_ranges``; for R = 2 ``shard_ranges`` alone."""
    from raglite_b200._dist import shard_ranges

    C = len(off) - 1
    if R == 2:
        return shard_ranges(off, 2)
    head = [(0, 1), (1, 1)]
    a = 1
    if R >= 4:
        b = a
        while b < C and off[b + 1] - off[a] < small_rows:
            b += 1
        head.append((a, b))
        a = b
    rest = shard_ranges(off[a:] - off[a], R - len(head))
    ranges = head + [(lo + a, hi + a) for lo, hi in rest]
    n_rows = [int(off[hi] - off[lo]) for lo, hi in ranges]
    assert len(ranges) == R and ranges[-1][1] == C and 0 in n_rows and (R < 4 or 0 < n_rows[2] < small_rows)
    return ranges


def _plant_duplicates(E, off, Q, num_hits, metric):
    """Copy the rows at ranks 3 and num_hits - 1 of query 0 (float64 order) over the first row of chunks spread across
    the corpus, so identical rows sit in different shards near the top and at / across the num_hits cut."""
    E = E.copy()
    order = np.argsort(ovs.vector_distances_f64(E, Q[0], metric), kind="stable")
    C = len(off) - 1
    targets = [int(off[int(C * f)]) for f in (0.31, 0.55, 0.77, 0.93)]
    for j, src in enumerate((order[3], order[num_hits - 1])):
        for t in targets[2 * j:2 * j + 2] + [targets[(2 * j + 3) % 4]]:
            E[t] = E[src]
    return E


def _shards(rl, E, off, ranges, bases, **kw):
    out = []
    for (lo, hi), base in zip(ranges, bases, strict=True):
        r0, r1 = int(off[lo]), int(off[hi])
        extra = {k: v[lo:hi] for k, v in kw.items() if isinstance(v, list)}
        fixed = {k: v for k, v in kw.items() if not isinstance(v, list)}
        out.append(rl.CorpusIndex(E[r0:r1], off[lo:hi + 1] - r0, chunk_base=base,
                                  chunk_ids=[f"c{g}" for g in range(lo, hi)], **extra, **fixed))
    return out


def _to_global(ids, ranges, bases):
    """Sharded chunk numbers -> the single index's: shard r's ``base_r + i`` is global chunk ``lo_r + i``."""
    out = ids.copy()
    for (lo, hi), base in zip(ranges, bases, strict=True):
        sel = (ids >= base) & (ids < base + (hi - lo))
        out[sel] = ids[sel] - base + lo
    return out


def _compare(got, want, E, off, Q, metric, ties):
    """Bit-identical (ids, sims, counts), except at a float32 tie of two different float64 values (counted in ``ties``)."""
    g_ids, g_sims, g_cnt = got
    w_ids, w_sims, w_cnt = want
    for b in range(len(Q)):
        same = (g_cnt[b] == w_cnt[b] and np.array_equal(g_ids[b], w_ids[b])
                and np.array_equal(g_sims[b].view(np.int32), w_sims[b].view(np.int32)))
        if same:
            continue
        n = min(g_cnt[b], w_cnt[b])
        diff = np.nonzero((g_ids[b, :n] != w_ids[b, :n]) | (g_sims[b, :n].view(np.int32) != w_sims[b, :n].view(np.int32)))[0]
        i = int(diff[0]) if len(diff) else n
        assert i < n and g_sims[b, i].view(np.int32) == w_sims[b, i].view(np.int32), (b, i, g_ids[b], w_ids[b], g_sims[b], w_sims[b])
        s64 = ovs.maxsim_scores(E, off, Q[b], metric, f64=True)
        assert s64[g_ids[b, i]] != s64[w_ids[b, i]], ("a tie of equal float64 values must follow global row order", b, i)
        ties.append((b, i))


def _host(t):
    return t.cpu().numpy()


def _scan_merge(rl, idx_list, Qd, R, *, k, num_hits, metric, algo):
    """Scan every shard (``scan_checked``), lay the packed lists end to end and merge them: what the all-gather and
    ``merge_packed`` of the sharded pipeline do."""
    import torch
    from raglite_b200._index import merge_packed

    res = [idx.scan_checked(Qd, k=k, num_hits=num_hits, metric=metric, algo=algo) for idx in idx_list]
    B, H = int(Qd.shape[0]), num_hits if num_hits > 0 else k
    sim, chunk, count = merge_packed(torch.cat([r.packed for r in res]), R, B, H, num_hits=num_hits, k=k)
    return _host(chunk), _host(sim), _host(count)


# ---- a. real scans, packed merge -----------------------------------------------------------------------------------
STORE = [("fp32", "auto"), ("fp32", "fp32"), ("fp16", "auto")]


@pytest.fixture(scope="module")
def corpus_a():
    E, off = make_corpus(2500, (1, 5), 64, seed=41, fp16_round=True)
    Q = make_queries(E, 8, seed=42)
    return E, off, Q


@pytest.mark.parametrize("mode", ["sql", "exact"])
@pytest.mark.parametrize("store", STORE, ids=lambda s: "-".join(s))
@pytest.mark.parametrize("metric", ["cosine", "dot", "l2"])
@pytest.mark.parametrize("layout", ["contiguous", "spaced+tombstones"])
@pytest.mark.parametrize("R", [2, 3, 8])
def test_shard_scans_merged_equal_the_single_index(rl, corpus_a, R, layout, metric, store, mode):
    import torch

    storage, algo = store
    k = 10
    num_hits = 40 if mode == "sql" else 0
    E0, off, Q = corpus_a
    E = _plant_duplicates(E0, off, Q, 40, metric)
    C = len(off) - 1
    ranges = _edge_ranges(off, R, small_rows=40)
    bases = ShardedIndex.shard_bases(R) if layout.startswith("spaced") else [lo for lo, _ in ranges]
    single = rl.CorpusIndex(E, off, chunk_ids=[f"c{g}" for g in range(C)], storage=storage)
    shards = _shards(rl, E, off, ranges, bases, storage=storage)
    alive = np.ones(C, dtype=bool)
    if "tombstones" in layout:   # every 7th chunk of the even-numbered shards
        for r, ((lo, hi), idx) in enumerate(zip(ranges, shards, strict=True)):
            dead = [g for g in range(lo, hi) if r % 2 == 0 and g % 7 == 3]
            if dead:
                assert idx.delete_chunks([f"c{g}" for g in dead]) == len(dead)
                single.delete_chunks([f"c{g}" for g in dead])
                alive[dead] = False
    Qd = torch.from_numpy(Q).cuda()
    want = _scan_merge(rl, [single], Qd, 1, k=k, num_hits=num_hits, metric=metric, algo=algo)
    ids, sims, cnt = _scan_merge(rl, shards, Qd, R, k=k, num_hits=num_hits, metric=metric, algo=algo)
    got = (_to_global(ids, ranges, bases), sims, cnt)
    ties = []
    _compare(got, want, E, off, Q, metric, ties)
    assert ties == []
    for b in range(len(Q)):
        n = int(cnt[b])
        if mode == "sql":
            check_sql_semantics(E, off, Q[b], got[0][b, :n], sims[b, :n], k=k, metric=metric,
                                allowed_chunks=None if alive.all() else alive)
        elif alive.all():
            check_exact_maxsim(E, off, Q[b], got[0][b, :n], sims[b, :n], k=k, metric=metric)


@pytest.mark.parametrize("num_hits", [1024, 1200])    # R * H = 8192 (shared-memory window) and 9600 (prefilter)
@pytest.mark.parametrize("spaced", [False, True])
def test_merge_window_edges_with_real_scans(rl, num_hits, spaced):
    import torch

    R, k = 8, 64
    E, off = make_corpus(9000, (1, 5), 64, seed=51, fp16_round=True)
    Q = make_queries(E, 6, seed=52)
    E = _plant_duplicates(E, off, Q, num_hits, "cosine")
    ranges = _edge_ranges(off, R, small_rows=num_hits)
    bases = ShardedIndex.shard_bases(R) if spaced else [lo for lo, _ in ranges]
    single = rl.CorpusIndex(E, off)
    shards = _shards(rl, E, off, ranges, bases)
    Qd = torch.from_numpy(Q).cuda()
    want = _scan_merge(rl, [single], Qd, 1, k=k, num_hits=num_hits, metric="cosine", algo="auto")
    ids, sims, cnt = _scan_merge(rl, shards, Qd, R, k=k, num_hits=num_hits, metric="cosine", algo="auto")
    ties = []
    _compare((_to_global(ids, ranges, bases), sims, cnt), want, E, off, Q, "cosine", ties)
    assert ties == []


@pytest.mark.parametrize("storage", ["fp32", "fp16"])
def test_wide_rows_and_256_query_groups(rl, storage):
    """d = 1024 and 256 queries (the wgmma scan's query groups) over 3 shards, one of them empty."""
    import torch

    R, k, num_hits = 3, 10, 40
    E, off = make_corpus(3000, (1, 3), 1024, seed=81, fp16_round=True)
    Q = make_queries(E, 256, seed=82)
    E = _plant_duplicates(E, off, Q, num_hits, "cosine")
    ranges = _edge_ranges(off, R, small_rows=num_hits)
    bases = ShardedIndex.shard_bases(R)
    single = rl.CorpusIndex(E, off, storage=storage)
    shards = _shards(rl, E, off, ranges, bases, storage=storage)
    Qd = torch.from_numpy(Q).cuda()
    for nh in (num_hits, 0):
        want = _scan_merge(rl, [single], Qd, 1, k=k, num_hits=nh, metric="cosine", algo="auto")
        ids, sims, cnt = _scan_merge(rl, shards, Qd, R, k=k, num_hits=nh, metric="cosine", algo="auto")
        ties = []
        _compare((_to_global(ids, ranges, bases), sims, cnt), want, E, off, Q, "cosine", ties)
        assert ties == []


# ---- b. merge edges on synthetic packed buffers ------------------------------------------------------------------
def _f2ord(s):
    u = np.asarray(s, np.float32).view(np.uint32)
    return np.where(u & 0x80000000, ~u, u | 0x80000000).astype(np.uint32)


def merge_reference(chunk, sim, count, num_hits, k):
    """``rl_topk_merge`` restated: the first min(count, H) entries of every list, ordered by sim descending (the
    order of the float's bits, so +0 > -0) and then by position ``r * H + i``; the best ``num_hits`` of them (all
    when num_hits = 0: exact MaxSim); GROUP BY chunk, the first occurrence carries the max; the first k chunks."""
    R, B, H = sim.shape
    ids = np.full((B, k), -1, np.int64)
    sims = np.full((B, k), -np.inf, np.float32)
    cnt = np.zeros(B, np.int32)
    for b in range(B):
        pos = np.concatenate([r * H + np.arange(min(int(count[r, b]), H)) for r in range(R)]).astype(np.int64)
        s = sim.transpose(1, 0, 2).reshape(B, R * H)[b, pos]
        c = chunk.transpose(1, 0, 2).reshape(B, R * H)[b, pos]
        o = np.lexsort((pos, -_f2ord(s).astype(np.int64)))
        if num_hits > 0:
            o = o[:num_hits]
        s, c = s[o], c[o]
        _, first = np.unique(c, return_index=True)
        keep = np.sort(first)[:k]
        n = len(keep)
        ids[b, :n], sims[b, :n], cnt[b] = c[keep], s[keep], n
    return ids, sims, cnt


def _synthetic(R, B, H, seed, *, counts="mixed", ties=False, big_ids=False, n_chunks=None):
    rng = np.random.default_rng(seed)
    if ties:
        sim = rng.choice(np.array([0.5, 0.25, -0.0, 0.0], np.float32), size=(R, B, H))
    else:
        sim = -np.sort(-rng.standard_normal((R, B, H)).astype(np.float32), axis=2)
    n_chunks = n_chunks or max(4, R * H // 3)
    chunk = rng.integers(0, n_chunks, size=(R, B, H)).astype(np.int64) + ((1 << 40) + 12345 if big_ids else 0)
    if counts == "full":
        count = np.full((R, B), H, np.int32)
    elif counts == "zero":
        count = np.zeros((R, B), np.int32)
    else:   # a mix: zero on some ranks, more than H (clamped) on others, anything in between
        count = rng.integers(0, H + 1, size=(R, B)).astype(np.int32)
        count[rng.random((R, B)) < 0.2] = 0
        count[rng.random((R, B)) < 0.2] = H + 1 + rng.integers(0, 1000)
        count[:, 0] = H + 7          # query 0: every list over-full
        count[:, 1] = 0              # query 1: every list empty
    for r in range(R):               # -inf padding behind each list's count, as the scan writes it
        for b in range(B):
            n = min(int(count[r, b]), H)
            sim[r, b, n:] = -np.inf
            chunk[r, b, n:] = -1
    if counts == "mixed" and H > 2:  # -inf hits inside a count: still hits, grouped under their chunk
        sim[0, 2, H - 1] = -np.inf
    return chunk, sim.astype(np.float32), count


def _pack(chunk, sim, count):
    import torch
    from raglite_b200._index import hits_views, new_scan_result

    R, B, H = sim.shape
    bufs = []
    for r in range(R):
        res = new_scan_result(B, H, H, 1, "cuda")
        res.hit_chunk.copy_(torch.from_numpy(chunk[r]))
        res.hit_sim.copy_(torch.from_numpy(sim[r]))
        res.hit_count.copy_(torch.from_numpy(count[r]))
        res.status.zero_()
        bufs.append(res.packed)
    allb = torch.cat(bufs)
    c, s, n, _ = hits_views(allb, R, B, H)
    assert np.array_equal(_host(c), chunk) and np.array_equal(_host(n), count)
    return allb


MERGE_CASES = [
    # (R, H, num_hits, k, counts, ties, big_ids)
    (1, 8191, 0, 64, "mixed", False, False),       # R*H = 8191: window, exact mode
    (1, 8191, 3000, 100, "mixed", True, True),
    (64, 128, 0, 300, "mixed", False, True),       # R*H = 8192: the largest window
    (64, 128, 4000, 64, "mixed", True, False),
    (3, 2731, 2000, 64, "mixed", False, True),     # R*H = 8193: prefilter
    (3, 2731, 8192, 4096, "mixed", True, False),
    (64, 200, 1500, 100, "mixed", True, True),     # prefilter, 64 ranks, ties across ranks
    (2, 7, 0, 50, "mixed", False, False),          # k > distinct chunks
    (5, 16, 30, 200, "full", True, True),
    (17, 40, 500, 10, "mixed", False, False),
    (9, 1000, 4096, 64, "mixed", False, True),     # prefilter with num_hits < R*H
    (4, 50, 80, 16, "zero", False, False),         # count 0 on every rank
    (64, 1, 0, 8, "mixed", True, False),
]


@pytest.mark.parametrize("case", MERGE_CASES, ids=lambda c: "R{}-H{}-nh{}-k{}-{}{}{}".format(
    *c[:5], "-ties" if c[5] else "", "-bigids" if c[6] else ""))
def test_packed_merge_matches_the_numpy_restatement(rl, case):
    from raglite_b200._index import merge_packed

    R, H, num_hits, k, counts, ties, big_ids = case
    B = 5
    chunk, sim, count = _synthetic(R, B, H, seed=R * 1000 + H, counts=counts, ties=ties, big_ids=big_ids,
                                   n_chunks=6 if k > 20 and R * H < 100 else None)
    out_sim, out_chunk, out_count = merge_packed(_pack(chunk, sim, count), R, B, H, num_hits=num_hits, k=k)
    w_ids, w_sims, w_cnt = merge_reference(chunk, sim, count, num_hits, k)
    assert np.array_equal(_host(out_count), w_cnt)
    assert np.array_equal(_host(out_chunk), w_ids)
    assert np.array_equal(_host(out_sim).view(np.int32), w_sims.view(np.int32))
    if counts != "zero":
        assert w_cnt.max() > 0
    if counts == "mixed":
        assert w_cnt[1] == 0


# ---- c. the whole pipeline through thread ranks ---------------------------------------------------------------------
def _unequal_ranges(C, R):
    cuts = np.round(np.cumsum([0] + [1 + r for r in range(R)]) / sum(1 + r for r in range(R)) * C).astype(int)
    return [(int(cuts[r]), int(cuts[r + 1])) for r in range(R)]


@pytest.fixture(scope="module")
def corpus_c():
    E, off = make_corpus(4000, (1, 5), 64, seed=61, fp16_round=True)
    Q = make_queries(E, 16, seed=62)
    return E, off, Q


@pytest.mark.parametrize("R", [2, 3, 4])
def test_thread_ranks_search_equals_the_single_index(rl, corpus_c, monkeypatch, R):
    install(monkeypatch)
    E, off, Q = corpus_c
    C = len(off) - 1
    ranges = _unequal_ranges(C, R)
    shards = _shards(rl, E, off, ranges, [lo for lo, _ in ranges])
    single = rl.CorpusIndex(E, off)
    cfg = rl.RAGLiteConfig(reranker=None)

    def rank_fn(r, g):
        sh = ShardedIndex(shards[r], g)
        return [rl.vector_search_batch(Q, num_results=10, index=sh, config=cfg, exact_maxsim=ex) for ex in (False, True)]

    results = run_ranks(R, rank_fn)
    for ex, mode in enumerate(("sql", "exact")):
        want = rl.vector_search_batch(Q, num_results=10, index=single, config=cfg, exact_maxsim=bool(ex))
        for r in range(R):
            for a, b in zip(results[r][ex], results[0][ex], strict=True):
                assert np.array_equal(a, b), f"rank {r} differs from rank 0 ({mode})"
        ties = []
        _compare(results[0][ex], want, E, off, Q, "cosine", ties)
        assert ties == [], mode


@pytest.mark.parametrize("R", [2, 3])
def test_thread_ranks_vector_search_returns_every_shards_ids(rl, corpus_c, monkeypatch, R):
    """``vector_search`` on a freshly built sharded index (spaced bases) returns the chunk ids of hits owned by other
    ranks, as the single index does."""
    install(monkeypatch)
    E, off, Q = corpus_c
    C = len(off) - 1
    ranges = _unequal_ranges(C, R)
    shards = _shards(rl, E, off, ranges, ShardedIndex.shard_bases(R))
    cfg1 = rl.RAGLiteConfig(db_url="threads://single", reranker=None)
    rl.register_index(cfg1, rl.CorpusIndex(E, off, chunk_ids=[f"c{g}" for g in range(C)]))
    try:
        want = [rl.vector_search(Q[b], num_results=10, config=cfg1) for b in range(len(Q))]
    finally:
        rl.unregister_index(cfg1)

    def rank_fn(r, g):
        cfg = rl.RAGLiteConfig(db_url=f"threads://rank{r}", reranker=None)
        rl.register_index(cfg, ShardedIndex(shards[r], g))
        try:
            return [rl.vector_search(Q[b], num_results=10, config=cfg) for b in range(len(Q))]
        finally:
            rl.unregister_index(cfg)

    for got in run_ranks(R, rank_fn):
        assert got == want
    owners = {int(i[1:]) for ids, _ in want for i in ids}
    assert any(lo <= g < hi for g in owners for lo, hi in ranges[1:]), "some hits must be owned by ranks > 0"


def test_thread_ranks_overflow_on_one_rank_retries_together(rl, monkeypatch):
    """Rank 1's shard is sorted by ascending similarity to the queries and scanned with a tiny candidate list: it
    overflows, the others do not.  Every rank must run the pipeline the same number of times, and the answer must be
    the single index's."""
    import torch
    from raglite_b200._index import run_until_no_overflow

    install(monkeypatch)
    R = 3
    E, off = make_corpus(12000, 1, 64, seed=71, fp16_round=True)
    Q = make_queries(E, 8, seed=72)
    ranges = [(0, 2000), (2000, 10000), (10000, 12000)]
    lo, hi = ranges[1]
    E = E.copy()
    E[lo:hi] = E[lo:hi][np.argsort((E[lo:hi] @ Q.T).max(1), kind="stable")]
    shards = _shards(rl, E, off, ranges, [lo for lo, _ in ranges])
    runs: dict[int, list[int]] = {}
    orig = ShardedIndex.search_pipeline

    def counting(self, *a, **kw):
        runs.setdefault(self.rank, []).append(int(kw.get("cand_cap", 0)))
        return orig(self, *a, **kw)

    monkeypatch.setattr(ShardedIndex, "search_pipeline", counting)
    kw = dict(k=10, num_hits=40, metric="cosine", algo="fp32", sample_stride=16)

    def rank_fn(r, g):
        sh = ShardedIndex(shards[r], g)
        Qd = torch.from_numpy(Q).cuda()
        out = None

        def run(flags, cand_cap):
            nonlocal out
            out = sh.search_pipeline(Qd, flags=flags, cand_cap=cand_cap, **kw)
            return out[3]

        with sh.local._lock:
            first = sh.local.scan(Qd, cand_cap=256 if r == 1 else 0, **kw)
            overflowed = bool((first.status & 1).any())
            run_until_no_overflow(sh.local, run, cand_cap=256 if r == 1 else 0)
        return overflowed, [_host(t) for t in (out[1], out[0], out[2])]

    results = run_ranks(R, rank_fn)
    assert [ov for ov, _ in results] == [False, True, False], "only rank 1's tiny list may overflow"
    assert len(runs[0]) == len(runs[1]) == len(runs[2]) >= 2, runs
    single = rl.CorpusIndex(E, off)
    want = _scan_merge(rl, [single], torch.from_numpy(Q).cuda(), 1, k=10, num_hits=40, metric="cosine", algo="fp32")
    for _, got in results:
        ties = []
        _compare(tuple(got), want, E, off, Q, "cosine", ties)
        assert ties == []


def _count_probes(rl, monkeypatch):
    calls = []
    lock = threading.Lock()
    orig = rl.CorpusIndex.count_at_least

    def counting(self, *a, **k):
        with lock:
            calls.append(self.chunk_base)
        return orig(self, *a, **k)

    monkeypatch.setattr(rl.CorpusIndex, "count_at_least", counting)
    return calls


def test_thread_ranks_rank_then_filter_fused_proof(rl, monkeypatch):
    """Many rows match and the filtered hits are nowhere near the 20_000-th nearest row: the bounds the filtered scans
    keep, summed over the shards, prove the filter-first answer; no counting pass runs (constants scaled: 100_000 ->
    1_000 matching rows, 1_000_000 -> 20_000 nearest vectors)."""
    import raglite_b200._search as S

    install(monkeypatch)
    monkeypatch.setattr(S, "FILTER_FIRST_MAX_ROWS", 1_000)
    monkeypatch.setattr(S, "RANK_FIRST_LIMIT", 20_000)
    R = 3
    E, off = make_corpus(20_000, 3, 64, seed=330, fp16_round=True)
    C = len(off) - 1
    tagged = np.arange(C) % 2 == 0
    meta = [{"half": int(t)} for t in tagged]
    ranges = _unequal_ranges(C, R)
    shards = _shards(rl, E, off, ranges, [lo for lo, _ in ranges], chunk_metadata=meta)
    Q = make_queries(E, 12, seed=331)
    cfg = rl.RAGLiteConfig(reranker=None)
    want = rl.vector_search_batch(Q, num_results=10, metadata_filter={"half": 1}, index=rl.CorpusIndex(E, off, chunk_metadata=meta),
                                  config=cfg)
    calls = _count_probes(rl, monkeypatch)

    def rank_fn(r, g):
        sh = ShardedIndex(shards[r], g)
        return rl.vector_search_batch(Q, num_results=10, metadata_filter={"half": 1}, index=sh, config=cfg)

    results = run_ranks(R, rank_fn)
    assert calls == [], "the summed fused bound must prove the filter-first answer"
    for got in results:
        ties = []
        _compare(got, want, E, off, Q, "cosine", ties)
        assert ties == []
    for b in range(len(Q)):
        check_sql_semantics(E, off, Q[b], want[0][b, :want[2][b]], want[1][b, :want[2][b]], k=10, allowed_chunks=tagged)


@pytest.mark.parametrize("R", [2, 3])
def test_thread_ranks_rank_then_filter_probe_cuts(rl, monkeypatch, R):
    """Query 0's filter keeps the far half of the corpus plus four chunks near it: the explicit probe, with its
    counts summed over the shards, cuts at the 400 nearest rows of the whole corpus and leaves only the near ones
    (constants scaled: 100_000 -> 60 matching rows, 1_000_000 -> 400 nearest vectors)."""
    import raglite_b200._search as S

    install(monkeypatch)
    monkeypatch.setattr(S, "FILTER_FIRST_MAX_ROWS", 60)
    monkeypatch.setattr(S, "RANK_FIRST_LIMIT", 400)
    k = 10
    E, off = make_corpus(600, (1, 5), 64, seed=320, fp16_round=True)
    C = len(off) - 1
    Q = make_queries(E, 3, seed=321, frac_random=0.0)
    order = np.argsort(-ovs.maxsim_scores(E, off, Q[0], "cosine", f64=True))
    tagged = np.zeros(C, dtype=bool)
    tagged[order[C // 2:]] = True
    tagged[order[[0, 2, 5, 30]]] = True
    meta = [{"topic": ["keep"] if t else ["drop"]} for t in tagged]
    ranges = _unequal_ranges(C, R)
    shards = _shards(rl, E, off, ranges, [lo for lo, _ in ranges], chunk_metadata=meta)
    cfg = rl.RAGLiteConfig(reranker=None)
    single = rl.vector_search_batch(Q, num_results=k, metadata_filter={"topic": "keep"},
                                    index=rl.CorpusIndex(E, off, chunk_metadata=meta), config=cfg)
    calls = _count_probes(rl, monkeypatch)

    def rank_fn(r, g):
        sh = ShardedIndex(shards[r], g)
        return rl.vector_search_batch(Q, num_results=k, metadata_filter={"topic": "keep"}, index=sh, config=cfg)

    results = run_ranks(R, rank_fn)
    assert len(calls) >= R, "the explicit rank probe must run on every rank"
    chunk, sim, count = results[0]
    for got in results[1:]:
        assert all(np.array_equal(a, b) for a, b in zip(got, results[0], strict=True)), "every rank must keep the same hits"
    took_rank_first = False
    for b in range(len(Q)):
        got = chunk[b, :count[b]].tolist()
        options = [ovs.vector_search_sql(E, off, Q[b], num_results=k, allowed_chunks=tagged, f64=True, filter_first_max=60,
                                         rank_first_limit=lim)[:2] for lim in (400, 399, 401)]   # the row at the cut may fall either way
        opt_ids = [o[0].tolist() for o in options]
        assert got in opt_ids, (b, got, opt_ids[0])
        assert np.allclose(sim[b, :count[b]], options[opt_ids.index(got)][1], atol=1e-4)
        if opt_ids[1] == opt_ids[0] == opt_ids[2]:    # no row at the cut: the single index must agree exactly
            assert got == single[0][b, :single[2][b]].tolist()
        first_ids, _, _ = ovs.vector_search_sql(E, off, Q[b], num_results=k, allowed_chunks=tagged, f64=True)
        took_rank_first |= got != first_ids.tolist()
    assert took_rank_first, "query 0 must differ from the filter-first answer"


def test_thread_ranks_async_searches_in_flight(rl, corpus_c, monkeypatch):
    install(monkeypatch)
    R = 3
    E, off, Q = corpus_c
    C = len(off) - 1
    ranges = _unequal_ranges(C, R)
    shards = _shards(rl, E, off, ranges, [lo for lo, _ in ranges])
    cfg = rl.RAGLiteConfig(reranker=None)
    batches = [Q[:5], Q[5:16], Q[2:9]]

    def rank_fn(r, g):
        sh = ShardedIndex(shards[r], g)
        pend = [rl.vector_search_batch_async(q, num_results=10, index=sh, config=cfg, exact_maxsim=(i == 1))
                for i, q in enumerate(batches)]
        got = [p.result() for p in pend]
        serial = [rl.vector_search_batch(q, num_results=10, index=sh, config=cfg, exact_maxsim=(i == 1))
                  for i, q in enumerate(batches)]
        return got, serial

    for got, serial in run_ranks(R, rank_fn):
        for a, b in zip(got, serial, strict=True):
            assert all(np.array_equal(x, y) for x, y in zip(a, b, strict=True))


def test_thread_ranks_delete_and_compact_on_one_rank(rl, corpus_c, monkeypatch):
    """Rank 1 deletes a third of its chunks and compacts; after ``refresh(chunk_ids=True)`` on every rank the sharded
    answer, in chunk ids, is that of a single index built fresh from the surviving rows."""
    install(monkeypatch)
    R = 3
    E, off, Q = corpus_c
    C = len(off) - 1
    ranges = _unequal_ranges(C, R)
    shards = _shards(rl, E, off, ranges, ShardedIndex.shard_bases(R))
    lo, hi = ranges[1]
    dead = {g for g in range(lo, hi) if g % 3 == 1}
    cfg = rl.RAGLiteConfig(reranker=None)

    def rank_fn(r, g):
        sh = ShardedIndex(shards[r], g)
        if r == 1:
            assert sh.local.delete_chunks([f"c{x}" for x in sorted(dead)]) == len(dead)
            sh.local.compact()
        sh.refresh(chunk_ids=True)
        ids, sims, cnt = rl.vector_search_batch(Q, num_results=10, index=sh, config=cfg)
        return [[sh.chunk_id_of(int(c)) for c in ids[b, :cnt[b]]] for b in range(len(Q))], sims, cnt

    keep = np.array([g not in dead for g in range(C)])
    rows = np.repeat(keep, np.diff(off))
    fresh = rl.CorpusIndex(E[rows], np.concatenate([[0], np.cumsum(np.diff(off)[keep])]),
                           chunk_ids=[f"c{g}" for g in range(C) if keep[g]])
    w_ids, w_sims, w_cnt = rl.vector_search_batch(Q, num_results=10, index=fresh, config=cfg)
    want = [[fresh.chunk_id_of(int(c)) for c in w_ids[b, :w_cnt[b]]] for b in range(len(Q))]
    for ids, sims, cnt in run_ranks(R, rank_fn):
        assert ids == want
        assert np.array_equal(cnt, w_cnt) and np.array_equal(sims.view(np.int32), w_sims.view(np.int32))


# ---- d. the fused bound of an empty shard ------------------------------------------------------------------------------
@pytest.mark.parametrize("storage", ["fp32", "fp16"])
def test_empty_shard_unfiltered_bound_is_zero(rl, storage):
    import torch
    from raglite_b200._lib import RL_FLAG_COUNT_UNFILTERED

    empty = rl.CorpusIndex(np.zeros((0, 64), np.float32), [0], storage=storage)
    Qd = torch.from_numpy(make_queries(np.eye(64, dtype=np.float32), 9, seed=3)).cuda()
    allowed = torch.ones(16, dtype=torch.uint8, device="cuda")[:0]
    res = empty.scan(Qd, k=10, num_hits=40, row_allowed=allowed, flags=RL_FLAG_COUNT_UNFILTERED)
    assert empty._ws, "the scan must have allocated this stream's workspace"
    for pattern in (0x7F, 0x00, 0xFF):
        for ws in empty._ws.values():
            ws.fill_(pattern)
        res = empty.scan(Qd, k=10, num_hits=40, row_allowed=allowed, flags=RL_FLAG_COUNT_UNFILTERED, out=res)
        assert _host(empty.unfiltered_bound()).tolist() == [0] * 9, hex(pattern)
        assert _host(res.hit_count).tolist() == [0] * 9 and _host(res.status).tolist() == [0] * 9


def test_empty_shard_takes_the_fused_branch_whatever_its_workspace_holds(rl, monkeypatch):
    """A sharded index with an empty shard: the rank-then-filter search must prove the filter-first answer from the
    fused bound (no counting pass) for any stale bytes in the empty shard's workspace, and give the single index's
    answer."""
    import raglite_b200._search as S

    install(monkeypatch)
    monkeypatch.setattr(S, "FILTER_FIRST_MAX_ROWS", 1_000)
    monkeypatch.setattr(S, "RANK_FIRST_LIMIT", 20_000)
    R = 3
    E, off = make_corpus(20_000, 3, 64, seed=330, fp16_round=True)
    C = len(off) - 1
    tagged = np.arange(C) % 2 == 0
    meta = [{"half": int(t)} for t in tagged]
    ranges = [(0, 9000), (9000, 9000), (9000, C)]
    shards = _shards(rl, E, off, ranges, [lo for lo, _ in ranges], chunk_metadata=meta)
    Q = make_queries(E, 12, seed=331)
    cfg = rl.RAGLiteConfig(reranker=None)
    want = rl.vector_search_batch(Q, num_results=10, metadata_filter={"half": 1}, index=rl.CorpusIndex(E, off, chunk_metadata=meta),
                                  config=cfg)
    calls = _count_probes(rl, monkeypatch)

    from raglite_b200 import _dist

    def rank_fn(r, g):
        sh = ShardedIndex(shards[r], g)
        out = []
        for pattern in (0x7F, 0x00):
            rl.vector_search_batch(Q, num_results=10, metadata_filter={"half": 1}, index=sh, config=cfg)   # workspaces exist
            for ws in sh.local._ws.values():
                ws.fill_(pattern)
            _dist.dist.barrier(group=g)
            out.append(rl.vector_search_batch(Q, num_results=10, metadata_filter={"half": 1}, index=sh, config=cfg))
        return out

    results = run_ranks(R, rank_fn)
    assert calls == [], f"the fused bound must prove the answer with an empty shard ({len(calls)} counting passes ran)"
    for per_pattern in results:
        for got in per_pattern:
            ties = []
            _compare(got, want, E, off, Q, "cosine", ties)
            assert ties == []
