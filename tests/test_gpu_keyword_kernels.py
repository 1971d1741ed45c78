"""The BM25 kernels at the C-ABI (``rl_bm25_topk_global``: score + select; ``rl_bm25_stats``: corpus + df) against the
NumPy restatement of ``keyword_oracle`` (``bm25_csr_scores`` / ``bm25_topk``), bit for bit, on postings built directly
(no text analysis, so any tf, doc_len, statistics and corpus size can be reached in seconds).

* Scores.  The kernels round every double as written, so a score differs from the restatement only through ``log10`` in
  the idf.  The device's own idf values are taken from a probe call at k1 = 0 (each posting then adds idf * (f * 1) /
  (f + 0 * norm) = idf exactly) and fed to the restatement: every score must then match to the last bit, every id list
  exactly -- ties, cut and order by (score desc, chunk asc) -- with exact counts, -1 / -inf padding and zeroed pad bytes.
* Cuts.  The select kernel is a radix select over the 96-bit composite (key, ~chunk) in nine digits, most significant
  first; the digit that decides a cut is the first one in which the k-th and (k+1)-th composites differ.  The cases
  below are built so that each of the nine digits decides at least one cut, and they say which digits they reach.
* Launch edges: score tiles of 4096 chunks, B > 65 535 queries (two launches), workspaces of 1, 7 and all queries,
  n_chunks = 0, 3.1 M chunks (the ~chunk digit at bits 21..31), chunk_base >= 2^40, shard statistics unrelated to the
  local postings, k1 / b other than 1.2 / 0.75, tf up to 10^6 and doc_len up to 2^30.
* ``rl_bm25_stats`` at 200 000 terms (the df kernel's grid-stride loop), against NumPy exactly."""

from __future__ import annotations

import collections

import numpy as np
import pytest

import keyword_oracle as ko

pytestmark = pytest.mark.gpu

KTILE = 4096                                     # chunks per score CTA
MAX_K = 4096
KEY_SHIFTS, CHUNK_SHIFTS = [53, 42, 31, 20, 9, 0], [21, 10, 0]   # the select's digits: key bits, then ~chunk bits
CUTS: collections.Counter = collections.Counter()   # cuts by the digit that decided them ("none": no cut needed)
IDF = {"values": 0, "differ": 0}                    # device idf against NumPy's log10


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print(f"\ncuts by deciding digit: {dict(sorted(CUTS.items(), key=str))}; device idf values differing from "
          f"NumPy's log10: {IDF['differ']} of {IDF['values']} (all within 1 ulp)")


def _lib():
    import torch

    from raglite_b200 import _lib as L

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return L


def _up(a, dtype):
    """A device copy of ``a``, one element longer (so that an empty array still has an address)."""
    import torch

    a = np.concatenate([np.asarray(a, dtype).ravel(), np.zeros(1, dtype)])
    return torch.from_numpy(a).cuda()


def _device_topk(csr, stats, q_off, q_terms, k, *, k1=1.2, b=0.75, mask=None, chunk_base=0, group=None):
    """``rl_bm25_topk_global`` on host arrays; ``group`` sizes the workspace (default: the whole batch).  The packed
    buffer starts filled with 0xA5, so its pad bytes are checked to be zeroed.  Returns (chunk, score, count)."""
    import torch

    L = _lib()
    lib = L.load()
    term_off, doc, tf, doc_len = csr
    B, C, V = len(q_off) - 1, len(doc_len), len(term_off) - 1
    keep = [_up(term_off, np.int64), _up(doc, np.int32), _up(tf, np.int32), _up(doc_len, np.int32) if C else None,
            _up(stats, np.int64), None if mask is None else _up(mask, np.uint8), _up(q_off, np.int32),
            _up(q_terms, np.int32)]
    ptr = [None if t is None else t.data_ptr() for t in keep]
    need = int(lib.rl_bm25_workspace_bytes(C, B if group is None else group))
    ws = torch.empty(need, dtype=torch.uint8, device="cuda") if need else None
    nbytes = int(lib.rl_bm25_packed_bytes(B, k))
    packed = torch.full((nbytes,), 0xA5, dtype=torch.uint8, device="cuda")
    L.check(lib.rl_bm25_topk_global(ptr[0], ptr[1], ptr[2], ptr[3], ptr[4], V, C, ptr[5], ptr[6], ptr[7], B, k, k1, b,
                                    chunk_base, packed.data_ptr(), None if ws is None else ws.data_ptr(), need,
                                    torch.cuda.current_stream().cuda_stream), "rl_bm25_topk_global")
    raw = packed.cpu().numpy()
    used = B * k * 16 + B * 4
    assert nbytes % 16 == 0 and (raw[used:] == 0).all(), "the packed buffer's pad bytes must be zeroed"
    return (raw[: B * k * 8].view(np.int64).reshape(B, k), raw[B * k * 8: B * k * 16].view(np.float64).reshape(B, k),
            raw[B * k * 16: used].view(np.int32))


def _numpy_idf(N, df):
    df = np.asarray(df, np.float64)
    return np.log10(((np.float64(N) - df) + 0.5) / (df + 0.5) + 1.0)


def _device_idf(N, dfs):
    """The device's idf of each df at N chunks: a one-chunk index with one term, one query per distinct df holding only
    that term, k1 = 0 -- every score is then idf * (1 * 1) / (1 + 0 * norm) = idf exactly."""
    dfs = np.asarray(dfs, np.int64)
    uniq = np.unique(dfs)
    csr = ko.csr_from_postings([([0], 1)], [1])
    stats = np.concatenate([[N, 1], uniq])
    _, score, count = _device_topk(csr, stats, np.arange(len(uniq) + 1), np.zeros(len(uniq)), 1, k1=0.0)
    assert (count == 1).all(), "every probe idf must be positive"
    idf = score[:, 0].copy()
    ulps = np.abs(idf.view(np.int64) - _numpy_idf(N, uniq).view(np.int64))
    assert ulps.max() <= 1, (N, uniq[ulps > 1])
    IDF["values"] += len(uniq)
    IDF["differ"] += int((ulps != 0).sum())
    return idf[np.searchsorted(uniq, dfs)]


def _ranked(scores_q, keep_q):
    """Every kept chunk by (score desc, chunk asc), with its composite key and ~chunk."""
    cand = np.flatnonzero(keep_q)
    c = cand[np.lexsort((cand, -scores_q[cand]))]
    return c, scores_q[c].view(np.uint64) | np.uint64(1 << 63), (~c.astype(np.uint32)).astype(np.uint64)


def _digit(key_a, lo_a, key_b, lo_b):
    """The select digit (0..8) that separates two composites: the first one, most significant first, where they differ."""
    x = int(key_a) ^ int(key_b)
    if x:
        return next(i for i, s in enumerate(KEY_SHIFTS) if x.bit_length() - 1 >= s)
    x = int(lo_a) ^ int(lo_b)
    assert x, "composites are unique"
    return 6 + next(i for i, s in enumerate(CHUNK_SHIFTS) if x.bit_length() - 1 >= s)


def _cut_digit(scores_q, keep_q, k):
    """The digit that decides the cut of the top k, or None when every kept chunk is taken (no cut)."""
    c, key, lo = _ranked(scores_q, keep_q)
    return None if len(c) <= k else _digit(key[k - 1], lo[k - 1], key[k], lo[k])


def _ks_by_digit(scores_q, keep_q):
    """For each digit, the values of k <= 4096 whose cut it decides."""
    c, key, lo = _ranked(scores_q, keep_q)
    out: dict[int, list[int]] = collections.defaultdict(list)
    for k in range(1, min(len(c) - 1, MAX_K) + 1):
        out[_digit(key[k - 1], lo[k - 1], key[k], lo[k])].append(k)
    return out


def _restate(csr, stats, q_off, q_terms, k1, b):
    """The restatement's dense scores and matched masks, with the device's idf of each entry."""
    idf = _device_idf(stats[0], stats[2:]) if len(q_terms) and stats[0] > 0 else None
    scores, matched = ko.bm25_csr_scores(*csr, stats, q_off, q_terms, k1, b, idf=idf)
    assert (scores[matched] > 0).all(), "a matched chunk must score above zero (the kernel's test for a result)"
    return scores, matched


def _compare(csr, stats, q_off, q_terms, ks, *, k1=1.2, b=0.75, mask=None, chunk_base=0, restated=None):
    """Device against restatement for every k: ids, score bits and counts exactly.  Returns {k: [deciding digit of each
    query]}."""
    scores, matched = restated if restated is not None else _restate(csr, stats, q_off, q_terms, k1, b)
    keep = matched if mask is None else matched & np.asarray(mask, bool)
    digits = {}
    for k in ks:
        got = _device_topk(csr, stats, q_off, q_terms, k, k1=k1, b=b, mask=mask, chunk_base=chunk_base)
        want = ko.bm25_topk(scores, matched, mask, k, chunk_base)
        assert np.array_equal(got[2], want[2]), ("counts", k)
        assert np.array_equal(got[0], want[0]), ("ids", k)
        assert np.array_equal(got[1].view(np.int64), want[1].view(np.int64)), ("score bits", k)
        digits[k] = [_cut_digit(scores[q], keep[q], k) for q in range(len(scores))]
        CUTS.update("none" if d is None else d for d in digits[k])
    return digits


def _plan(queries):
    q_off = np.concatenate([[0], np.cumsum([len(q) for q in queries])]).astype(np.int32)
    return q_off, np.asarray([t for q in queries for t in q], np.int32)


def _stats(N, total, df_of_term, q_terms):
    """stats int64 [2 + J] = {N, sum of doc_len, df of each entry} (0 for an entry of -1), as the host plan uploads it."""
    q_terms = np.asarray(q_terms, np.int64)
    df = np.where(q_terms >= 0, np.asarray(df_of_term, np.int64)[np.maximum(q_terms, 0)], 0)
    return np.concatenate([[N, total], df]).astype(np.int64)


def _local_stats(csr, q_terms):
    """The statistics of a single index: its own N, sum of doc_len and postings counts."""
    term_off, _, _, doc_len = csr
    return _stats(len(doc_len), int(doc_len.astype(np.int64).sum()), np.diff(term_off), q_terms)


# ---- tile edges ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, KTILE - 1, KTILE, KTILE + 1, 3 * KTILE + 17])
def test_tile_edges(n):
    rng = np.random.default_rng(n)
    edges = [c for c in (0, KTILE - 1, KTILE, n - 1) if c < n]
    spread = np.union1d(edges, rng.choice(n, size=min(n, 900), replace=False))        # several tiles
    last = (n - 1) // KTILE * KTILE
    inside = rng.choice(np.arange(last, n), size=min(n - last, 300), replace=False)   # one tile
    half = rng.choice(n, size=max(n // 2, 1), replace=False)
    doc_len = rng.integers(1, 200, size=n)
    csr = ko.csr_from_postings([(spread, rng.integers(1, 4, size=len(spread))), (inside, 1),
                                (half, rng.integers(1, 6, size=len(half))), (np.arange(n), 1)], doc_len)
    queries = [[0], [1], [0, 1, 2], [2, 0, 3, 1], [3], [], [-1, 0]]
    q_off, q_terms = _plan(queries)
    stats = _local_stats(csr, q_terms)
    restated = _restate(csr, stats, q_off, q_terms, 1.2, 0.75)
    _compare(csr, stats, q_off, q_terms, [1, 7, 4096], restated=restated)
    ids, _, count = _device_topk(csr, stats, q_off, q_terms, 4096)
    assert count[0] == len(spread) and set(edges) <= set(ids[0, : count[0]].tolist())   # the edge chunks come back
    assert len({c // KTILE for c in spread}) == (n + KTILE - 1) // KTILE                  # ... from every tile
    assert len({c // KTILE for c in inside}) == 1
    assert count[5] == 0 and count[4] == min(n, 4096)


# ---- every radix digit decides a cut ----------------------------------------------------------------------------------
def _digit_case(kind, rng):
    """(csr, queries, stats, target digits) of one family of cuts."""
    if kind == "equal":                 # one score: only ~chunk decides
        n = 50_000
        csr = ko.csr_from_postings([(rng.choice(n, size=3000, replace=False), 1), ([], 1)], np.full(n, 10))
        queries = [[0], [1], [-1]]      # valid = 3000, a term without postings, an unknown entry (valid = 0)
        return csr, queries, _local_stats(csr, _plan(queries)[1]), {7, 8}
    if kind == "last_bits":             # avgdl = 0.75 * 2^54: one more doc_len moves norm by about one ulp
        n, N = 12_000, 512              # N * avgdl fits int64; N and df need not be the local counts
        doc_len = np.empty(n, np.int64)
        doc_len[:4000] = 1 + rng.integers(0, 1 << 12, size=4000)        # scores within ~2^10 ulps: low key bits decide
        doc_len[4000:8000] = 1 + rng.integers(0, 1 << 22, size=4000)
        doc_len[8000:] = 1 + rng.integers(0, 1 << 30, size=4000)        # up to 2^30
        csr = ko.csr_from_postings([(np.arange(0, 4000), 1), (np.arange(4000, 8000), 1), (np.arange(8000, n), 1)],
                                   doc_len)
        queries = [[0], [1], [2]]
        return csr, queries, _stats(N, N * 3 * (1 << 52), [40, 40, 40], _plan(queries)[1]), {3, 4, 5}
    n, N = 30_000, 1_000_000            # distinct scores: exponents and leading mantissa bits decide
    rare = rng.choice(n, size=300, replace=False)
    common = rng.choice(n, size=6000, replace=False)
    doc_len = rng.integers(1, 3000, size=n)
    csr = ko.csr_from_postings([(rare, rng.integers(1, 1000, size=300)), (common, rng.integers(1, 100, size=6000))],
                               doc_len)
    queries = [[0, 1], [1], [0]]
    return csr, queries, _stats(N, N * 1500, [1, N], _plan(queries)[1]), {0, 1, 2}


@pytest.mark.parametrize("kind", ["equal", "last_bits", "distinct"])
def test_every_radix_digit_decides_a_cut(kind):
    csr, queries, stats, targets = _digit_case(kind, np.random.default_rng(len(kind)))
    q_off, q_terms = _plan(queries)
    scores, matched = _restate(csr, stats, q_off, q_terms, 1.2, 0.75)
    valid = matched.sum(axis=1)
    ks = {1, MAX_K}
    for q in range(len(queries)):
        ks |= {v for v in (valid[q] - 1, valid[q], valid[q] + 1) if 1 <= v <= MAX_K}
    reached = set()
    for q in range(len(queries)):
        by_digit = _ks_by_digit(scores[q], matched[q])
        for d in targets & by_digit.keys():
            ks |= set(by_digit[d][:: max(1, len(by_digit[d]) // 4)][:4])   # a few cuts of every reachable target digit
        if kind == "last_bits" and q == 0:   # cut pairs one ulp apart, the upper one odd: only the key's bit 0 decides
            _, key, _ = _ranked(scores[q], matched[q])
            bit0 = np.flatnonzero((key[:-1] ^ key[1:])[:MAX_K] == 1) + 1
            assert len(bit0) >= 8
            ks |= set(bit0[:: len(bit0) // 8][:8].tolist())
    digits = _compare(csr, stats, q_off, q_terms, sorted(int(k) for k in ks), restated=(scores, matched))
    for k, per_query in digits.items():
        reached |= {d for d in per_query if d is not None}
        if kind == "last_bits":
            for q, d in enumerate(per_query):
                if d == 5:              # the cut pair shares the top 55 key bits
                    _, key, _ = _ranked(scores[q], matched[q])
                    assert (int(key[k - 1]) ^ int(key[k])) >> 9 == 0
    assert targets <= reached, (kind, sorted(reached))
    assert any(d is None for per in digits.values() for d in per), "valid <= k: no cut"
    if kind == "equal":
        assert len(np.unique(scores[0][matched[0]])) == 1 and valid[2] == 0 and valid[1] == 0


# ---- past 2^21 chunks -----------------------------------------------------------------------------------------------
def test_past_two_to_the_21_chunks():
    """3.1 M chunks: the ~chunk digit at bits 21..31 takes two values, so it decides cuts that straddle 2^21."""
    n = 3_100_000
    rng = np.random.default_rng(21)
    every = np.arange(0, n, 1024)                                     # equal scores; 2048 of them below 2^21
    scattered = rng.choice(n, size=4000, replace=False)
    csr = ko.csr_from_postings([(every, 1), (scattered, rng.integers(1, 20, size=4000))], np.full(n, 7))
    queries = [[0], [1], [1, 0]]
    q_off, q_terms = _plan(queries)
    stats = _local_stats(csr, q_terms)
    restated = _restate(csr, stats, q_off, q_terms, 1.2, 0.75)
    assert len(every) > 2048 and (every < 1 << 21).sum() == 2048
    digits = _compare(csr, stats, q_off, q_terms, [1000, 2048, 2100, 4096], restated=restated, chunk_base=(1 << 40) + 3)
    assert every[2099] >= 1 << 21 > every[999]                       # the cut chunk of k = 2100 above 2^21, of 1000 below
    assert digits[2048][0] == 6 and digits[4096][0] is None
    # a mask around the cuts
    mask = np.ones(n, bool)
    mask[every[2040:2060]] = False
    mask[every[995:1003]] = False
    mask[every[2097:2101]] = False
    got = _compare(csr, stats, q_off, q_terms, [1000, 2048, 2100], mask=mask, restated=restated)
    assert got[2048][0] == 7                                         # the masked chunks moved the cut past 2^21


# ---- statistics as a shard receives them ------------------------------------------------------------------------------
def _shard_case(rng, n=9000, V=300, B=200):
    sizes = np.minimum((rng.pareto(1.0, size=V) * 40).astype(int), n // 3)
    sizes[:5] = [0, 1, 0, n // 3, 2]
    doc_len = rng.integers(1, 30, size=n)
    post = [(rng.choice(n, size=s, replace=False), rng.integers(1, 4, size=s)) for s in sizes]
    csr = ko.csr_from_postings(post, doc_len)
    N, total = 4 * n + 123, 4 * int(doc_len.sum()) + 99_999            # global N and sum of doc_len above the local ones
    df = np.minimum(sizes + rng.integers(0, 3 * n, size=V), N)        # global df >= local postings
    df[0], df[1], df[3] = 50, N, N                                     # df without local postings; df = N
    queries = []
    for _ in range(B):
        m = int(rng.integers(1, 13))
        q = rng.choice(V, size=m, replace=False).tolist()             # any order: the sharded plan's sorted stems
        if rng.random() < 0.3:
            q.insert(int(rng.integers(0, m + 1)), -1)                  # a stem this shard never saw
        queries.append(q)
    queries[:4] = [[0], [1, 3], [3, 2, 1, 0, -1], [-1]]
    q_off, q_terms = _plan(queries)
    stats = np.concatenate([[N, total], np.where(q_terms >= 0, df[np.maximum(q_terms, 0)], 7)]).astype(np.int64)
    return csr, stats, q_off, q_terms


def test_statistics_unrelated_to_the_local_postings():
    csr, stats, q_off, q_terms = _shard_case(np.random.default_rng(5))
    term_off = csr[0]
    local = np.diff(term_off)[np.maximum(q_terms, 0)]
    assert (stats[2:][q_terms >= 0] > local[q_terms >= 0]).any() and (stats[2:] == stats[0]).any()
    assert (np.diff(q_terms[q_off[2]:q_off[3] - 1]) < 0).all()        # entries [3, 2, 1, 0, -1]: descending
    digits = _compare(csr, stats, q_off, q_terms, [1, 10, 100, 4096], chunk_base=12345)
    assert any(d is not None and d >= 6 for per in digits.values() for d in per)   # ties cut by ~chunk


# ---- parameters ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k1,b", [(1.2, 0.75), (0.0, 0.75), (1.2, 0.0), (1.2, 1.0), (2.5, 0.3)])
def test_parameters(k1, b):
    rng = np.random.default_rng(int(k1 * 10 + b * 100))
    n, V = 20_000, 50
    doc_len = np.exp(rng.uniform(0, np.log(2.0**30), size=n)).astype(np.int64)          # 1 .. 2^30
    doc_len[:2] = [1, 1 << 30]
    post = []
    for _ in range(V):
        s = int(rng.integers(500, 3000))
        tf = np.exp(rng.uniform(0, np.log(1e6), size=s)).astype(np.int64)               # 1 .. 10^6
        tf[0] = 1_000_000
        post.append((rng.choice(n, size=s, replace=False), tf))
    csr = ko.csr_from_postings(post, doc_len)
    queries = [rng.choice(V, size=int(rng.integers(1, 9)), replace=False).tolist() for _ in range(64)]
    q_off, q_terms = _plan(queries)
    stats = _local_stats(csr, q_terms)
    assert csr[2].max() == 1_000_000 and csr[3].max() == 1 << 30
    _compare(csr, stats, q_off, q_terms, [1, 50, 4096], k1=k1, b=b)


# ---- query groups ----------------------------------------------------------------------------------------------------
def test_query_groups_are_bit_identical():
    csr, stats, q_off, q_terms = _shard_case(np.random.default_rng(9), n=6000, V=200, B=40)
    _compare(csr, stats, q_off, q_terms, [64])
    full = _device_topk(csr, stats, q_off, q_terms, 64)
    for group in (1, 7):                                               # 7: a partial last group
        got = _device_topk(csr, stats, q_off, q_terms, 64, group=group)
        assert all(np.array_equal(a.view(np.int64), c.view(np.int64)) for a, c in zip(got, full, strict=True)), group


def test_more_queries_than_one_launch_holds():
    """B = 65 537 on a tiny corpus: the grid's y limit makes two launches (groups of 65 535 and 2)."""
    rng = np.random.default_rng(65537)
    n, V, B = 37, 6, 65_537
    csr = ko.csr_from_postings([(rng.choice(n, size=int(s), replace=False), rng.integers(1, 3, size=int(s)))
                                for s in (5, 20, 37, 1, 12, 30)], rng.integers(1, 5, size=n))
    queries = [rng.permutation(V)[: int(rng.integers(0, V + 1))].tolist() for _ in range(B)]
    queries[-2:] = [[2], [5, 0, 1]]
    q_off, q_terms = _plan(queries)
    stats = _local_stats(csr, q_terms)
    # the restatement once per distinct query
    uniq = sorted({tuple(q) for q in queries})
    u_off, u_terms = _plan([list(q) for q in uniq])
    u_stats = _local_stats(csr, u_terms)
    scores, matched = _restate(csr, u_stats, u_off, u_terms, 1.2, 0.75)
    row = {q: i for i, q in enumerate(uniq)}
    pick = np.asarray([row[tuple(q)] for q in queries])
    k = 5
    want = ko.bm25_topk(scores, matched, None, k)
    got = _device_topk(csr, stats, q_off, q_terms, k)
    assert np.array_equal(got[2], want[2][pick]) and np.array_equal(got[0], want[0][pick])
    assert np.array_equal(got[1].view(np.int64), want[1][pick].view(np.int64))
    assert B > 65_535 and (got[2][-2:] > 0).all()


def test_empty_shard():
    """n_chunks = 0 with a NULL workspace (and NULL doc_len): every row empty."""
    term_off = np.zeros(4, np.int64)
    csr = (term_off, np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(0, np.int32))
    q_off, q_terms = _plan([[0, 1], [], [2, -1]])
    ids, scores, count = _device_topk(csr, np.asarray([100, 500, 3, 4, 5, 6], np.int64), q_off, q_terms, 5,
                                      chunk_base=1 << 41)
    assert (count == 0).all() and (ids == -1).all() and np.isneginf(scores).all()


# ---- rl_bm25_stats -----------------------------------------------------------------------------------------------------
def test_stats_kernel_matches_numpy():
    import torch

    L = _lib()
    lib = L.load()
    rng = np.random.default_rng(200_000)
    V, n = 200_000, 150_001                                            # n is not a multiple of 1024
    term = rng.integers(0, V, size=300_000)
    chunk = rng.integers(0, n, size=300_000)
    special = {0: 0, 70_001: 1, 65_536: 255, 131_072: 256, 199_999: 257, 100_000: 120_000, 3: 120_001}
    for t, s in special.items():
        drop = term == t
        term, chunk = term[~drop], chunk[~drop]
        term = np.concatenate([term, np.full(s, t)])
        chunk = np.concatenate([chunk, rng.choice(n, size=s, replace=False)])
    pairs = np.unique((term.astype(np.int64) << 32) | chunk)
    term, doc = pairs >> 32, (pairs & 0xFFFFFFFF).astype(np.int32)
    term_off = np.concatenate([[0], np.cumsum(np.bincount(term, minlength=V))]).astype(np.int64)
    assert all(term_off[t + 1] - term_off[t] == s for t, s in special.items())
    doc_len = rng.integers(0, 1 << 30, size=n).astype(np.int32)
    d_term_off, d_doc, d_len = _up(term_off, np.int64), _up(doc, np.int32), _up(doc_len, np.int32)
    for name, alive in (("none", None), ("random", rng.random(n) < 0.7), ("dead", np.zeros(n, bool))):
        live = np.ones(n, bool) if alive is None else alive
        df = torch.full((V,), -7, dtype=torch.int32, device="cuda")
        corpus = torch.full((3,), -7.0, dtype=torch.float64, device="cuda")
        d_alive = None if alive is None else _up(alive, np.uint8)
        L.check(lib.rl_bm25_stats(d_term_off.data_ptr(), d_doc.data_ptr(), d_len.data_ptr(),
                                  None if d_alive is None else d_alive.data_ptr(), V, n, df.data_ptr(), corpus.data_ptr(),
                                  torch.cuda.current_stream().cuda_stream), "rl_bm25_stats")
        want_df = np.bincount(term, weights=live[doc], minlength=V).astype(np.int64)
        got_df, got = df.cpu().numpy(), corpus.cpu().numpy()
        N, total = int(live.sum()), int(doc_len[live].astype(np.int64).sum())
        assert total < 2**53 and (name != "none" or total > 2**32)
        assert np.array_equal(got_df, want_df), (name, np.flatnonzero(got_df != want_df)[:5])
        assert got[0] == N and got[1] == total, name
        with np.errstate(invalid="ignore"):
            avgdl = np.float64(total) / np.float64(N)
        assert got[2].view(np.int64) == avgdl.view(np.int64) or (np.isnan(got[2]) and np.isnan(avgdl)), name
        if name == "dead":
            assert N == 0 and total == 0 and np.isnan(got[2]) and (got_df == 0).all()
