"""Which rows vector search returns when similarities tie, held bit for bit to ``vector_exact_oracle``.

Rows and queries have small integer entries, so every returned sim is a known float32 value and every hit list a known
function of (sim desc, row asc).  Ids, the bits of every sim, counts and the -inf / -1 padding must match exactly, at the
scan (``CorpusIndex.scan`` / ``scan_checked``), after ``merge_hits``, and through the public ``vector_search_batch``.

The corpora reach the code random ones never do: ties at the ``num_hits`` cut, ``select_kernel``'s fallback over the
whole sample (more than 8192 tied sample rows), ``finalize_kernel``'s streaming rescoring past 4096 survivors and every
digit of its radix select (``block_gather_top``), exact MaxSim's GROUP BY over more than 512 survivors, masks that
remove the lowest tied rows, chunk ids past 2^40, candidate-list overflow retries and an R = 3 split of one corpus.
The ``~row`` bits 28..31 of the streaming composite are not covered: telling them apart needs more than 2^28 rows."""

from __future__ import annotations

import numpy as np
import pytest
import vector_exact_oracle as vo

pytestmark = pytest.mark.gpu

DIGIT_CUTS: dict[int, int] = {s: 0 for s in vo.SHIFTS}


@pytest.fixture(scope="module")
def rl():
    import torch

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import raglite_b200

    return raglite_b200


@pytest.fixture(scope="module", autouse=True)
def _digit_report():
    yield
    print("\nblock_gather_top cuts per digit (shift: count):", DIGIT_CUTS)


def _dev(x):
    import torch

    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _row_chunk(off, n):
    return np.repeat(np.arange(len(off) - 1), np.diff(off)).astype(np.int64)[:n]


def _same(got, want, what):
    gs, gc, gn = got
    ws, wc, wn = want
    assert int(gn) == int(wn), (what, "count", int(gn), int(wn))
    assert np.array_equal(np.asarray(gc), wc), (what, "ids", np.nonzero(np.asarray(gc) != wc)[0][:8], gc[:8], wc[:8])
    assert np.array_equal(np.asarray(gs, np.float32).view(np.uint32), ws.view(np.uint32)), (
        what, "sim bits", np.nonzero(np.asarray(gs, np.float32).view(np.uint32) != ws.view(np.uint32))[0][:8])


def _check_scan(idx, res, E, Q, off, metric, *, num_hits, k, allowed=None, base=0, what="", sims=None):
    """Scan output (per query) and its ``merge_hits`` against the restatement.  ``sims`` (``[B, N]``, from
    ``vo.exact_sims_batch``) is computed when not given; returns it, so a caller checks several passes over one corpus
    with one restatement of the sims."""
    from raglite_b200._index import merge_hits

    if sims is None:
        sims = vo.exact_sims_batch(E, Q, metric)
    rc = _row_chunk(off, len(E))
    hs, hc, hn = res.hit_sim.cpu().numpy(), res.hit_chunk.cpu().numpy(), res.hit_count.cpu().numpy()
    assert np.all(res.status.cpu().numpy() == 0), what
    H = num_hits if num_hits > 0 else k
    want = np.zeros((1, len(Q), H), np.float32), np.zeros((1, len(Q), H), np.int64), np.zeros((1, len(Q)), np.int32)
    for b in range(len(Q)):
        w = (vo.sql_hits(sims[b], rc, num_hits, allowed=allowed, chunk_base=base) if num_hits > 0
             else vo.exact_hits(sims[b], rc, k, allowed=allowed, chunk_base=base))
        _same((hs[b], hc[b], hn[b]), w, f"{what} scan b={b}")
        want[0][0, b], want[1][0, b], want[2][0, b] = w
    ms, mc, mn = merge_hits(res.hit_sim, res.hit_chunk, res.hit_count, num_hits=num_hits, k=k)
    ws, wc, wn = vo.merge_hits(*want, num_hits, k)
    ms, mc, mn = ms.cpu().numpy(), mc.cpu().numpy(), mn.cpu().numpy()
    for b in range(len(Q)):
        _same((ms[b], mc[b], mn[b]), (ws[b], wc[b], wn[b]), f"{what} merge b={b}")
    return sims


def _int_corpus(n, d, pool, seed, lo=-3, hi=3):
    """``n`` rows drawn from ``pool`` distinct integer rows (each repeated n / pool times, shuffled): every sim ties."""
    rng = np.random.default_rng(seed)
    P = rng.integers(lo, hi + 1, size=(pool, d)).astype(np.float32)
    P[np.abs(P).sum(1) == 0, 0] = 1
    return P[rng.permutation(np.arange(n) % pool)]


def _queries(B, d, seed):
    rng = np.random.default_rng(seed)
    Q = rng.integers(-3, 4, size=(B, d)).astype(np.float32)
    Q[np.abs(Q).sum(1) == 0, 0] = 1
    return Q


# ---- the matrix: every metric, storage, scan and width, ties at the cut ------------------------------------------
def _matrix():
    out = []
    Bs = (1, 7, 129, 300)
    i = 0
    for metric in ("cosine", "dot", "l2", "l1"):
        paths = [("fp32", "fp32"), ("fp16", "fp32")] if metric == "l1" else [("fp32", "fp32"), ("fp32", "tcgen05"), ("fp16", "tcgen05")]
        for storage, algo in paths:
            for d in (4, 8, 50, 64, 1024):
                if (storage == "fp16" and d % 8) or (algo == "tcgen05" and d % 4) or (d == 50 and (storage, algo) != ("fp32", "fp32")):
                    continue
                B = Bs[i % 4] if d < 1024 else 7
                i += 1
                out.append((metric, storage, algo, d, B))
    out.append(("cosine", "fp32", "tcgen05", 1024, 300))    # 256-query groups of the fp32 tensor-core scan
    out.append(("dot", "fp32", "tcgen05", 1024, 300))
    return out


@pytest.mark.parametrize("case", _matrix(), ids=lambda c: "-".join(map(str, c)))
def test_ties_match_the_restatement(rl, case):
    metric, storage, algo, d, B = case
    n = 3000
    E = _int_corpus(n, d, pool=n // 2, seed=d + B)                 # every row has exactly one twin
    Q = _queries(B, d, seed=d * 7 + B)
    rng = np.random.default_rng(d)
    off = np.r_[0, np.cumsum(rng.integers(1, 5, size=n))]
    off = off[off < n]
    off = np.r_[off, n].astype(np.int64)
    idx = rl.CorpusIndex(E, off, storage=storage)
    Qd = _dev(Q)
    sims = vo.exact_sims_batch(E, Q, metric)
    for num_hits, k in ((100, 10), (0, 10)):
        res = idx.scan_checked(Qd, k=k, num_hits=num_hits, metric=metric, algo=algo)
        _check_scan(idx, res, E, Q, off, metric, num_hits=num_hits, k=k, sims=sims, what=f"{case} num_hits={num_hits}")


# ---- tied sets at the cut: a few rows, a window's worth, more than 4096 rows -------------------------------------
@pytest.mark.parametrize("algo", ["fp32", "tcgen05"])
@pytest.mark.parametrize("group", [2, 4096 - 100 + 1, 5000])
def test_tied_group_at_the_cut(rl, group, algo):
    E, Q, K, (n_above, n_tied) = vo.tied_group_case(group)
    off = np.arange(len(E) + 1, dtype=np.int64)
    idx = rl.CorpusIndex(E, off)
    Qd = _dev(Q)
    sims = vo.exact_sims_batch(E, Q, "dot")
    for num_hits, k in ((K, 20), (0, K)):
        res = idx.scan_checked(Qd, k=k, num_hits=num_hits, metric="dot", algo=algo)
        _check_scan(idx, res, E, Q, off, "dot", num_hits=num_hits, k=k, sims=sims, what=f"group={group} {algo} nh={num_hits}")
        if group > 2:   # query 0's survivors are the rows at or above its cut: the window edge, then past it
            assert idx.scan_stats()["survivors_max"] == n_above + n_tied, (idx.scan_stats(), n_above, n_tied)


# ---- fully tied corpus: select_kernel's fallback over the whole sample, masks, size limits -----------------------
@pytest.mark.parametrize("metric", ["cosine", "l1"])
def test_fully_tied_corpus(rl, metric):
    n, d = 20_000, 8
    E = np.tile(np.array([[1, 2, 0, -1, 3, 0, 1, 1]], np.float32), (n, 1))
    Q = _queries(2, d, seed=5)
    off = np.arange(n + 1, dtype=np.int64)
    idx = rl.CorpusIndex(E, off, chunk_ids=[f"c{i}" for i in range(n)], chunk_base=2 ** 40 + 3)
    Qd = _dev(Q)
    base = 2 ** 40 + 3
    sims = vo.exact_sims_batch(E, Q, metric)
    for stride in (1, 0):             # stride 1: all 20000 tied rows in the sample (> 8192: the fallback)
        for num_hits, k in ((1, 1), (100, 10), (4096, 50), (0, 1), (0, 1000), (0, 4096)):
            res = idx.scan_checked(Qd, k=k, num_hits=num_hits, metric=metric, sample_stride=stride)
            if stride == 1:   # every sample row ties with the sel_k-th: more than the select's 8192-entry lists
                st = idx.scan_stats()
                assert st["sample_stride"] == 1 and st["n_sample_rows"] >= n > vo.SEL_LIST_CAP, st
            _check_scan(idx, res, E, Q, off, metric, num_hits=num_hits, k=k, base=base, sims=sims,
                        what=f"stride={stride} nh={num_hits} k={k}")
    # a filter that removes the lowest tied rows, then tombstones of the next ones: the rows after them come back
    allowed = np.ones(n, bool)
    allowed[:300] = False
    res = idx.scan_checked(Qd, k=10, num_hits=100, metric=metric, row_allowed=_dev(allowed.astype(np.uint8)))
    _check_scan(idx, res, E, Q, off, metric, num_hits=100, k=10, allowed=allowed, base=base, sims=sims, what="filter")
    idx.delete_chunks([f"c{i}" for i in range(0, 5000, 2)])
    alive = np.ones(n, bool)
    alive[0:5000:2] = False
    for num_hits, k in ((100, 10), (0, 700)):
        res = idx.scan_checked(Qd, k=k, num_hits=num_hits, metric=metric)
        _check_scan(idx, res, E, Q, off, metric, num_hits=num_hits, k=k, allowed=alive, base=base, sims=sims, what="tombstones")
    res = idx.scan_checked(Qd, k=10, num_hits=100, metric=metric, row_allowed=_dev(allowed.astype(np.uint8)) & idx._alive,
                   mask_has_tombstones=True)
    _check_scan(idx, res, E, Q, off, metric, num_hits=100, k=10, allowed=allowed & alive, base=base, sims=sims,
                what="filter+tombstones")


def test_exact_selection_size_limit(rl):
    """Exact MaxSim selects (k - 1) max_vecs + 1 rows: 4096 is accepted (one tied 4095-vector chunk), 4097 refused."""
    from raglite_b200._lib import RagliteB200Error

    d = 8
    row = np.array([[2, 1, 0, 0, 1, 0, 0, 1]], np.float32)
    for mv, ok in ((4095, True), (4096, False)):
        E = np.tile(row, (mv + 3000, 1))
        off = np.r_[0, np.arange(mv, mv + 3001)].astype(np.int64)    # one chunk of mv tied rows, 3000 single-row chunks
        idx = rl.CorpusIndex(E, off)
        Q = _queries(3, d, seed=mv)
        if ok:
            res = idx.scan_checked(_dev(Q), k=2, num_hits=0, metric="cosine")
            _check_scan(idx, res, E, Q, off, "cosine", num_hits=0, k=2, what=f"max_vecs={mv}")
        else:
            with pytest.raises(RagliteB200Error, match="exceeds the 4096-survivor"):
                idx.scan(_dev(Q), k=2, num_hits=0, metric="cosine")


# ---- every digit of block_gather_top ------------------------------------------------------------------------------
@pytest.mark.parametrize("algo", ["fp32", "tcgen05"])
@pytest.mark.parametrize("shift", vo.SHIFTS)
def test_streaming_select_every_digit(rl, shift, algo):
    E, q, K, planted = vo.digit_case(shift)
    n = len(E)
    Q = np.tile(q, (2, 1))
    off = np.arange(n + 1, dtype=np.int64)
    idx = rl.CorpusIndex(E, off)
    sims = vo.exact_sims_batch(E, Q, "dot")
    want_shift, _ = vo.gather_top(vo.composites(sims[0], planted), K)
    assert want_shift == shift
    for num_hits, k in ((K, 10), (0, K)):
        res = idx.scan_checked(_dev(Q), k=k, num_hits=num_hits, metric="dot", algo=algo)
        _check_scan(idx, res, E, Q, off, "dot", num_hits=num_hits, k=k, sims=sims, what=f"digit {shift} {algo} nh={num_hits}")
        st = idx.scan_stats()
        assert st["survivors_max"] == len(planted) and st["survivors_total"] == len(Q) * len(planted), st
        DIGIT_CUTS[shift] += len(Q)


# ---- exact MaxSim: a chunk that spans two sampled blocks ----------------------------------------------------------
@pytest.mark.parametrize("stride", [0, 2, 4, 16])
def test_exact_maxsim_chunk_spanning_sampled_blocks(rl, stride):
    """Chunk C's first row ends sampled block 0 and its last row starts sampled block S: C must count once in the
    sample's order statistic, or the emit threshold lands above the second chunk and only C comes back."""
    S = stride or 2
    E, q, off, _ = vo.spanning_chunk_case(S)
    Q = q[None, :].copy()
    idx = rl.CorpusIndex(E, off)
    res = idx.scan_checked(_dev(Q), k=2, num_hits=0, metric="cosine", algo="fp32", sample_stride=stride)
    assert idx.scan_stats()["sample_stride"] == S
    _check_scan(idx, res, E, Q, off, "cosine", num_hits=0, k=2, what=f"spanning chunk S={S}")
    assert int(res.hit_count[0]) == 2


def test_public_vector_search_batch(rl):
    """One public call per mode on a tied corpus, against the restatement through the merge."""
    E, q, off, _ = vo.spanning_chunk_case(2)
    E[4000:6000] = E[3000]                           # 2000 tied rows
    Q = np.stack([q, E[3000]])
    idx = rl.CorpusIndex(E, off)
    from raglite_b200._search import num_hits_rule

    cfg = rl.RAGLiteConfig(reranker=None)
    rc = _row_chunk(off, len(E))
    nr = 12
    for exact in (True, False):
        ids, sims, counts = rl.vector_search_batch(Q, num_results=nr, config=cfg, index=idx, exact_maxsim=exact)
        nh = 0 if exact else num_hits_rule(nr, 4, cfg.chunk_max_size)
        H = nh or nr
        lists = np.zeros((1, len(Q), H), np.float32), np.zeros((1, len(Q), H), np.int64), np.zeros((1, len(Q)), np.int32)
        s = vo.exact_sims_batch(E, Q, cfg.vector_search_distance_metric)
        for b in range(len(Q)):
            lists[0][0, b], lists[1][0, b], lists[2][0, b] = (vo.sql_hits(s[b], rc, nh) if nh else vo.exact_hits(s[b], rc, nr))
        ws, wc, wn = vo.merge_hits(*lists, nh, nr)
        for b in range(len(Q)):
            _same((sims[b], ids[b], counts[b]), (ws[b], wc[b], wn[b]), f"public exact={exact} b={b}")


# ---- candidate-list overflow: both retries end bit-exact -----------------------------------------------------------
@pytest.mark.parametrize("tied", [200, 3000])
def test_overflow_retries(rl, tied):
    """``cand_cap`` = 256 and the retries of ``run_until_no_overflow``, one pass at a time.  200 tied rows at the top of
    query 0, all in odd 128-row blocks, which no sample stride > 1 samples: the sample's k-th value is a background row,
    the first pass emits several hundred rows and overflows, and its finalize cut (the tied value) makes the
    threshold-reuse retry fit the same 256 slots.  3000 tied rows never fit 256: the reuse retry overflows again and a
    4096-entry list ends it."""
    from raglite_b200._lib import RL_FLAG_REUSE_THRESHOLDS, RL_STATUS_CAND_OVERFLOW

    n, d = 20_000, 8
    rng = np.random.default_rng(tied)
    E = rng.integers(-3, 4, size=(n, d)).astype(np.float32)
    E[np.abs(E).sum(1) == 0, 0] = 1
    Q = _queries(2, d, seed=tied)
    odd_block_rows = np.nonzero((np.arange(n) // 128) % 2 == 1)[0]
    E[rng.choice(odd_block_rows, size=tied, replace=False)] = Q[0] * 2       # tied rows at the top for query 0
    off = np.arange(n + 1, dtype=np.int64)
    idx = rl.CorpusIndex(E, off)
    Qd = _dev(Q)
    sims = vo.exact_sims_batch(E, Q, "cosine")
    want = [RL_STATUS_CAND_OVERFLOW, 0] if tied < 256 else [RL_STATUS_CAND_OVERFLOW, RL_STATUS_CAND_OVERFLOW, 0]
    for num_hits, k in ((10, 10), (0, 10)):
        kw = dict(k=k, num_hits=num_hits, metric="cosine", algo="fp32")
        res = idx.scan(Qd, **kw, cand_cap=256)
        assert idx.scan_stats()["sample_stride"] > 1
        statuses = [int(res.status.max())]
        res = idx.scan(Qd, **kw, cand_cap=256, flags=RL_FLAG_REUSE_THRESHOLDS, out=res)   # re-uses the failed pass's cut
        statuses.append(int(res.status.max()))
        if statuses[-1] == 0:
            _check_scan(idx, res, E, Q, off, "cosine", num_hits=num_hits, k=k, sims=sims, what=f"reuse tied={tied}")
        else:
            res = idx.scan(Qd, **kw, cand_cap=4096, out=res)                           # a list that holds the tied rows
            statuses.append(int(res.status.max()))
            if statuses[-1] == 0:
                _check_scan(idx, res, E, Q, off, "cosine", num_hits=num_hits, k=k, sims=sims, what=f"larger list tied={tied}")
        print(f"overflow tied={tied} num_hits={num_hits}: statuses {statuses}")
        assert statuses == want, statuses
        res = idx.scan_checked(Qd, **kw, cand_cap=256)
        _check_scan(idx, res, E, Q, off, "cosine", num_hits=num_hits, k=k, sims=sims, what=f"scan_checked tied={tied}")


# ---- sharding: an R = 3 split of one tied corpus ----------------------------------------------------------------
@pytest.mark.parametrize("metric", ["cosine", "l2"])
def test_three_shards_of_a_tied_corpus(rl, metric):
    import torch

    from raglite_b200._index import merge_hits

    n, d = 9000, 64
    E = _int_corpus(n, d, pool=40, seed=11)            # 225 copies of every row
    Q = _queries(5, d, seed=12)
    off = np.arange(n + 1, dtype=np.int64)
    cuts = [0, 2000, 5500, n]
    sims = vo.exact_sims_batch(E, Q, metric)
    for num_hits, k in ((1000, 30), (0, 300)):
        H = num_hits or k
        parts = []
        for r in range(3):
            lo, hi = cuts[r], cuts[r + 1]
            sh = rl.CorpusIndex(E[lo:hi], off[lo:hi + 1] - lo, chunk_base=lo)
            res = sh.scan_checked(_dev(Q), k=k, num_hits=num_hits, metric=metric)
            parts.append((res.hit_sim.clone(), res.hit_chunk.clone(), res.hit_count.clone()))
        hs, hc, hn = (torch.stack([p[i] for p in parts]) for i in range(3))
        ms, mc, mn = (x.cpu().numpy() for x in merge_hits(hs, hc, hn, num_hits=num_hits, k=k))
        rc = _row_chunk(off, n)
        lists = np.zeros((1, len(Q), H), np.float32), np.zeros((1, len(Q), H), np.int64), np.zeros((1, len(Q)), np.int32)
        for b in range(len(Q)):
            lists[0][0, b], lists[1][0, b], lists[2][0, b] = (vo.sql_hits(sims[b], rc, num_hits) if num_hits
                                                              else vo.exact_hits(sims[b], rc, k))
        ws, wc, wn = vo.merge_hits(*lists, num_hits, k)
        for b in range(len(Q)):
            _same((ms[b], mc[b], mn[b]), (ws[b], wc[b], wn[b]), f"R=3 {metric} nh={num_hits} b={b}")
