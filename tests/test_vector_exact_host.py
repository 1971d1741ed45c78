"""The bit-exact restatement of vector search (``vector_exact_oracle``) against the float64 oracle and the rounding
chains of ``test_gpu_rescoring``, and the path and digit every device construction of ``test_gpu_vector_ties`` reaches,
decided from the data alone.  CPU only."""

from __future__ import annotations

import numpy as np
import pytest
import rounding as rd
import vector_exact_oracle as vo
from test_gpu_rescoring import CHAINS

from oracle import vector_search as ovs

CHAINS_ALL = {**CHAINS, "l1": lambda x: vo.ONE - rd.f32(x)}   # sim = 1 - (float)sum |e - q|


def _int_rows(n, d, seed, lo=-3, hi=3):
    rng = np.random.default_rng(seed)
    E = rng.integers(lo, hi + 1, size=(n, d)).astype(np.float32)
    E[np.abs(E).sum(1) == 0, 0] = 1
    return E


@pytest.mark.parametrize("metric", ["cosine", "dot", "l2", "l1"])
def test_sims_follow_the_rescoring_chains(metric):
    E = _int_rows(4000, 64, seed=1)
    q = _int_rows(1, 64, seed=2)[0]
    got = vo.exact_sims(E, q, metric)
    E64, q64 = E.astype(np.float64), q.astype(np.float64)
    if metric == "cosine":
        v = (E64 @ q64) / np.sqrt(np.einsum("ij,ij->i", E64, E64) * (q64 @ q64))
    elif metric == "dot":
        v = E64 @ q64
    elif metric == "l2":
        v = np.einsum("ij,ij->i", E64 - q64, E64 - q64)
    else:
        v = np.abs(E64 - q64).sum(1)
    want = CHAINS_ALL[metric](v)
    assert np.array_equal(got.view(np.uint32), np.asarray(want, np.float32).view(np.uint32))


def test_refuses_inputs_whose_sums_would_round():
    with pytest.raises(AssertionError, match="integers"):
        vo.exact_sims(np.full((2, 4), 0.5, np.float32), np.ones(4, np.float32), "dot")
    with pytest.raises(AssertionError, match="would round"):
        vo.exact_sims(np.full((2, 4), 2.0 ** 26, np.float32), np.full(4, 2.0 ** 26, np.float32), "cosine")


@pytest.mark.parametrize("metric", ["cosine", "dot", "l2"])
def test_sql_list_equals_the_float64_oracle_with_float32_ties(metric):
    """The restated num_hits list is the oracle's ``ORDER BY dist LIMIT num_hits`` with float32 ties by row, and its
    GROUP BY is ``group_hits``.  For cosine the oracle rounds 1 - (1 - s), the kernel s: the rows where the two float32
    sims differ are counted and named; outside them the lists agree."""
    n, d, num_hits = 3000, 16, 200
    rng = np.random.default_rng(3)
    P = _int_rows(600, d, seed=4)
    E = P[rng.permutation(np.arange(n) % 600)]         # five copies of every row: every sim ties
    off = np.arange(n + 1, dtype=np.int64)
    rc = np.arange(n)
    differ = []
    for b in range(6):
        q = _int_rows(1, d, seed=10 + b)[0]
        sims = vo.exact_sims(E, q, metric)
        s, c, cnt = vo.sql_hits(sims, rc, num_hits)
        ids, gsims, rows = ovs.vector_search_sql(E, off, q, num_results=num_hits, oversample=1, metric=metric,
                                                 f64=True, f32_ties=True)
        dist32 = ovs.float_distance_of_f64(ovs.vector_distances_f64(E, q, metric), metric)
        osim = vo.ONE - dist32
        bad = np.nonzero(osim.view(np.uint32) != sims.view(np.uint32))[0]
        differ.append(len(bad))
        if metric != "cosine" or len(bad) == 0:
            assert cnt == num_hits and np.array_equal(c, rows)
            assert np.array_equal(s.view(np.uint32), osim[rows].view(np.uint32))
            w_ids, w_sims = ovs.group_hits(dist32[rows], rc[rows], num_hits)
            assert np.array_equal(w_ids, c[: len(w_ids)]) and np.array_equal(w_sims, s[: len(w_sims)])
        else:   # name the rows: float32(1 - (1 - s)) != float32(s) only where 1 - (1 - s) loses bits of s
            s64 = (E.astype(np.float64) @ q) / np.sqrt(np.einsum("ij,ij->i", E.astype(np.float64), E.astype(np.float64)) * (q.astype(np.float64) @ q))
            assert np.all(rd.f32(1.0 - (1.0 - s64[bad])) != rd.f32(s64[bad]))
            assert np.all(np.abs(s64[bad]) < 0.5)
    print(f"{metric}: rows where float_distance_of_f64's sim differs from exact_sim's, per query: {differ}")
    if metric != "cosine":
        assert not any(differ)


def test_exact_mode_equals_maxsim_topk_exact():
    n, d = 4000, 16
    rng = np.random.default_rng(5)
    E = _int_rows(n, d, seed=6, lo=-2, hi=2)
    off = np.r_[0, np.cumsum(rng.integers(1, 6, size=n))]
    off = np.r_[off[off < n], n].astype(np.int64)
    rc = np.repeat(np.arange(len(off) - 1), np.diff(off))
    for b in range(4):
        q = _int_rows(1, d, seed=20 + b)[0]
        sims = vo.exact_sims(E, q, "dot")
        s, c, cnt = vo.exact_hits(sims, rc, 50)
        ids, s64 = ovs.maxsim_topk_exact(E, off, q, 50, "dot")
        assert cnt == 50 and np.array_equal(c, ids) and np.array_equal(s, rd.f32(s64))   # s64 = 1 + dot, exact


def test_merge_restatement_groups_the_sql_list():
    """``merge_hits`` of one SQL list is ``group_hits`` over it (the first occurrence of a chunk carries its max)."""
    n, d = 3000, 8
    rng = np.random.default_rng(7)
    E = _int_rows(n, d, seed=8, lo=-1, hi=1)
    off = np.r_[0, np.cumsum(rng.integers(1, 4, size=n))]
    off = np.r_[off[off < n], n].astype(np.int64)
    rc = np.repeat(np.arange(len(off) - 1), np.diff(off))
    q = _int_rows(1, d, seed=9)[0]
    sims = vo.exact_sims(E, q, "l2")
    s, c, cnt = vo.sql_hits(sims, rc, 300)
    ms, mc, mn = vo.merge_hits(s[None, None], c[None, None], np.array([[cnt]]), 300, 40)
    w_ids, w_sims = ovs.group_hits(vo.ONE - s[:cnt], c[:cnt], 40)
    # group_hits breaks chunk ties by chunk index, the device by first occurrence (row order): equal where no two
    # chunks tie, and the same set of sims always
    assert np.array_equal(np.sort(ms[0, :mn[0]]), np.sort(vo.ONE - (vo.ONE - w_sims)))
    first = {}
    for i in range(cnt):
        first.setdefault(int(c[i]), i)
    want = sorted(first, key=first.get)[:40]
    assert mn[0] == 40 and mc[0, :40].tolist() == want


# ---- the device constructions: path and digit from the data ----------------------------------------------------------
@pytest.mark.parametrize("shift", vo.SHIFTS)
def test_digit_cases_reach_their_digit(shift):
    E, q, K, planted = vo.digit_case(shift)
    sims = vo.exact_sims(E, q, "dot")
    rest = np.setdiff1d(np.arange(len(E)), planted)
    assert sims[planted].min() - sims[rest].max() > 2 ** 22    # every other row far below the cut: survivors = planted
    assert len(planted) > vo.WINDOW                              # more survivors than the window: the streaming path
    got_shift, gathered = vo.gather_top(vo.composites(sims, planted), K)
    assert got_shift == shift
    assert K <= len(gathered) <= vo.WINDOW
    best = vo.order(sims)[:K]                                    # the K best are among the gathered composites
    assert np.isin(vo.composites(sims, best), gathered).all()
    if shift in (52, 40, 28):                                    # decided by sims one float step apart
        s = np.unique(sims[planted])
        assert len(s) == 2 and np.nextafter(s[0], np.float32(np.inf)) == s[1]
    else:                                                        # decided by the row order of one tied sim
        assert len(np.unique(sims[planted])) == 1


def test_gather_top_full_resolution_and_short_sets():
    rng = np.random.default_rng(0)
    comps = rng.choice(2 ** 62, size=10_000, replace=False).astype(np.uint64) + np.uint64(1)
    shift, got = vo.gather_top(comps, 100)
    assert shift == 52 and np.array_equal(np.sort(got)[-100:], np.sort(comps)[-100:])
    shift, got = vo.gather_top(comps[:50], 100)                 # fewer than K: everything, first digit
    assert shift == 52 and len(got) == 50


@pytest.mark.parametrize("S", [2, 4, 16])
def test_spanning_chunk_case(S):
    """C starts at the last row of sampled block 0 and ends at the first row of sampled block S; the second best chunk
    is a single row far below C.  At auto stride the layout picks S = 2 (8 cut to 2 by the 8 sel_k rows_per_sel rule)."""
    E, q, off, (lo, hi) = vo.spanning_chunk_case(S)
    assert lo == 127 and hi - 1 == S * 128 and hi - lo == 128 * (S - 1) + 2
    sims = vo.exact_sims(E, q, "cosine")
    rc = np.repeat(np.arange(len(off) - 1), np.diff(off))
    s, c, cnt = vo.exact_hits(sims, rc, 2)
    assert cnt == 2 and c[0] == rc[lo] and sims[lo:hi].min() > 0.85 and s[1] < 0.6
    if S == 2:   # make_layout's automatic stride for n = 8200, k = 2, max_vecs = 130
        n_blocks, sel = (len(E) + 127) // 128, 2 * (hi - lo)
        f = np.sqrt(2 * (hi - lo) * 16.0 / (len(E) * 4.0))
        auto = 1 << int(np.floor(np.log2(4.0 / f)))
        while auto > 1 and (n_blocks // auto) * 128 < 8 * sel:
            auto //= 2
        assert n_blocks >= 64 and auto == 2


@pytest.mark.parametrize("group", [2, 4096 - 100 + 1, 5000])
def test_tied_group_case_sizes(group):
    """The tied set at query 0's cut (planted copies plus natural twins), and the rows at or above the cut: inside the
    window, exactly the window, past it (the streaming rescoring)."""
    E, Q, K, (above, tied) = vo.tied_group_case(group)
    assert above < K <= above + tied and tied >= group
    assert {2: above + tied < vo.WINDOW, 3997: above + tied == vo.WINDOW, 5000: above + tied > vo.WINDOW}[group]
    print(f"group {group}: {above} rows above the cut, {tied} tied at it")


def test_batched_sims_equal_per_query_sums():
    """``exact_sims_batch`` forms l2's ``sum (e - q)^2`` as ``ne + nq - 2 dot``: exact for integers, so equal bits."""
    E = _int_rows(500, 33, seed=30)
    Q = _int_rows(7, 33, seed=31)
    for metric in ("cosine", "dot", "l2", "l1"):
        got = vo.exact_sims_batch(E, Q, metric)
        E64 = E.astype(np.float64)
        for b, q in enumerate(Q.astype(np.float64)):
            t = E64 - q
            v = {"cosine": (E64 @ q) / np.sqrt(np.einsum("ij,ij->i", E64, E64) * (q @ q)), "dot": E64 @ q,
                 "l2": np.einsum("ij,ij->i", t, t), "l1": np.abs(t).sum(1)}[metric]
            assert np.array_equal(got[b].view(np.uint32), np.asarray(CHAINS_ALL[metric](v), np.float32).view(np.uint32))
