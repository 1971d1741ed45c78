"""The emission restatement (``emit_oracle``) on the CPU: block maps, ``sel_count``, R within A, and the float32
arithmetic of the online refinement's refresh edge."""

from __future__ import annotations

import emit_oracle as eo
import numpy as np
import pytest

F32 = np.float32


@pytest.mark.parametrize("S", [1, 2, 3, 4, 7, 16, 64, 255, 256])
@pytest.mark.parametrize("n_rows", [1, 127, 128, 129, 128 * 257 + 5, 128 * 1024])
def test_block_maps_cover_every_block_once(S, n_rows):
    nb = eo.n_blocks(n_rows)
    smp, main = eo.sample_blocks(n_rows, S), eo.main_blocks(n_rows, S)
    both = np.concatenate([smp, main])
    assert len(both) == nb and np.array_equal(np.sort(both), np.arange(nb))
    assert np.all(smp % S == 0) and (S == 1 or np.all(main % S != 0))
    assert np.all(np.diff(main) > 0)
    rows = eo.sample_rows(len(smp) * eo.BLOCK_ROWS, S)
    assert np.array_equal(rows, (smp[:, None] * 128 + np.arange(128)).ravel())
    cover = np.concatenate([eo.block_rows(smp, n_rows), eo.block_rows(main, n_rows)])
    assert np.array_equal(np.sort(cover), np.arange(n_rows))


def test_sel_count_both_modes():
    assert eo.sel_count(k=10, num_hits=64, max_vecs=7) == 64
    assert eo.sel_count(k=10, num_hits=0, max_vecs=3) == 28
    assert eo.sel_count(k=1, num_hits=0, max_vecs=9) == 1


def test_kth_key_counts_ties_with_multiplicity():
    keys = np.array([[5, 3, 3, 3, 1, -np.inf]], F32)
    valid = np.array([True, True, True, True, True, False])
    assert eo.kth_key(keys, valid[None, :], 2)[0] == 3 and eo.kth_key(keys, valid[None, :], 4)[0] == 3
    assert eo.kth_key(keys, valid[None, :], 5)[0] == 1
    assert eo.kth_key(keys, valid[None, :], 6)[0] == -np.inf          # fewer valid rows than sel: everything required
    v2 = valid.copy()
    v2[0] = False                                                     # a masked row does not count
    assert eo.kth_key(keys, v2[None, :], 1)[0] == 3


@pytest.mark.parametrize("seed", range(6))
def test_required_within_allowed_on_synthetic_keys(seed):
    rng = np.random.default_rng(seed)
    B, n, sel = 7, 3000, [1, 17, 200][seed % 3]
    keys = rng.normal(size=(B, n)).astype(F32)
    keys[:, ::11] = keys[:, :1]                                       # ties
    keys[:, 5::97] = (keys[:, :1] - F32(0.01) * rng.integers(0, 4, size=(B, 1))).astype(F32)
    valid = rng.random((B, n)) > 0.2
    eps = F32(10.0 ** rng.uniform(-4, -2, size=B))
    R, ks = eo.required(keys, valid, sel, eps)
    assert np.all((valid & (keys >= ks[:, None])).sum(1) >= sel)      # K_sel really is the sel-th largest
    assert np.all((valid & (keys > ks[:, None])).sum(1) < sel)
    # any threshold at or below K_sel - 2 eps -- in particular the select kernel's T - 2 eps with T <= K_sel -- allows R
    for T in (ks, np.nextafter(ks, F32(-np.inf)), ks - F32(1.0)):
        thr = (T.astype(F32) - F32(2.0) * eps).astype(F32)
        A = eo.allowed(keys, valid, thr)
        assert not np.any(R & ~A)
    # one ulp above K_sel - 2 eps drops a required row when one sits on the limit
    limit_rows = valid & (keys.astype(np.float64) == ks.astype(np.float64)[:, None] - 2.0 * eps.astype(np.float64)[:, None])
    assert eo.allowed(keys, valid, np.nextafter((ks - F32(2) * eps).astype(F32), F32(np.inf)))[limit_rows].sum() == 0


def _edge_cases(n: int, seed: int):
    """(thr0, inv_w, eps) as select_kernel makes them: w = 4 eps or wider, inv_w = 1 / w in float32."""
    rng = np.random.default_rng(seed)
    for _ in range(n):
        eps = F32(10.0 ** rng.uniform(-6.5, -1))
        thr0 = F32(rng.choice([rng.uniform(-1, 1), rng.uniform(-300, 300), -rng.uniform(0, 1e4)]))
        w = F32(F32(4) * eps) * F32(rng.choice([1.0, 1.0, rng.uniform(1, 40)]))
        yield thr0, F32(F32(1) / F32(w)), eps


def test_naive_refresh_edge_misbins_keys_one_ulp_below():
    """The float32 arithmetic of ``thr0 + best / inv_w`` can put the edge one ulp above a key that ``hist_bin`` already
    counts in bin ``best``: the count at the edge then includes a key below it, the edge can exceed K_sel, and the
    threshold ``edge - 2 eps`` can pass over a row at ``K_sel - 2 eps``.  This happens on a few percent of edges."""
    hits = total = 0
    for thr0, inv_w, _ in _edge_cases(3000, 1):
        for best in range(1, eo.HIST_BINS):
            e = eo.naive_edge(thr0, inv_w, best)
            below = np.nextafter(e, F32(-np.inf), dtype=F32)
            total += 1
            hits += int(eo.hist_bin(below, thr0, inv_w) >= best)
    assert 0.005 * total < hits < 0.2 * total, (hits, total)


def test_refresh_edge_lies_at_or_below_every_key_it_counts():
    """The refresh's edge lies at or below the least key that ``hist_bin`` counts in bin ``best`` or above (found by
    bisection), and at most a few ulps of ``g + |edge|`` below the naive edge, so the threshold it raises a query to
    never passes over a row at ``K_sel - 2 eps`` when K_sel is a counted key."""
    with np.errstate(over="ignore", invalid="ignore"):
        for thr0, inv_w, eps in _edge_cases(1500, 2):
            for best in range(1, eo.HIST_BINS):
                naive = eo.naive_edge(thr0, inv_w, best)
                e = eo.refresh_edge(thr0, inv_w, best)
                k_min = eo.least_key_in_bin(thr0, inv_w, best)
                assert e <= k_min, (thr0, inv_w, best, e, k_min)
                g = float(best) / float(inv_w)
                assert float(naive) - float(e) <= 2.0**-19 * (g + abs(float(naive))), (thr0, inv_w, best)
                t = eo.refreshed_threshold(thr0, inv_w, eps, best)
                assert float(t) <= float(k_min) - 2.0 * float(eps), (thr0, inv_w, eps, best)


def test_refresh_edge_at_large_thr0_and_edge_near_zero():
    """Edges near 0 behind a large |thr0| (dot and l2 keys): the rounding of ``key - thr0`` is an ulp of thr0, many ulps
    of the edge, and the margin scales with it."""
    with np.errstate(over="ignore", invalid="ignore"):
        for thr0 in (F32(-300.0), F32(-0.42144415), F32(-1e4), F32(-3.0)):
            for best in range(1, eo.HIST_BINS):
                inv_w = F32(F32(best) / -thr0)          # the edge of bin `best` at 0
                for iw in (inv_w, np.nextafter(inv_w, F32(0)), np.nextafter(inv_w, F32(1e9))):
                    e = eo.refresh_edge(thr0, iw, best)
                    assert e <= eo.least_key_in_bin(thr0, iw, best), (thr0, iw, best)
