"""The emission contract, checked row by row: every scan's candidate list against the full key dump.

Finalize rescores only the band ``[T' - 2 eps, inf)`` of the list the scan emitted, so a row the emission misses is
dropped without a trace.  ``emit_oracle`` states what the list must hold (R: every valid row with key >= K_sel - 2 eps)
and what it may hold (A: valid rows with key >= the select kernel's threshold).  Each case runs the scan twice on the
same index and queries: with ``sample_stride=1`` for the dump of every key, and with S > 1 for the emission, whose list,
count, threshold and histogram width come back through ``debug_candidates``.  Per query:

* every candidate row is valid (in range, not masked, not tombstoned) and appears once;
* its key equals the row's dump key bit for bit (both go through the same epilogue arithmetic);
* R is within the list and the list within A, or the list overflowed: ``RL_STATUS_CAND_OVERFLOW`` and ``cand_cnt > cap``;
* the search result equals the float64 similarities' top hits to the float32 rounding of a sim.

The corpora steer the tensor-core scan's online refinement through tile order (persistent CTA c walks main-pass tiles
c, c + grid, ...): the best rows in each CTA's first tiles (the threshold rises early), in its last tiles (it rises
late), all in one CTA, or across the CTAs of one lane (B > 128).  Corpora are large enough that CTAs walk more than 16
tiles, so the periodic refresh runs.  Cuts are built from ties at K_sel and from dense ladders of keys across
``[K_sel - 4 eps, K_sel + 4 eps]``; a tied block under a low threshold sends more than 1024 hits through one tile (the
direct-emit branch and the rank packing); a forced overflow is followed by the ``RL_FLAG_REUSE_THRESHOLDS`` retry; a
metadata mask with tombstones under ``RL_FLAG_COUNT_UNFILTERED`` holds ``cnt_all`` to its restated bounds.  The worst
margins per case go to ``scan_emit_margins.jsonl`` in the temporary directory.
"""

from __future__ import annotations

import json
import tempfile
import zlib
from pathlib import Path

import emit_oracle as eo
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rl():
    import torch

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import raglite_b200

    return raglite_b200


@pytest.fixture(scope="module")
def sms(rl):
    import ctypes

    from raglite_b200 import _lib

    n = ctypes.c_int(0)
    _lib.check(_lib.load().rl_device_info(ctypes.byref(n), None, None, None), "rl_device_info")
    return int(n.value)


def _record(name: str, payload: dict) -> None:
    with (Path(tempfile.gettempdir()) / "scan_emit_margins.jsonl").open("a") as f:
        f.write(json.dumps({"test": name, **payload}) + "\n")


def _unit(x):
    return x / x.norm(dim=1, keepdim=True)


# ---- tile orders ---------------------------------------------------------------------------------------------------
def _grid(n_main: int, B: int, sms: int, d: int, storage: str) -> tuple[int, int]:
    """(lanes, tiles per lane step) of the wgmma launch that holds query 0: tile t of lane L is main ordinal L + t*lanes."""
    nq = 256 if (B > 128 and storage != "fp16" and (d + 63) // 64 >= 16) else 128
    groups = min((B + nq - 1) // nq, max(1, min(sms // 2, 1024 // nq)))
    lanes = sms // groups
    return min(n_main, lanes), groups


def _order_ords(order: str, n_main: int, lanes: int, count: int) -> np.ndarray:
    """Main-pass ordinals of ``count`` tiles placed in the given order."""
    tiles = -(-n_main // lanes)          # tiles of the longest lanes
    if order == "early":                 # the first tile of each lane, then the second, ...
        o = np.arange(count)
    elif order == "late":                # the last tile of each lane
        last = np.array([L + ((n_main - 1 - L) // lanes) * lanes for L in range(lanes)])
        o = np.concatenate([last, last - lanes, last - 2 * lanes])[:count]
    elif order == "one_cta":             # every tile of lane 3, from its last one down
        o = (3 + np.arange(tiles) * lanes)[::-1]
        o = o[o < n_main][:count]
    elif order == "lane":                # lane 0's tiles, spread over its whole walk
        o = (np.arange(tiles) * lanes)
        o = o[o < n_main][np.linspace(0, min(tiles, n_main // lanes) - 1, count).astype(int)]
    else:
        raise AssertionError(order)
    assert len(o) == count and len(np.unique(o)) == count and np.all(o < n_main)
    return o.astype(np.int64)


# ---- cases ---------------------------------------------------------------------------------------------------------
# name: (metric, storage, algo, d, n_rows, B, S, num_hits, k, vecs, order, plant, extra)
N_BIG = 128 * 132 * 96 + 37    # 96 tiles per CTA at B <= 128: the periodic refresh runs six times
CASES = {
    "nq128_cos_early": ("cosine", "fp32", "tcgen05", 64, N_BIG, 17, 16, 64, 10, 1, "early", "near", ""),
    "nq128_cos_late": ("cosine", "fp32", "tcgen05", 64, N_BIG, 17, 16, 64, 10, 1, "late", "near", ""),
    "nq128_cos_one_cta": ("cosine", "fp32", "tcgen05", 64, N_BIG, 1, 16, 32, 10, 1, "one_cta", "near", ""),
    "nq128_cos_lane_b300": ("cosine", "fp32", "tcgen05", 64, 128 * 3000 + 3, 300, 4, 32, 10, 1, "lane", "near", "rpq16"),
    "nq128_cos_ties_b129": ("cosine", "fp32", "tcgen05", 128, 128 * 1300, 129, 8, 64, 10, 1, "early", "ties", ""),
    "nq128_cos_ladder": ("cosine", "fp32", "tcgen05", 64, 128 * 2600 + 37, 17, 16, 80, 10, 1, "late", "ladder", ""),
    "nq128_cos_burst": ("cosine", "fp32", "tcgen05", 64, 128 * 2600, 17, 16, 64, 10, 1, "early", "burst", ""),
    "nq128_cos_scaled_rows": ("cosine", "fp32", "tcgen05", 64, 128 * 4400 + 9, 17, 2, 64, 10, 1, "late", "near", "norm03"),
    "nq128_dot_b1": ("dot", "fp32", "tcgen05", 128, 128 * 2600, 1, 16, 64, 10, 1, "late", "near", ""),
    "nq128_l2_b129": ("l2", "fp32", "tcgen05", 64, 128 * 1500 + 100, 129, 4, 64, 10, 1, "late", "ladder", ""),
    "nq128_b1100": ("cosine", "fp32", "tcgen05", 64, 128 * 500 + 1, 1100, 4, 16, 10, 1, "early", "near", ""),
    "nq256_cos_b300": ("cosine", "fp32", "tcgen05", 1024, 128 * 1400, 300, 16, 64, 10, 1, "early", "near", ""),
    "nq256_l2_b256_ladder": ("l2", "fp32", "tcgen05", 1024, 128 * 2300 + 77, 256, 0, 64, 10, 1, "late", "ladder", ""),
    "fp16_cos_b129": ("cosine", "fp16", "tcgen05", 128, 128 * 2200 + 5, 129, 16, 64, 10, 1, "late", "ladder", ""),
    "fp16_dot_b17_ties": ("dot", "fp16", "tcgen05", 64, 128 * 2600, 17, 0, 64, 10, 1, "early", "ties", ""),
    "maxsim_cos_s4": ("cosine", "fp32", "tcgen05", 64, 3 * 128 * 1000, 17, 4, 0, 10, 3, "late", "near", ""),
    "maxsim_fp16_ladder": ("cosine", "fp16", "tcgen05", 64, 3 * 128 * 900, 17, 16, 0, 10, 3, "early", "ladder", ""),
    "fp32scan_dot_s4": ("dot", "fp32", "fp32", 64, 128 * 400 + 11, 17, 4, 64, 10, 1, "late", "ladder", ""),
    "fp32scan_cos_maxsim": ("cosine", "fp32", "fp32", 48, 3 * 128 * 200, 129, 2, 0, 10, 3, "early", "ties", ""),
    "l1_fp32": ("l1", "fp32", "fp32", 64, 128 * 400 + 7, 17, 4, 64, 10, 1, "late", "near", ""),
    "l1_fp16_maxsim": ("l1", "fp16", "fp32", 64, 3 * 128 * 200, 17, 16, 0, 10, 3, "early", "ties", ""),
}


def _make(rl, name: str, sms: int):
    """(index, Q, planted tile ordinals, planted rows) for a case; everything seeded."""
    import torch

    metric, storage, algo, d, n, B, S, num_hits, k, vecs, order, plant, extra = CASES[name]
    seed = zlib.crc32(name.encode()) % (1 << 30)
    g = torch.Generator(device="cuda").manual_seed(seed)
    Q = _unit(torch.randn((B, d), generator=g, device="cuda"))
    E = _unit(torch.randn((n, d), generator=g, device="cuda"))
    if metric in ("dot", "l2", "l1"):
        E *= 1.0 + 0.5 * torch.rand((n, 1), generator=g, device="cuda")
    S_eff = S if S > 0 else eo.auto_stride(n, k=k, num_hits=num_hits, max_vecs=vecs)
    main = eo.main_blocks(n, S_eff)
    lanes, _ = _grid(len(main), B, sms, d, storage)
    sel = eo.sel_count(k=k, num_hits=num_hits, max_vecs=vecs)
    rpq = {"near": 16 if extra == "rpq16" else 2 * sel, "ties": 3 * sel, "ladder": 2 * sel, "burst": 0}[plant]
    n_tiles = max(1, -(-B * rpq // 128))
    ords = _order_ords(order, len(main), lanes, n_tiles)
    rows = torch.from_numpy(eo.block_rows(main[ords], n)).cuda()
    if plant != "burst":
        rows = rows[: B * rpq]
    qb = torch.arange(len(rows), device="cuda") // max(rpq, 1)    # the query each planted row belongs to
    j = (torch.arange(len(rows), device="cuda") % max(rpq, 1)).double()
    noise = _unit(torch.randn((len(rows), d), generator=g, device="cuda"))
    if plant == "near":          # near-duplicates of the query, cosine ~0.89
        E[rows] = E[rows].norm(dim=1, keepdim=True) * _unit(Q[qb] + 0.5 * noise)
    elif plant == "ties":        # 3 sel bitwise-identical rows per query
        E[rows] = _unit(Q + 0.5 * _unit(torch.randn((B, d), generator=g, device="cuda")))[qb]
    elif plant == "ladder":      # per query, unit rows whose cosines step evenly over ~8 eps around the sel-th
        q = Q[qb]
        u = _unit(noise - (noise * q).sum(1, keepdim=True) * q)
        eps_est = (1.25e-3 if algo == "tcgen05" else 0.0) + (d + 8) * 1.2e-7
        c = 0.9 + (j - rpq / 2) * (8 * eps_est / rpq)
        E[rows] = (c[:, None] * q.double() + (1 - c * c).sqrt()[:, None] * u.double()).float()
    elif plant == "burst":       # one tile of rows near every query: the queries share a direction
        v = _unit(torch.randn((1, d), generator=g, device="cuda"))
        Q = _unit(v + 0.25 * _unit(torch.randn((B, d), generator=g, device="cuda")))
        E[rows] = v + 1e-3 * noise
    if extra == "norm03":        # one row of norm 0.3: the cosine loader scales rows itself
        E[n // 2] *= 0.3
    if storage == "fp16":
        E = E.half()
    kw = {"vecs_per_chunk": vecs} if vecs > 1 else {}
    idx = rl.CorpusIndex(E.contiguous(), storage=storage, **kw)
    return idx, Q.contiguous(), ords, rows


def _exact_sims(E, Q, metric: str):
    """Float64 similarity of every (query, row) as finalize computes it before its float32 rounding."""
    import torch

    Ed, Qd = E.double(), Q.double()
    if metric == "l1":
        return 1.0 - torch.cdist(Qd, Ed, p=1)
    G = Qd @ Ed.T
    if metric == "dot":
        return 1.0 + G
    ne2 = (Ed * Ed).sum(1)
    if metric == "l2":
        d2 = (ne2[None, :] + (Qd * Qd).sum(1)[:, None] - 2.0 * G).clamp(min=0)
        return 1.0 - d2.sqrt()
    return (G / (ne2.sqrt()[None, :] * Qd.norm(dim=1)[:, None])).clamp(-1, 1)


def _check_result(res, E, Q, metric: str, valid, row_chunk, num_hits: int, k: int, rows_ok) -> None:
    """The hit list against the float64 sims: the sorted sims agree to a float32 rounding and every returned chunk's
    exact similarity is the sim reported for it."""
    import torch

    sims = _exact_sims(E, Q, metric)
    sims = torch.where(valid, sims, torch.full_like(sims, -float("inf")))
    if num_hits > 0:
        want = sims.topk(num_hits, dim=1).values
        got = res.hit_sim.double()
    else:
        n_chunks = int(row_chunk.max()) + 1
        ch = torch.full((sims.shape[0], n_chunks), -float("inf"), dtype=torch.float64, device=sims.device)
        ch.scatter_reduce_(1, row_chunk[None, :].expand_as(sims), sims, reduce="amax")
        want = ch.topk(k, dim=1).values
        got = res.hit_sim.double()
        sims = ch
    ok = torch.from_numpy(rows_ok).cuda()
    tol = 2.0**-22 * want.abs().clamp(min=1.0)
    fin = torch.isfinite(want)
    diff = torch.where(fin, (got - want).abs(), torch.zeros_like(want))
    assert bool(torch.all(torch.isfinite(got) == fin)), "hit counts differ"
    assert bool(torch.all(diff[ok] <= tol[ok])), ("sims", float(diff[ok].max()))
    own = sims.gather(1, res.hit_chunk.clamp(min=0))      # one vector per chunk in SQL cases: chunk == row
    d2 = torch.where(fin, (own - got).abs(), torch.zeros_like(got))
    assert bool(torch.all(d2[ok] <= tol[ok])), ("chunk sims", float(d2[ok].max()))


def _host(t):
    return t.cpu().numpy()


def _emission(idx, Q, kw: dict, S: int, *, valid_np, keys, eps, sel, name, flags=0, cand_cap=0, row_allowed=None,
              expect_overflow=None):
    """One emission run and every per-query check; returns (result, candidates, stats, R, A, C, K_sel, overflowed)."""
    import torch

    from raglite_b200 import _lib

    res = idx.scan(Q, **kw, sample_stride=S, flags=flags, cand_cap=cand_cap, row_allowed=row_allowed)
    st = idx.scan_stats()
    cd = {key: _host(v) for key, v in idx.debug_candidates().items()}
    status = _host(res.status)
    torch.cuda.synchronize()
    B, n = keys.shape
    cap = st["cand_cap"]
    assert st["sample_stride"] > 1, (name, st)
    R, ksel = eo.required(keys, valid_np, sel, eps)
    A = eo.allowed(keys, valid_np, cd["thr"])
    assert not np.any(R & ~A), (name, "select threshold above K_sel - 2 eps", np.nonzero((R & ~A).any(1))[0][:8])
    cnt = cd["cand_cnt"]
    over = (status & _lib.RL_STATUS_CAND_OVERFLOW) != 0
    assert np.array_equal(over, cnt > cap), (name, "overflow flag", np.nonzero(over != (cnt > cap))[0][:8])
    if expect_overflow is not None:
        assert bool(over.any()) == expect_overflow, (name, "overflow", int(over.sum()), int(cnt.max()), cap)
    C = np.zeros((B, n), bool)
    for b in range(B):
        m = min(int(cnt[b]), cap)
        r = cd["row"][b, :m]
        assert np.all((r >= 0) & (r < n)), (name, b, "row out of range")
        assert len(np.unique(r)) == m, (name, b, "duplicate rows", m - len(np.unique(r)))
        bad = ~valid_np[b, r]
        assert not bad.any(), (name, b, "masked, tombstoned or padding rows", r[bad][:8])
        kb = cd["key"][b, :m].view(np.uint32)
        want = keys[b, r].view(np.uint32)
        assert np.array_equal(kb, want), (name, b, "key bits", r[kb != want][:8], cd["key"][b, :m][kb != want][:4],
                                          keys[b, r][kb != want][:4])
        C[b, r] = True
    missing = R & ~C & ~over[:, None]
    if missing.any():
        b = int(np.nonzero(missing.any(1))[0][0])
        r = np.nonzero(missing[b])[0]
        lim = float(ksel[b]) - 2.0 * float(eps[b])
        raise AssertionError((name, "required rows missing", "query", b, "rows", r[:8].tolist(), "tiles",
                              (r[:8] // 128).tolist(), "keys", keys[b, r[:8]].tolist(), "K_sel", float(ksel[b]),
                              "limit", lim, "thr", float(cd["thr"][b])))
    assert not np.any(C & ~A), (name, "candidates below the select threshold")
    return res, cd, st, R, A, C, ksel, over


@pytest.mark.parametrize("name", list(CASES))
def test_emission_holds_required_rows(rl, sms, name):
    import torch

    metric, storage, algo, d, n, B, S, num_hits, k, vecs, order, plant, extra = CASES[name]
    idx, Q, ords, _ = _make(rl, name, sms)
    kw = dict(k=k, num_hits=num_hits, metric=metric, algo=algo)
    idx.scan(Q, **kw, sample_stride=1)
    keys = _host(idx.debug_dump()[:, :n])
    eps = _host(idx.debug_eps())
    valid = np.isfinite(keys)
    assert valid.all()
    sel = eo.sel_count(k=k, num_hits=num_hits, max_vecs=vecs)
    res, cd, st, R, A, C, ksel, over = _emission(idx, Q, kw, S, valid_np=valid, keys=keys, eps=eps, sel=sel, name=name)
    assert st["sample_stride"] == (S or eo.auto_stride(n, k=k, num_hits=num_hits, max_vecs=vecs))
    assert not over.any(), (name, "unexpected overflow")
    _check_result(res, idx.E.float(), Q, metric, torch.from_numpy(valid).cuda(), idx.row_chunk.long(), num_hits, k,
                  np.ones(B, bool))
    lim = ksel.astype(np.float64) - 2.0 * eps
    margin = np.where(R, (keys - lim[:, None]) / eps[:, None], np.inf).min()
    n_a, n_c = A.sum(1), C.sum(1)
    S_eff = st["sample_stride"]
    main = eo.main_blocks(n, S_eff)
    n_main_tiles = len(main)
    lanes, _ = _grid(n_main_tiles, B, sms, d, storage)
    _record(name, {"S": S_eff, "B": B, "n_rows": n, "cap": st["cand_cap"], "min_required_margin_eps": float(margin),
                   "cand_over_allowed": float(n_c.sum() / max(1, n_a.sum())), "required": int(R.sum()),
                   "candidates": int(n_c.sum()), "allowed": int(n_a.sum()),
                   "unrequired_cut": float((n_a.sum() - n_c.sum()) / max(1, n_a.sum() - R.sum())), "tiles_per_lane": n_main_tiles / lanes})
    # what each case exists for
    if algo == "tcgen05":
        assert n_main_tiles / lanes > 16, (name, "the periodic refresh needs > 16 tiles per CTA")
    if plant == "ladder":        # keys dense across the cut: a required row within an eps of the limit
        assert margin < 1.0, (name, margin)
    if plant == "ties":
        assert np.all((keys == ksel[:, None]).sum(1) >= 2), (name, "no tie at K_sel")
    if plant == "burst":         # the burst tile is tile 0 of its CTA: every key >= thr there is a hit of that tile
        blk_rows = eo.block_rows(main[ords[:1]], n)
        hits = int(A[:, blk_rows].sum())
        assert hits > 1024, (name, "hits in the burst tile", hits)
    if name == "nq128_cos_one_cta":
        # all best rows in one lane: no CTA stages 192 hits before its last tile, so no flush feeds the global histogram,
        # the threshold stays the select kernel's and every allowed row is emitted (by the end-of-scan flushes)
        assert n_c.sum() == n_a.sum(), (name, int(n_c.sum()), int(n_a.sum()))
    if name == "nq128_cos_late":
        # best rows in every lane's last tile: flushes come only at the end, so the threshold rises too late to keep
        # out more than a few allowed rows
        assert n_c.sum() >= 0.95 * n_a.sum(), (name, int(n_c.sum()), int(n_a.sum()))
    if order == "lane":          # the lane's CTAs flush and refresh: some allowed rows outside R were never emitted
        assert (n_a.sum() - n_c.sum()) / max(1, n_a.sum() - R.sum()) > 0.1, (name, int(n_c.sum()), int(n_a.sum()))
    if algo == "tcgen05" and order == "early" and plant == "near":
        # the threshold rose while the scan ran: a good share of the allowed rows that are not required was never emitted
        cut = (n_a.sum() - n_c.sum()) / max(1, n_a.sum() - R.sum())
        assert cut > 0.2, (name, "the refinement did not tighten the threshold", int(n_c.sum()), int(n_a.sum()), int(R.sum()))


def test_overflow_then_reused_threshold_retry(rl, sms):
    """A forced overflow (cand_cap = 256) on the float32 scan, which never refines, then the retry with the thresholds
    finalize wrote: the overflowing list is still within A, and the retry's list satisfies the whole contract."""
    import torch

    from raglite_b200 import _lib

    n, d, B = 128 * 800 + 3, 64, 17
    g = torch.Generator(device="cuda").manual_seed(99)
    Q = _unit(torch.randn((B, d), generator=g, device="cuda"))
    E = _unit(torch.randn((n, d), generator=g, device="cuda"))
    idx = rl.CorpusIndex(E.contiguous())
    kw = dict(k=10, num_hits=64, metric="cosine", algo="fp32")
    idx.scan(Q, **kw, sample_stride=1)
    keys, eps = _host(idx.debug_dump()[:, :n]), _host(idx.debug_eps())
    valid = np.isfinite(keys)
    first = _emission(idx, Q, kw, 16, valid_np=valid, keys=keys, eps=eps, sel=64, name="overflow", cand_cap=256,
                      expect_overflow=True)
    retry = _emission(idx, Q, kw, 16, valid_np=valid, keys=keys, eps=eps, sel=64, name="retry", cand_cap=256,
                      flags=_lib.RL_FLAG_REUSE_THRESHOLDS)
    assert np.all(retry[1]["thr"] >= first[1]["thr"]), "the retry did not start from the tighter thresholds"
    assert np.any(retry[1]["thr"] > first[1]["thr"])
    ok = ~retry[7]
    assert ok.any()
    _check_result(retry[0], idx.E, Q, "cosine", torch.from_numpy(valid).cuda(), idx.row_chunk.long(), 64, 10, ok)
    _record("overflow_retry", {"first_cnt_max": int(first[1]["cand_cnt"].max()), "retry_overflowed": int((~ok).sum()),
                               "retry_cnt_max": int(retry[1]["cand_cnt"].max())})


@pytest.mark.parametrize("metric", ["cosine", "l2", "l1"])
def test_unfiltered_counter_within_bounds(rl, sms, metric):
    """A metadata mask with tombstones under RL_FLAG_COUNT_UNFILTERED.  Allowed rows near each query fill the first
    sample blocks, so the select kernel's threshold already lies near the cut; masked rows from the same distribution
    come in the last tiles.  For cosine they have norm 0.55: the scan keys them without scaling rows in the loader, and
    their key without the 1/|e| lies far under the threshold while their key does not.  ``cnt_all`` must lie within
    its restated bounds, and the unfiltered bound must cover every live row at least as near as the worst filtered
    hit."""
    import torch

    n, d, B, S, H = 128 * 2600 + 37, 64, 17, 16, 32
    g = torch.Generator(device="cuda").manual_seed(7 + len(metric))
    Q = _unit(torch.randn((B, d), generator=g, device="cuda"))
    E = _unit(torch.randn((n, d), generator=g, device="cuda"))
    main = eo.main_blocks(n, S)
    lanes, _ = _grid(len(main), B, sms, d, "fp32")
    near_ok = torch.from_numpy(eo.block_rows(eo.sample_blocks(n, S), n)[: 2 * H * B]).cuda()
    near_masked = torch.from_numpy(eo.block_rows(main[_order_ords("late", len(main), lanes, 40)], n)).cuda()
    m_scale = 0.55 if metric == "cosine" else 1.0
    for rows, scale in ((near_ok, 1.0), (near_masked, m_scale)):
        qb = torch.arange(len(rows), device="cuda") % B
        E[rows] = scale * _unit(Q[qb] + 0.5 * _unit(torch.randn((len(rows), d), generator=g, device="cuda")))
    allowed = (torch.rand(n, generator=g, device="cuda") < 0.5).to(torch.uint8)
    allowed[near_ok] = 1
    allowed[near_masked] = 0
    ids = [f"c{i}" for i in range(n)]
    algo = "fp32" if metric == "l1" else "tcgen05"
    idx = rl.CorpusIndex(E.contiguous(), chunk_ids=ids)
    dead = np.arange(11, n, 89)
    idx.delete_chunks([ids[i] for i in dead])
    kw = dict(k=10, num_hits=H, metric=metric, algo=algo)
    idx.scan(Q, **kw, sample_stride=1)                       # tombstones only: the key of every live row
    keys, eps = _host(idx.debug_dump()[:, :n]), _host(idx.debug_eps())
    alive = np.ones(n, bool)
    alive[dead] = False
    allowed_np = _host(allowed).astype(bool)
    valid = np.isfinite(keys) & allowed_np[None, :]
    assert np.array_equal(np.isfinite(keys[0]), alive)
    from raglite_b200 import _lib

    res, cd, st, R, A, C, ksel, over = _emission(idx, Q, kw, S, valid_np=valid, keys=keys, eps=eps, sel=H,
                                                 name=f"unfiltered_{metric}", flags=_lib.RL_FLAG_COUNT_UNFILTERED,
                                                 row_allowed=allowed)
    assert not over.any()
    bound = _host(idx.unfiltered_bound())
    cnt_all = bound - cd["cand_cnt"] - st["n_sample_rows"]
    main_mask = np.zeros(n, bool)
    main_mask[eo.block_rows(main, n)] = True
    lo, hi = eo.cnt_all_bounds(keys, alive & ~allowed_np, main_mask, ksel, eps, cd["thr"])
    assert np.all(lo > 0), "no masked row reaches the cut: the case does not test the counter"
    if metric == "cosine":   # rows a count against the key without 1/|e| would miss
        mrows = _host(near_masked)
        km = keys[:, mrows]
        assert np.all(((km >= cd["thr"][:, None]) & (km * m_scale < cd["thr"][:, None])).sum(1) > 0)
    assert np.all((lo <= cnt_all) & (cnt_all <= hi)), (metric, lo.tolist(), cnt_all.tolist(), hi.tolist())
    sims = _exact_sims(idx.E, Q, metric)
    worst = res.hit_sim.double()[:, H - 1]
    live = torch.from_numpy(alive).cuda()
    near = ((sims >= (worst + 2.0**-20 * worst.abs().clamp(min=1.0))[:, None]) & live[None, :]).sum(1)
    assert bool(torch.all(near.cpu() <= torch.from_numpy(bound))), (near.tolist(), bound.tolist())
    _check_result(res, idx.E, Q, metric, torch.from_numpy(valid).cuda(), idx.row_chunk.long(), H, 10, np.ones(B, bool))
    _record(f"unfiltered_{metric}", {"cnt_all": cnt_all.tolist(), "lo": lo.tolist(), "hi": hi.tolist()})


# ---- keys planted at the refresh edge and at the sample's statistic --------------------------------------------------
def _at_cos(q, c, g, d: int):
    """Unit rows whose cosine to the unit query q is c (one row per entry of c)."""
    import torch

    u = torch.randn((len(c), d), generator=g, device="cuda", dtype=torch.float64)
    qd = q.double()[None, :]
    u = u - (u * qd).sum(1, keepdim=True) * qd
    u = u / u.norm(dim=1, keepdim=True)
    c = torch.as_tensor(c, dtype=torch.float64, device="cuda")[:, None]
    return (c * qd + (1 - c * c).sqrt() * u).float()


@pytest.mark.parametrize("kind", ["edge_sql", "edge_maxsim", "sample_stat"])
def test_planted_cut_at_refresh_edge_and_sample_statistic(rl, sms, kind):
    """Keys placed where the threshold arithmetic decides, B = 1, cosine, S = 16.

    The sample blocks hold ``sel_k`` identical rows at cosine c0, so the select kernel's statistic T sits on c0, its
    threshold is thr0 = T - 2 eps and the histogram's bins are 4 eps wide (the sample's tail has no spread).  ``thr0``
    and ``hist_inv_w`` are read back from a first scan; the sample is the same in the scan under test, so they are too.
    Candidate rows are keyed once in a calibration index (dump), and each one is then placed by its key.

    ``edge_*``: 200 rows far above (bin 15) in tiles 0 and 1 of lane 0, plus X in bin 6 just above its edge, make X the
    ``sel_count``-th key K_sel; tile 1 flushes (more than 192 staged hits) and the refresh raises the threshold to
    edge_6 - 2 eps.  Required rows Y under edge_6 but above K_sel - 2 eps come in lane 0's later tiles, together with
    decoys Z under edge_6 - 2 eps that the raised threshold must keep out.  ``edge_maxsim`` is the same in exact MaxSim
    mode with two vectors per chunk (``sel_count`` = 201 vectors for k = 101 chunks).

    ``sample_stat``: nothing lies above the sample's tie, so K_sel = c0, and required rows Y between c0 - 2 eps and
    T - eps come in the main pass: they need the select kernel's full 2 eps guard."""
    import torch

    d, S, n, j = 64, 16, 128 * 1600, 6
    maxsim = kind == "edge_maxsim"
    vecs = 2 if maxsim else 1
    k, num_hits = (101, 0) if maxsim else (10, 201)
    sel = eo.sel_count(k=k, num_hits=num_hits, max_vecs=vecs)
    assert sel == 201
    kw = dict(k=k, num_hits=num_hits, metric="cosine", algo="tcgen05")
    ikw = {"vecs_per_chunk": vecs} if maxsim else {}
    g = torch.Generator(device="cuda").manual_seed(4242 + len(kind))
    q = _unit(torch.randn((1, d), generator=g, device="cuda"))
    Q = q.contiguous()
    E0 = _unit(torch.randn((n, d), generator=g, device="cuda"))
    c0 = 0.7
    smp_rows = torch.from_numpy(eo.block_rows(eo.sample_blocks(n, S), n)[:sel]).cuda()
    E0[smp_rows] = _at_cos(q[0], [c0], g, d).expand(sel, d)       # one vector: bitwise-tied sample keys
    main = eo.main_blocks(n, S)
    lanes, _ = _grid(len(main), 1, sms, d, "fp32")
    lane0 = [eo.block_rows(main[[t * lanes]], n) for t in range(8)]   # lane 0's tiles 0..7
    scratch = eo.block_rows(main[[lanes // 2 + t * lanes for t in range(4)]], n)   # another lane: calibration only

    def run(E, S_run):
        idx = rl.CorpusIndex(E.contiguous(), **ikw)
        res = idx.scan(Q, **kw, sample_stride=S_run)
        return idx, res

    # 1) the select kernel's threshold and bin width (the main pass does not change them)
    idx, _ = run(E0, S)
    cd = idx.debug_candidates()
    thr0, inv_w, eps = float(cd["thr"][0]), float(cd["hist_inv_w"][0]), float(idx.debug_eps()[0])
    assert abs(1.0 / inv_w - 4 * eps) < 1e-3 * eps, "the sample tail should leave the bins 4 eps wide"
    T = thr0 + 2 * eps
    edge = thr0 + j / inv_w
    # 2) calibration: a fine ladder of candidate rows in another lane's tiles, keyed by a dump
    lo_c, hi_c = (edge - 4 * eps, edge + 2 * eps) if kind != "sample_stat" else (c0 - 3 * eps, c0)
    ladder = _at_cos(q[0], np.linspace(lo_c, hi_c, len(scratch)), g, d)
    E1 = E0.clone()
    sc_t = torch.from_numpy(scratch).cuda()
    E1[sc_t] = ladder
    idx, _ = run(E1, 1)
    lk = _host(idx.debug_dump()[0, torch.from_numpy(scratch).cuda()]).astype(np.float64)

    def pick(lo, hi, m):
        i = np.nonzero((lk >= lo) & (lk <= hi))[0]
        assert len(i) >= m, (kind, "no ladder keys in", lo, hi, len(i))
        return ladder[torch.from_numpy(i[np.linspace(0, len(i) - 1, m).astype(int)]).cuda()]

    E = E0.clone()
    if kind == "sample_stat":
        ks = c0                                               # K_sel: the tie
        Y = pick(ks - 1.9 * eps, T - 1.1 * eps, 16)           # required, below T - eps
        E[torch.from_numpy(lane0[3][:16]).cuda()] = Y
    else:
        hi_rows = _at_cos(q[0], np.full(200, 0.95), g, d)
        E[torch.from_numpy(np.concatenate([lane0[0][:100], lane0[1][:100]])).cuda()] = hi_rows
        X = pick(edge + 0.3 * eps, edge + 0.6 * eps, 1)
        E[int(lane0[1][100])] = X[0]
        Y = pick(edge - 1.35 * eps, edge - 0.3 * eps, 16)     # required (>= K_sel - 2 eps) and under the edge
        Zd = pick(edge - 4 * eps, edge - 2.6 * eps, 16)       # allowed (>= thr0) but under edge - 2 eps
        E[torch.from_numpy(lane0[3][:32:2]).cuda()] = Y       # every other row: chunks of two hold one planted row
        E[torch.from_numpy(lane0[5][:32:2]).cuda()] = Zd
    # 3) the scan under test against its own dump
    idx, _ = run(E, 1)
    keys, eps_a = _host(idx.debug_dump()[:, :n]), _host(idx.debug_eps())
    valid = np.isfinite(keys)
    res, cd, st, R, A, C, ksel, over = _emission(idx, Q, kw, S, valid_np=valid, keys=keys, eps=eps_a, sel=sel, name=kind)
    assert not over.any()
    assert float(cd["thr"][0]) == np.float32(thr0) and float(cd["hist_inv_w"][0]) == np.float32(inv_w)
    _check_result(res, idx.E, Q, "cosine", torch.from_numpy(valid).cuda(), idx.row_chunk.long(), num_hits, k, np.ones(1, bool))
    y_rows = lane0[3][:16] if kind == "sample_stat" else lane0[3][:32:2]
    ky = keys[0, y_rows].astype(np.float64)
    lim = float(ksel[0]) - 2.0 * float(eps_a[0])
    assert np.all(R[0, y_rows]), (kind, "planted rows are not required")
    if kind == "sample_stat":                                 # the case exists for rows a T - eps threshold would drop
        assert float(ksel[0]) == np.float32(_host(idx.debug_dump()[0, smp_rows[:1]])[0])
        assert np.all(ky < T - eps), (kind, ky.max(), T - eps)
    else:
        x_row = int(lane0[1][100])
        assert keys[0, x_row] == ksel[0], (kind, "X is not K_sel")
        assert int(eo.hist_bin(keys[0, x_row], np.float32(thr0), np.float32(inv_w))) == j
        assert np.all(ky < edge) and np.all(ky >= lim)        # dropped by a threshold of edge, or of edge_{j+1} - 2 eps
        z_rows = lane0[5][:32:2]
        assert np.all(A[0, z_rows]) and not np.any(C[0, z_rows]), (kind, "the refresh did not raise the threshold")
    _record(f"planted_{kind}", {"thr0": thr0, "inv_w": inv_w, "eps": eps, "K_sel": float(ksel[0]),
                                "required_margin_eps": float((ky.min() - lim) / eps),
                                "candidates": int(C.sum()), "allowed": int(A.sum())})
