"""Bit-exact NumPy restatement of ``rl_maxsim_topk`` on integer-valued corpora (TEST INFRASTRUCTURE).

When every row entry and query entry is a small integer, every float64 sum the finalize pass forms while rescoring a
survivor (``dot``, ``ne``, ``nq``, ``d2``, ``d1`` in ``exact_row_sim``) is exact, whatever order the warp adds in.
``sqrt`` and ``/`` in float64 round correctly, and the float32 steps of ``exact_sim`` are fixed, so every similarity the
device returns is a known float32 value and every hit list is a known function of the order (sim desc, row asc): sims
compare by their order-preserving bits (``f2ord``, so +0 ranks above -0), equal sims by ascending row.

``exact_sims``    the float32 sim of every row through ``exact_sim``'s chain (cosine, dot, l2, l1); ``exact_sims_batch``
                  for a batch of queries.
``sql_hits``      SQL mode (``num_hits > 0``): the ``num_hits`` best allowed rows, as ``chunk_base + row_chunk``, padded with
                  -inf / -1, and the count.
``exact_hits``    exact MaxSim mode: the same order, the first occurrence of each chunk, cut at k.
``gather_top``    ``block_gather_top`` (the streaming rescoring past 4096 survivors): which of its six digits (shifts 52,
                  40, 28, 16, 4, 0) ends the radix select over the composites ``(f2ord(sim) << 32) | ~row``.
``merge_hits``    ``rl_topk_merge`` over the shard lists: ``merge_reference`` of ``test_gpu_sharded_threads``.
"""

from __future__ import annotations

import numpy as np

ONE = np.float32(1.0)
WINDOW = 4096                       # RL_MAX_SURVIVORS: the finalize window
SEL_LIST_CAP = 8192                 # kSelListCap: select_kernel's short lists; more sample rows at the bound fall back
SHIFTS = (52, 40, 28, 16, 4, 0)     # block_gather_top's digits, 12 bits each but the last (4 bits)
EXACT_LIMIT = 2.0 ** 53


def f2ord(s) -> np.ndarray:
    """The order-preserving uint32 image of float32 ``s`` (``f2ord`` in common.cuh)."""
    u = np.asarray(s, np.float32).view(np.uint32)
    return np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000)).astype(np.uint32)


def exact_sims_batch(E: np.ndarray, Q: np.ndarray, metric: str) -> np.ndarray:
    """Float32 sim of every row for every query, ``[B, N]``, as ``exact_sim`` returns it (``select_finalize.cu``).

    The float64 sums are asserted exact: integer entries, and ``ne * nq`` and ``sum (e - q)^2`` below 2^53 (which bound
    ``|dot|`` and ``sum |e - q|`` too).  Then ``d2 = ne + nq - 2 dot`` is the kernel's ``sum (e - q)^2`` exactly, so one
    product ``E Q^T`` serves every metric but l1, whose ``sum |e - q|`` is formed per query."""
    E64 = np.asarray(E, np.float32).astype(np.float64)
    Q64 = np.atleast_2d(np.asarray(Q, np.float32)).astype(np.float64)
    assert np.all(E64 == np.round(E64)) and np.all(Q64 == np.round(Q64)), "entries must be integers"
    ne = np.einsum("ij,ij->i", E64, E64)
    nq = np.einsum("ij,ij->i", Q64, Q64)
    ne_max, nq_max = float(ne.max(initial=0.0)), float(nq.max(initial=0.0))
    assert max(ne_max * nq_max, (np.sqrt(ne_max) + np.sqrt(nq_max)) ** 2) < EXACT_LIMIT, \
        "float64 sums (or ne * nq) would round"
    dot = Q64 @ E64.T                                                # [B, N]
    with np.errstate(invalid="ignore", divide="ignore"):
        if metric == "l1":
            d1 = np.stack([np.abs(E64 - q).sum(1) for q in Q64])
            return ONE - d1.astype(np.float32)                       # 1.0f - (float)d1
        if metric == "cosine":
            s = np.fmin(1.0, np.fmax(-1.0, dot / np.sqrt(ne[None, :] * nq[:, None])))   # a NaN ratio clamps to -1
            return ONE - (ONE - s.astype(np.float32))                # dist = 1.0f - (float)s, sim = 1.0f - dist
        if metric == "dot":
            return ONE - (-dot).astype(np.float32)
        if metric == "l2":
            d2 = ne[None, :] + nq[:, None] - 2.0 * dot
            return ONE - np.sqrt(d2).astype(np.float32)
    raise ValueError(metric)


def exact_sims(E: np.ndarray, q: np.ndarray, metric: str) -> np.ndarray:
    """``exact_sims_batch`` of one query: ``[N]``."""
    return exact_sims_batch(E, np.ravel(q)[None, :], metric)[0]


def order(sims: np.ndarray, allowed: np.ndarray | None = None) -> np.ndarray:
    """Rows in the device's order, (sim desc by float bits, row asc); disallowed rows left out."""
    rows = np.arange(len(sims)) if allowed is None else np.nonzero(np.asarray(allowed, bool))[0]
    return rows[np.lexsort((rows, ~f2ord(sims[rows])))]


def sql_hits(sims, row_chunk, num_hits: int, *, allowed=None, chunk_base: int = 0):
    """SQL mode hit list: ``(sim float32 [H], chunk int64 [H], count)``."""
    o = order(sims, allowed)[:num_hits]
    s = np.full(num_hits, -np.inf, np.float32)
    c = np.full(num_hits, -1, np.int64)
    s[: len(o)], c[: len(o)] = sims[o], chunk_base + np.asarray(row_chunk, np.int64)[o]
    return s, c, len(o)


def exact_hits(sims, row_chunk, k: int, *, allowed=None, chunk_base: int = 0):
    """Exact MaxSim hit list: the first occurrence of each chunk in the device's order, the first k of them."""
    o = order(sims, allowed)
    ch = np.asarray(row_chunk, np.int64)[o]
    _, first = np.unique(ch, return_index=True)
    keep = o[np.sort(first)[:k]]
    s = np.full(k, -np.inf, np.float32)
    c = np.full(k, -1, np.int64)
    s[: len(keep)], c[: len(keep)] = sims[keep], chunk_base + np.asarray(row_chunk, np.int64)[keep]
    return s, c, len(keep)


def composites(sims: np.ndarray, rows: np.ndarray) -> np.ndarray:
    """The streaming rescoring's composite of each survivor: ``(f2ord(sim) << 32) | ~row`` (larger = better)."""
    rows = np.asarray(rows, np.int64)
    return (f2ord(sims[rows]).astype(np.uint64) << np.uint64(32)) | (~rows.astype(np.uint32)).astype(np.uint64)


def gather_top(comps: np.ndarray, K: int, window: int = WINDOW) -> tuple[int, np.ndarray]:
    """``block_gather_top`` restated: the shift of the digit that ends the loop and the composites it gathers (those
    whose top bits are at least the K-th largest's, ``window`` at most when the loop ends inside it)."""
    comps = np.asarray(comps, np.uint64)
    comps = comps[comps != 0]
    prefix, bits, need, shift = 0, 0, K, 64
    while bits < 64:
        w = min(12, 64 - bits)
        shift = 64 - bits - w
        live = comps if bits == 0 else comps[(comps >> np.uint64(64 - bits)) == np.uint64(prefix)]
        hist = np.bincount(((live >> np.uint64(shift)) & np.uint64((1 << w) - 1)).astype(np.int64), minlength=1 << w)
        above_incl = np.cumsum(hist[::-1])[::-1]          # elements in this bin and every bin above it
        if above_incl[0] < need:                          # fewer than `need` left: take everything
            bits += w
            prefix = prefix << w
            break
        b = int(np.nonzero(above_incl >= need)[0][-1])
        above = int(above_incl[b] - hist[b])
        prefix = (prefix << w) | b
        bits += w
        need -= above
        if (K - need) + int(hist[b]) <= window:
            break
    got = comps[(comps >> np.uint64(64 - bits)) >= np.uint64(prefix)]
    return shift, got


def merge_hits(sim, chunk, count, num_hits: int, k: int):
    """``rl_topk_merge`` over ``[R, B, H]`` lists -> ``(sim [B, k], chunk [B, k], count [B])`` (the restatement lives
    with the sharded-merge tests)."""
    from test_gpu_sharded_threads import merge_reference

    ids, sims, cnt = merge_reference(np.asarray(chunk), np.asarray(sim, np.float32), np.asarray(count), num_hits, k)
    return sims, ids, cnt


# ---- constructions ---------------------------------------------------------------------------------------------------
# Every one places the rows it is about (the planted rows) far above all others, so the finalize pass's survivors are
# exactly the planted rows whatever the scan's key error: which path and which digit a case reaches follows from the
# data alone (``test_vector_exact_host.py`` asserts it; the device tests assert the survivor counts).
DIGIT_D = 8
DIGIT_BASE = 2 ** 23          # dot metric, q = ones: sim = 1 + dot, adjacent integers are adjacent floats in [2^23, 2^24)


def digit_case(shift: int) -> tuple[np.ndarray, np.ndarray, int, np.ndarray]:
    """A dot-metric corpus whose streaming rescoring ends ``block_gather_top`` at digit ``shift``:
    ``(E float32 [N, 8], q float32 [8], K, planted rows)``.  Rows are ``[v, 0, ..]`` with integer v, q is all ones,
    so each row's sim is ``1 + v``.  Planted rows sit at sims 2^23 + m for a few m, one float step (one unit) apart;
    every other row has |sim| < 2^10.  Shifts 52 / 40 / 28 are decided by the sims (m = 2^20 vs 2^20 - 1, 256 vs 255,
    257 vs 256: adjacent floats that first differ in the digit's bits), 16 / 4 / 0 by the row order of one tied sim:
    3000 tied rows below 2^16 and 3000 above (16); 6000 in one 2^16-row range (4); 6000 from row 8 with K = 4096, so
    the 16-row group of the K-th holds rows on both sides of it (0)."""
    rng = np.random.default_rng(1000 + shift)
    n = 70_000 if shift == 16 else 12_000
    E = np.zeros((n, DIGIT_D), np.float32)
    E[:] = rng.integers(-60, 61, size=(n, DIGIT_D))
    K = 1000
    if shift in (52, 40, 28):
        m_hi = {52: 2 ** 20, 40: 256, 28: 257}[shift]
        planted = np.sort(rng.choice(n, size=6000, replace=False))
        vals = np.where(np.arange(6000) % 2 == 0, m_hi, m_hi - 1)
    elif shift == 16:
        planted = np.r_[np.arange(1000, 4000), np.arange(66_000, 69_000)]
        vals = np.full(6000, 256)
    elif shift == 4:
        planted = np.arange(2000, 8000)
        vals = np.full(6000, 256)
    elif shift == 0:
        planted, vals, K = np.arange(8, 6008), np.full(6000, 256), WINDOW
    else:
        raise ValueError(shift)
    E[planted] = 0
    E[planted, 0] = DIGIT_BASE + vals - 1
    return E, np.ones(DIGIT_D, np.float32), K, planted


def spanning_chunk_case(S: int) -> tuple[np.ndarray, np.ndarray, np.ndarray, tuple[int, int]]:
    """Exact MaxSim, k = 2: one chunk C of ``128 (S - 1) + 2`` near-copies of the query from row 127, so that with
    sample stride S its first row is the last row of sampled block 0 and its last row the first of sampled block S;
    every other chunk holds one random row.  ``(E float32 [8200, 64], q float32 [64], chunk_off, C's rows)``."""
    n, d = 8200, 64
    rng = np.random.default_rng(77 + S)
    E = rng.integers(-3, 4, size=(n, d)).astype(np.float32)
    E[np.abs(E).sum(1) == 0, 0] = 1
    q = rng.integers(-3, 4, size=d).astype(np.float32)
    q[0] = 3
    lo, hi = 127, 127 + 128 * (S - 1) + 2
    E[lo:hi] = q
    E[lo:hi, 1:] += rng.integers(-1, 2, size=(hi - lo, d - 1))   # sim ~ 0.9 -- 1
    off = np.r_[np.arange(0, lo + 1), np.arange(hi, n + 1)].astype(np.int64)
    return E, q, off, (lo, hi)


def tied_group_case(group: int, K: int = 100) -> tuple[np.ndarray, np.ndarray, int, tuple[int, int]]:
    """Dot metric, 12 000 random rows with entries in [-3, 3], d = 64, three queries: query 0's K-th best row and
    ``group - 1`` copies of it planted far below.  Random integer dots tie naturally too, so the tied set at query 0's
    cut is the copies plus the row's natural twins.  ``(E, Q, K, (rows above the cut, rows tied at it))`` for query 0;
    distinct dots differ by at least 1, far more than the scan's error bound, so these are the finalize survivors."""
    n, d = 12_000, 64
    rng = np.random.default_rng(group)
    E = rng.integers(-3, 4, size=(n, d)).astype(np.float32)
    Q = np.random.default_rng(group + 1).integers(-3, 4, size=(3, d)).astype(np.float32)
    Q[np.abs(Q).sum(1) == 0, 0] = 1
    o = order(exact_sims(E, Q[0], "dot"))
    src = o[K - 1]
    dst = rng.choice(o[K + group + 500:], size=group - 1, replace=False)
    E[dst] = E[src]
    sims = exact_sims(E, Q[0], "dot")
    s_cut = sims[src]
    return E, Q, K, (int((sims > s_cut).sum()), int((sims == s_cut).sum()))
