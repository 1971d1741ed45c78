"""Restatements of ``split_chunklets`` and ``split_chunks`` (TEST INFRASTRUCTURE).

* ``chunklet_cuts``: the reference's chunklet dynamic program (``_split_chunklets.py:138-171``) as its loop, j
  descending with ``<=``, in Python floats (IEEE double); ``square="mul"`` is the device's d * d, ``square="pow"`` the
  reference's NumPy scalar power (C ``pow``).
* ``chunk_costs_f32``: ``_split_chunks.py:53-83`` in NumPy float32, the cost vector the reference hands to ``linprog``;
  ``linprog_cuts`` the reference's integer program on it; ``chunk_cuts`` the same windowed loop over those costs
  (``rl_chunk_partition``).
* ``chunk_costs_f64``: the cost formula in float64, with the quantities the device's error bound needs.
* ``fma64`` and ``chunk_costs_device``: ``rl_chunk_similarities`` restated lane by lane in its own float32 and float64
  order, for bit-exact checks at the C-ABI.
"""

from __future__ import annotations

import math
import re

import numpy as np
from sentences_oracle import fmaf

EPS32 = float(np.finfo(np.float32).eps)
U32 = 2.0**-24
SQRT_EPS32 = np.float32(3.4526698300124390840e-4)   # the kernel's kSqrtEps: sqrt(FLT_EPSILON) rounded to float32


def _window_dp(n: int, lens, max_size: int, cost) -> list[int]:
    pl = [0]
    for x in lens:
        pl.append(pl[-1] + int(x))
    dp = [math.inf] * (n + 1)
    dp[0] = 0.0
    back = [-1] * (n + 1)
    for i in range(1, n + 1):
        for j in range(i - 1, -1, -1):
            if pl[i] - pl[j] > max_size:
                break
            c = dp[j] + cost(j, i)
            if c <= dp[i]:
                dp[i] = c
                back[i] = j
    cuts = []
    i = back[n]
    while i > 0:
        cuts.append(i)
        i = back[i]
    return cuts[::-1]


def chunklet_cuts(p, statements, lens, max_size: int, square: str = "mul") -> list[int]:
    p = [float(x) for x in p]
    pb, ps = [0.0], [0.0]
    for k, (a, b) in enumerate(zip(p, statements, strict=True)):
        pb.append(a if k == 0 else pb[-1] + a)
        ps.append(float(b) if k == 0 else ps[-1] + float(b))

    def cost(j: int, i: int) -> float:
        s = ps[i] - ps[j]
        d = s - 3.0
        sq = d * d if square == "mul" else math.pow(d, 2.0)
        return ((1.0 - p[j]) + (pb[i] - pb[j + 1])) + sq / math.sqrt(max(s, 1e-6)) / 2.0

    return _window_dp(len(p), lens, max_size, cost)


def chunk_cuts(costs, lens, max_size: int) -> list[int]:
    c = [float(x) for x in np.asarray(costs, dtype=np.float32)]
    return _window_dp(len(lens), lens, max_size, lambda j, i: c[j - 1] if j > 0 else 0.0)


def is_heading(chunklet: str) -> bool:
    return re.match(r"^#+\s", chunklet.replace("\n", "").strip()) is not None


def nonoutlying(sizes) -> np.ndarray:
    sizes = np.asarray(sizes)
    q15, q85 = np.quantile(sizes, [0.15, 0.85])
    return (q15 <= sizes) & (sizes <= q85)


def _heading_rule(sim: np.ndarray, heading) -> np.ndarray:
    prev = True
    for i in range(len(heading) - 1):
        h = bool(heading[i])
        if h:
            if not prev:
                sim[i - 1] = sim[i - 1] / 4
            sim[i] = 1.0
        prev = h
    return sim


def chunk_costs_f32(chunklets, emb) -> np.ndarray:
    """float32 NumPy, step by step as the reference computes them."""
    return chunk_costs_f32_flags(emb, nonoutlying([len(c) for c in chunklets]), [is_heading(c) for c in chunklets])


def chunk_costs_f32_flags(emb, keep, heading) -> np.ndarray:
    """``chunk_costs_f32`` with the selected rows and the heading flags given instead of derived from the chunklets."""
    X = np.asarray(emb).astype(np.float32)
    X = X / np.linalg.norm(X, axis=1, keepdims=True)
    keep = np.asarray(keep, bool)
    if np.any(keep):
        disc = np.mean(X[keep, :], axis=0)
        disc = disc / np.linalg.norm(disc)
        Y = X - np.outer(X @ disc, disc)
        if not np.any(np.linalg.norm(Y, axis=1) <= np.finfo(np.float32).eps):
            X = Y / np.linalg.norm(Y, axis=1, keepdims=True)
    sim = np.sum(X[:-1] * X[1:], axis=1)
    sim = np.maximum((sim + 1) / 2, np.sqrt(np.finfo(np.float32).eps))
    return _heading_rule(sim, heading)


def chunk_costs_f64(emb, keep, heading) -> tuple[np.ndarray, dict]:
    """The same formula in float64 (rows, mask and heading flags given), plus what the error bound needs: whether the
    projection is kept, |mean|, and each row's projected norm."""
    X = np.asarray(emb, dtype=np.float64)
    X = X / np.linalg.norm(X, axis=1, keepdims=True)
    info = {"proj": False, "mu": 1.0, "pn": np.ones(len(X))}
    keep = np.asarray(keep, bool)
    if keep.any():
        mu = X[keep].mean(axis=0)
        info["mu"] = float(np.linalg.norm(mu))
        disc = mu / info["mu"]
        Y = X - np.outer(X @ disc, disc)
        pn = np.linalg.norm(Y, axis=1)
        info["pn_all"] = pn
        if not np.any(pn <= EPS32):
            X = Y / pn[:, None]
            info["proj"], info["pn"] = True, pn
    sim = np.maximum((np.sum(X[:-1] * X[1:], axis=1) + 1) / 2, math.sqrt(EPS32))
    prev = True
    for i in range(len(X) - 1):
        if heading[i]:
            if not prev:
                sim[i - 1] /= 4
            sim[i] = 1.0
        prev = bool(heading[i])
    return sim, info


def chunk_cost_bound(d: int, m: int, info: dict) -> np.ndarray:
    """Bound on |device cost - float64 cost| per cut, from the float32 steps of ``rl_chunk_similarities`` (u = 2^-24,
    g(k) = k u / (1 - k u), unit vectors, errors to first order, every factor rounded up):

    * row norm: a d-term sum of squares, sqrt, then one division per element: each normalised row is within
      e_x = g(d) / 2 + 2u of the exact one (2-norm, relative to 1);
    * mean of the m selected rows: e_x + g(m + 1) (the sum of m unit-norm rows has norm at most m); normalising it
      amplifies that by 2 / |mean| and adds g(d) / 2 + 2u: e_disc;
    * c = x . disc: e_x + e_disc + g(d); the projection y = x - c disc adds e_x + 2 e_disc + e_c + 2u per unit of its
      norm: e_y; dividing by |y| (itself within e_y + g(d)) gives 2 (e_y + g(d)) / |y| + u;
    * the dot of two such rows: the sum of their errors + g(d); (s + 1) / 2 halves it and adds u; the max with
      sqrt(eps), the heading rule's 1 and its division by 4 never widen it.
    Without the projection, the rows' errors are e_x."""
    g = lambda k: k * U32 / (1 - k * U32)  # noqa: E731
    e_x = g(d) / 2 + 2 * U32
    if info["proj"]:
        e_disc = 2 * (e_x + g(m + 1)) / info["mu"] + g(d) / 2 + 2 * U32
        e_c = e_x + e_disc + g(d)
        e_y = e_x + 2 * e_disc + e_c + 2 * U32
        e_row = 2 * (e_y + g(d)) / info["pn"] + U32
    else:
        e_row = np.full(len(info["pn"]), e_x)
    return 2 * ((e_row[:-1] + e_row[1:] + g(d)) / 2 + U32)   # a factor 2 for the first-order truncation


def linprog_cuts(costs, sizes, max_size: int) -> tuple[list[int], float]:
    """The reference's integer program (``_split_chunks.py:85-116``) on ``costs``: its cuts and objective."""
    from scipy.optimize import linprog
    from scipy.sparse import coo_matrix

    csum = np.cumsum(sizes)
    rows, cols = [], []
    for i in range(len(sizes) - 1):
        r = csum[i - 1] if i > 0 else 0
        idx = np.searchsorted(csum - r, max_size, side="right")
        if idx == len(csum):
            break
        cols.extend(range(i, idx))
        rows.extend([i] * (idx - i))
    A = coo_matrix((np.ones(len(rows)), (rows, cols)), shape=(max(rows) + 1, len(sizes) - 1), dtype=np.float32)
    res = linprog(costs, A_ub=-A, b_ub=-np.ones(A.shape[0], dtype=np.float32), bounds=(0, 1),
                  integrality=[1] * A.shape[1])
    assert res.success
    cuts = (np.where(res.x)[0] + 1).tolist()
    return cuts, objective(costs, cuts)


def objective(costs, cuts) -> float:
    return float(sum(float(costs[c - 1]) for c in cuts))


# ---- rl_chunk_similarities in its own order ----------------------------------------------------------------------------
def _two_sum(a, b):
    s = a + b
    bp = s - a
    return s, (a - (s - bp)) + (b - bp)


def _split(a):
    t = 134217729.0 * a                                   # 2^27 + 1
    hi = t - (t - a)
    return hi, a - hi


def fma64(a, b, c) -> np.ndarray:
    """IEEE ``fma(a, b, c)`` of float64 arrays: a b + c rounded once.

    Dekker's TwoProduct gives p + e = a b and Knuth's TwoSum s + t = p + c and v + w = t + e, all exactly; a last
    TwoSum gives r + q = s + v, so a b + c = r + q + w with r = RN(s + v).  That r is the answer except where q puts
    s + v exactly on the midpoint between r and its neighbour on q's side and w pulls the exact value past it (then
    the neighbour), and where q = 0 (then RN(r + w)).  w lies far below the distance from q to any midpoint otherwise.
    An exact zero takes IEEE's sign: -0 only for (-0) + (-0).  Exact for finite inputs when Veltkamp's split cannot
    overflow (|a|, |b| <= 2^995) and the product's error term does not underflow (|a b| >= 2^-969, or a b = 0); the
    kernels' operands are unit-scale and stay far inside that range.  Non-finite results are a b + c as NumPy gives
    them (NaN stays NaN; the kernel's NaN is compared only as NaN)."""
    a, b, c = np.broadcast_arrays(*(np.asarray(x, np.float64) for x in (a, b, c)))
    with np.errstate(over="ignore", invalid="ignore"):
        p = a * b
        ah, al = _split(a)
        bh, bl = _split(b)
        e = ((ah * bh - p) + ah * bl + al * bh) + al * bl
        s, t = _two_sum(p, c)
        v, w = _two_sum(t, e)
        r, q = _two_sum(s, v)
        nb = np.nextafter(r, np.where(q > 0, np.inf, -np.inf))
        toward = (q != 0) & (q == (nb - r) / 2) & (w != 0) & ((w > 0) == (q > 0))
        out = np.where(toward, nb, np.where(q == 0, r + w, r))
        out = np.where((r == 0) & (q == 0) & (w == 0), np.where(p == 0, p + c, 0.0), out)
        naive = p + c
    return np.where(np.isfinite(naive), out, naive)


_LANES = np.arange(32)


def _butterfly(acc: np.ndarray):
    """``warp_sum``: lane l adds lane l ^ o for o = 16 ... 1 in acc's dtype; every lane ends with lane 0's sum."""
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[..., _LANES ^ o]
    return acc[..., 0]


def _strided(dim: int, step: int):
    """The columns thread t of ``step`` threads visits at each trip of ``for (k = t; k < dim; k += step)``."""
    for k0 in range(0, dim, step):
        yield slice(k0, min(k0 + step, dim)), min(step, dim - k0)


def chunk_costs_device(X, dim: int, doc_off, nonoutlying, is_heading, fill=np.float32(np.nan)
                       ) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """``chunk_similarity_kernel`` step by step: (costs [N] float32 with ``fill`` where nothing is written, status [D],
    whether each document's costs use the projection [D]).
    ``X`` [N, ld] float16 or float32, of which the first ``dim`` columns are the rows; flags uint8 or bool.

    1. Norms: lane l of a row's warp runs ``fmaf(x, x, ss)`` over k = l, l + 32, ...; float32 butterfly; ``sqrtf``.
       A zero norm gives status 1 and nothing else for its document.  xn = fl32(x / |x|).
    2. Discourse: thread t of 256 sums (double) xn over the selected rows in row order for k = t, t + 256, ..., divides
       by m and accumulates ``fma64(mu, mu, part)``; double butterfly per warp; the 8 warp sums from 0.0 in warp order;
       ``sqrt``; disc = mu / |mu|.
    3. Projection (m > 0): per row ``c = fma64(xn, disc, c)`` per lane, butterfly; ``y = fma64(-c, disc, xn)``,
       ``ss = fma64(y, y, ss)``, butterfly, ``sqrt``; any pn <= FLT_EPSILON (in double) skips the projection.
    4. Costs: with the projection each row is fl32(fl32(xn - fl32(c_f32 disc_f32)) / pn_f32); ``fmaf`` per lane, float32
       butterfly, fl32(fl32(s + 1) * 0.5), then ``v < kSqrtEps ? kSqrtEps : v`` (NaN stays NaN).
    5. The heading rule in row order, the division by 4 a float32 division."""
    doc_off = np.asarray(doc_off, np.int64)
    D, N = len(doc_off) - 1, int(doc_off[-1])
    x = np.asarray(X)[:N, :dim].astype(np.float32)
    n = np.diff(doc_off)
    doc = np.repeat(np.arange(D), n)
    costs = np.full(N, fill, np.float32)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        acc = np.zeros((N, 32), np.float32)
        for sl, k in _strided(dim, 32):
            acc[:, :k] = fmaf(x[:, sl], x[:, sl], acc[:, :k])
        nrm = np.sqrt(_butterfly(acc))
        status = (np.bincount(doc, weights=nrm == 0, minlength=D) > 0).astype(np.int32)
        live = status == 0
        xn = x / nrm[:, None]
        xn64 = xn.astype(np.float64)

        sel = np.asarray(nonoutlying)[:N] != 0
        m = np.bincount(doc, weights=sel, minlength=D).astype(np.int64)
        mu = np.zeros((D, dim))
        for j in range(int(n.max()) if D else 0):
            d = np.nonzero(n > j)[0]
            d = d[sel[doc_off[d] + j]]
            mu[d] = mu[d] + xn64[doc_off[d] + j]
        mu = np.where(m[:, None] > 0, mu / np.maximum(m, 1)[:, None], 0.0)
        part = np.zeros((D, 256))
        for sl, k in _strided(dim, 256):
            part[:, :k] = fma64(mu[:, sl], mu[:, sl], part[:, :k])
        red = _butterfly(part.reshape(D, 8, 32))
        dn = np.zeros(D)
        for w in range(8):
            dn = dn + red[:, w]
        disc = mu / np.sqrt(dn)[:, None]

        pr = np.nonzero((m[doc] > 0) & live[doc])[0]
        dr, xp = disc[doc[pr]], xn64[pr]
        c = np.zeros((len(pr), 32))
        for sl, k in _strided(dim, 32):
            c[:, :k] = fma64(xp[:, sl], dr[:, sl], c[:, :k])
        c = _butterfly(c)
        ss = np.zeros((len(pr), 32))
        for sl, k in _strided(dim, 32):
            y = fma64(-c[:, None], dr[:, sl], xp[:, sl])
            ss[:, :k] = fma64(y, y, ss[:, :k])
        pn = np.sqrt(_butterfly(ss))
        dot, pnrm = np.zeros(N, np.float32), np.ones(N, np.float32)
        dot[pr], pnrm[pr] = c.astype(np.float32), pn.astype(np.float32)
        proj = (m > 0) & ~(np.bincount(doc[pr], weights=pn <= EPS32, minlength=D) > 0)

        i = np.nonzero(live[doc] & (np.arange(N) - doc_off[doc] < n[doc] - 1))[0]
        a, b = xn[i], xn[i + 1]
        pj = proj[doc[i]]
        dk = disc[doc[i[pj]]].astype(np.float32)
        for rows, r in ((a, i), (b, i + 1)):
            rows[pj] = (rows[pj] - dot[r[pj], None] * dk) / pnrm[r[pj], None]
        s = np.zeros((len(i), 32), np.float32)
        for sl, k in _strided(dim, 32):
            s[:, :k] = fmaf(a[:, sl], b[:, sl], s[:, :k])
        v = (_butterfly(s) + np.float32(1)) * np.float32(0.5)
        costs[i] = np.where(v < SQRT_EPS32, SQRT_EPS32, v)

    head = np.asarray(is_heading)[:N] != 0
    for d in np.nonzero(live & (np.bincount(doc, weights=head, minlength=D) > 0))[0]:
        o, prev = int(doc_off[d]), True
        for k in range(int(n[d]) - 1):
            if head[o + k]:
                if not prev:
                    costs[o + k - 1] = costs[o + k - 1] / np.float32(4)
                costs[o + k] = 1.0
            prev = head[o + k]
    return costs, status, proj & live


# the projection test's edge: (delta of the third row, whether the projection is kept) per row dtype; fp16 has no
# float32 step above eps, so its second row sits one fp16 subnormal step above it
EPS_EDGE = {np.dtype(np.float32): ((2.0**-23, False), (2.0**-23 * (1 + 2.0**-23), True)),
            np.dtype(np.float16): ((2 * 2.0**-24, False), (3 * 2.0**-24, True))}


def eps_edge_rows(delta: float, dim: int, dtype) -> np.ndarray:
    """Two selected rows (1, 1, 0, ...) and (1, -1, 0, ...), whose discourse vector is exactly e0 in float32 and float64
    alike, then an unselected row (1, delta, 0, ...), whose projected norm is exactly delta, and an unselected row
    (1, 1/2, 0, ...) for a second cut.  Select with ``EPS_EDGE_KEEP``."""
    X = np.zeros((4, dim), dtype)
    X[:, 0] = 1
    X[0, 1], X[1, 1], X[2, 1], X[3, 1] = 1, -1, delta, 0.5
    assert float(X[2, 1]) == delta
    return X


EPS_EDGE_KEEP = np.array([1, 1, 0, 0], np.uint8)
