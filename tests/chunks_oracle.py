"""Restatements of ``split_chunklets`` and ``split_chunks`` (TEST INFRASTRUCTURE).

* ``chunklet_cuts``: the reference's chunklet dynamic program (``_split_chunklets.py:138-171``) as its loop, j
  descending with ``<=``, in Python floats (IEEE double); ``square="mul"`` is the device's d * d, ``square="pow"`` the
  reference's NumPy scalar power (C ``pow``).
* ``chunk_costs_f32``: ``_split_chunks.py:53-83`` in NumPy float32, the cost vector the reference hands to ``linprog``;
  ``linprog_cuts`` the reference's integer program on it; ``chunk_cuts`` the same windowed loop over those costs
  (``rl_chunk_partition``).
* ``chunk_costs_f64``: the cost formula in float64, with the quantities the device's error bound needs.
"""

from __future__ import annotations

import math
import re

import numpy as np

EPS32 = float(np.finfo(np.float32).eps)
U32 = 2.0**-24


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


def _heading_rule(sim: np.ndarray, chunklets) -> np.ndarray:
    prev = True
    for i in range(len(chunklets) - 1):
        h = is_heading(chunklets[i])
        if h:
            if not prev:
                sim[i - 1] = sim[i - 1] / 4
            sim[i] = 1.0
        prev = h
    return sim


def chunk_costs_f32(chunklets, emb) -> np.ndarray:
    """float32 NumPy, step by step as the reference computes them."""
    X = np.asarray(emb).astype(np.float32)
    X = X / np.linalg.norm(X, axis=1, keepdims=True)
    keep = nonoutlying([len(c) for c in chunklets])
    if np.any(keep):
        disc = np.mean(X[keep, :], axis=0)
        disc = disc / np.linalg.norm(disc)
        Y = X - np.outer(X @ disc, disc)
        if not np.any(np.linalg.norm(Y, axis=1) <= np.finfo(np.float32).eps):
            X = Y / np.linalg.norm(Y, axis=1, keepdims=True)
    sim = np.sum(X[:-1] * X[1:], axis=1)
    sim = np.maximum((sim + 1) / 2, np.sqrt(np.finfo(np.float32).eps))
    return _heading_rule(sim, chunklets)


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
