"""Returned similarities to the last rounding: the finalize pass rescoring every survivor in float64
(``exact_row_sim`` / ``exact_sim`` in ``select_finalize.cu``) against a float64 NumPy recomputation of the owning
row, through the kernel's own chain of float32 roundings (``tests/rounding.py``).

Searches go through ``CorpusIndex.scan_checked`` + ``merge_hits`` with hundreds to thousands of hits per query, in
SQL mode (``num_hits``) and exact MaxSim mode, one vector per chunk so that every hit names its row."""

from __future__ import annotations

import numpy as np
import pytest
import rounding as rd

pytestmark = pytest.mark.gpu

ONE = np.float32(1.0)
CHAINS = {
    "cosine": lambda x: ONE - (ONE - rd.f32(np.clip(x, -1.0, 1.0))),   # dist = 1 - (float)s, sim = 1 - dist
    "dot": lambda x: ONE - rd.f32(-x),                                  # sim = 1 - (float)(-dot)
    "l2": lambda x: ONE - rd.f32(np.sqrt(np.maximum(x, 0.0))),          # sim = 1 - (float)sqrt(sum (e - q)^2)
}


@pytest.fixture(scope="module")
def rl():
    import torch

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import raglite_b200

    return raglite_b200


@pytest.fixture(scope="module", autouse=True)
def _two_value_report():
    yield
    print("\ntwo-value branch maxima (count, entries):", dict(sorted(rd.TWO_VALUE_MAX.items())))


def oracle(E: np.ndarray, q: np.ndarray, metric: str) -> tuple[np.ndarray, np.ndarray]:
    """(float64 value before the float32 roundings, bound b on its float64 difference from the kernel's value) for
    rows E (as stored) and query q (float32).  Both sides form their sums of d terms in different orders, each
    within gamma_d of the exact sum of the (identically rounded) terms."""
    d = E.shape[1]
    E64, q64 = E.astype(np.float64), q.astype(np.float64)
    g = rd.gamma(d)
    if metric == "l2":
        # terms fl(fl(e - q)^2) are nonnegative (a fused multiply-add only removes a rounding): 2 gamma_d v
        t = E64 - q64
        v = np.einsum("ij,ij->i", t, t)
        return v, 2 * g * v
    dot = E64 @ q64                           # products of two float32 values are exact in float64
    a = np.abs(E64) @ np.abs(q64)
    if metric == "dot":
        return dot, 2 * g * a
    ne = np.einsum("ij,ij->i", E64, E64)
    nq = q64 @ q64
    den = np.sqrt(ne * nq)
    s = dot / den
    # dot within 2 gamma_d a; ne, nq within 2 gamma_d relative (halved by the sqrt); ne * nq, sqrt and the division
    # round once each per side
    return s, 2 * rd.gamma(d + 3) * (a / den + np.abs(s))


def _corpus(n: int, d: int, storage: str, metric: str, seed: int, B: int):
    """Rows with norms from 1e-3 to 1e3 (fp16 cosine: 0.5 to 30, what its fast path accepts); queries that are
    near-duplicates of planted rows (|e - q| ~ 1e-6 |q|) or random directions with a planted opposite row."""
    rng = np.random.default_rng(seed)
    E = rng.standard_normal((n, d), dtype=np.float32)
    E /= np.linalg.norm(E, axis=1, keepdims=True)
    lo, hi = (np.log10(0.5), np.log10(30.0)) if (storage == "fp16" and metric == "cosine") else (-3.0, 3.0)
    E *= (10.0 ** rng.uniform(lo, hi, size=(n, 1))).astype(np.float32)
    if storage == "fp16":
        E = E.astype(np.float16).astype(np.float32)
    Q = rng.standard_normal((B, d), dtype=np.float32)
    Q *= (10.0 ** rng.uniform(-3.0, 3.0, size=(B, 1)) / np.linalg.norm(Q, axis=1, keepdims=True)).astype(np.float32)
    for b in range(B // 2):
        r = int(rng.integers(0, n))
        u = rng.standard_normal(d).astype(np.float32)
        Q[b] = E[r] + np.float32(1e-6) * np.linalg.norm(E[r]) * u / np.linalg.norm(u)
        if storage == "fp32":      # two more rows near the same query
            E[(r + 1) % n] = Q[b] + np.float32(2e-6) * np.linalg.norm(Q[b]) * u[::-1] / np.linalg.norm(u)
            E[(r + 2) % n] = Q[b] - np.float32(1e-6) * np.linalg.norm(Q[b]) * u / np.linalg.norm(u)
    for b in range(B // 2, B):     # sim -1 for cosine
        anti = -2.0 * Q[b] / np.linalg.norm(Q[b])
        E[int(rng.integers(0, n))] = anti.astype(np.float16) if storage == "fp16" else anti
    return E, Q


def _search(idx, Q: np.ndarray, *, metric: str, algo: str, sql: bool, H: int):
    import torch

    from raglite_b200._index import merge_hits

    Qd = torch.from_numpy(np.ascontiguousarray(Q)).cuda()
    res = idx.scan_checked(Qd, k=H, num_hits=H if sql else 0, metric=metric, algo=algo)
    sim, chunk, cnt = merge_hits(res.hit_sim, res.hit_chunk, res.hit_count, num_hits=H if sql else 0, k=H)
    return sim.cpu().numpy(), chunk.cpu().numpy(), cnt.cpu().numpy()


def _check_hits(E, Q, sim, chunk, cnt, metric: str, what: str) -> np.ndarray:
    """Every returned (chunk, sim) against the bracket; returns the checked sims."""
    allsims = []
    for b in range(len(Q)):
        n = int(cnt[b])
        rows = chunk[b, :n]
        assert n > 0 and np.all(rows >= 0) and len(np.unique(rows)) == n
        assert np.all(np.diff(sim[b, :n]) <= 0)                       # descending
        v, bound = oracle(E[rows], Q[b], metric)
        rd.check(sim[b, :n], v, bound, CHAINS[metric], what=what)
        allsims.append(sim[b, :n])
    return np.concatenate(allsims)


PATHS = [("fp32", 64, "fp32"), ("fp32", 64, "tcgen05"), ("fp32", 50, "fp32"), ("fp16", 64, "tcgen05")]


@pytest.mark.parametrize("sql", [True, False], ids=["sql", "exact"])
@pytest.mark.parametrize("path", PATHS, ids=lambda p: f"{p[0]}-d{p[1]}-{p[2]}")
@pytest.mark.parametrize("metric", ["cosine", "dot", "l2"])
def test_returned_sims_to_the_last_rounding(rl, metric, path, sql):
    storage, d, algo = path
    n, B = 3000, 8
    H = n                                   # every row comes back: sims span the whole range
    E, Q = _corpus(n, d, storage, metric, seed=d + 3 * len(metric) + (7 if sql else 0), B=B)
    idx = rl.CorpusIndex(E, np.arange(n + 1, dtype=np.int64), storage=storage)
    sim, chunk, cnt = _search(idx, Q, metric=metric, algo=algo, sql=sql, H=H)
    assert np.all(cnt == H)
    sims = _check_hits(E, Q, sim, chunk, cnt, metric, what=f"rescore {metric} {storage} d={d} {algo}")
    if metric == "cosine":   # returned sims span [-1, 1], many below 0.5 where the 1 - dist round trip moves them
        assert sims.min() < -0.999 and sims.max() > 0.999 and (sims < 0.5).sum() > 1000


@pytest.mark.parametrize("storage,algo", [("fp32", "fp32"), ("fp32", "tcgen05"), ("fp16", "tcgen05")])
@pytest.mark.parametrize("metric", ["cosine", "l2"])
def test_streaming_rescoring_past_4096_survivors(rl, metric, storage, algo):
    d, n_cluster, n_other = 64, 5000, 1000
    rng = np.random.default_rng(99)
    c = rng.standard_normal(d).astype(np.float32)
    c /= np.linalg.norm(c)
    spread = 1e-3 if storage == "fp16" else 1e-4
    E = np.concatenate([c + (spread / np.sqrt(d)) * rng.standard_normal((n_cluster, d)).astype(np.float32),
                        rng.standard_normal((n_other, d)).astype(np.float32) / np.sqrt(d)]).astype(np.float32)
    E = E[rng.permutation(len(E))]
    if storage == "fp16":
        E = E.astype(np.float16).astype(np.float32)
    Q = (c + 0.01 * rng.standard_normal((4, d)).astype(np.float32) / np.sqrt(d)).astype(np.float32)
    idx = rl.CorpusIndex(E, np.arange(len(E) + 1, dtype=np.int64), storage=storage)
    for sql in (True, False):
        sim, chunk, cnt = _search(idx, Q, metric=metric, algo=algo, sql=sql, H=100)
        assert idx.scan_stats()["survivors_max"] > 4096              # the streaming rescoring ran
        assert np.all(cnt == 100)
        _check_hits(E, Q, sim, chunk, cnt, metric, what=f"rescore streaming {metric} {storage} {algo}")
        # and the 100 returned rows are the 100 best (ties at the float32 cut may swap rows with equal sims)
        for b in range(len(Q)):
            v, _ = oracle(E, Q[b], metric)
            allsim = CHAINS[metric](v)
            assert np.sort(allsim)[::-1][99] == sim[b, 99]


@pytest.mark.parametrize("algo", ["fp32", "tcgen05"])
@pytest.mark.parametrize("scale", ["unscaled", "scaled"])
def test_l2_sims_within_1e4_of_the_direct_distance(rl, scale, algo):
    """The library's 1e-4 score contract for l2 against sqrt(sum (e - q)^2), with queries that duplicate corpus rows
    exactly or to within float32 steps: there ne + nq - 2 dot would cancel to its rounding error.  For dot and l2 the
    tensor-core scan multiplies rows by one global power of two that brings max |x| into (0.5, 1] (``pow2_scale`` in
    scan_wgmma.cu; the cosine gate on stats[1] <= 1024 does not apply to them).  "unscaled": max |x| = 1, so that
    factor is 1, at nearly the largest norm it allows (|x| in [0.9, 1]: |e| ~ 30 of sqrt(d) = 32).  "scaled":
    |e| = 1e4."""
    d, n, B = 1024, 4000, 16
    rng = np.random.default_rng(7 if scale == "scaled" else 8)
    E = rng.standard_normal((n, d), dtype=np.float32)
    if scale == "unscaled":
        E = (np.sign(E) * rng.uniform(0.9, 1.0, size=E.shape)).astype(np.float32)
        E[:, 0] = np.where(E[:, 0] < 0, -1.0, 1.0)             # max |x| = 1 exactly
    else:
        E *= (1e4 / np.linalg.norm(E, axis=1, keepdims=True)).astype(np.float32)
    rows = rng.choice(n, size=B, replace=False)
    Q = E[rows].copy()
    Q[B // 2:] = np.nextafter(Q[B // 2:], np.float32(np.inf))           # one float32 step away in every entry
    idx = rl.CorpusIndex(E, np.arange(n + 1, dtype=np.int64), storage="fp32")
    for sql in (True, False):
        sim, chunk, cnt = _search(idx, Q, metric="l2", algo=algo, sql=sql, H=50)
        near_err = []
        for b in range(B):
            hit = chunk[b, : cnt[b]]
            t = E[hit].astype(np.float64) - Q[b].astype(np.float64)
            direct = 1.0 - np.sqrt(np.einsum("ij,ij->i", t, t))
            err = np.abs(sim[b, : cnt[b]] - direct)
            near = np.abs(direct - 1.0) <= 1.0       # (near-)duplicates; far rows are checked relative to |sim|,
            near_err.append(err[near].max())         # where float32 itself resolves no better than 6e-8 |sim|
            assert hit[0] == rows[b] and near[0]
            assert np.all(err[~near] <= 1e-4 * np.abs(direct[~near])), (scale, algo, sql, b)
        print(f"l2 {scale} {algo} sql={sql}: largest error at (near-)duplicates {max(near_err):.3g}")
        assert max(near_err) <= 1e-4, (scale, algo, sql, near_err)
