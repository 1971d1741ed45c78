"""Certified reference and a control-flow port for ``rl_adapter_targets`` (``csrc/adapter_fit.cu``), host only.

The kernel projects q onto the cone ``{t : D t >= 0}``, ``D = {p_i - c n_j}`` with ``c = 1 + alpha``: it runs
Lawson-Hanson NNLS on ``min |q + D^T mu|, mu >= 0`` and returns ``t = q + D^T mu*``.

* :func:`project` is the reference.  SciPy's ``nnls`` proposes the active set A.  t* = q - Pi_span(D_A) q is then
  computed by Gram-Schmidt applied twice in ``np.longdouble`` (64-bit significand) and certified:
  - primal, ``D t* >= -tau``;
  - complementary, ``|D_A t*| <= tau``;
  - dual, ``t* - q = D_A^T lam`` with ``lam >= 0`` to a residual ``<= tau'``.
  tau is relative to ``|q| max_j |d_j|`` and tau' to ``|q|``, never to |t|: t* = 0 is a legitimate answer.  An
  instance whose certificate fails raises :class:`Uncertified`; such an instance is unusable, whatever the kernel says.
* :func:`kernel_port` restates the kernel's control flow in float64 NumPy: the same pick order, iteration count, pivot
  test, fresh-column safeguard, step-back and re-admission.  nvcc contracts to FMA and the port does not, so its
  roundings differ from the device's.  What it pins are the kernel's decisions.  It counts each branch, and it records
  how close a decision came to flipping: the smallest relative gap at a pick, and the closest pivot to its threshold.
* :func:`families` builds the instance families that the host and the GPU tests share.
"""

from __future__ import annotations

import dataclasses
import math
from collections import Counter

import numpy as np
from scipy.optimize import nnls

LD = np.longdouble
assert np.finfo(LD).eps <= 2.0 ** -63, "project() needs an 80-bit long double"

PIVOT_REL = 1e-14          # the kernel's Cholesky pivot threshold, relative to the diagonal entry
TAU_PRIMAL = 1e-13         # certificate tolerances of the reference, see project()
TAU_DUAL = 1e-10


class Uncertified(AssertionError):
    """The reference could not certify its own answer: the instance is rejected."""


@dataclasses.dataclass
class Projection:
    t: np.ndarray              # t* in longdouble
    active: np.ndarray         # generator indices with mu > 0 in SciPy's nnls
    basis: np.ndarray          # the independent subset of them that Gram-Schmidt kept
    cond: float                # cond(H_BB), H = D D^T on the basis (1.0 for an empty basis)
    scale: float               # |q| max_j |d_j|
    qnorm: float


def generators(P, N, alpha, dtype=np.float64) -> np.ndarray:
    """D, one row p_i - c n_j per pair, pair (i, j) at row i |N| + j (the kernel's generator order)."""
    c = dtype(1.0 + float(alpha))      # the kernel's c = 1.0 + alpha, rounded to double first
    P, N = np.asarray(P).astype(dtype), np.asarray(N).astype(dtype)
    return (P[:, None, :] - c * N[None, :, :]).reshape(-1, P.shape[1])


def _gram_schmidt_twice(V: np.ndarray, rel: float = 1e-12):
    """Orthonormal basis (rows) of the rows of V (longdouble), and the indices of the rows it kept."""
    Qb, keep = [], []
    for k, v0 in enumerate(V):
        n0 = np.sqrt(v0 @ v0)
        if n0 == 0:
            continue
        v = v0.copy()
        for _ in range(2):
            for u in Qb:
                v -= (u @ v) * u
        nv = np.sqrt(v @ v)
        if nv <= rel * n0:
            continue
        Qb.append(v / nv)
        keep.append(k)
    return (np.array(Qb, dtype=LD).reshape(len(Qb), V.shape[1]), np.array(keep, dtype=np.int64))


def dual_residual(D_A: np.ndarray, t: np.ndarray, q: np.ndarray) -> float:
    """min over lam >= 0 of |D_A^T lam - (t - q)|: 0 when t - q lies in the cone of the active generators."""
    r = np.asarray(t, np.float64) - np.asarray(q, np.float64)
    if len(D_A) == 0:
        return float(np.linalg.norm(r))
    return float(nnls(np.asarray(D_A, np.float64).T, r, maxiter=50 * max(len(D_A), 10))[1])


def project(q, P, N, alpha) -> Projection:
    """t*, the projection of q onto {t : D t >= 0}, with its certificate (see the module docstring)."""
    q64 = np.asarray(q, np.float64)
    D64 = generators(P, N, alpha)
    m = len(D64)
    mu, _ = nnls(D64.T, -q64, maxiter=200 * max(m, 10))
    active = np.flatnonzero(mu > 0)
    Dl = generators(P, N, alpha, LD)
    ql = q64.astype(LD)
    Qb, kept = _gram_schmidt_twice(Dl[active])
    t = ql.copy()
    for _ in range(2):
        t -= Qb.T @ (Qb @ t) if len(Qb) else 0
    basis = active[kept]
    qn = float(np.sqrt(ql @ ql))
    dmax = float(np.max(np.sqrt(np.einsum("ij,ij->i", Dl, Dl)))) if m else 0.0
    scale = qn * dmax
    Dt = Dl @ t
    if m and Dt.min() < -TAU_PRIMAL * scale:
        raise Uncertified(f"primal: min D t* = {float(Dt.min()):.3g}, scale {scale:.3g}")
    if len(active) and np.abs(Dt[active]).max() > TAU_PRIMAL * scale:
        raise Uncertified(f"complementarity: max |D_A t*| = {float(np.abs(Dt[active]).max()):.3g}, scale {scale:.3g}")
    res = dual_residual(D64[active], t, q64)
    if res > TAU_DUAL * qn:
        raise Uncertified(f"dual: residual {res:.3g}, |q| {qn:.3g}")
    if len(basis):
        B = D64[basis]
        cond = float(np.linalg.cond(B @ B.T))
    else:
        cond = 1.0
    return Projection(t=t, active=active, basis=basis, cond=cond, scale=scale, qnorm=qn)


@dataclasses.dataclass
class PortResult:
    t: np.ndarray
    iters: int
    mu: np.ndarray
    branches: Counter
    pick_gap: float            # smallest (best - runner-up) / best over every pick, and (tol - max w) / tol at the stop
    pivot_margin: float        # smallest |log10(dg / (1e-14 H_cc))| over every pivot with dg > 0


def kernel_port(q, P, N, alpha, *, relative_tol: bool = True) -> PortResult:
    """``adapter_targets_kernel`` for one eval in float64 NumPy (the kernel's inputs are float32).

    ``relative_tol=False`` is the stopping rule before it was made scale-free: ``1e-13 (gmax + 1)``."""
    q = np.asarray(q, np.float32).astype(np.float64)
    P = np.asarray(P, np.float32).astype(np.float64)
    N = np.asarray(N, np.float32).astype(np.float64)
    nP, nN = len(P), len(N)
    r, m = nP + nN, nP * nN
    W = np.concatenate([P, N])
    G = W @ W.T
    wq = W @ q
    c = 1.0 + float(alpha)
    jj = np.arange(m)
    i1, j1 = jj // nN, nP + jj % nN
    H = (G[i1][:, i1] - c * G[i1][:, j1]) - c * G[j1][:, i1] + (c * c) * G[j1][:, j1]
    g = wq[i1] - c * wq[j1]
    gmax = float(np.abs(g).max())
    tol = 1e-13 * gmax if relative_tol else 1e-13 * (gmax + 1.0)
    max_iter = 6 * m + 64
    mu = np.zeros(m)
    inS = np.zeros(m, np.uint8)
    ever_rejected = np.zeros(m, bool)
    S: list[int] = []
    br: Counter = Counter()
    it = 0
    pick_gap, pivot_margin = math.inf, math.inf
    while True:
        w = -g.copy()
        for a in S:
            w = w - H[:, a] * mu[a]
        w = np.where(inS != 0, -1.0, w)
        cand = w > tol
        it += 1
        if cand.any():
            pick = int(np.argmax(np.where(cand, w, -np.inf)))    # first maximum, as the serial scan's strict '>'
            best = w[pick]
            rest = np.delete(w, pick)
            second = max(float(rest.max()) if len(rest) else -math.inf, tol)
            pick_gap = min(pick_gap, (best - second) / best)
        else:
            pick = -1
            mx = float(w.max())
            if mx > 0 and tol > 0:
                pick_gap = min(pick_gap, (tol - mx) / tol)
        if pick < 0:
            br["stop_optimal"] += 1
            w_rej = -g.copy()
            for a in S:
                w_rej = w_rej - H[:, a] * mu[a]
            if ((inS == 2) & (w_rej > tol)).any():
                br["stop_with_rejected"] += 1   # the rejected columns were never re-examined: the face is not optimal
            break
        if len(S) >= r:
            br["stop_full"] += 1
            break
        if it > max_iter:
            br["stop_cap"] += 1
            break
        if ever_rejected[pick]:
            br["readmitted"] += 1
        S.append(pick)
        inS[pick] = 1
        fresh = True
        while True:
            s = len(S)
            Hs = H[np.ix_(S, S)]
            L = np.zeros((s, s))
            flag = 0
            for col in range(s):
                dg = Hs[col, col] - L[col, :col] @ L[col, :col]
                hcc = abs(Hs[col, col])
                if dg > 0 and hcc > 0:
                    pivot_margin = min(pivot_margin, abs(math.log10(dg / (PIVOT_REL * hcc))))
                if dg <= PIVOT_REL * hcc or dg <= 0.0:
                    flag = 1
                    break
                L[col, col] = math.sqrt(dg)
                if col + 1 < s:
                    L[col + 1:, col] = (Hs[col + 1:, col] - L[col + 1:, :col] @ L[col, :col]) / L[col, col]
            if flag:
                br["pivot_reject"] += 1
                j = S.pop()
                inS[j] = 2
                ever_rejected[j] = True
                break
            rhs = -g[S]
            z = np.zeros(s)
            for a in range(s):
                z[a] = (rhs[a] - L[a, :a] @ z[:a]) / L[a, a]
            for a in range(s - 1, -1, -1):
                z[a] = (z[a] - L[a + 1:, a] @ z[a + 1:]) / L[a, a]
            if fresh and z[s - 1] <= 0.0:
                flag = 2
            fresh = False
            step, feasible = 1.0, True
            for a in range(s):
                if z[a] <= 0.0:
                    feasible = False
                    cur = mu[S[a]]
                    step = min(step, cur / (cur - z[a]))
            if flag == 2:
                br["fresh_reject"] += 1
                j = S.pop()
                inS[j] = 2
                ever_rejected[j] = True
                break
            if feasible:
                mu[S] = z
                if (inS == 2).any():
                    br["rejected_cleared"] += 1
                inS[inS == 2] = 0
                br["step_full"] += 1
                break
            br["step_back"] += 1
            keep = []
            for a in range(s):
                j = S[a]
                v = mu[j] + step * (z[a] - mu[j])
                if v <= 1e-300 or (z[a] <= 0.0 and mu[j] / (mu[j] - z[a]) <= step):
                    v = 0.0
                mu[j] = v
                if v > 0.0:
                    keep.append(j)
                else:
                    inS[j] = 0
            dropped = s - len(keep)
            br["dropped"] += dropped
            if dropped > 1:
                br["step_back_multi"] += 1
            S = keep
            if not S:
                br["emptied"] += 1
                break
    a = np.zeros(r)
    for i in range(nP):
        a[i] = mu[i * nN:(i + 1) * nN].sum()
    for j in range(nN):
        a[nP + j] = mu[j::nN].sum()
    t = q.copy()
    for i in range(nP):
        t = t + a[i] * P[i]
    for j in range(nN):
        t = t - (c * a[nP + j]) * N[j]
    return PortResult(t=t, iters=it, mu=mu, branches=br, pick_gap=pick_gap, pivot_margin=pivot_margin)


def device_bound(proj: Projection) -> float:
    """The |T - t*|_inf allowance of the device answer: 1e-12 |q| up to cond(H_BB) = 1e4, then growing with cond."""
    return max(1e-12, 1e-16 * proj.cond) * proj.qnorm


def check_certificate(T, q, P, N, alpha, proj: Projection, *, primal: float = 1e-12, dual: float = 1e-9) -> tuple[float, float]:
    """The certificate for an answer T that is not the reference's own: D T >= -primal |q| dmax, and T - q in the
    cone of the reference's active generators (lam >= 0) to a residual <= dual |q|.  Returns the two margins used."""
    D = generators(P, N, alpha)
    T = np.asarray(T, np.float64)
    dt = D @ T
    worst = float(-dt.min()) / proj.scale if proj.scale > 0 else 0.0
    assert worst <= primal, f"primal: min D T = {-worst:.3g} x |q| dmax"
    res = dual_residual(D[proj.active], T, q) / proj.qnorm if proj.qnorm > 0 else 0.0
    assert res <= dual, f"dual: residual {res:.3g} x |q|"
    return worst, res


# ---------------------------------------------------------------------------------------------------------------- #
# instance families

SHAPES = [(1, 1), (1, 63), (63, 1), (16, 48), (33, 31), (32, 32)]
DIMS = [1, 4, 8, 31, 33, 384, 1024]
ALPHAS = [0.0, 0.05, 1.0, 10.0]
KINDS = ["random", "correlated", "feasible", "polar", "duplicates", "zero_generators", "zero_vectors",
         "near_duplicates", "fp16", "norm_spread"]


@dataclasses.dataclass
class Instance:
    name: str
    q: np.ndarray              # float32 [d]
    P: np.ndarray              # float32 [|P|, d]
    N: np.ndarray              # float32 [|N|, d]
    alpha: float


def _unit(x):
    n = np.linalg.norm(x, axis=-1, keepdims=True)
    return x / np.where(n == 0, 1, n)


def make_instance(kind: str, nP: int, nN: int, d: int, alpha: float, seed: int, pair_eps: float | None = None) -> Instance:
    rng = np.random.default_rng(seed)
    q = _unit(rng.standard_normal(d))
    P = _unit(rng.standard_normal((nP, d)))
    N = _unit(rng.standard_normal((nN, d)))
    if kind == "correlated":                      # retrieved vectors resemble the query, as a real fit sees them
        P, N = 0.6 * P + 0.4 * q, 0.6 * N + 0.4 * q
    elif kind == "feasible":                      # every p_i . q >= c n_j . q already: t = q
        P, N = 0.3 * P + 2.0 * q, 0.3 * N - 2.0 * q
    elif kind == "polar":                         # q = -D^T lam exactly (small integers, c in {1, 2}): t* = 0
        P = rng.integers(-3, 4, size=(nP, d)).astype(np.float64)
        N = rng.integers(-3, 4, size=(nN, d)).astype(np.float64)
        D = generators(P, N, alpha)
        lam = np.zeros(len(D))
        lam[rng.choice(len(D), size=min(3, len(D)), replace=False)] = rng.integers(1, 4, size=min(3, len(D)))
        q = -(lam @ D)
        if not q.any():
            q = -D[0] if D[0].any() else q
    elif kind == "duplicates":                    # p_1 = p_0, n_1 = n_0 and p_i = n_j across
        P, N = 0.6 * P + 0.4 * q, 0.6 * N + 0.4 * q
        if nP > 1:
            P[1] = P[0]
        if nN > 1:
            N[1] = N[0]
        N[-1] = P[-1]
    elif kind == "zero_generators":               # alpha = 0 and p_i = n_j: the generator is exactly 0
        P, N = 0.6 * P + 0.4 * q, 0.6 * N + 0.4 * q
        N[0] = P[0]
        N[-1] = P[-1]
    elif kind == "zero_vectors":
        P, N = 0.6 * P + 0.4 * q, 0.6 * N + 0.4 * q
        P[-1] = 0.0
        N[0] = 0.0
    elif kind == "near_duplicates":               # pairs 1e-3 ... 1e-7 apart, or all pairs eps apart
        eps = [1e-3, 1e-4, 1e-5, 1e-6, 1e-7] if pair_eps is None else [pair_eps]
        for k in range(1, nP, 2):
            P[k] = P[k - 1] + eps[(k // 2) % len(eps)] * _unit(rng.standard_normal(d))
        for k in range(1, nN, 2):
            N[k] = N[k - 1] + eps[(k // 2 + 1) % len(eps)] * _unit(rng.standard_normal(d))
    elif kind == "fp16":                          # what fp16 storage hands the fit; q too
        P, N = 0.6 * P + 0.4 * q, 0.6 * N + 0.4 * q
        P = P.astype(np.float16).astype(np.float64)
        N = N.astype(np.float16).astype(np.float64)
        q = q.astype(np.float16).astype(np.float64)
    elif kind == "norm_spread":                   # norms 2^-10 ... 2^10 within one eval
        P, N = 0.6 * P + 0.4 * q, 0.6 * N + 0.4 * q
        P *= np.exp2(rng.integers(-10, 11, size=(nP, 1)))
        N *= np.exp2(rng.integers(-10, 11, size=(nN, 1)))
    elif kind != "random":
        raise ValueError(kind)
    return Instance(f"{kind}-{nP}x{nN}-d{d}-a{alpha:g}-s{seed}", q.astype(np.float32), P.astype(np.float32),
                    N.astype(np.float32), float(alpha))


def families() -> list[Instance]:
    """Every kind at every shape: d and alpha rotate with the shape, so each kind meets every d and alpha, and the
    kinds that need a particular alpha get it (0 for the zero generators, an exact c for the polar cone)."""
    out = []
    for k, kind in enumerate(KINDS):
        for s, (nP, nN) in enumerate(SHAPES):
            d = DIMS[(s + 2 * k) % len(DIMS)]
            alpha = ALPHAS[(s + k) % len(ALPHAS)]
            if kind == "zero_generators":
                alpha = 0.0
            elif kind == "polar":
                alpha = (0.0, 1.0)[s % 2]
            out.append(make_instance(kind, nP, nN, d, alpha, seed=1000 * k + s))
    # every pair 1e-7 apart: the pivot test rejects columns that still have a real gradient, and they come back
    out.append(make_instance("near_duplicates", 16, 48, 33, 0.05, seed=0, pair_eps=1e-7))
    # pairs 1e-3 ... 1e-7 apart where the kernel stops with rejected columns whose gradient is still above tol
    out.append(make_instance("near_duplicates", 32, 32, 33, 0.05, seed=83))
    return out
