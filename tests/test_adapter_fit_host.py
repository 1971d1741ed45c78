"""The adapter fit's references on the host: ``adapter_oracle.project`` against 50-digit mpmath and the reference's
golden targets, ``adapter_oracle.kernel_port`` against ``project`` and across every branch, and the C-ABI refusals of
``rl_adapter_targets`` / ``rl_best_vectors`` before any CUDA call (no GPU needed)."""

from __future__ import annotations

import ctypes
from collections import Counter

import mpmath
import numpy as np
import pytest

import adapter_oracle as ao


def _mp_projection(q, P, N, alpha, basis):
    """t = q + D_B^T lam with D_B t = 0, solved at 50 digits; returns t, lam and min_j d_j . t (all mpmath)."""
    mpmath.mp.dps = 50
    c = mpmath.mpf(float(1.0 + alpha))
    D = [[mpmath.mpf(float(p)) - c * mpmath.mpf(float(n)) for p, n in zip(pi, nj)] for pi in P for nj in N]
    qm = [mpmath.mpf(float(x)) for x in q]
    B = [D[j] for j in basis]
    t = list(qm)
    lam = []
    if B:
        H = mpmath.matrix([[mpmath.fsum(a * b for a, b in zip(u, v)) for v in B] for u in B])
        rhs = mpmath.matrix([-mpmath.fsum(a * b for a, b in zip(u, qm)) for u in B])
        lam = list(mpmath.lu_solve(H, rhs))
        t = [qm[i] + mpmath.fsum(lam[k] * B[k][i] for k in range(len(B))) for i in range(len(qm))]
    dt = min(mpmath.fsum(a * b for a, b in zip(dj, t)) for dj in D)
    return t, lam, dt


@pytest.mark.parametrize("seed", range(12))
def test_project_agrees_with_mpmath_at_50_digits(seed):
    rng = np.random.default_rng(seed)
    d = int(rng.integers(1, 17))
    nP = int(rng.integers(1, 5))
    nN = int(rng.integers(1, 9 - nP))
    alpha = float(rng.choice(ao.ALPHAS))
    inst = ao.make_instance(["random", "correlated", "polar", "near_duplicates"][seed % 4], nP, nN, d,
                            alpha if seed % 4 != 2 else float(seed % 2), seed)
    proj = ao.project(inst.q, inst.P, inst.N, inst.alpha)
    t, lam, dt = _mp_projection(inst.q, inst.P, inst.N, inst.alpha, proj.basis)
    qn = proj.qnorm
    # the 50-digit answer on the reference's face is feasible, and where the face's generators are independent its
    # multipliers are unique and >= 0 (with dependent ones, project's own nnls certificate covers the sign)
    assert dt >= -1e-40 * max(qn, 1)
    if len(proj.basis) == len(proj.active):
        assert all(x >= -1e-40 * max(abs(y) for y in lam) for x in lam)   # exact zeros come out as +-1e-50
    hi = proj.t.astype(np.float64)
    lo = (proj.t - hi.astype(ao.LD)).astype(np.float64)                  # a long double is exactly hi + lo
    diff = max(abs(float(mpmath.mpf(float(h)) + mpmath.mpf(float(w)) - b)) for h, w, b in zip(hi, lo, t))
    assert diff <= 1e-17 * max(qn, 1e-300) * max(1.0, proj.cond), (diff, proj.cond)


def test_project_agrees_with_the_reference_golden(golden_dir):
    """The golden targets are the reference's SciPy iterate cast to the query dtype: equal to 1 ulp of that dtype."""
    z = np.load(golden_dir / "adapter_target.npz")
    for i in range(3):
        q, P, N, t = z[f"q{i}"], z[f"P{i}"], z[f"N{i}"], z[f"t{i}"]
        got = ao.project(q.astype(np.float32), P, N, 0.05).t.astype(np.float64).astype(q.dtype)
        it = np.int16 if q.dtype == np.float16 else np.int32
        ulp = np.abs(got.view(it).astype(np.int64) - t.view(it).astype(np.int64))
        assert ulp.max() <= 1, (i, ulp.max())


def test_certificate_rejects_a_wrong_face():
    """d = 1, q = 1, one generator 1: t = 1 (mu = 0).  t' = 0 (mu = -1) is feasible, in the span and has the lower
    objective, so only the dual sign tells it apart."""
    q, P, N = np.array([1.0], np.float32), np.array([[1.0]], np.float32), np.array([[0.0]], np.float32)
    proj = ao.project(q, P, N, 0.0)
    assert proj.t[0] == 1 and len(proj.active) == 0
    ao.check_certificate(np.array([1.0]), q, P, N, 0.0, proj)
    with pytest.raises(AssertionError, match="dual"):
        ao.check_certificate(np.array([0.0]), q, P, N, 0.0, proj)


def test_kernel_port_agrees_with_project():
    for inst in ao.families():
        proj = ao.project(inst.q, inst.P, inst.N, inst.alpha)
        port = ao.kernel_port(inst.q, inst.P, inst.N, inst.alpha)
        err = float(np.abs(port.t - proj.t.astype(np.float64)).max())
        stalled = port.branches["stop_with_rejected"] > 0 or port.pivot_margin < 1
        bound = 1e-6 * proj.qnorm if stalled else ao.device_bound(proj)
        assert err <= bound, (inst.name, err, bound)
        if inst.name.startswith("feasible-"):
            assert port.iters == 1 and np.array_equal(port.t, inst.q.astype(np.float64))


def test_families_reach_every_branch():
    total: Counter = Counter()
    for inst in ao.families():
        total += ao.kernel_port(inst.q, inst.P, inst.N, inst.alpha).branches
    for branch in ("step_full", "step_back", "pivot_reject", "rejected_cleared", "readmitted", "stop_optimal",
                   "stop_with_rejected"):
        assert total[branch] > 0, (branch, total)
    # never reached, by construction or in practice (DESIGN 5): rank(D) <= r - 1, so r independent columns cannot
    # fill the passive set; the fresh column stays positive through a step-back, so the set never empties; the
    # iteration cap, the fresh-column safeguard and a step-back that drops two columns at once need rounding ties
    for branch in ("stop_full", "emptied", "stop_cap"):
        assert total[branch] == 0, (branch, total)


def test_scale_free_stopping_rule_in_the_port():
    """The port at 2^-16 scale: the relative rule keeps the unit-scale answer, the old absolute floor stops early."""
    inst = next(i for i in ao.families() if i.name == "random-32x32-d384-a0.05-s5")
    base = ao.kernel_port(inst.q, inst.P, inst.N, inst.alpha)
    s = np.float32(2.0 ** -16)
    rel = ao.kernel_port(inst.q * s, inst.P * s, inst.N * s, inst.alpha)
    old = ao.kernel_port(inst.q * s, inst.P * s, inst.N * s, inst.alpha, relative_tol=False)
    assert rel.iters == base.iters and np.array_equal(rel.t, base.t * (2.0 ** -16))
    assert old.iters < base.iters


def _lib():
    from raglite_b200 import _lib as L

    return L.load()


@pytest.mark.parametrize("n_slots,d,alpha", [(0, 8, 0.05), (65, 8, 0.05), (4, 0, 0.05), (4, 8, -1e-300), (4, 8, float("nan"))])
def test_adapter_targets_refuses_bad_arguments(n_slots, d, alpha):
    lib = _lib()
    p = ctypes.c_void_p(16)
    assert lib.rl_adapter_targets(p, p, 3, n_slots, d, p, alpha, p, p, p, None) == -1
    assert "rl_adapter_targets" in lib.rl_last_error().decode()


def test_adapter_targets_refuses_null_pointers():
    lib = _lib()
    p = ctypes.c_void_p(16)
    args = [p, p, 3, 4, 8, p, 0.05, p, p, p, None]
    for k in (0, 1, 5, 7, 8, 9):
        a = list(args)
        a[k] = None
        assert lib.rl_adapter_targets(*a) == -1, k
        assert "null pointer" in lib.rl_last_error().decode()
    assert lib.rl_adapter_targets(None, None, 0, 4, 8, None, 0.05, None, None, None, None) == 0   # no evals: nothing to do


@pytest.mark.parametrize("e_dtype,ld,d,n_slots", [(0, 8, 8, 0), (0, 8, 0, 4), (0, 7, 8, 4), (2, 8, 8, 4)])
def test_best_vectors_refuses_bad_arguments(e_dtype, ld, d, n_slots):
    lib = _lib()
    p = ctypes.c_void_p(16)
    assert lib.rl_best_vectors(p, e_dtype, ld, d, p, p, 3, n_slots, p, p, p, None) == -1
    assert "rl_best_vectors" in lib.rl_last_error().decode()


def test_best_vectors_refuses_null_pointers():
    lib = _lib()
    p = ctypes.c_void_p(16)
    args = [p, 0, 8, 8, p, p, 3, 4, p, p, p, None]
    for k in (0, 4, 5, 8, 9, 10):
        a = list(args)
        a[k] = None
        assert lib.rl_best_vectors(*a) == -1, k
        assert "null pointer" in lib.rl_last_error().decode()
    assert lib.rl_best_vectors(None, 0, 8, 8, None, None, 0, 4, None, None, None, None) == 0
