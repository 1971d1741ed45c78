"""Rounding-bracket oracle for kernels that compute in float64 and round a fixed number of times.

Such a kernel's answer is exact apart from the order of its float64 sums.  Given the float64 NumPy value ``v`` of the
same quantity, a proven bound ``b`` on the float64 difference between the kernel's value and ``v`` (both sides'
summation errors), and the kernel's chain of roundings, every value in ``[v - b, v + b]`` goes through the (monotone)
chain to one of two results: ``chain(v - b)`` and ``chain(v + b)``.  The kernel's output must be one of them.  They
are equal unless a rounding boundary lies inside the interval; the number of entries where they differ (the
two-value branch) is counted and kept small, so that a loose ``b`` cannot make a check pass vacuously.
"""

from __future__ import annotations

import numpy as np

U = 2.0 ** -53          # unit roundoff of float64
TWO_VALUE_MAX: dict[str, tuple[int, int]] = {}   # what -> (largest two-value count seen, size of that check)


def gamma(n) -> np.ndarray:
    """``gamma_n = n u / (1 - n u)``: the relative error bound of a float64 sum of n terms (or dot product of length
    n) in any order, relative to the sum of the terms' absolute values (Higham, Accuracy and Stability, 3.1)."""
    n = np.asarray(n, dtype=np.float64)
    return n * U / (1.0 - n * U)


def f32(x):
    return np.asarray(x, np.float64).astype(np.float32)


def f16(x):
    """float64 -> float16 in one rounding (NumPy converts directly, without a float32 step)."""
    with np.errstate(over="ignore"):
        return np.asarray(x, np.float64).astype(np.float16)


def bracket(v, b, chain) -> tuple[np.ndarray, np.ndarray]:
    """``(chain(v - b), chain(v + b))``: the two acceptable outputs of each entry."""
    v = np.asarray(v, np.float64)
    b = np.broadcast_to(np.asarray(b, np.float64), v.shape)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        return np.asarray(chain(v - b)), np.asarray(chain(v + b))


def _same(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return (a == b) | (np.isnan(a) & np.isnan(b))


def check(out, v, b, chain, *, what: str, max_two: int | None = None) -> int:
    """Assert ``out`` (any float dtype; compared by value, NaN equal to NaN) is ``chain(v - b)`` or ``chain(v + b)``
    entry by entry (anything between them where the bound spans several rounding steps), and that they differ at no
    more than ``max_two`` entries (default: 1 % of the entries, at least 4).  Returns that two-value count."""
    out = np.asarray(out)
    v = np.asarray(v, np.float64)
    assert out.shape == v.shape, (what, out.shape, v.shape)
    lo, hi = bracket(v, b, chain)
    two = ~_same(lo, hi)
    n_two = int(two.sum())
    ok = _same(out, lo) | _same(out, hi)
    if n_two:
        # a worst-case bound can span several rounding steps where the value cancels (|v| much smaller than the sum
        # of |terms|): there every output between the two ends is acceptable; such entries count as two-value ones
        with np.errstate(over="ignore"):
            wide = two & (np.nextafter(lo, hi) != hi)
        o = np.asarray(out, np.float64)
        ok |= wide & (o >= np.minimum(lo, hi)) & (o <= np.maximum(lo, hi))
    if not ok.all():
        bad = np.argwhere(~ok)[:5]
        bb = np.broadcast_to(np.asarray(b, np.float64), v.shape)
        rows = [(tuple(int(i) for i in ix), float(v[tuple(ix)]), float(bb[tuple(ix)]), float(lo[tuple(ix)]),
                 float(hi[tuple(ix)]), float(out[tuple(ix)])) for ix in bad]
        raise AssertionError(f"{what}: {int((~ok).sum())} of {out.size} outside the rounding bracket; "
                             f"(index, v, b, chain(v-b), chain(v+b), got): {rows}")
    limit = max(4, out.size // 100) if max_two is None else max_two
    assert n_two <= limit, f"{what}: {n_two} of {out.size} entries on the two-value branch (limit {limit}): b is too loose"
    seen = TWO_VALUE_MAX.get(what, (0, 0))
    if n_two >= seen[0]:
        TWO_VALUE_MAX[what] = (n_two, out.size)
    return n_two
