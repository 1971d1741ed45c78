"""``rl_chunk_similarities`` at the C-ABI, bit for bit against ``chunks_oracle.chunk_costs_device``, its lane-exact
restatement: every written cost, every status and the untouched last slot of each document, compared as bit patterns
(a NaN the kernel computes compares as NaN; the guard behind every slot is a NaN of its own payload, so an unwritten
slot is told apart from a NaN cost).  Cases: widths off and on the multiples of 32 and 256 up to the shared-memory
opt-in, row strides wider than the row (odd for fp16), 0 to 300 rows, every kind of selection mask and heading
pattern, fp16 subnormals and values near 65504, rows of very different norms; a launch of more than three grid
strides with planted zero-row, unselected and skipped-projection documents in the same CTAs; the projection test's
eps edge; the sqrt(eps) clamp and a NaN through it."""

from __future__ import annotations

import chunks_oracle as co
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
SENT = -7
GUARD_BITS = 0x7FC0BEEF                                  # a quiet NaN no float operation produces
GUARD = np.array([GUARD_BITS], np.uint32).view(np.float32)[0]
SIM_MAX_BLOCKS = 4096                                    # kSimMaxBlocks of csrc/chunks.cu


def _lib():
    from raglite_b200 import _lib

    return _lib.load()


def _dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _similarities(X: np.ndarray, dim: int, off, non, head) -> tuple[np.ndarray, np.ndarray]:
    """One launch on the rows X [N, ld] (ld = X.shape[1]): (costs [N], status [D]), after checking the guards behind
    both outputs."""
    import torch

    lib = _lib()
    off = np.asarray(off, np.int64)
    D, N = len(off) - 1, int(off[-1])
    costs = _dev(np.full(N + 64, GUARD, np.float32))
    status = torch.full((D + 32,), SENT, dtype=torch.int32, device="cuda")
    ws = torch.empty(int(lib.rl_chunk_similarities_workspace_bytes(N)), dtype=torch.uint8, device="cuda")
    d_x = _dev(X if N else np.zeros((1, X.shape[1]), X.dtype))
    d_off, d_non, d_head = _dev(off), _dev(np.asarray(non, np.uint8)), _dev(np.asarray(head, np.uint8))
    rc = lib.rl_chunk_similarities(d_x.data_ptr(), 1 if X.dtype == np.float16 else 0, X.shape[1], dim,
                                   d_off.data_ptr(), D, N, d_non.data_ptr(), d_head.data_ptr(), costs.data_ptr(),
                                   status.data_ptr(), ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, lib.rl_last_error()
    got, st = costs.cpu().numpy(), status.cpu().numpy()
    assert (got[N:].view(np.uint32) == GUARD_BITS).all() and (st[D:] == SENT).all()
    return got[:N], st[:D]


def _assert_bits(got: np.ndarray, want: np.ndarray, what) -> None:
    """Equal bit patterns; computed NaNs (any NaN but the guard) compare as one value."""
    g, w = got.view(np.uint32).copy(), want.view(np.uint32).copy()
    for a, v in ((g, got), (w, want)):
        a[np.isnan(v) & (a != GUARD_BITS)] = 0x7FFFFFFF
    bad = np.nonzero(g != w)[0]
    assert not len(bad), (what, len(bad), [(int(i), float(got[i]), float(want[i])) for i in bad[:6]])


def _check(X, dim, off, non, head, what):
    got, st = _similarities(X, dim, off, non, head)
    want, wst, proj = co.chunk_costs_device(X, dim, off, non, head, fill=GUARD)
    assert st.tolist() == wst.tolist(), what
    _assert_bits(got, want, what)
    return got, st, proj


# ---- every width and dtype --------------------------------------------------------------------------------------------
NS = (0, 1, 2, 3, 8, 9, 33, 300)
MASKS = ("quantile", "none", "one", "all")
HEADS = ("none", "all", "first", "second_to_last", "runs", "alternating")


def _mask(kind: str, n: int, rng) -> np.ndarray:
    if kind == "quantile":
        return co.nonoutlying(rng.integers(10, 400, size=n)) if n else np.zeros(0, bool)
    m = np.zeros(n, bool)
    if kind == "one" and n:
        m[rng.integers(0, n)] = True                       # m = 1: that row's exact projection is zero
    if kind == "all":
        m[:] = True
    return m


def _heads(kind: str, n: int, rng) -> np.ndarray:
    h = np.zeros(n, bool)
    if kind == "all":
        h[:] = True
    elif kind == "first" and n:
        h[0] = True
    elif kind == "second_to_last" and n >= 2:
        h[n - 2] = True
    elif kind == "runs":
        h = (np.arange(n) // 3) % 2 == 1
    elif kind == "alternating":
        h = np.arange(n) % 2 == 1
    return h


def _rows(rng, n: int, dim: int, dtype, style: str) -> np.ndarray:
    X = rng.standard_normal((3, dim))[rng.integers(0, 3, size=n)] + rng.standard_normal((n, dim))
    if style == "norms":                                   # rows of very different norms in one document
        X *= 2.0 ** rng.integers(-12, 13, size=(n, 1))
    elif style == "big" and dtype == np.float16:           # values near 65504
        X = np.clip(X * 30000, -65504, 65504)
        X[:, : min(dim, 3)] = 65504 * np.sign(X[:, : min(dim, 3)] + 0.5)
    elif style == "tiny" and dtype == np.float16:          # subnormal entries (multiples of 2^-24)
        X = np.where(rng.random((n, dim)) < 0.5, rng.integers(-1023, 1024, size=(n, dim)) * 2.0**-24, X * 1e-3)
    elif style == "big":
        X *= 1e12
    elif style == "tiny":
        X *= 1e-12
    X = X.astype(dtype)
    zero = ~X.astype(np.float32).any(axis=1)
    X[zero, 0] = 1                                         # zero rows belong to the zero-row cases only
    return X


@pytest.mark.parametrize("dtype", [np.float16, np.float32])
@pytest.mark.parametrize("dim", [1, 2, 31, 33, 255, 257, 384, 1000, 1024, 6144, 6145, 8192])
def test_similarities_bit_exact(dtype, dim):
    rng = np.random.default_rng(dim * 2 + (dtype == np.float16))
    if dtype == np.float16:
        ld = dim + (2 if dim % 2 else 3)                  # an odd row stride: rows start on odd halves
    else:
        ld = dim + (2 if dim % 3 else 0)
    docs = []
    for k in range(32):                                    # every row count with every mask
        n = NS[k % 8]
        style = ("plain", "norms", "big", "tiny")[(k // 2) % 4]
        docs.append((_rows(rng, n, dim, dtype, style), _mask(MASKS[k // 8], n, rng), _heads(HEADS[k % 6], n, rng)))
    off = np.concatenate([[0], np.cumsum([len(x) for x, _, _ in docs])])
    X = np.zeros((int(off[-1]), ld), dtype)
    X[:, :dim] = np.concatenate([x for x, _, _ in docs])
    if ld > dim:
        X[:, dim:] = np.nan                                # the stride's padding must never be read
    non = np.concatenate([m for _, m, _ in docs])
    head = np.concatenate([h for _, _, h in docs])
    got, st, proj = _check(X, dim, off, non, head, (dtype, dim))
    assert (st == 0).all()
    n = np.diff(off)
    assert (got[off[1:][n > 0] - 1].view(np.uint32) == GUARD_BITS).all()   # the last row's slot keeps its guard
    if dim >= 2:
        assert proj.any() and not proj[n >= 2].all()       # both sides of the projection decision


# ---- the grid-stride loop ----------------------------------------------------------------------------------------------
def test_similarities_grid_stride_resets():
    """12 296 documents: every CTA runs three trips, some four.  CTAs 5 and 6 meet a zero-row document, a document with
    no selected row and one whose projection is skipped, in turn and in other orders, with ordinary documents after;
    each later document must find its flags reset.  Only the zero-row documents report status 1."""
    rng = np.random.default_rng(21)
    dim, D = 40, 3 * SIM_MAX_BLOCKS + 8
    docs = []
    for _ in range(D):
        n = int(rng.integers(0, 7))
        docs.append([_rows(rng, n, dim, np.float32, "plain"), co.nonoutlying(rng.integers(10, 400, size=n))
                     if n else np.zeros(0, bool), rng.random(n) < 0.2])

    def zero(n=5):
        X = _rows(rng, n, dim, np.float32, "plain")
        X[2] = 0
        return [X, np.ones(n, bool), np.zeros(n, bool)]

    def unselected(n=5):
        return [_rows(rng, n, dim, np.float32, "plain"), np.zeros(n, bool), np.zeros(n, bool)]

    def skipped(n=5):
        X = np.repeat(_rows(rng, 1, dim, np.float32, "plain"), n, axis=0)
        X[-1] = _rows(rng, 1, dim, np.float32, "plain")[0]
        return [X, np.r_[np.ones(n - 1, bool), False], np.zeros(n, bool)]   # identical selected rows: |y| = 0

    def ordinary(n=6):
        return [_rows(rng, n, dim, np.float32, "plain"), np.ones(n, bool), np.zeros(n, bool)]

    plan = {5: (zero, unselected, skipped, ordinary), 6: (skipped, ordinary, zero, ordinary),
            7: (unselected, zero, ordinary, skipped)}
    for cta, kinds in plan.items():
        for trip, make in enumerate(kinds):
            docs[cta + trip * SIM_MAX_BLOCKS] = make()
    off = np.concatenate([[0], np.cumsum([len(x) for x, _, _ in docs])])
    X = np.concatenate([x for x, _, _ in docs])
    got, st, proj = _check(X, dim, off, np.concatenate([m for _, m, _ in docs]),
                           np.concatenate([h for _, _, h in docs]), "grid stride")
    zeros = {cta + trip * SIM_MAX_BLOCKS for cta, kinds in plan.items() for trip, make in enumerate(kinds)
             if make is zero}
    assert set(np.nonzero(st)[0].tolist()) == zeros
    assert D > 3 * SIM_MAX_BLOCKS
    for cta, kinds in plan.items():
        for trip, make in enumerate(kinds):
            d = cta + trip * SIM_MAX_BLOCKS
            assert proj[d] == (make is ordinary), (cta, trip)
            if make is not zero:
                assert not np.isnan(got[off[d]:off[d + 1] - 1]).any(), (cta, trip)


# ---- the projection test's edge ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float16, np.float32])
def test_similarities_projection_eps_edge(dtype):
    """Projected norms of exactly FLT_EPSILON (skipped: the test is <=) and one step above it (kept), in one launch
    among ordinary documents; the reference's float32 NumPy takes the same decisions and gives the same costs."""
    rng = np.random.default_rng(31)
    dim = 40
    edge = co.EPS_EDGE[np.dtype(dtype)]
    docs = [(_rows(rng, 7, dim, dtype, "plain"), np.ones(7, bool))]
    for delta, _ in edge:
        docs += [(co.eps_edge_rows(delta, dim, dtype), co.EPS_EDGE_KEEP.astype(bool)),
                 (_rows(rng, 5, dim, dtype, "plain"), np.ones(5, bool))]
    off = np.concatenate([[0], np.cumsum([len(x) for x, _ in docs])])
    X = np.concatenate([x for x, _ in docs])
    non = np.concatenate([m for _, m in docs])
    head = np.zeros(len(X), bool)
    got, st, proj = _check(X, dim, off, non, head, "eps edge")
    assert (st == 0).all()
    for k, (delta, kept) in enumerate(edge):
        d = 1 + 2 * k
        assert proj[d] == kept and proj[d + 1], delta
        want = co.chunk_costs_f32_flags(docs[d][0], docs[d][1], head[:4])
        np.testing.assert_array_equal(got[off[d]:off[d + 1] - 1], want)
    assert [kept for _, kept in edge] == [False, True]    # both sides of the edge reached


# ---- the clamp -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float16, np.float32])
def test_similarities_clamp(dtype):
    """Adjacent antiparallel rows without a selected row: (s + 1) / 2 falls below sqrt(eps) and the cost is exactly
    float32 sqrt(eps), and a quarter of it where the next chunklet is a heading.  A NaN entry passes the host's zero-norm
    check (its norm is NaN, not 0); its costs stay NaN through the clamp, as NumPy's maximum keeps them."""
    rng = np.random.default_rng(41)
    dim = 33
    x = _rows(rng, 3, dim, dtype, "plain")
    anti = np.stack([x[0], -x[0], x[1], -x[1], x[2]])
    nan_rows = x.copy()
    nan_rows[1, 5] = np.nan
    docs = [(anti, np.array([0, 0, 0, 0, 0], bool)), (anti, np.array([0, 1, 0, 0, 0], bool)),
            (nan_rows, np.array([0, 0, 0], bool))]
    off = np.concatenate([[0], np.cumsum([len(x) for x, _ in docs])])
    X = np.concatenate([x for x, _ in docs])
    head = np.concatenate([h for _, h in docs])
    non = np.zeros(len(X), bool)
    got, st, _ = _check(X, dim, off, non, head, "clamp")
    assert (st == 0).all()
    sq = np.sqrt(np.float32(np.finfo(np.float32).eps))
    assert sq == co.SQRT_EPS32
    assert got[0] == sq and got[2] == sq                   # x0 . -x0 and x1 . -x1
    assert got[5] == sq / 4 and got[6] == 1                # the cut before the heading, then the heading's own
    assert np.isnan(got[10]) and np.isnan(got[11])
    for d, (rows, h) in enumerate(docs):
        want = co.chunk_costs_f32_flags(rows, non[off[d]:off[d + 1]], h)
        g = got[off[d]:off[d + 1] - 1]
        assert (np.isnan(g) == np.isnan(want)).all() and (g[want == sq] == sq).all(), d
