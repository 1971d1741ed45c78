"""``split_chunklets`` / ``split_chunks`` on the host: the restatements against the reference's own outputs
(``tests/golden/split_chunklets.npz`` and ``split_chunks.npz``), the windowed dynamic program against ``linprog``, the
``pow`` against ``d * d`` difference, every refusal before any CUDA call, and the restatement of
``rl_chunk_similarities`` that ``test_gpu_chunk_similarity_exact.py`` relies on (``fma64`` against exact fractions, the
restatement against float64 and the reference's costs, the planted rows of the projection test's edge)."""

from __future__ import annotations

import ctypes as C
import json
import math
import random
from fractions import Fraction

import chunks_oracle as co
import numpy as np
import pytest

from raglite_b200 import _chunks as K


def _cases(golden_dir, name: str):
    z = np.load(golden_dir / name)
    return json.loads(bytes(z["cases"]).decode()), z


def _cuts_of(pieces: list[str]) -> list[int]:
    return np.cumsum([len(p) for p in pieces])[:-1].tolist()


def _sentence_cuts(sentences: list[str], chunklets: list[str]) -> list[int]:
    ends = np.cumsum([len(s) for s in sentences]).tolist()
    return [ends.index(c) + 1 for c in _cuts_of(chunklets)]


# ---- chunklets -----------------------------------------------------------------------------------------------------------
def test_chunklet_restatement_reproduces_reference(golden_dir):
    cases, _ = _cases(golden_dir, "split_chunklets.npz")
    assert len(cases) > 40
    for c in cases:
        s = c["sentences"]
        if c["error"] is not None:
            with pytest.raises(ValueError, match=c["error"]):
                K.markdown_chunklet_boundaries(s)
            continue
        md = K.markdown_chunklet_boundaries(s)
        st = K.num_statements(s)
        assert md.tolist() == c["md"] and st.tolist() == c["statements"], c["name"]
        for square in ("mul", "pow"):
            cuts = co.chunklet_cuts(md, st, [len(x) for x in s], c["max_size"], square=square)
            assert ["".join(s[a:b]) for a, b in zip([0, *cuts], [*cuts, len(s)])] == c["chunklets"], (c["name"], square)


def test_chunklet_golden_covers_the_cases(golden_dir):
    cases, _ = _cases(golden_dir, "split_chunklets.npz")
    names = {c["name"] for c in cases}
    assert {"atx", "setext", "lists", "quotes", "consecutive", "whitespace", "long_middle", "long_first", "one",
            "empty"} <= names
    by = {(c["name"], c["max_size"]): c["chunklets"] for c in cases}
    assert [len(x) for x in by[("long_middle", 20)]] == [75, 5, 20]
    assert [len(x) for x in by[("long_first_short", 20)]] == [50, 5, 20]
    assert len({c["max_size"] for c in cases}) >= 4


def test_pow_and_square_differ_only_towards_the_correct_rounding():
    """The reference squares with NumPy's scalar power (C pow); the device multiplies.  They differ on a few values in
    a thousand, and the product, correctly rounded, is never the farther one."""
    rng = random.Random(5)
    xs = [rng.uniform(-5.0, 10.0) for _ in range(100_000)]
    diff = [x for x in xs if math.pow(x, 2.0) != x * x]
    assert np.float64(xs[0]) ** 2 == math.pow(xs[0], 2.0)    # NumPy's scalar power is C pow here
    assert diff, "pow is correctly rounded on this host: the difference this test pins is gone"
    for x in diff:
        exact = Fraction(x) ** 2
        assert abs(Fraction(x * x) - exact) <= abs(Fraction(math.pow(x, 2.0)) - exact)


# ---- chunks ----------------------------------------------------------------------------------------------------------
def test_chunk_restatement_reproduces_reference(golden_dir):
    cases, z = _cases(golden_dir, "split_chunks.npz")
    solved = 0
    for i, c in enumerate(cases):
        if not c["solved"]:
            continue
        solved += 1
        costs = co.chunk_costs_f32(c["chunklets"], z[f"emb{i}"])
        assert costs.dtype == np.float32 and np.array_equal(costs, z[f"cost{i}"]), c["name"]
        cuts, _ = co.linprog_cuts(costs, [len(x) for x in c["chunklets"]], c["max_size"])
        assert cuts == _cuts_of_chunks(c["chunklets"], c["chunks"]), c["name"]
    assert solved >= 40


def _cuts_of_chunks(chunklets: list[str], chunks: list[str]) -> list[int]:
    return _sentence_cuts(chunklets, chunks)


def test_window_dp_equals_linprog(golden_dir):
    cases, z = _cases(golden_dir, "split_chunks.npz")
    ties = 0
    for i, c in enumerate(cases):
        if not c["solved"]:
            continue
        costs, sizes = z[f"cost{i}"], [len(x) for x in c["chunklets"]]
        want = _cuts_of_chunks(c["chunklets"], c["chunks"])
        got = co.chunk_cuts(costs, sizes, c["max_size"])
        assert all(sum(sizes[a:b]) <= c["max_size"] for a, b in zip([0, *got], [*got, len(sizes)]))
        if got != want:
            a, b = co.objective(costs, got), co.objective(costs, want)
            assert a <= b and math.isclose(a, b, rel_tol=4 * co.EPS32), (c["name"], a, b)    # a tie
            ties += 1
        else:
            assert co.objective(costs, got) <= co.linprog_cuts(costs, sizes, c["max_size"])[1]
    assert ties <= 2


def test_chunk_golden_covers_the_cases(golden_dir):
    cases, z = _cases(golden_dir, "split_chunks.npz")
    errors = {c["name"]: c["error"] for c in cases if c["error"]}
    assert errors == {"too_long": K.CHUNKLET_TOO_LARGE, "zero_norm": K.ZERO_NORM}
    skipped = [c for i, c in enumerate(cases) if c["name"].startswith("identical")]
    assert skipped and all(c["solved"] for c in skipped)
    assert {z[f"emb{i}"].dtype for i in range(len(cases))} == {np.dtype(np.float16), np.dtype(np.float32)}
    assert any(co.is_heading(x) for c in cases for x in c["chunklets"])


def test_is_heading_matches_restatement():
    for s in ("# A", "## B\n", "\n# C", "#nospace", " # D ", "text # E", "#\tF", "####### G"):
        assert K.is_heading(s) == co.is_heading(s), s


# ---- refusals before any CUDA call ----------------------------------------------------------------------------------------
@pytest.fixture
def no_cuda(monkeypatch):
    import torch

    from raglite_b200 import _lib

    def boom(*a, **k):
        raise AssertionError("CUDA reached")

    monkeypatch.setattr(_lib, "load", boom)
    monkeypatch.setattr(torch.cuda, "current_device", boom)
    monkeypatch.setattr(torch.Tensor, "to", boom)


def test_refusals_before_cuda(no_cuda, golden_dir):
    with pytest.raises(NotImplementedError, match="boundary_cost / statement_cost"):
        K.split_chunklets(["a. ", "b. "], boundary_cost=lambda p: 0.0)
    with pytest.raises(NotImplementedError, match="boundary_cost / statement_cost"):
        K.split_chunklets(["a. ", "b. "], statement_cost=lambda s: 0.0)
    with pytest.raises(ValueError, match=K.EMPTY_DOCUMENT):
        K.split_chunklets([])
    with pytest.raises(ValueError, match=K.EMPTY_DOCUMENT):
        K.split_chunklets_batch([["a. "], []])
    cases, z = _cases(golden_dir, "split_chunks.npz")
    for i, c in enumerate(cases):
        if c["error"] is not None:
            with pytest.raises(ValueError, match=c["error"]):
                K.split_chunks(c["chunklets"], z[f"emb{i}"], max_size=c["max_size"])
    # both errors at once: the size check comes first, as in the reference
    e = np.zeros((2, 4), np.float16)
    with pytest.raises(ValueError, match=K.CHUNKLET_TOO_LARGE):
        K.split_chunks(["x" * 10, "y"], e, max_size=5)
    with pytest.raises(ValueError, match="max_size"):
        K.split_chunklets(["a. "], max_size=-1)


def test_early_exits_without_cuda(no_cuda, golden_dir):
    cases, z = _cases(golden_dir, "split_chunks.npz")
    for i, c in enumerate(cases):
        if c["error"] is None and not c["solved"]:
            chunks, embs = K.split_chunks(c["chunklets"], z[f"emb{i}"], max_size=c["max_size"])
            assert chunks == c["chunks"] and len(embs) == 1 and np.array_equal(embs[0], z[f"emb{i}"])
    chunks, embs = K.split_chunks([], np.zeros((0, 4), np.float16))
    assert chunks == [] and len(embs) == 1 and embs[0].shape == (0, 4)


RL_EINVAL, RL_ENOSPACE = -1, -3


def _abi():
    from raglite_b200 import _lib

    return _lib.load(), C.c_void_p(256)


def test_partition_refusals():
    lib, d = _abi()
    need = lib.rl_chunklet_partition_workspace_bytes(100, 3)
    assert need == 4 * 1024 + 512 == lib.rl_chunk_partition_workspace_bytes(100, 3)
    assert lib.rl_chunklet_partition_workspace_bytes(-1, 3) == 0 and lib.rl_chunk_partition_workspace_bytes(1, -1) == 0
    names = ("a", "b", "lens", "off", "max", "cuts", "counts", "status", "ws")

    def chunklet(D=3, N=100, ws_bytes=need, **ptr):
        p = {k: d for k in names} | ptr
        return lib.rl_chunklet_partition(p["a"], p["b"], p["lens"], p["off"], p["max"], D, N, p["cuts"], p["counts"],
                                         p["status"], p["ws"], ws_bytes, None)

    def chunk(D=3, N=100, ws_bytes=need, **ptr):
        p = {k: d for k in names} | ptr
        return lib.rl_chunk_partition(p["a"], p["lens"], p["off"], p["max"], D, N, p["cuts"], p["counts"],
                                      p["status"], p["ws"], ws_bytes, None)

    for f, used in ((chunklet, names), (chunk, ("a", "lens", "off", "max", "cuts", "counts", "status", "ws"))):
        assert f(D=-1) == RL_EINVAL and f(N=-1) == RL_EINVAL
        for k in used:
            assert f(**{k: None}) == RL_EINVAL, k
            assert "null pointer" in lib.rl_last_error().decode()
        assert f(ws_bytes=need - 1) == RL_ENOSPACE
        assert "workspace too small" in lib.rl_last_error().decode()
        assert f(D=0, ws_bytes=0, **{k: None for k in names}) == 0


def test_similarities_refusals():
    lib, d = _abi()
    need = lib.rl_chunk_similarities_workspace_bytes(100)
    assert need == 3 * 512 and lib.rl_chunk_similarities_workspace_bytes(-1) == 0
    names = ("X", "off", "non", "head", "costs", "status", "ws")

    def sim(dtype=1, ld=64, dim=64, D=3, N=100, ws_bytes=need, **ptr):
        p = {k: d for k in names} | ptr
        return lib.rl_chunk_similarities(p["X"], dtype, ld, dim, p["off"], D, N, p["non"], p["head"], p["costs"],
                                         p["status"], p["ws"], ws_bytes, None)

    for bad in (dict(dtype=2), dict(dtype=-1), dict(D=-1), dict(N=-1), dict(dim=0), dict(ld=63), dict(dim=8193, ld=8193)):
        assert sim(**bad) == RL_EINVAL, bad
    assert "dim <= 8192" in lib.rl_last_error().decode()
    for k in names:
        assert sim(**{k: None}) == RL_EINVAL, k
    assert sim(ws_bytes=need - 1) == RL_ENOSPACE
    assert sim(D=0, ws_bytes=0, **{k: None for k in names}) == 0


# ---- the lane-exact restatement of rl_chunk_similarities -------------------------------------------------------------
def _fma_exact64(a, b, c) -> np.ndarray:
    """a b + c in exact rational arithmetic, rounded once (``float`` of a Fraction is correctly rounded, ties to even)."""
    return np.array([float(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z)))
                     for x, y, z in zip(a, b, c, strict=True)])


def test_fma64_against_fractions():
    """``chunks_oracle.fma64`` is a correctly rounded a b + c: random triples with magnitudes from 2^-60 to 2^60, c
    close to -a b (cancellation), and planted triples whose exact value is a float64 midpoint, or one ulp of the
    product's error term off it."""
    rng = np.random.default_rng(11)
    n = 6000
    a, b, c = (rng.standard_normal(n) * 2.0 ** rng.integers(-60, 61, n) for _ in range(3))
    near = rng.random(n) < 0.4
    c[near] = -(a[near] * b[near]) * (1 + rng.standard_normal(near.sum()) * 2.0 ** rng.integers(-52, -20, near.sum()))
    np.testing.assert_array_equal(co.fma64(a, b, c), _fma_exact64(a, b, c))
    # midpoints: a b within a rounding of half an ulp of c, a with a 26-bit significand, so a (h / a) = h (1 + delta)
    # with |delta| <= 2^-53: exactly on the midpoint (a a power of two) or just off it, on either side
    c = rng.standard_normal(n) * 2.0 ** rng.integers(-40, 41, n)
    h = (np.nextafter(np.abs(c), np.inf) - np.abs(c)) / 2 * np.where(rng.random(n) < 0.5, -1.0, 1.0)
    a = np.ldexp(rng.integers(2**25, 2**26, n).astype(np.float64), -25) * 2.0 ** rng.integers(-20, 21, n)
    a[: n // 4] = 2.0 ** rng.integers(-20, 21, n // 4)
    b = h / a
    step = rng.integers(-1, 2, n)
    b = np.where(step > 0, np.nextafter(b, np.inf), np.where(step < 0, np.nextafter(b, -np.inf), b))
    want = _fma_exact64(a, b, c)
    np.testing.assert_array_equal(co.fma64(a, b, c), want)
    assert ((a * b + c) != want).sum() > n // 20               # the two-rounding answer is often wrong here
    # an exact zero: +0 but for (-0) + (-0), as IEEE round-to-nearest gives
    z = co.fma64([2.0, -0.0, 0.0, 3.0], [3.0, 1.0, -1.0, 2.0**-30], [-6.0, -0.0, -0.0, -3.0 * 2.0**-30])
    assert z.view(np.uint64).tolist() == [0, 1 << 63, 1 << 63, 0]


def _random_doc(rng, n: int, dim: int, dtype):
    centers = rng.standard_normal((3, dim))
    X = centers[rng.integers(0, 3, size=n)] + rng.standard_normal((n, dim))
    return (X * 2.0 ** rng.integers(-6, 7, size=(n, 1))).astype(dtype)


def test_chunk_costs_device_within_float64_bound():
    """The restatement computes the cost formula: within ``chunk_cost_bound`` of ``chunk_costs_f64`` per document (the
    rows of each document at their own scale), fp16 and fp32 rows, widths off and on the multiples of 32 and 256."""
    rng = np.random.default_rng(12)
    for dtype in (np.float16, np.float32):
        for dim in (2, 31, 33, 257, 1000):
            docs = [_random_doc(rng, int(n), dim, dtype) for n in rng.integers(2, 40, size=12)]
            keeps = [rng.random(len(X)) < 0.7 for X in docs]
            heads = [rng.random(len(X)) < 0.2 for X in docs]
            off = np.concatenate([[0], np.cumsum([len(X) for X in docs])])
            got, status, proj = co.chunk_costs_device(np.concatenate(docs), dim, off, np.concatenate(keeps),
                                                      np.concatenate(heads))
            assert (status == 0).all()
            for i, (X, keep, head) in enumerate(zip(docs, keeps, heads, strict=True)):
                want, info = co.chunk_costs_f64(X, keep, head)
                g = got[off[i]:off[i + 1]]
                assert np.isnan(g[-1]) and proj[i] == info["proj"], (dtype, dim, i)
                err = np.abs(g[:-1] - want)
                assert (err <= co.chunk_cost_bound(dim, int(keep.sum()), info)).all(), (dtype, dim, i)


def test_chunk_costs_device_on_golden_cases(golden_dir):
    """On the reference's own cases, the restatement's costs are within the bound of the reference's float32 costs
    wherever both take the same projection decision (every case but those where a row's exact projection is zero)."""
    cases, z = _cases(golden_dir, "split_chunks.npz")
    checked = 0
    for i, c in enumerate(cases):
        if not c["solved"]:
            continue
        X = z[f"emb{i}"]
        keep = co.nonoutlying([len(x) for x in c["chunklets"]])
        head = np.array([co.is_heading(x) for x in c["chunklets"]])
        got, status, proj = co.chunk_costs_device(X, X.shape[1], [0, len(X)], keep, head)
        _, info = co.chunk_costs_f64(X, keep, head)
        assert status[0] == 0 and proj[0] == info["proj"], c["name"]
        if keep.any() and float(info["pn_all"].min()) < 1e-9:
            continue                                                      # the reference's test follows rounding
        err = np.abs(got[:-1].astype(np.float64) - z[f"cost{i}"])
        assert (err <= co.chunk_cost_bound(X.shape[1], int(keep.sum()), info)).all(), c["name"]
        checked += 1
    assert checked >= 40



@pytest.mark.parametrize("dtype", [np.float16, np.float32])
def test_projection_edge_rows_decide_alike(dtype):
    """The planted rows of the projection test's edge: the restatement skips the projection at |y| = eps and keeps it
    one step above, and the reference's float32 NumPy (run on the same mask) takes the same decisions and costs."""
    for delta, kept in co.EPS_EDGE[np.dtype(dtype)]:
        X = co.eps_edge_rows(delta, 40, dtype)
        head = np.zeros(4, bool)
        got, status, proj = co.chunk_costs_device(X, 40, [0, 4], co.EPS_EDGE_KEEP, head)
        assert status[0] == 0 and proj[0] == kept, delta
        want = co.chunk_costs_f32_flags(X, co.EPS_EDGE_KEEP, head)
        np.testing.assert_array_equal(got[:-1], want)
        assert (want[:2] == co.SQRT_EPS32).all() == kept       # kept: rows 0 and 1 project onto -e1 and e1
