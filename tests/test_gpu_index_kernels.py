"""The index-side kernels against float64 NumPy, to the last rounding (``tests/rounding.py``): ``rl_row_stats`` /
``rl_row_stats_f16``, ``rl_chunk_row_map``, ``rl_row_mask``, ``rl_adapter_apply``, ``rl_segment_mean_pool`` and
``rl_best_vectors``, called through the C-ABI at the shapes, strides, alignments and values where their code paths
split (vector body / scalar path / ragged tail / grid-stride loop / shared-memory opt-in / size limits)."""

from __future__ import annotations

import numpy as np
import pytest
import rounding as rd
from synth import make_corpus, make_queries, random_orthogonal

from oracle import vector_search as ovs

pytestmark = pytest.mark.gpu

RL_EINVAL, RL_EUNSUPPORTED = -1, -4
STATS_WARPS = 132 * 16 * 8          # rl_row_stats: grid cap x warps per block = rows before the grid-stride loop wraps
MASK_ROWS = 132 * 8 * 256 * 16      # rl_row_mask: rows one pass of the capped grid covers


@pytest.fixture(scope="module")
def lib():
    import torch

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from raglite_b200 import _lib

    return _lib.load()


@pytest.fixture(scope="module", autouse=True)
def _two_value_report():
    yield
    print("\ntwo-value branch maxima (count, entries):", dict(sorted(rd.TWO_VALUE_MAX.items())))


def _stream():
    import torch

    return torch.cuda.current_stream().cuda_stream


def _dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _check(rc, what):
    from raglite_b200 import _lib

    _lib.check(rc, what)


# ---- rl_row_stats / rl_row_stats_f16 --------------------------------------------------------------------------------
def _strided(rows: np.ndarray, ld: int, offset: int, fill) -> tuple[np.ndarray, np.ndarray]:
    """``rows`` laid out with leading dimension ``ld`` behind ``offset`` elements; padding and prefix hold ``fill``
    (NaN: a kernel that reads outside the d columns of a row gets a NaN statistic)."""
    n, d = rows.shape
    flat = np.full(offset + n * ld, fill, dtype=rows.dtype)
    flat[offset:].reshape(n, ld)[:, :d] = rows
    return flat, flat[offset:].reshape(n, ld)[:, :d]


def _run_row_stats(lib, flat: np.ndarray, offset: int, n: int, d: int, ld: int):
    import torch

    f16 = flat.dtype == np.float16
    E = _dev(flat)
    inv = torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")
    sq = torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")
    st = torch.zeros(4, dtype=torch.float32, device="cuda")
    fn = lib.rl_row_stats_f16 if f16 else lib.rl_row_stats
    _check(fn(E.data_ptr() + offset * flat.itemsize, n, d, ld, inv.data_ptr(), sq.data_ptr(), st.data_ptr(), _stream()),
           "rl_row_stats")
    return inv.cpu().numpy(), sq.cpu().numpy(), st.cpu().numpy()


def _sum_sq_bound(X: np.ndarray, S: np.ndarray) -> np.ndarray:
    """Bound on the difference of two float64 sums of a row's exact squares S = sum x^2 taken in different orders.
    Every square is a multiple of m^2, m = the row's smallest ulp(x) over its non-zero entries: when S < 2^53 m^2 every
    partial sum of either order is exact, and the bound is 0 (such sums often sit exactly on a float32 midpoint, which
    any positive bound would turn into a two-value case).  Otherwise no term passes through more than d - 1
    additions: 2 gamma_{d-1} S."""
    A = np.abs(X)
    m = np.where(A > 0, np.spacing(A).astype(np.float64), np.inf).min(axis=1)
    return np.where(S < 2.0 ** 53 * m * m, 0.0, 2 * rd.gamma(X.shape[1] - 1) * S)


def _check_row_stats(X: np.ndarray, inv: np.ndarray, sq: np.ndarray, st: np.ndarray, tag: str) -> None:
    """X: the n rows as stored (float32 or float16); the sum of squares within ``_sum_sq_bound``.  1/|e| and |e| add
    a sqrt and a division per side, and the sqrt halves the relative error of S: 2 gamma_{d+4} |value| bounds those."""
    d = X.shape[1]
    X64 = X.astype(np.float64)
    S = np.einsum("ij,ij->i", X64, X64)
    rd.check(sq, S, _sum_sq_bound(X, S), rd.f32, what=f"row_stats sq_norm {tag}")
    nz = S > 0
    with np.errstate(divide="ignore"):
        inv_v = np.where(nz, 1.0 / np.sqrt(S), 0.0)
    rd.check(inv, inv_v, 2 * rd.gamma(d + 4) * inv_v, rd.f32, what=f"row_stats inv_norm {tag}")
    nmax = np.sqrt(S.max())
    rd.check(st[0], nmax, 2 * rd.gamma(d + 4) * nmax, rd.f32, what=f"row_stats stats[0] {tag}")
    assert st[1] == np.abs(X).max().astype(np.float32), (tag, st[1])
    imax = 1.0 / np.sqrt(S[nz].min()) if nz.any() else 0.0
    rd.check(st[2], imax, 2 * rd.gamma(d + 4) * imax, rd.f32, what=f"row_stats stats[2] {tag}")
    assert st[3] == (0.0 if nz.all() else 1.0), (tag, st[3])


def _stats_rows(n: int, d: int, variant: str, dtype, seed: int) -> np.ndarray:
    """Rows whose statistics are set by planted rows at positions handled by warps other than a block's first one,
    in the first pass of the grid and in later ones."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d), dtype=np.float32)
    X /= np.maximum(np.linalg.norm(X, axis=1, keepdims=True), 1e-30)
    if variant == "gate":        # unit-ish rows + a zero row, a row of norm 0.4, a row holding 1024.5 (1025 in fp16)
        X *= rng.uniform(0.6, 1.5, size=(n, 1)).astype(np.float32)
        plant = {59: 0.0, 406: 0.4, 1234: None}
        big = 1025.0 if dtype == np.float16 else 1024.5
    else:                        # norms log-uniform over the type's range, a zero row
        lo, hi = (-3.0, 3.0) if dtype == np.float16 else (-20.0, 18.0)
        X *= (10.0 ** rng.uniform(lo, hi, size=(n, 1))).astype(np.float32)
        plant = {8 * 97 + 5: 0.0, STATS_WARPS + 8 * 11 + 3: 0.0}
        big = None
    for r, nrm in plant.items():
        if r >= n:
            continue
        if nrm is None:
            X[r] = X[r] * 0.5
            X[r, r % d] = big
        else:
            X[r] *= nrm / max(float(np.linalg.norm(X[r])), 1e-30)
    extreme = {n - 1: 3.0, STATS_WARPS + 8 * 40 + 6: 2.5}          # largest norms, later grid-stride passes
    if variant == "range":
        extreme = {n - 1: 1e18 if dtype == np.float32 else 5e3, 8 * 300 + 7: 1e-20 if dtype == np.float32 else 2e-3}
    for r, nrm in extreme.items():
        if 0 <= r < n and r not in plant:
            X[r] *= nrm / max(float(np.linalg.norm(X[r])), 1e-30)
    return X.astype(dtype)


@pytest.mark.parametrize("variant", ["gate", "range"])
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("pad", [0, 3])
@pytest.mark.parametrize("d", [1, 3, 4, 100, 1024, 1027])
def test_row_stats_fp32_against_float64(lib, d, pad, offset, variant):
    ld = d + pad
    n_max = 40000 if d <= 100 else STATS_WARPS + 1
    X = _stats_rows(n_max, d, variant, np.float32, seed=d * 10 + pad + offset)
    flat, _ = _strided(X, ld, offset, np.float32(np.nan))
    for n in (1, STATS_WARPS, STATS_WARPS + 1, 40000):
        if n > n_max:
            continue
        inv, sq, st = _run_row_stats(lib, flat[: offset + n * ld], offset, n, d, ld)
        _check_row_stats(X[:n], inv, sq, st, f"fp32 d={d} ld={ld} off={offset} n={n} {variant}")


@pytest.mark.parametrize("variant", ["gate", "range"])
@pytest.mark.parametrize("pad", [0, 8])
@pytest.mark.parametrize("d", [8, 72, 1024])
def test_row_stats_fp16_against_float64(lib, d, pad, variant):
    ld = d + pad
    n_max = 40000 if d <= 72 else STATS_WARPS + 1
    X = _stats_rows(n_max, d, variant, np.float16, seed=d + pad)
    flat, _ = _strided(X, ld, 0, np.float16(np.nan))
    for n in (1, STATS_WARPS, STATS_WARPS + 1, 40000):
        if n > n_max:
            continue
        inv, sq, st = _run_row_stats(lib, flat[: n * ld], 0, n, d, ld)
        _check_row_stats(X[:n], inv, sq, st, f"fp16 d={d} ld={ld} n={n} {variant}")


def test_row_stats_fp16_refuses_unaligned_layouts(lib):
    import torch

    E = torch.zeros(64 * 40, dtype=torch.float16, device="cuda")
    out = torch.zeros(64, dtype=torch.float32, device="cuda")
    st = torch.zeros(4, dtype=torch.float32, device="cuda")
    for d, ld, off in ((12, 16, 0), (16, 20, 0), (16, 16, 1)):
        rc = lib.rl_row_stats_f16(E.data_ptr() + 2 * off, 8, d, ld, out.data_ptr(), out.data_ptr(), st.data_ptr(), _stream())
        assert rc == RL_EUNSUPPORTED, (d, ld, off, rc)
    assert lib.rl_row_stats(E.data_ptr(), 8, 16, 8, out.data_ptr(), out.data_ptr(), st.data_ptr(), _stream()) == RL_EINVAL


def test_row_stats_fold_across_append_and_compact():
    import raglite_b200 as rl

    d = 64
    E, off = make_corpus(3000, 1, d, seed=21)
    ids = [f"c{i}" for i in range(3000)]
    idx = rl.CorpusIndex(E, off, chunk_ids=ids, storage="fp32")
    assert idx.rows_unit_scale
    st0 = idx.stats.cpu().numpy().copy()
    q = make_queries(E, 1, seed=22)[0]
    small = (0.4 * q / np.linalg.norm(q)).astype(np.float32)        # the nearest row by cosine, norm 0.4
    idx.append(small[None], chunk_ids=["small"])
    both = np.concatenate([E, small[None]])
    _check_row_stats(both, idx.inv_norm.cpu().numpy(), idx.sq_norm.cpu().numpy(), idx.stats.cpu().numpy(), "append")
    assert abs(idx.stats.cpu().numpy()[2] - 2.5) < 1e-5 and not idx.rows_unit_scale
    cfg = rl.RAGLiteConfig(reranker=None)
    for algo in ("fp32", "auto"):
        got, sims, _ = rl.vector_search_batch(q[None], num_results=3, config=cfg, index=idx, algo=algo)
        assert got[0, 0] == 3000 and abs(sims[0, 0] - 1.0) < 1e-5, (algo, got[0], sims[0])
    idx.delete_chunks(["small"])
    idx.compact()
    assert idx.rows_unit_scale and idx.n_rows == 3000
    assert np.array_equal(idx.stats.cpu().numpy(), st0)
    _check_row_stats(E, idx.inv_norm.cpu().numpy(), idx.sq_norm.cpu().numpy(), idx.stats.cpu().numpy(), "compact")
    # the max-|x| gate: 1024 keeps rows unscaled, 1024.5 does not
    for big, unit in ((1024.0, True), (1024.5, False)):
        row = np.zeros((1, d), np.float32)
        row[0, 5] = big
        j = rl.CorpusIndex(np.concatenate([E, row]), storage="fp32")
        assert j.stats.cpu().numpy()[1] == np.float32(big) and j.rows_unit_scale == unit, (big, j.stats)


# ---- rl_chunk_row_map -----------------------------------------------------------------------------------------------
def test_chunk_row_map_against_row_to_chunk(lib):
    import torch

    rng = np.random.default_rng(31)
    C = 132 * 8 * 256 + 5000                                    # more chunks than one pass of the capped grid
    counts = rng.integers(0, 4, size=C).astype(np.int64)        # a quarter of the chunks are empty
    counts[:3] = 0
    counts[-2:] = 0
    counts[1234] = 70000                                        # one long chunk: a single thread writes its rows
    for off in (np.array([0, 0, 3, 3, 5, 5], np.int64), np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)):
        n = int(off[-1])
        rc_dev = torch.full((n + 64,), -7, dtype=torch.int32, device="cuda")
        off_dev = _dev(off)
        _check(lib.rl_chunk_row_map(off_dev.data_ptr(), len(off) - 1, rc_dev.data_ptr(), _stream()), "rl_chunk_row_map")
        got = rc_dev.cpu().numpy()
        assert np.array_equal(got[:n], ovs.row_to_chunk(off).astype(np.int32))
        assert np.all(got[n:] == -7)


# ---- rl_row_mask ----------------------------------------------------------------------------------------------------
ALIVE_BYTES = np.array([0, 1, 0x02, 0x80, 0xFF], np.uint8)
OK_BYTES = np.array([0, 1, 2, 255], np.uint8)


def _run_row_mask(lib, chunk_ok, row_chunk, alive, n, *, out_off=0, rc_off=0):
    import torch

    guard = 48
    out = torch.full((n + guard + 16,), 0xA5, dtype=torch.uint8, device="cuda")
    ptr = lambda t, o=0: None if t is None else t.data_ptr() + o   # noqa: E731
    rc = lib.rl_row_mask(ptr(chunk_ok), ptr(row_chunk, rc_off), ptr(alive), n, out.data_ptr() + out_off, _stream())
    return rc, out.cpu().numpy()


@pytest.mark.parametrize("n", [1, 15, 16, 17, MASK_ROWS + 17])
def test_row_mask_bit_exact(lib, n):
    rng = np.random.default_rng(n)
    n_chunks = max(1, n // 3)
    rotations = range(5) if n < 64 else range(1)
    for rot in rotations:
        row_chunk = rng.integers(0, n_chunks, size=n).astype(np.int32)
        chunk_ok = OK_BYTES[rng.integers(0, 4, size=n_chunks)]
        if n < 64:     # every alive byte value in every byte lane of a 16-byte word across the rotations
            alive = ALIVE_BYTES[(np.arange(n) + rot) % 5]
        else:
            alive = ALIVE_BYTES[rng.integers(0, 5, size=n)]
        dev = {"ok": _dev(chunk_ok), "rc": _dev(row_chunk), "alive": _dev(alive)}
        for use_ok in (True, False):
            for use_alive in (True, False):
                want = np.ones(n, bool)
                if use_ok:
                    want &= chunk_ok[row_chunk] != 0
                if use_alive:
                    want &= alive != 0
                rc, out = _run_row_mask(lib, dev["ok"] if use_ok else None, dev["rc"] if use_ok else None,
                                        dev["alive"] if use_alive else None, n)
                assert rc == 0
                tag = (n, rot, use_ok, use_alive)
                bad = np.flatnonzero(out[:n] != want.astype(np.uint8))
                assert bad.size == 0, (tag, bad[:8], out[bad[:8]], want[bad[:8]])
                assert np.all(out[n:] == 0xA5), tag                       # nothing written past n_rows


def test_row_mask_refuses_misaligned_pointers(lib):
    n = 40
    ok = _dev(np.ones(4, np.uint8))
    row_chunk = _dev(np.zeros(n + 8, np.int32))
    alive = _dev(np.ones(n + 16, np.uint8))
    rc, out = _run_row_mask(lib, ok, row_chunk, alive, n, out_off=1)
    assert rc == RL_EINVAL and np.all(out == 0xA5)
    rc, out = _run_row_mask(lib, ok, row_chunk, alive, n, rc_off=4)
    assert rc == RL_EINVAL and np.all(out == 0xA5)


# ---- rl_adapter_apply -----------------------------------------------------------------------------------------------
def _run_adapter(lib, A_dev, Q: np.ndarray, mode: int) -> np.ndarray:
    import torch

    B, d = Q.shape
    out = torch.full((B, d), float("nan"), dtype=torch.float32, device="cuda")
    Q_dev = _dev(Q)
    _check(lib.rl_adapter_apply(A_dev.data_ptr(), Q_dev.data_ptr(), out.data_ptr(), B, d, mode, _stream()),
           "rl_adapter_apply")
    return out.cpu().numpy()


@pytest.mark.parametrize("d", [1, 31, 96, 1536, 1537, 4096, 6400])
def test_adapter_apply_both_round_modes_against_float64(lib, d):
    rng = np.random.default_rng(d)
    A = rng.standard_normal((d, d)) / np.sqrt(d)
    Q = rng.standard_normal((300, d)).astype(np.float32)
    Q[::7] *= np.float32(30000.0)                 # some outputs beyond the fp16 range: +-inf, like astype(float16)
    want = Q.astype(np.float64) @ A.T
    # Both sides form a length-d float64 dot product.  The kernel's lane runs ceil(d/32) fused multiply-adds, then a
    # 5-level shuffle tree: no term passes through more than ceil(d/32) + 5 roundings.  NumPy's BLAS: at most d.
    # So b = (gamma_{ceil(d/32)+5} + gamma_d) sum_j |A_ij q_j|.
    b = (rd.gamma(-(-d // 32) + 5) + rd.gamma(d)) * (np.abs(Q).astype(np.float64) @ np.abs(A).T)
    A_dev = _dev(A)
    for B in (1, 7, 8, 9, 300):
        for mode, chain in ((0, rd.f32), (1, rd.f16)):
            got = _run_adapter(lib, A_dev, Q[:B], mode)
            rd.check(got, want[:B], b[:B], chain, what=f"adapter_apply mode={mode} d={d}")


def test_adapter_apply_fp16_overflow_and_double_rounding(lib):
    d = 96
    rng = np.random.default_rng(5)
    A = rng.standard_normal((d, d)) / np.sqrt(d)
    A[:8, :] = 0.0
    t = 2.0 ** -11
    A[0, 0] = 65520.0                              # exactly the fp16 overflow threshold: rounds to inf
    A[1, 0] = -65520.0
    A[2, 0] = np.nextafter(65520.0, 0.0)           # just below it: 65504
    A[3, :3] = [1.0, t, 2.0 ** -40]                # just past the midpoint 1 + 2^-11; float32 would land on it
    A[4, :3] = [-1.0, -t, -(2.0 ** -40)]
    A[5, :3] = [1.0, 3 * t, -(2.0 ** -40)]         # just below the midpoint 1 + 3 2^-11; float32 would tie up
    A[6, :2] = [2.0 ** -25, 2.0 ** -70]            # just past half the smallest fp16 subnormal
    A[7, :2] = [3 * 2.0 ** -25, -(2.0 ** -70)]     # just below 1.5 subnormals
    Q = rng.standard_normal((9, d)).astype(np.float32)
    Q[:, :3] = np.array([1.0, -1.0, 2.0, 4.0, 1.0, -2.0, 1.0, 1.0, 8.0], np.float32)[:, None]
    exact = Q.astype(np.float64) @ A[:8].T        # powers of two times <= 3 terms: every partial sum exact
    got16 = _run_adapter(lib, _dev(A), Q, 1)
    assert np.array_equal(got16[:, :8], rd.f16(exact).astype(np.float32), equal_nan=True), (got16[:, :8], rd.f16(exact))
    via_f32 = exact.astype(np.float32).astype(np.float16).astype(np.float32)
    assert (via_f32 != got16[:, :8]).sum() >= 9      # the cases do separate one rounding from two
    assert np.isinf(got16[:, :2]).all()
    got32 = _run_adapter(lib, _dev(A), Q, 0)
    assert np.array_equal(got32[:, :8], exact.astype(np.float32))


def test_adapter_apply_refuses_d_6401(lib):
    import torch

    d = 6401
    A = torch.zeros((d, d), dtype=torch.float64, device="cuda")
    Q = torch.zeros((1, d), dtype=torch.float32, device="cuda")
    out = torch.full((1, d), 7.0, dtype=torch.float32, device="cuda")
    for mode in (0, 1):
        assert lib.rl_adapter_apply(A.data_ptr(), Q.data_ptr(), out.data_ptr(), 1, d, mode, _stream()) == RL_EUNSUPPORTED
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())


def test_adapter_through_search_with_fp16_queries():
    from dataclasses import replace

    import torch

    import raglite_b200 as rl

    d = 64
    E, off = make_corpus(3000, 1, d, seed=41, fp16_round=True)
    A = random_orthogonal(d, seed=42)
    idx = rl.CorpusIndex(E, off)
    idx.set_query_adapter(A)
    Qh = make_queries(E, 16, seed=43).astype(np.float16)
    Q32 = Qh.astype(np.float32)                                         # float32 values exactly representable in fp16
    oracle_q = np.stack([ovs.apply_query_adapter(A, q) for q in Qh])    # (A @ q).astype(float16)
    got_q = idx.apply_adapter(torch.from_numpy(Q32).cuda(), round_fp16=True).cpu().numpy()
    b = (rd.gamma(-(-d // 32) + 5) + rd.gamma(d)) * (np.abs(Q32).astype(np.float64) @ np.abs(A).T)
    rd.check(got_q, Q32.astype(np.float64) @ A.T, b, rd.f16, what="adapter_apply search queries")
    assert np.array_equal(got_q, oracle_q.astype(np.float32))
    cfg = rl.RAGLiteConfig(reranker=None)
    r32 = rl.vector_search_batch(Q32, num_results=10, config=cfg, index=idx, queries_are_fp16=True)
    r16 = rl.vector_search_batch(Qh, num_results=10, config=cfg, index=idx)
    plain = rl.vector_search_batch(oracle_q.astype(np.float32), num_results=10, index=idx,
                                   config=replace(cfg, vector_search_query_adapter=False))
    for got in (r32, r16):
        for x, y in zip(got, plain, strict=True):
            assert np.array_equal(x, y)


# ---- rl_segment_mean_pool -------------------------------------------------------------------------------------------
def _pool_oracle(X: np.ndarray, rb: np.ndarray, re: np.ndarray, normalize: int) -> tuple[np.ndarray, np.ndarray]:
    """The kernel's arithmetic restated in float64: a sequential row sum per column (NumPy's axis-0 order, the same
    adds in the same order: the means match bit for bit), the mean, then the norm (summation order differs: each
    side within gamma_d of sum m^2, plus a sqrt and a division each -> 2 gamma_{d+4} |value|), clamped to eps at
    normalize = 2."""
    X64 = X.astype(np.float64)
    S, d = len(rb), X.shape[1]
    means = np.empty((S, d))
    lens = re - rb
    with np.errstate(invalid="ignore", divide="ignore"):
        for L in np.unique(lens):
            sel = np.flatnonzero(lens == L)
            acc = np.zeros((len(sel), d))
            for j in range(int(L)):
                acc += X64[rb[sel] + j]
            means[sel] = acc / float(L)
        if normalize == 0:
            return means, np.zeros_like(means)
        nrm = np.sqrt((means * means).sum(axis=1))
        if normalize == 2:
            nrm = np.where(np.isnan(nrm), nrm, np.maximum(nrm, 2.220446049250313e-16))
        v = means / nrm[:, None]
    return v, 2 * rd.gamma(d + 4) * np.abs(v)


def _run_pool(lib, flat: np.ndarray, offset: int, ld: int, d: int, rb, re, normalize: int) -> np.ndarray:
    import torch

    S = len(rb)
    out = torch.full((S, d), float("nan"), dtype=torch.float16, device="cuda")
    X, rb_dev, re_dev = _dev(flat), _dev(rb.astype(np.int32)), _dev(re.astype(np.int32))   # alive until the kernel ran
    _check(lib.rl_segment_mean_pool(X.data_ptr() + 4 * offset, ld, d, rb_dev.data_ptr(), re_dev.data_ptr(), S, normalize,
                                         out.data_ptr(), _stream()), "rl_segment_mean_pool")
    return out.cpu().numpy()


def _segments(n_rows: int, long: int, rng) -> tuple[np.ndarray, np.ndarray]:
    segs = [(10, 10), (5, 6), (10, 13), (3, 7), (7, 12), (2, 9), (4, 11), (20, 22), (0, 1)]   # empty, 1, 3, 4, 5 rows; overlaps
    if long:
        segs.append((n_rows - long, n_rows))
    for _ in range(12):
        a = int(rng.integers(0, n_rows - 6))
        segs.append((a, a + int(rng.integers(0, 6))))
    segs = segs[::-1]                                                               # out of order
    rb, re = (np.array(x, np.int64) for x in zip(*segs, strict=True))
    return rb, re


@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("pad", [0, 1])
@pytest.mark.parametrize("d", [3, 4, 1024, 4097, 25600])
def test_segment_mean_pool_against_float64(lib, d, pad, offset):
    rng = np.random.default_rng(d + 7 * pad + offset)
    long = 3000 if d <= 4097 else 0
    n_rows = long + 40
    X = rng.standard_normal((n_rows, d), dtype=np.float32)
    X[21] = -X[20]                                       # segment (20, 22): mean exactly zero
    ld = d + pad
    flat, _ = _strided(X, ld, offset, np.float32(np.nan))
    rb, re = _segments(n_rows, long, rng)
    for normalize in (0, 1, 2):
        got = _run_pool(lib, flat, offset, ld, d, rb, re, normalize)
        v, b = _pool_oracle(X, rb, re, normalize)
        rd.check(got, v, b, rd.f16, what=f"segment_mean_pool normalize={normalize} d={d}")
        z = int(np.flatnonzero((rb == 20) & (re == 22))[0])
        e = int(np.flatnonzero(rb == re)[0])
        assert np.isnan(got[e]).all()                                   # empty sentence: NaN, like np.mean
        if normalize == 1:
            assert np.isnan(got[z]).all()                               # 0 / 0
        else:
            assert (got[z] == 0).all()                                  # normalize=2 clamps the norm to eps


@pytest.mark.parametrize("d", [3, 4])
def test_segment_mean_pool_70000_segments(lib, d):
    rng = np.random.default_rng(70 + d)
    X = rng.standard_normal((1000, d), dtype=np.float32)
    S = 70000
    rb = rng.integers(0, 995, size=S)
    re = rb + rng.integers(0, 6, size=S)
    for normalize in (0, 2):
        got = _run_pool(lib, X.ravel(), 0, d, d, rb, re, normalize)
        v, b = _pool_oracle(X, rb, re, normalize)
        rd.check(got, v, b, rd.f16, what=f"segment_mean_pool S=70000 normalize={normalize}")


def test_segment_mean_pool_refuses_d_25601(lib):
    import torch

    d = 25601
    X = torch.zeros((1, d), dtype=torch.float32, device="cuda")
    r = torch.zeros(1, dtype=torch.int32, device="cuda")
    out = torch.full((1, d), 7.0, dtype=torch.float16, device="cuda")
    rc = lib.rl_segment_mean_pool(X.data_ptr(), d, d, r.data_ptr(), r.data_ptr(), 1, 1, out.data_ptr(), _stream())
    assert rc == RL_EUNSUPPORTED
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())                     # refused before any launch: nothing written


# ---- rl_best_vectors ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,ld,fp16", [(1, 3, False), (33, 40, False), (1024, 1030, False), (8, 8, True), (1024, 1032, True)])
def test_best_vectors_pick_first_maxsim_row(lib, d, ld, fp16):
    import torch

    rng = np.random.default_rng(d + ld)
    n_evals, n_slots = 3, 10
    n_chunks = n_evals * n_slots
    counts = rng.integers(1, 701, size=n_chunks)
    counts[:6] = [1, 2, 4, 5, 9, 700]
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    N = int(off[-1])
    X = rng.standard_normal((N, d), dtype=np.float32)
    Q = rng.standard_normal((n_evals, d), dtype=np.float32)
    chunks = np.arange(n_chunks, dtype=np.int64).reshape(n_evals, n_slots)
    chunks[1, 7:] = -1
    dup = {}                                          # chunk -> row that must win (the first of two equal maxima)
    for e in range(n_evals):
        for s in range(n_slots):
            c = int(chunks[e, s])
            if c < 0 or counts[c] < 6 or c % 3 == 2:
                continue
            gap = 4 if c % 3 == 0 else 1              # 4 apart: one warp's rows; 1 apart: two warps
            p = int(rng.integers(0, counts[c] - gap))
            r0 = int(off[c])
            big = (1.0 + np.linalg.norm(X[r0:off[c + 1]], axis=1).max()) * Q[e] / np.linalg.norm(Q[e])
            X[r0 + p] = X[r0 + p + gap] = big          # strictly above every other row by Cauchy-Schwarz
            dup[c] = r0 + p
    dt = np.float16 if fp16 else np.float32
    Xs = X.astype(dt)
    flat, _ = _strided(Xs, ld, 0, dt(np.nan))
    best = torch.full((n_evals, n_slots, d), float("nan"), dtype=torch.float32, device="cuda")
    rows = torch.full((n_evals, n_slots), -9, dtype=torch.int64, device="cuda")
    E_dev, off_dev, ch_dev, Q_dev = _dev(flat), _dev(off), _dev(chunks), _dev(Q)            # alive until the kernel ran
    _check(lib.rl_best_vectors(E_dev.data_ptr(), 1 if fp16 else 0, ld, d, off_dev.data_ptr(), ch_dev.data_ptr(),
                                    n_evals, n_slots, Q_dev.data_ptr(), best.data_ptr(), rows.data_ptr(), _stream()),
           "rl_best_vectors")
    best, rows = best.cpu().numpy(), rows.cpu().numpy()
    X64 = Xs.astype(np.float64)
    for e in range(n_evals):
        for s in range(n_slots):
            c = int(chunks[e, s])
            if c < 0:
                assert rows[e, s] == -1 and not best[e, s].any()
                continue
            r0, r1 = int(off[c]), int(off[c + 1])
            sc = X64[r0:r1] @ Q[e].astype(np.float64)
            b = 2 * rd.gamma(d) * (np.abs(X64[r0:r1]) @ np.abs(Q[e]).astype(np.float64))
            if c in dup:
                assert rows[e, s] == dup[c], (c, rows[e, s], dup[c])
            else:
                m = int(np.argmax(sc))
                near = np.flatnonzero(sc + b >= sc[m] - b[m])     # rows the float64 summation order may put first
                if len(near) == 1:
                    assert rows[e, s] == r0 + m, (c, rows[e, s], r0 + m)
                else:
                    assert rows[e, s] - r0 in near
            assert np.array_equal(best[e, s], Xs[rows[e, s]].astype(np.float32))
