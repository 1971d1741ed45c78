"""The GGUF kernels at the C-ABI against the float64 statement of ggml's arithmetic (``gguf_exact``): the dequantized
rows bit for bit on every edge block, the quantized linear's own dequantizer values read back through one-hot
activations, the linear against float64 at bge-m3's shapes, and the quantized images byte for byte."""

from __future__ import annotations

import ctypes as C
import json
import tempfile
from pathlib import Path

import gguf_exact as gx
import numpy as np
import pytest
import torch
from gguf_fixtures import random_blocks

pytestmark = pytest.mark.gpu

Q8_0, Q4_K, Q6_K = gx.Q8_0, gx.Q4_K, gx.Q6_K
TYPES = [Q8_0, Q4_K, Q6_K]
F16_NAN_GUARD = 0x7E5A   # a NaN no kernel writes


@pytest.fixture(scope="module")
def lib():  # noqa: ANN201
    from raglite_b200 import _lib

    return _lib.load()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _record(name: str, payload: dict) -> None:
    """Append a line (case + measured error) to xenc_bounds.jsonl in the temporary directory."""
    with (Path(tempfile.gettempdir()) / "xenc_bounds.jsonl").open("a") as f:
        f.write(json.dumps({"test": name, **payload}) + "\n")


def _assert_f16_equal(got: np.ndarray, want: np.ndarray, what: str) -> None:
    """fp16 ``got`` against float64 fp16 values: NaN as NaN, everything else bit for bit."""
    nan = np.isnan(want)
    bad = (np.isnan(got) != nan) | (~nan & (got.view(np.uint16) != gx.f16_value_bits(np.where(nan, 0.0, want))))
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.size} differ, first at {np.argwhere(bad)[:4].tolist()}: " \
                          f"got {got[bad][:4]} want {want[bad][:4]}"


def _dequant(lib, ty: int, raw: np.ndarray, rows: int, K: int, guard: int = 256) -> np.ndarray:  # noqa: ANN001
    out = torch.full((rows * K + guard,), F16_NAN_GUARD, dtype=torch.int16, device="cuda")
    assert lib.rl_dequant_rows_f16(ty, torch.from_numpy(raw).cuda().data_ptr(), rows, K, out.data_ptr(), _stream()) == 0, \
        lib.rl_last_error()
    o = out.cpu().numpy().view(np.uint16)
    assert (o[rows * K:] == F16_NAN_GUARD).all(), "written behind the output"
    return o[:rows * K].view(np.float16).reshape(rows, K)


# ---- rl_dequant_rows_f16 ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ty", TYPES)
def test_dequant_rows_on_every_edge_block(lib, ty) -> None:  # noqa: ANN001
    """Every edge block, including +-inf and NaN scale fields, one block per row and tiled into rows of 1024 and 4096."""
    blocks = gx.edge_blocks(ty, nonfinite=True)
    be, _ = gx.BLOCK[ty]
    want_blocks = gx.dequant_exact(ty, blocks)
    for K in (be, 1024, 4096):
        per_row = K // be
        rows = (len(blocks) + per_row - 1) // per_row
        for shift in (0, len(blocks) // 3):
            raw = gx.tile_blocks(blocks, ty, rows, K, shift)
            idx = (np.arange(rows * per_row) + shift) % len(blocks)
            _assert_f16_equal(_dequant(lib, ty, raw, rows, K), want_blocks[idx].reshape(rows, K), f"K={K} shift={shift}")
    out = torch.full((512,), F16_NAN_GUARD, dtype=torch.int16, device="cuda")   # rows = 0 writes nothing
    assert lib.rl_dequant_rows_f16(ty, torch.from_numpy(blocks.reshape(-1)).cuda().data_ptr(), 0, be, out.data_ptr(),
                                   _stream()) == 0
    assert (out.cpu().numpy().view(np.uint16) == F16_NAN_GUARD).all()


@pytest.mark.parametrize("ty", [Q6_K, Q8_0])
def test_dequant_rows_full_vocabulary_table(lib, ty) -> None:  # noqa: ANN001
    """bge-m3's token table shape, 250 002 x 1024 (the grid-stride loop's many trips), with edge blocks at both ends:
    the first and last rows and a seeded sample against the statement."""
    rows, K = 250_002, 1024
    rng = np.random.default_rng(ty)
    be, bb = gx.BLOCK[ty]
    raw = random_blocks(ty, rows, K, rng, scale=30.0).reshape(-1, bb)
    edges = gx.edge_blocks(ty, nonfinite=True)
    raw[:len(edges)] = edges
    raw[-len(edges):] = edges
    out = torch.full((rows * K + 256,), F16_NAN_GUARD, dtype=torch.int16, device="cuda")
    assert lib.rl_dequant_rows_f16(ty, torch.from_numpy(raw.reshape(-1)).cuda().data_ptr(), rows, K, out.data_ptr(),
                                   _stream()) == 0, lib.rl_last_error()
    assert (out[rows * K:] == F16_NAN_GUARD).all()
    pick = np.unique(np.r_[np.arange(80), rows - 80 + np.arange(80), rng.integers(0, rows, 2000)])   # edges: 80 rows
    got = out[:rows * K].view(rows, K)[torch.from_numpy(pick).cuda()].cpu().numpy().view(np.float16)
    per_row = K // be
    want = gx.dequant_exact(ty, raw.reshape(rows, per_row, bb)[pick].reshape(-1, bb)).reshape(len(pick), K)
    _assert_f16_equal(got, want, "full table")


# ---- the quantized linear --------------------------------------------------------------------------------------------
def _q_image(lib, parts: list[tuple[int, np.ndarray, int]], K: int) -> torch.Tensor:  # noqa: ANN001
    """Quantized image of (type, GGUF bytes, rows) parts: one pack per part, concatenated when there are several."""
    imgs = []
    for ty, raw, N in parts:
        img = torch.empty(int(lib.rl_xenc_qlinear_image_bytes(ty, N, K)), dtype=torch.uint8, device="cuda")
        assert img.numel() > 0
        assert lib.rl_xenc_pack_qlinear(ty, torch.from_numpy(raw).cuda().data_ptr(), N, K, img.data_ptr(), _stream()) == 0
        imgs.append(img)
    if len(imgs) == 1:
        return imgs[0]
    out = torch.empty(sum(i.numel() for i in imgs), dtype=torch.uint8, device="cuda")
    ptrs = (C.c_void_p * len(imgs))(*[i.data_ptr() for i in imgs])
    assert lib.rl_xenc_concat_qlinear(ptrs, len(imgs), out.data_ptr(), _stream()) == 0, lib.rl_last_error()
    torch.cuda.synchronize()
    return out


def _linear_q(lib, X: torch.Tensor, img: torch.Tensor, bias: torch.Tensor, N: int, K: int, act: int) -> torch.Tensor:  # noqa: ANN001
    Y = torch.full((X.shape[0], N), float("nan"), dtype=torch.float16, device="cuda")
    assert lib.rl_xenc_linear_q(X.data_ptr(), img.data_ptr(), bias.data_ptr(), Y.data_ptr(), X.shape[0], N, K, act,
                                _stream()) == 0, lib.rl_last_error()
    return Y


_FINITE: dict[int, tuple[np.ndarray, np.ndarray]] = {}


def _finite_edges(ty: int) -> tuple[np.ndarray, np.ndarray]:
    """The finite edge blocks and their statement values (cached per type)."""
    if ty not in _FINITE:
        b = gx.finite_blocks(ty, gx.edge_blocks(ty))
        _FINITE[ty] = (b, gx.dequant_exact(ty, b))
    return _FINITE[ty]


def _edge_part(ty: int, N: int, K: int, shift: int) -> tuple[tuple[int, np.ndarray, int], np.ndarray]:
    """A part of N rows tiled from the finite edge blocks, and its float64 values [N, K]."""
    b, vals = _finite_edges(ty)
    be, _ = gx.BLOCK[ty]
    idx = (np.arange(N * K // be) + shift) % len(b)
    return (ty, np.ascontiguousarray(b[idx]).reshape(-1), N), vals[idx].reshape(N, K)


def _read_back(lib, parts, W: np.ndarray, K: int) -> None:  # noqa: ANN001
    """X = one-hot rows e_0 .. e_{K-1}, then e_0 .. e_36 again (a ragged last token tile); bias 0, act 0.  Then
    Y[t, n] = 1 * W[n, t] + exact zeros: the dequantizer warps' fp16 value, which must be the statement's."""
    N = W.shape[0]
    eye = torch.eye(K, dtype=torch.float16, device="cuda")
    X = torch.cat([eye, eye[:37]]).contiguous()
    Y = _linear_q(lib, X, _q_image(lib, parts, K), torch.zeros(N, dtype=torch.float32, device="cuda"), N, K, 0)
    Wt = torch.from_numpy(W.astype(np.float16)).cuda().T          # exact: W holds fp16 values
    want = torch.cat([Wt, Wt[:37]])
    bad = Y != want                                               # +-0 compare equal: the epilogue adds a +0 bias
    if bad.any():
        sub = bad & (want != 0) & (want.abs() < 2.0**-14)
        raise AssertionError(f"{int(bad.sum())} of {bad.numel()} differ ({int(sub.sum())} at subnormal weights); "
                             f"first {bad.nonzero()[:4].tolist()}: got {Y[bad][:4].tolist()} want {want[bad][:4].tolist()}")


ONE_HOT = [(ty, N, K) for ty in TYPES for N in (32, 96, 160, 8192) for K in ((128,) if ty == Q8_0 else ()) + (256, 1024, 4096)]


@pytest.mark.parametrize(("ty", "N", "K"), ONE_HOT)
def test_linear_q_one_hot_reads_back_the_dequantized_weights(lib, ty, N, K) -> None:  # noqa: ANN001
    part, W = _edge_part(ty, N, K, shift=N + K)
    _read_back(lib, [part], W, K)


@pytest.mark.parametrize("layout", ["qkv", "64 parts"])
def test_linear_q_one_hot_read_back_of_mixed_images(lib, layout) -> None:  # noqa: ANN001
    K = 1024
    if layout == "qkv":
        spec = [(Q4_K, 1024), (Q4_K, 1024), (Q6_K, 1024)]
    else:   # every type, one pass each, the last one short
        spec = [(TYPES[i % 3], 128) for i in range(63)] + [(Q6_K, 96)]
    parts, Ws = [], []
    for i, (ty, n) in enumerate(spec):
        p, w = _edge_part(ty, n, K, shift=37 * i)
        parts.append(p)
        Ws.append(w)
    _read_back(lib, parts, np.concatenate(Ws), K)


# bge-m3's four linears: (name, N, K, act)
BGE_M3 = [("qkv", 3072, 1024, 0), ("o", 1024, 1024, 0), ("up", 4096, 1024, 1), ("down", 1024, 4096, 0)]
Q4_K_M = {"qkv": [Q4_K, Q4_K, Q6_K], "o": [Q4_K], "up": [Q4_K], "down": [Q6_K]}


def _check_float64(Y: torch.Tensor, X: torch.Tensor, W: torch.Tensor, b: torch.Tensor, act: int) -> float:
    """Worst |Y - ref| / bound over Y, with ref = act(X W^T + b) in float64 from the fp16 X and W; an infinite output
    must have the reference's sign and a reference within its bound of fp16's overflow threshold (65520)."""
    K = X.shape[1]
    worst = 0.0
    for t0 in range(0, X.shape[0], 8192):
        Xd = X[t0:t0 + 8192].double()
        ref = Xd @ W.T + b
        if act:
            ref = 0.5 * ref * (1.0 + torch.erf(ref / 2.0**0.5))
        bound = 2.0**-11 * ref.abs() + (K + 2) * 2.0**-23 * (Xd.abs() @ W.abs().T) + 1e-6
        y = Y[t0:t0 + 8192].double()
        inf = torch.isinf(y)
        ok_inf = (torch.sign(y) == torch.sign(ref)) & (ref.abs() + bound >= 65520.0)
        assert bool((~inf | ok_inf).all()), "an overflow to inf the reference does not reach"
        r = ((y - ref).abs() / bound)[~inf]                       # NaN: an output never written
        worst = max(worst, float(r.max()) if r.numel() else 0.0)
        assert not torch.isnan(r).any()
    return worst


@pytest.mark.parametrize("weights", ["Q8_0", "Q4_K", "Q6_K", "Q4_K_M"])
@pytest.mark.parametrize(("name", "N", "K", "act"), BGE_M3)
def test_linear_q_matches_float64_at_bge_m3_shapes(lib, weights, name, N, K, act) -> None:  # noqa: ANN001
    """X W^T + b (exact GELU on up) in float64 from the statement's fp16 weights, at T = 1, 129, 20 000 and 65 536
    tokens (one call of the engine), within test_linear_layer_matches_torch's bound."""
    rng = np.random.default_rng(hash((weights, name)) % 2**32)
    types = Q4_K_M[name] if weights == "Q4_K_M" else [{"Q8_0": Q8_0, "Q4_K": Q4_K, "Q6_K": Q6_K}[weights]]
    n = N // len(types)
    parts = [(t, random_blocks(t, n, K, rng), n) for t in types]
    W = np.concatenate([gx.dequant_rows_exact(t, raw, n, K) for t, raw, n in parts])
    Wd = torch.from_numpy(W).cuda()
    img = _q_image(lib, parts, K)
    b = torch.from_numpy(rng.standard_normal(N).astype(np.float32) * 0.1).cuda()
    g = torch.Generator(device="cuda").manual_seed(len(name))
    worst, worst_at = 0.0, None
    for T in (1, 129, 20000, 65536):
        X = (torch.randn((T, K), generator=g, device="cuda") * 2.0).half()
        Y = _linear_q(lib, X, img, b, N, K, act)
        r = _check_float64(Y, X, Wd, b.double(), act)
        assert r <= 1.0, (T, r)
        if r > worst:
            worst, worst_at = r, T
        del X, Y
    _record("linear_q", {"weights": weights, "linear": name, "max_err_over_bound": worst, "at_T": worst_at})


@pytest.mark.parametrize("ty", TYPES)
def test_linear_q_overflows_to_inf_like_float64(lib, ty) -> None:  # noqa: ANN001
    """Outputs past fp16's range: inf with the reference's sign, the rest within the bound."""
    N, K, T = 1024, 1024, 129
    rng = np.random.default_rng(40 + ty)
    raw = random_blocks(ty, N, K, rng, scale={Q8_0: 2e4, Q4_K: 3e4, Q6_K: 1e5}[ty])
    W = torch.from_numpy(gx.dequant_rows_exact(ty, raw, N, K)).cuda()
    assert torch.isfinite(W).all()
    X = torch.from_numpy(rng.standard_normal((T, K)).astype(np.float16) * 4).cuda()
    b = torch.zeros(N, dtype=torch.float32, device="cuda")
    Y = _linear_q(lib, X, _q_image(lib, [(ty, raw, N)], K), b, N, K, 0)
    n_inf = int(torch.isinf(Y).sum())
    assert 0.05 * Y.numel() < n_inf < 0.95 * Y.numel(), n_inf
    assert _check_float64(Y, X, W, b.double(), 0) <= 1.0


# ---- images byte for byte ------------------------------------------------------------------------------------------------
def _raw(ty: int, N: int, K: int, rng: np.random.Generator) -> np.ndarray:
    """Every byte random: packing moves bytes, and each must land where the layout says."""
    be, bb = gx.BLOCK[ty]
    return rng.integers(0, 256, N * K // be * bb, dtype=np.uint8)


def _pack(lib, ty: int, raw: np.ndarray, N: int, K: int) -> torch.Tensor:  # noqa: ANN001
    img = torch.full((int(lib.rl_xenc_qlinear_image_bytes(ty, N, K)),), 0xA5, dtype=torch.uint8, device="cuda")
    assert lib.rl_xenc_pack_qlinear(ty, torch.from_numpy(raw).cuda().data_ptr(), N, K, img.data_ptr(), _stream()) == 0
    return img


PACK = [(ty, N, K) for ty in TYPES for N, K in ((32, 256), (96, 1024), (160, 256), (8160, 1024), (8192, 4096))]
PACK += [(Q8_0, 32, 128), (Q8_0, 160, 128)]


@pytest.mark.parametrize(("ty", "N", "K"), PACK)
def test_pack_qlinear_equals_the_image_restatement(lib, ty, N, K) -> None:  # noqa: ANN001
    """Header, pass descriptors, per-slice rows and zero padding rows; N 8192 x K 4096 has 2^18 (pass, slice, row)
    items, two per thread of the 1024 x 128 grid, so the grid-stride loop's second trip is compared too."""
    raw = _raw(ty, N, K, np.random.default_rng(N + K + ty))
    got = _pack(lib, ty, raw, N, K).cpu().numpy()
    want = gx.image([(ty, raw, N)], K)
    assert got.size == want.size
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{bad.size} bytes differ, first at {bad[:8].tolist()}"


def _concat(lib, imgs: list[torch.Tensor], fill: int = 0x5A) -> tuple[int, torch.Tensor]:  # noqa: ANN001
    out = torch.full((sum(i.numel() for i in imgs),), fill, dtype=torch.uint8, device="cuda")
    ptrs = (C.c_void_p * len(imgs))(*[i.data_ptr() for i in imgs])
    rc = lib.rl_xenc_concat_qlinear(ptrs, len(imgs), out.data_ptr(), _stream())
    torch.cuda.synchronize()
    return rc, out


def test_concat_qlinear_equals_the_image_restatement(lib) -> None:  # noqa: ANN001
    rng = np.random.default_rng(7)
    K = 1024
    spec = [(Q4_K, 1024), (Q8_0, 256), (Q6_K, 128), (Q4_K, 384), (Q8_0, 160)]
    parts = [(ty, _raw(ty, n, K, rng), n) for ty, n in spec]
    imgs = [_pack(lib, ty, raw, n, K) for ty, raw, n in parts]
    want = gx.image(parts, K)

    def check(out: torch.Tensor) -> None:   # the image, then the rest of the buffer (the parts' other headers) untouched
        o = out.cpu().numpy()
        assert np.array_equal(o[:want.size], want) and (o[want.size:] == 0x5A).all()

    rc, flat = _concat(lib, imgs)
    assert rc == 0, lib.rl_last_error()
    check(flat)
    # a concatenation of concatenations is the flat one
    rc, a = _concat(lib, imgs[:2])
    assert rc == 0
    rc, b = _concat(lib, imgs[2:])
    assert rc == 0
    rc, ab = _concat(lib, [a, b])
    assert rc == 0
    check(ab)
    # one part is itself
    for img in imgs:
        rc, one = _concat(lib, [img])
        assert rc == 0 and torch.equal(one, img)
    # 64 one-pass parts
    parts64 = [(TYPES[i % 3], _raw(TYPES[i % 3], 128, 256, rng), 128) for i in range(63)] + [(Q6_K, _raw(Q6_K, 32, 256, rng), 32)]
    rc, img64 = _concat(lib, [_pack(lib, ty, raw, n, 256) for ty, raw, n in parts64])
    want = gx.image(parts64, 256)
    assert rc == 0
    check(img64)


def test_concat_qlinear_refusals(lib) -> None:  # noqa: ANN001
    rng = np.random.default_rng(8)
    q = _pack(lib, Q4_K, _raw(Q4_K, 128, 256, rng), 128, 256)
    q512 = _pack(lib, Q4_K, _raw(Q4_K, 128, 512, rng), 128, 512)
    q96 = _pack(lib, Q8_0, _raw(Q8_0, 96, 256, rng), 96, 256)
    W = torch.randn((128, 256), device="cuda")
    f16 = torch.empty(int(lib.rl_xenc_linear_image_bytes(128, 256)), dtype=torch.uint8, device="cuda")
    assert lib.rl_xenc_pack_linear(W.data_ptr(), 128, 256, f16.data_ptr(), _stream()) == 0
    for imgs, code, msg in (([q, f16], -1, "part 1 is not a quantized image"), ([f16], -1, "part 0 is not a quantized image"),
                            ([q, q512], -1, "parts differ in K"), ([q96, q], -4, "every part but the last")):
        rc, out = _concat(lib, imgs, fill=0x5A)
        assert rc == code and msg in lib.rl_last_error().decode(), (rc, lib.rl_last_error())
        assert (out == 0x5A).all(), "a refused concatenation wrote its output"
    rc, _ = _concat(lib, [q, q96])   # the short part last is fine
    assert rc == 0
