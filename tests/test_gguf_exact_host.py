"""The float64 statement of GGUF dequantization (``gguf_exact``) against the ggml-order restatement and, where it
imports, ``gguf.quants``; the image restatement's sizes against the library; and the quantized-weight entry points'
refusals before any CUDA call (no GPU)."""

from __future__ import annotations

import ctypes as C

import gguf_exact as gx
import numpy as np
import pytest
from gguf_fixtures import Q4_K, Q6_K, Q8_0, dequant, random_blocks

TYPES = [Q8_0, Q4_K, Q6_K]
EINVAL, EUNSUPPORTED = -1, -4


def _same_f16(stmt: np.ndarray, f16: np.ndarray) -> bool:
    """float64 fp16 values against fp16 bits: NaN as NaN, every other value bit for bit (signed zeros included)."""
    f16 = np.asarray(f16, np.float16).reshape(stmt.shape)
    nan = np.isnan(stmt)
    return np.array_equal(nan, np.isnan(f16)) and np.array_equal(gx.f16_value_bits(stmt[~nan]), f16[~nan].view(np.uint16))


def _fixture_f16(ty: int, blocks: np.ndarray) -> np.ndarray:
    be, _ = gx.BLOCK[ty]
    with np.errstate(over="ignore", invalid="ignore"):
        return dequant(ty, blocks.reshape(-1), len(blocks), be).astype(np.float16)


def test_rounding_helpers() -> None:
    bits = np.arange(65536)
    v = gx.f16_bits_value(bits)
    assert np.array_equal(np.isnan(v), np.isnan(np.arange(65536, dtype=np.uint16).view(np.float16)))
    fin = ~np.isnan(v)
    assert np.array_equal(v[fin], np.arange(65536, dtype=np.uint16).view(np.float16)[fin].astype(np.float64))
    assert np.array_equal(gx.f16_value_bits(v[fin]), bits[fin].astype(np.uint16))
    # ties: halfway between fp16 neighbours goes to the even one, at every binade including the subnormals
    mid = (v[0:0x7BFF:2] + v[1:0x7C00:2]) / 2
    assert np.array_equal(gx.to_f16(mid), v[0:0x7BFF:2])
    mid2 = (v[1:0x7BFF:2] + v[2:0x7C00:2]) / 2
    assert np.array_equal(gx.to_f16(mid2), v[2:0x7C00:2])
    assert gx.to_f16(np.array([65519.99, 65520.0, -65520.0]))[1:].tolist() == [np.inf, -np.inf]
    assert gx.to_f16(np.array([65519.99]))[0] == 65504
    assert np.signbit(gx.to_f16(np.array([-2.0**-26]))[0]) and gx.to_f16(np.array([2.0**-25 * 3]))[0] == 2.0**-23
    r = np.random.default_rng(0).standard_normal(100000) * np.exp2(np.random.default_rng(1).integers(-140, 120, 100000))
    assert np.array_equal(gx.to_f32(r), r.astype(np.float32).astype(np.float64))


@pytest.mark.parametrize("ty", TYPES)
def test_builders_round_trip(ty) -> None:  # noqa: ANN001
    rng = np.random.default_rng(ty)
    if ty == Q4_K:
        for _ in range(20):
            sc, m, q = rng.integers(0, 64, 8), rng.integers(0, 64, 8), rng.integers(0, 16, 256)
            b = gx.q4_k_block(0x3C00, 0x4000, sc, m, q)[None]
            for e in range(256):
                assert [int(x[0]) for x in gx.q4k_fields(b, e)] == [sc[e // 32], m[e // 32], q[e]]
    elif ty == Q6_K:
        for _ in range(20):
            sc, q = rng.integers(-128, 128, 16), rng.integers(0, 64, 256)
            b = gx.q6_k_block(0x3C00, sc, q)[None]
            for e in range(256):
                h, g, l = e // 128, (e % 128) // 32, e % 32
                assert [int(x[0]) for x in gx.q6k_fields(b, e)] == [sc[8 * h + 2 * g + l // 16], q[e]]
    else:
        q = rng.integers(-128, 128, 32)
        assert np.array_equal(gx.q8_0_block(0x3C00, q)[2:].view(np.int8), q)


@pytest.mark.parametrize("ty", TYPES)
def test_edge_blocks_cover_their_fields(ty) -> None:  # noqa: ANN001
    b = gx.edge_blocks(ty, nonfinite=True)
    if ty == Q8_0:
        d = gx._u16(b, 0)
        assert set(d.tolist()) == set(gx.EDGE_F16 + gx.NONFINITE_F16)
        for x in set(d.tolist()):
            assert set(b[d == x, 2:].view(np.int8).reshape(-1).tolist()) == set(range(-128, 128))
    elif ty == Q4_K:
        pairs = set(zip(gx._u16(b, 0).tolist(), gx._u16(b, 2).tolist(), strict=True))
        assert len(pairs) == len(gx.EDGE_F16 + gx.NONFINITE_F16) ** 2
        for j in range(8):
            e = 32 * j
            sc, m, _ = gx.q4k_fields(b, e)
            assert set(sc.tolist()) == set(range(64)) and set(m.tolist()) == set(range(64))
            for blk in b[-64:]:   # every nibble in every sub-block
                assert {int(gx.q4k_fields(blk[None], e + i)[2][0]) for i in range(32)} == set(range(16))
    else:
        assert set(gx._u16(b, 208).tolist()) == set(gx.EDGE_F16 + gx.NONFINITE_F16)
        for p in range(16):
            assert set(b[:, 192 + p].view(np.int8).tolist()) == set(range(-128, 128))
        for h in range(2):
            for g in range(4):
                codes = np.concatenate([gx.q6k_fields(b, 128 * h + 32 * g + l)[1] for l in range(32)])
                assert set(codes.tolist()) == set(range(64))
    # the edges the kernels must meet: fp16 overflow, subnormal results, and exact ties rounded both ways to even
    y = gx.dequant_exact(ty, b)
    assert np.isposinf(y).any() and np.isneginf(y).any() and np.isnan(y).any()
    sub = (y != 0) & (np.abs(y) < 2.0**-14)
    assert sub.sum() > 100 and np.signbit(y[y == 0]).any() and (~np.signbit(y[y == 0])).any()
    fin = gx.finite_blocks(ty, gx.edge_blocks(ty))
    assert len(fin) >= 0.5 * len(gx.edge_blocks(ty)) and np.isfinite(gx.dequant_exact(ty, fin)).all()
    assert (np.abs(gx.dequant_exact(ty, fin)) > 32768).any()
    if ty == Q8_0:   # e.g. d = 1 + 2^-10 times q = 3: ties between fp16 neighbours, settled to the even neighbour
        d = gx._u16(b, 0)
        with np.errstate(invalid="ignore"):
            exact = gx.f16_bits_value(d)[:, None] * b[:, 2:].view(np.int8)
        rounded = gx.to_f16(exact)
        ulp = np.exp2(np.maximum(np.frexp(np.where(np.isfinite(exact), exact, 1.0))[1] - 1, -14) - 10)
        tie = np.isfinite(exact) & (np.abs(np.where(np.isfinite(exact), exact, 0.0) / ulp) % 1 == 0.5)
        assert tie.sum() > 8 and tie[d == 0x3C01].any()
        bits = gx.f16_value_bits(np.abs(rounded[tie]))
        assert (bits % 2 == 0).all()
        assert (np.abs(rounded[tie]) > np.abs(exact[tie])).any() and (np.abs(rounded[tie]) < np.abs(exact[tie])).any()


@pytest.mark.parametrize("ty", TYPES)
def test_statement_equals_the_ggml_order_restatement(ty) -> None:  # noqa: ANN001
    """Bit for bit on every edge block (the exactness claims asserted on each) and on seeded random blocks at several
    scales."""
    b = gx.edge_blocks(ty, nonfinite=True)
    assert _same_f16(gx.dequant_exact(ty, b), _fixture_f16(ty, b))
    rng = np.random.default_rng(10 + ty)
    be, bb = gx.BLOCK[ty]
    for scale in (1.0, 100.0, 1e4):
        r = random_blocks(ty, 64, 1024, rng, scale=scale).reshape(-1, bb)
        assert _same_f16(gx.dequant_exact(ty, r), _fixture_f16(ty, r))
    r = rng.integers(0, 256, (4000, bb), dtype=np.uint8)   # every byte random: fp16 scales over their whole range
    assert _same_f16(gx.dequant_exact(ty, r), _fixture_f16(ty, r))


@pytest.mark.parametrize("ty", TYPES)
def test_statement_equals_gguf_package(ty) -> None:  # noqa: ANN001
    quants = pytest.importorskip("gguf.quants")
    import gguf

    b = gx.edge_blocks(ty)
    be, bb = gx.BLOCK[ty]
    with np.errstate(over="ignore", invalid="ignore"):
        want = quants.dequantize(b.reshape(len(b), bb), gguf.GGMLQuantizationType(ty)).astype(np.float16)
    assert _same_f16(gx.dequant_exact(ty, b), want)


@pytest.mark.parametrize("ty", TYPES)
def test_image_sizes_equal_the_library(ty) -> None:  # noqa: ANN001
    from raglite_b200 import _lib

    lib = _lib.load()
    for N in (32, 96, 128, 160, 8160, 8192):
        for K in (128, 256, 1024, 4096):
            legal = K % gx.BLOCK[ty][0] == 0
            n_pass = (N + 127) // 128
            want = gx.image_bytes([ty] * n_pass, N, K) if legal else 0
            assert lib.rl_xenc_qlinear_image_bytes(ty, N, K) == want, (N, K)
    rng = np.random.default_rng(ty)
    for N, K in ((32, 256), (160, 512), (96, 256)):
        raw = random_blocks(ty, N, K, rng)
        img = gx.image([(ty, raw, N)], K)
        assert img.size == lib.rl_xenc_qlinear_image_bytes(ty, N, K)
        h = img[:16].view("<i4")
        assert h.tolist() == [(N + 127) // 128, N, K, 0x51494D47]


def test_image_restatement_layout() -> None:
    """Hand-checked offsets of a two-part Q4_K (128 rows) | Q6_K (48 rows) image at K 256."""
    rng = np.random.default_rng(3)
    a, b = random_blocks(Q4_K, 128, 256, rng), random_blocks(Q6_K, 48, 256, rng)
    img = gx.image([(Q4_K, a, 128), (Q6_K, b, 48)], 256)
    d = img[16:48].view(np.uint8)
    assert d[:8].view("<i4").tolist() == [Q4_K, 76] and int(d[8:16].view("<i8")[0]) == 2048
    assert d[16:24].view("<i4").tolist() == [Q6_K, 108] and int(d[24:32].view("<i8")[0]) == 2048 + 2 * 128 * 76
    assert img.size == 2048 + 2 * 128 * 76 + 2 * 48 * 108
    p1 = img[2048 + 2 * 128 * 76:].reshape(2, 48, 108)
    blk = b.reshape(48, 210)
    assert np.array_equal(p1[1, 5, :64], blk[5, 64:128]) and np.array_equal(p1[1, 5, 104:106], blk[5, 208:210])
    assert (p1[:, :, 106:] == 0).all()
    p0 = img[2048:2048 + 2 * 128 * 76].reshape(2, 128, 76)
    q = a.reshape(128, 144)
    assert np.array_equal(p0[0, 7, :4], q[7, :4]) and np.array_equal(p0[1, 7, 12:], q[7, 80:144])
    assert p0[1, 7, 4] == gx.q4k_fields(q[7:8], 128)[0][0] and p0[1, 7, 11] == gx.q4k_fields(q[7:8], 255)[1][0]


# ---- C-ABI refusals -----------------------------------------------------------------------------------------------------
def _lib():  # noqa: ANN202
    from raglite_b200 import _lib as L

    return L.load()


def _err(lib) -> str:  # noqa: ANN001
    return lib.rl_last_error().decode()


def test_qlinear_image_bytes_refusals() -> None:
    lib = _lib()
    assert lib.rl_xenc_qlinear_image_bytes(Q4_K, 128, 256) > 0
    for ty in (0, 1, 2, 13):
        assert lib.rl_xenc_qlinear_image_bytes(ty, 128, 256) == 0
    for N in (0, 48, 8224, -32):
        assert lib.rl_xenc_qlinear_image_bytes(Q8_0, N, 256) == 0
    for K in (0, 96, -128):
        assert lib.rl_xenc_qlinear_image_bytes(Q8_0, 128, K) == 0
    assert lib.rl_xenc_qlinear_image_bytes(Q4_K, 128, 384) == 0   # K % 128 == 0 but half a super-block
    assert lib.rl_xenc_qlinear_image_bytes(Q6_K, 128, 384) == 0
    assert lib.rl_xenc_qlinear_image_bytes(Q8_0, 128, 384) > 0


def test_quantized_entry_points_refuse_before_any_cuda_call() -> None:
    lib = _lib()
    d, odd = C.c_void_p(256), C.c_void_p(264)
    pack = lib.rl_xenc_pack_qlinear
    assert pack(Q8_0, None, 128, 256, d, None) == EINVAL and "null pointer" in _err(lib)
    assert pack(Q8_0, d, 128, 256, None, None) == EINVAL
    for ty, N, K in ((13, 128, 256), (Q8_0, 48, 256), (Q8_0, 0, 256), (Q8_0, 8224, 256), (Q8_0, 128, 96),
                     (Q4_K, 128, 384), (Q6_K, 128, 128), (Q8_0, 128, 0)):
        assert pack(ty, d, N, K, d, None) == EUNSUPPORTED, (ty, N, K)
        assert "rl_xenc_pack_qlinear" in _err(lib)

    deq = lib.rl_dequant_rows_f16
    assert deq(Q8_0, None, 1, 256, d, None) == EINVAL and deq(Q8_0, d, 1, 256, None, None) == EINVAL
    assert deq(Q8_0, d, -1, 256, d, None) == EINVAL
    for ty, K in ((13, 256), (0, 256), (Q8_0, 0), (Q8_0, 48), (Q4_K, 128), (Q6_K, 384), (Q4_K, -256)):
        assert deq(ty, d, 4, K, d, None) == EUNSUPPORTED, (ty, K)
    assert deq(Q4_K, d, 0, 256, d, None) == 0                           # rows = 0: nothing to do

    lin = lib.rl_xenc_linear_q   # (X, image, bias, Y, T, N, K, act, stream)
    for args in ((None, d, d, d), (d, None, d, d), (d, d, None, d), (d, d, d, None)):
        assert lin(*args, 1, 128, 256, 0, None) == EINVAL
    assert lin(d, d, d, d, -1, 128, 256, 0, None) == EINVAL
    assert lin(d, d, odd, d, 1, 128, 256, 0, None) == EINVAL and "bias must be 16-byte aligned" in _err(lib)
    for N, K in ((48, 256), (128, 192), (0, 256), (-32, 256), (128, 0), (8224, 256)):
        assert lin(d, d, d, d, 1, N, K, 0, None) == EUNSUPPORTED, (N, K)
        assert "rl_xenc_linear_q" in _err(lib)
    assert lin(d, d, d, d, 0, 128, 256, 0, None) == 0                   # T = 0: nothing to do

    cat = lib.rl_xenc_concat_qlinear
    parts = (C.c_void_p * 65)(*([256] * 65))
    assert cat(parts, 0, d, None) == EINVAL
    assert cat(None, 1, d, None) == EINVAL and cat(parts, 1, None, None) == EINVAL
    assert cat(parts, 65, d, None) == EUNSUPPORTED and "too many parts" in _err(lib)
    nulls = (C.c_void_p * 2)(None, 256)
    assert cat(nulls, 2, d, None) == EINVAL and "null part" in _err(lib)


def _weights(layer_types: tuple[int, int, int, int], *, H: int = 1024, F: int = 4096, nh: int = 16, n_layers: int = 2,
             bad_layer: int = 1):  # noqa: ANN202
    """Host weights with dummy device pointers; layer ``bad_layer`` gets ``layer_types`` (the others fp16 images)."""
    from raglite_b200._lib import XencLayer, XencWeights

    layers = (XencLayer * n_layers)()
    for i, L in enumerate(layers):
        for name, _ in XencLayer._fields_[:12]:
            setattr(L, name, 256)
        if i == bad_layer:
            L.qkv_type, L.o_type, L.up_type, L.down_type = layer_types
    w = XencWeights(n_layers=n_layers, hidden=H, n_heads=nh, ffn=F, vocab=1000, max_pos=514, type_vocab=1, ln_eps=1e-5)
    for name in ("word_emb", "pos_emb", "type_emb", "emb_ln_g", "emb_ln_b", "pooler_w", "pooler_b", "cls_w", "cls_b"):
        setattr(w, name, 256)
    w.layers = layers
    w._keep = layers
    return w


@pytest.mark.parametrize("fn", ["encode", "score"])
def test_encoder_refuses_bad_layer_image_types_before_any_cuda_call(fn) -> None:  # noqa: ANN001
    """An image type other than RL_XENC_IMAGE_F16 (0) / RL_XENC_IMAGE_QUANT (1) is RL_EINVAL, and a quantized linear
    whose K is not a multiple of 128 (or whose N is over 8192) RL_EUNSUPPORTED, from the entry checks: no kernel of the
    forward runs first.  The pointers are dummies and no device is needed."""
    lib = _lib()
    d = C.c_void_p(256)
    T, P, max_len = 64, 2, 32

    def call(w) -> int:  # noqa: ANN001
        ws = lib.rl_xenc_workspace_bytes(C.byref(w), T)
        if fn == "encode":
            return lib.rl_xenc_encode(C.byref(w), d, d, d, d, P, T, max_len, d, d, ws, None)
        return lib.rl_xenc_score(C.byref(w), d, d, d, d, P, T, max_len, d, d, d, ws, None)

    for types in ((2, 0, 0, 0), (0, -1, 0, 0), (0, 0, 7, 0), (0, 0, 0, 0x7FFFFFFF), (1, 1, 1, 3)):
        assert call(_weights(types)) == EINVAL, types
        assert "image type" in _err(lib) and f"rl_xenc_{fn}" in _err(lib)
    # H = 320 (10 heads of 32): qkv, o and up read K = H; down reads K = F
    for types in ((1, 0, 0, 0), (0, 1, 0, 0), (0, 0, 1, 0)):
        assert call(_weights(types, H=320, F=1280, nh=10)) == EUNSUPPORTED, types
        assert "K % 128 == 0" in _err(lib)
    assert call(_weights((0, 0, 0, 1), H=512, F=1568, nh=16)) == EUNSUPPORTED
    assert call(_weights((0, 0, 1, 0), H=512, F=8224, nh=16)) == EUNSUPPORTED   # up: N = F over 8192
