"""GGUF Q8_0 / Q4_K / Q6_K dequantization stated in float64 from each element's integer fields, edge blocks, and the
quantized linear image restated byte for byte.  NumPy only.

The statement does not follow ggml's array code.  Per element it decodes ``d`` / ``dmin`` from their fp16 bits, ``sc`` /
``m`` by a bit extraction of sub-block j and ``q`` from ``ql`` / ``qh`` by the element's index, then forms the value in
float64 and rounds to float32 only where ggml's float32 evaluation rounds:

* Q8_0 ``d q``: exact in float32 (11 + 8 bits), so the value is fp16(d q).
* Q4_K ``a = (d sc) q`` and ``b = dmin m``: exact in float32 (at most 21 bits).  The value is fp16(f32(a - b)): the
  float64 difference rounded once to float32 is the float32 difference, because 53 >= 2 * 24 + 2.
* Q6_K ``d sc``: exact.  The value is fp16(f32((d sc)(q - 32))), a product of at most 25 bits, exact in float64.

``dequant_exact`` asserts every exactness claim above on the blocks it is given, so a false claim fails the caller.
Rounding to fp16 and float32 is done here too (``round_float``), by scaling to the format's unit in the last place and
``np.rint`` (round half to even), so no NumPy cast decides a tie.
"""

from __future__ import annotations

import numpy as np

Q8_0, Q4_K, Q6_K = 8, 12, 14
BLOCK = {Q8_0: (32, 34), Q4_K: (256, 144), Q6_K: (256, 210)}   # (elements, bytes)

# fp16 bit patterns of the scale fields: +-0, the smallest and largest subnormal, the smallest normal, 1, 1 + 2^-10 and
# 65504, with their negatives; the non-finite ones only for rl_dequant_rows_f16 (an infinity poisons a linear's column).
EDGE_F16 = [s | b for s in (0x0000, 0x8000) for b in (0x0000, 0x0001, 0x03FF, 0x0400, 0x3C00, 0x3C01, 0x7BFF)]
NONFINITE_F16 = [0x7C00, 0xFC00, 0x7E00]


# ---- rounding and fp16 fields ---------------------------------------------------------------------------------------
def round_float(x: np.ndarray, p: int, emin: int, fmax: float) -> np.ndarray:
    """float64 ``x`` rounded to nearest even in a binary format with ``p`` significand bits, least normal exponent
    ``emin`` and largest finite value ``fmax`` (gradual underflow, overflow to +-inf); signed zeros, inf and NaN kept."""
    x = np.asarray(x, np.float64)
    fin = np.isfinite(x)
    xf = np.where(fin, x, 0.0)
    e = np.maximum(np.frexp(xf)[1] - 1, emin)                 # floor(log2 |x|), at least emin
    ulp = np.ldexp(1.0, e - (p - 1))
    r = np.rint(xf / ulp) * ulp                               # both steps exact: scaling by powers of two
    r = np.where(np.abs(r) > fmax, np.copysign(np.inf, x), r)
    return np.where(fin, r, x)


def to_f16(x: np.ndarray) -> np.ndarray:
    return round_float(x, 11, -14, 65504.0)


def to_f32(x: np.ndarray) -> np.ndarray:
    return round_float(x, 24, -126, float(np.finfo(np.float32).max))


def f16_bits_value(bits: np.ndarray) -> np.ndarray:
    """float64 value of fp16 bit patterns, decoded from sign, exponent and mantissa."""
    bits = np.asarray(bits, np.int64)
    sign = np.where(bits & 0x8000, -1.0, 1.0)
    e, m = (bits >> 10) & 31, (bits & 1023).astype(np.float64)
    mag = np.where(e == 0, np.ldexp(m, -24), np.ldexp(1024.0 + m, np.maximum(e, 1) - 25))
    mag = np.where(e == 31, np.where(m == 0, np.inf, np.nan), mag)
    return sign * mag


def f16_value_bits(v: np.ndarray) -> np.ndarray:
    """fp16 bit patterns (uint16) of float64 values that are already fp16 values (NaN as 0x7E00, sign kept)."""
    v = np.asarray(v, np.float64)
    sign = np.where(np.signbit(v), 0x8000, 0).astype(np.int64)
    a = np.abs(np.where(np.isnan(v), 0.0, v))
    fin = np.isfinite(a)
    af = np.where(fin, a, 1.0)
    e = np.maximum(np.frexp(af)[1] - 1, -14)
    m = np.ldexp(af, 10 - e).astype(np.int64)                  # 1024 + mantissa (normal) or the subnormal's mantissa
    bits = np.where(m >= 1024, ((e + 15) << 10) | (m - 1024), m)
    bits = np.where(fin, bits, 0x7C00)
    bits = np.where(np.isnan(v), 0x7E00, bits | sign)
    assert np.array_equal(f16_bits_value(bits)[~np.isnan(v)], v[~np.isnan(v)]), "not fp16 values"
    return bits.astype(np.uint16)


def _u16(b: np.ndarray, off: int) -> np.ndarray:
    return b[:, off].astype(np.int64) | (b[:, off + 1].astype(np.int64) << 8)


def _assert_f32_exact(x: np.ndarray, what: str) -> None:
    f = x[np.isfinite(x)]
    assert np.array_equal(to_f32(f), f), f"{what} is not exact in float32"


# ---- per-element fields -------------------------------------------------------------------------------------------
# Q4_K's 12 scale bytes hold sub-block j's 6-bit scale and min as bit fields (byte, low bit, width), low part first.
Q4K_SC_FIELDS = [[(j, 0, 6)] if j < 4 else [(j + 4, 0, 4), (j - 4, 6, 2)] for j in range(8)]
Q4K_M_FIELDS = [[(j + 4, 0, 6)] if j < 4 else [(j + 4, 4, 4), (j, 6, 2)] for j in range(8)]


def _field(s: np.ndarray, fields: list[tuple[int, int, int]]) -> np.ndarray:
    out, shift = np.zeros(len(s), np.int64), 0
    for byte, lo, width in fields:
        out |= ((s[:, byte].astype(np.int64) >> lo) & ((1 << width) - 1)) << shift
        shift += width
    return out


def q4k_fields(b: np.ndarray, e: int) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(sc, m, q) of element e (0..255) of Q4_K blocks ``b`` [n, 144].  Sub-block j = e // 32; its 32 codes are the low
    (j even) or high (j odd) nibbles of qs bytes 32 (j // 2) .. + 31."""
    j, l = e // 32, e % 32
    s = b[:, 4:16]
    q = (b[:, 16 + 32 * (j // 2) + l].astype(np.int64) >> (4 * (j % 2))) & 15
    return _field(s, Q4K_SC_FIELDS[j]), _field(s, Q4K_M_FIELDS[j]), q


def q6k_fields(b: np.ndarray, e: int) -> tuple[np.ndarray, np.ndarray]:
    """(sc, q) of element e (0..255) of Q6_K blocks ``b`` [n, 210].  Half h = e // 128, group g = (e % 128) // 32 and
    lane l = e % 32: the code's low 4 bits are nibble g // 2 of ql[64 h + 32 (g % 2) + l], its high 2 bits are bits
    2 g .. 2 g + 1 of qh[32 h + l]; the int8 scale is scales[8 h + 2 g + l // 16]."""
    h, g, l = e // 128, (e % 128) // 32, e % 32
    lo = (b[:, 64 * h + 32 * (g % 2) + l].astype(np.int64) >> (4 * (g // 2))) & 15
    hi = (b[:, 128 + 32 * h + l].astype(np.int64) >> (2 * g)) & 3
    sc = b[:, 192 + 8 * h + 2 * g + l // 16].astype(np.int8).astype(np.int64)
    return sc, lo | (hi << 4)


def dequant_exact(ty: int, raw: np.ndarray) -> np.ndarray:
    """float64 [n_blocks, block_elems] of fp16 values (see the module docstring); asserts the exactness claims."""
    be, bb = BLOCK[ty]
    b = np.asarray(raw, np.uint8).reshape(-1, bb)
    y = np.empty((len(b), be), np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        if ty == Q8_0:
            d = f16_bits_value(_u16(b, 0))
            for e in range(32):
                v = d * b[:, 2 + e].astype(np.int8)
                _assert_f32_exact(v, "Q8_0 d q")
                y[:, e] = to_f16(v)
        elif ty == Q4_K:
            d, dmin = f16_bits_value(_u16(b, 0)), f16_bits_value(_u16(b, 2))
            for e in range(256):
                sc, m, q = q4k_fields(b, e)
                ds = d * sc
                a, c = ds * q, dmin * m
                for v, what in ((ds, "Q4_K d sc"), (a, "Q4_K (d sc) q"), (c, "Q4_K dmin m")):
                    _assert_f32_exact(v, what)
                y[:, e] = to_f16(to_f32(a - c))
        elif ty == Q6_K:
            d = f16_bits_value(_u16(b, 208))
            for e in range(256):
                sc, q = q6k_fields(b, e)
                ds = d * sc
                _assert_f32_exact(ds, "Q6_K d sc")
                y[:, e] = to_f16(to_f32(ds * (q - 32)))
        else:
            raise ValueError(ty)
    return y


def dequant_rows_exact(ty: int, raw: np.ndarray, rows: int, K: int) -> np.ndarray:
    return dequant_exact(ty, raw).reshape(rows, K)


# ---- block builders -------------------------------------------------------------------------------------------------
def _f16_bytes(bits: np.ndarray) -> np.ndarray:
    return np.asarray(bits, "<u2").reshape(-1, 1).view(np.uint8)


def q8_0_block(d: int, q: np.ndarray) -> np.ndarray:
    return np.concatenate([_f16_bytes(d)[0], np.asarray(q, np.int8).view(np.uint8)])


def q4_k_block(d: int, dmin: int, sc: np.ndarray, m: np.ndarray, q: np.ndarray) -> np.ndarray:
    """One Q4_K block from its fields: 8 sub-block scales / mins (0..63) and 256 codes (0..15) in element order."""
    b = np.zeros(144, np.uint8)
    b[0:2], b[2:4] = _f16_bytes(d)[0], _f16_bytes(dmin)[0]
    for fields, vals in ((Q4K_SC_FIELDS, sc), (Q4K_M_FIELDS, m)):
        for j in range(8):
            v, shift = int(vals[j]), 0
            for byte, lo, width in fields[j]:
                b[4 + byte] |= ((v >> shift) & ((1 << width) - 1)) << lo
                shift += width
    for e in range(256):
        j, l = e // 32, e % 32
        b[16 + 32 * (j // 2) + l] |= int(q[e]) << (4 * (j % 2))
    return b


def q6_k_block(d: int, sc: np.ndarray, q: np.ndarray) -> np.ndarray:
    """One Q6_K block from its fields: 16 int8 scales and 256 codes (0..63) in element order."""
    b = np.zeros(210, np.uint8)
    for e in range(256):
        h, g, l = e // 128, (e % 128) // 32, e % 32
        b[64 * h + 32 * (g % 2) + l] |= (int(q[e]) & 15) << (4 * (g // 2))
        b[128 + 32 * h + l] |= (int(q[e]) >> 4) << (2 * g)
    b[192:208] = np.asarray(sc, np.int8).view(np.uint8)
    b[208:210] = _f16_bytes(d)[0]
    return b


def edge_blocks(ty: int, *, nonfinite: bool = False) -> np.ndarray:
    """uint8 [n, block_bytes]: every scale-field edge value (every pair of them for Q4_K's d and dmin), every quant code,
    and (Q4_K) every 6-bit scale and min in each of the 8 sub-block positions, (Q6_K) every int8 scale in each of the 16
    positions and every 6-bit code in each group of both halves.  ``nonfinite`` adds +-inf and NaN scale fields."""
    scales = EDGE_F16 + (NONFINITE_F16 if nonfinite else [])
    out = []
    if ty == Q8_0:
        codes = np.arange(-128, 128)
        for d in scales:                      # every int8 code with every d
            out += [q8_0_block(d, codes[32 * i:32 * i + 32]) for i in range(8)]
            out.append(q8_0_block(d, np.resize([-1, 0, 1], 32)))   # finite even at d = 65504
    elif ty == Q4_K:
        e = np.arange(256)
        i = 0
        for d in scales:
            for dmin in scales:
                k = i % 64
                sc = (k + 9 * np.arange(8)) % 64          # over 64 consecutive blocks: every value in every position
                m = (5 * k + 17 * np.arange(8) + 1) % 64
                q = (e + 3 * k) % 16                      # every nibble twice per sub-block
                out.append(q4_k_block(d, dmin, sc, m, q))
                i += 1
                # the same scales on codes that stay finite even at 65504: d q (j even) and -dmin (j odd)
                out.append(q4_k_block(d, dmin, np.arange(8) % 2 == 0, np.arange(8) % 2, (e // 3) % 2))
        for k in range(64):                               # the 6-bit fields once more at d = dmin = 1
            out.append(q4_k_block(0x3C00, 0x3C00, (k + 9 * np.arange(8)) % 64, (k + 23 * np.arange(8)) % 64, e % 16))
    elif ty == Q6_K:
        e = np.arange(256)
        scs = np.arange(-128, 128)
        for i, d in enumerate(scales):
            for k in range(16):                           # every int8 scale in each of the 16 positions
                sc = scs[(16 * k + 7 * np.arange(16) + 3 * i) % 256]
                q = (e + 5 * k + i) % 64                  # every code in each group of 32 of both halves
                out.append(q6_k_block(d, sc, q))
            out.append(q6_k_block(d, np.resize([1, -1], 16), 31 + e % 3))   # +-d, 0: finite even at 65504
    else:
        raise ValueError(ty)
    return np.stack(out)


def finite_blocks(ty: int, blocks: np.ndarray) -> np.ndarray:
    """The blocks whose every element is finite (an infinity would poison a linear's column with 0 * inf)."""
    return blocks[np.isfinite(dequant_exact(ty, blocks)).all(axis=1)]


def tile_blocks(blocks: np.ndarray, ty: int, N: int, K: int, shift: int = 0) -> np.ndarray:
    """uint8 GGUF bytes of an N x K tensor whose blocks cycle through ``blocks`` from index ``shift``."""
    be, _ = BLOCK[ty]
    idx = (np.arange(N * K // be) + shift) % len(blocks)
    return np.ascontiguousarray(blocks[idx]).reshape(-1)


# ---- the quantized linear image ---------------------------------------------------------------------------------------
IMG_DATA = 2048            # where the passes' rows start
IMG_MAGIC = 0x51494D47     # "QIMG"
PASS_N = 128
SLICE_K = 128
ROW_BYTES = {Q8_0: 136, Q4_K: 76, Q6_K: 108}


def _nb16(N: int, p: int) -> int:
    return (min(PASS_N, N - PASS_N * p) + 15) // 16 * 16


def image_bytes(types: list[int], N: int, K: int) -> int:
    """Size of the image of N rows whose pass p has type types[p]."""
    return IMG_DATA + sum((K // SLICE_K) * _nb16(N, p) * ROW_BYTES[t] for p, t in enumerate(types))


def _slice_rows(ty: int, rows: np.ndarray, s: int) -> np.ndarray:
    """[n, row_bytes]: each row's bytes of K slice s, as the image lays them out (include/raglite_b200.h, csrc/xenc.cu)."""
    be, bb = BLOCK[ty]
    blk = rows.reshape(len(rows), -1, bb)
    if ty == Q8_0:
        b = blk[:, 4 * s:4 * s + 4]
        return np.concatenate([b[:, :, :2].reshape(len(rows), -1), b[:, :, 2:].reshape(len(rows), -1)], axis=1)
    b, h = blk[:, s // 2], s % 2
    if ty == Q4_K:
        sm = [_field(b[:, 4:16], f[4 * h + i])[:, None] for f in (Q4K_SC_FIELDS, Q4K_M_FIELDS) for i in range(4)]
        return np.concatenate([b[:, 0:4], np.concatenate(sm, axis=1).astype(np.uint8), b[:, 16 + 64 * h:80 + 64 * h]], axis=1)
    return np.concatenate([b[:, 64 * h:64 * h + 64], b[:, 128 + 32 * h:160 + 32 * h], b[:, 192 + 8 * h:200 + 8 * h],
                           b[:, 208:210], np.zeros((len(rows), 2), np.uint8)], axis=1)


def image(parts: list[tuple[int, np.ndarray, int]], K: int) -> np.ndarray:
    """The image of the row-wise concatenation of (type, GGUF bytes, rows) parts: what rl_xenc_pack_qlinear writes for
    one part and rl_xenc_concat_qlinear for several (every part but the last a whole number of passes).  Header: n_pass,
    N, K, magic (int32), then per pass its type, row_bytes (int32) and offset from the image's start (int64)."""
    passes = []   # (type, rows of the pass)
    for ty, raw, n in parts:
        r = np.asarray(raw, np.uint8).reshape(n, -1)
        passes += [(ty, r[PASS_N * p:PASS_N * (p + 1)]) for p in range((n + PASS_N - 1) // PASS_N)]
    N = sum(n for _, _, n in parts)
    head = np.zeros(IMG_DATA, np.uint8)
    head[:16] = np.array([len(passes), N, K, IMG_MAGIC], "<i4").view(np.uint8)
    off, body = IMG_DATA, []
    for p, (ty, pr) in enumerate(passes):
        nb16, rb = (len(pr) + 15) // 16 * 16, ROW_BYTES[ty]
        head[16 + 16 * p:24 + 16 * p] = np.array([ty, rb], "<i4").view(np.uint8)
        head[24 + 16 * p:32 + 16 * p] = np.array([off], "<i8").view(np.uint8)
        run = np.zeros((K // SLICE_K, nb16, rb), np.uint8)   # padding rows up to nb16: zero bytes
        for s in range(K // SLICE_K):
            run[s, :len(pr)] = _slice_rows(ty, pr, s)
        body.append(run.reshape(-1))
        off += run.size
    out = np.concatenate([head, *body])
    assert out.size == image_bytes([t for t, _ in passes], N, K)
    return out
