"""The decoder's kernels at the C-ABI against float64: the quantized GEMV, the embedding gather, QK-norm + RoPE, causal
GQA attention (prefill chunks and decode across key-range splits) and the sampler token for token."""

from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

from gguf_fixtures import Q4_K, Q6_K, Q8_0, dequant, random_blocks
from llm_oracle import attention_ref, rms_norm_ref, rope_ref, sample, sample_margin

pytestmark = pytest.mark.gpu

TYPES = {"Q8_0": Q8_0, "Q4_K": Q4_K, "Q6_K": Q6_K}


@pytest.fixture(scope="module")
def lib():
    from raglite_b200 import _lib

    return _lib.load()


def _stream() -> int:
    return int(torch.cuda.current_stream().cuda_stream)


def _linear(lib, ty: int, raw: np.ndarray, N: int, K: int, keep: list):
    from raglite_b200._lib import LlmLinear

    lin = LlmLinear()
    row = raw.nbytes // N
    parts = range(0, N, 8192)
    for i, r0 in enumerate(parts):
        n = min(8192, N - r0)
        blocks = torch.from_numpy(raw[r0 * row:(r0 + n) * row].copy()).cuda()
        img = torch.empty(int(lib.rl_xenc_qlinear_image_bytes(ty, n, K)), dtype=torch.uint8, device="cuda")
        assert lib.rl_xenc_pack_qlinear(ty, blocks.data_ptr(), n, K, img.data_ptr(), _stream()) == 0
        keep += [blocks, img]
        lin.parts[i] = img.data_ptr()
    lin.n_parts, lin.N, lin.K = len(parts), N, K
    return lin


@pytest.mark.parametrize("ty", list(TYPES))
@pytest.mark.parametrize("N,K", [(128, 256), (1024, 4096), (8192, 512), (8224, 256), (151936, 256)])
def test_qgemv_against_float64(lib, ty, N, K):
    t = TYPES[ty]
    rng = np.random.default_rng(N + K + t)
    raw = random_blocks(t, N, K, rng)
    W = dequant(t, raw, N, K).astype(np.float64)
    x = rng.standard_normal(K).astype(np.float16)
    keep: list = []
    lin = _linear(lib, t, raw, N, K, keep)
    ws = torch.empty(max(1, int(lib.rl_llm_qgemv_workspace_bytes(N, K))), dtype=torch.uint8, device="cuda")
    xd = torch.from_numpy(x).cuda()
    y = torch.empty(N, dtype=torch.float32, device="cuda")
    assert lib.rl_llm_qgemv(C.byref(lin), xd.data_ptr(), y.data_ptr(), 1, ws.data_ptr(), ws.numel(), _stream()) == 0
    got = y.cpu().numpy().astype(np.float64)
    want = W @ x.astype(np.float64)
    # fp32 products and sums over K: each term's error below K 2^-23 of the sum of |w x|
    bound = K * 2.0 ** -23 * (np.abs(W) @ np.abs(x.astype(np.float64))) + 1e-30
    assert np.all(np.abs(got - want) <= bound), float(np.max(np.abs(got - want) / bound))
    y16 = torch.empty(N, dtype=torch.float16, device="cuda")
    assert lib.rl_llm_qgemv(C.byref(lin), xd.data_ptr(), y16.data_ptr(), 0, ws.data_ptr(), ws.numel(), _stream()) == 0
    assert np.array_equal(y16.cpu().numpy(), y.cpu().numpy().astype(np.float16))


@pytest.mark.parametrize("ty", list(TYPES))
def test_embed_rows_equal_ggml_values(lib, ty):
    t = TYPES[ty]
    N, K = 8192 + 640, 512
    rng = np.random.default_rng(t)
    raw = random_blocks(t, N, K, rng)
    W = dequant(t, raw, N, K)
    keep: list = []
    lin = _linear(lib, t, raw, N, K, keep)
    ids = np.array([0, 1, 8191, 8192, 8192 + 639, 4000], dtype=np.int32)
    out = torch.empty((len(ids), K), dtype=torch.float32, device="cuda")
    assert lib.rl_llm_embed(C.byref(lin), torch.from_numpy(ids).cuda().data_ptr(), len(ids), out.data_ptr(), _stream()) == 0
    assert np.array_equal(out.cpu().numpy().view(np.uint32), W[ids].view(np.uint32))


@pytest.mark.parametrize("T,p0", [(1, 0), (5, 37), (40, 100)])
def test_qk_norm_rope_against_float64(lib, T, p0):
    nh, nkv, n_ctx, eps, base = 8, 2, 256, 1e-6, 1e6
    rng = np.random.default_rng(T)
    qkv = rng.standard_normal((T, nh + 2 * nkv, 128)).astype(np.float16)
    qn = (1 + 0.2 * rng.standard_normal(128)).astype(np.float32)
    kn = (1 + 0.2 * rng.standard_normal(128)).astype(np.float32)
    dq = torch.empty((T, nh, 128), dtype=torch.float16, device="cuda")
    kc = torch.zeros((n_ctx, nkv, 128), dtype=torch.float16, device="cuda")
    vc = torch.zeros_like(kc)
    qn_d, kn_d = torch.from_numpy(qn).cuda(), torch.from_numpy(kn).cuda()
    assert lib.rl_llm_qk_norm_rope(torch.from_numpy(qkv).cuda().data_ptr(), T, p0, nh, nkv, qn_d.data_ptr(), kn_d.data_ptr(),
                                   eps, base, n_ctx, dq.data_ptr(), kc.data_ptr(), vc.data_ptr(), _stream()) == 0
    pos = np.arange(p0, p0 + T)[:, None]
    q_want = rope_ref(rms_norm_ref(qkv[:, :nh], qn, eps), np.broadcast_to(pos, (T, nh)), base)
    k_want = rope_ref(rms_norm_ref(qkv[:, nh:nh + nkv], kn, eps), np.broadcast_to(pos, (T, nkv)), base)
    # fp16 output rounding (2^-11 relative) plus fp32 angle error: pos * 2^-23 rad at most a few ulps
    tol = 2.0 ** -10 * np.abs(q_want).max() + (p0 + T) * 2.0 ** -21 * np.abs(q_want).max()
    assert np.abs(dq.cpu().numpy() - q_want).max() <= tol
    assert np.abs(kc.cpu().numpy()[p0:p0 + T] - k_want).max() <= tol
    assert np.array_equal(vc.cpu().numpy()[p0:p0 + T], qkv[:, nh + nkv:])
    assert not kc.cpu().numpy()[:p0].any() and not kc.cpu().numpy()[p0 + T:].any()


def _attention(lib, q, k, v, p0, nh, nkv, splits):
    T = q.shape[0]
    ws = torch.empty(max(1, int(lib.rl_llm_attention_workspace_bytes(T, nh, nkv, p0 + T, splits))), dtype=torch.uint8,
                     device="cuda")
    out = torch.empty((T, nh, 128), dtype=torch.float16, device="cuda")
    qd, kd, vd = (torch.from_numpy(a).cuda() for a in (q, k, v))
    rc = lib.rl_llm_attention(qd.data_ptr(), kd.data_ptr(), vd.data_ptr(), T, p0, nh, nkv, splits, out.data_ptr(),
                              ws.data_ptr(), ws.numel(), _stream())
    assert rc == 0
    return out.cpu().numpy().astype(np.float64)


@pytest.mark.parametrize("group", [1, 2, 4, 5, 8])
@pytest.mark.parametrize("T,p0", [(1, 0), (1, 63), (1, 64), (1, 65), (1, 511), (7, 0), (33, 90), (130, 17)])
def test_attention_against_float64(lib, group, T, p0):
    nkv = 2
    nh = group * nkv
    rng = np.random.default_rng(group * 1000 + T + p0)
    n_keys = p0 + T
    q = rng.standard_normal((T, nh, 128)).astype(np.float16)
    k = rng.standard_normal((n_keys, nkv, 128)).astype(np.float16)
    v = rng.standard_normal((n_keys, nkv, 128)).astype(np.float16)
    want = attention_ref(q, k, v, p0)
    for splits in (0, 1, 3):
        got = _attention(lib, q, k, v, p0, nh, nkv, splits)
        # fp16 output (2^-11 relative of |out| <= max|v|) + fp32 softmax and sums
        assert np.abs(got - want).max() <= 2.0 ** -10 * np.abs(v).max() + 1e-4, splits


def test_attention_splits_combine_every_range(lib):
    """A long decode whose keys all matter: a dropped key range moves the output."""
    nh, nkv, n_keys = 8, 8, 2048
    rng = np.random.default_rng(5)
    q = rng.standard_normal((1, nh, 128)).astype(np.float16) * np.float16(0.05)
    k = rng.standard_normal((n_keys, nkv, 128)).astype(np.float16)
    v = rng.standard_normal((n_keys, nkv, 128)).astype(np.float16)
    want = attention_ref(q, k, v, n_keys - 1)
    got = _attention(lib, q, k, v, n_keys - 1, nh, nkv, 0)
    assert np.abs(got - want).max() <= 2.0 ** -10 * np.abs(v).max() + 1e-4


def _sample_dev(lib, logits, hist, **kw):
    V = len(logits)
    ws = torch.empty(int(lib.rl_llm_sample_workspace_bytes(V)), dtype=torch.uint8, device="cuda")
    ld = torch.from_numpy(np.asarray(logits, np.float32)).cuda()
    hd = torch.from_numpy(np.asarray(hist, np.int32) if len(hist) else np.zeros(1, np.int32)).cuda()
    out = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    rc = lib.rl_llm_sample(ld.data_ptr(), V, hd.data_ptr(), len(hist), kw["temperature"], kw["top_k"], kw["top_p"],
                           kw["min_p"], kw["penalty"], kw["u"], out.data_ptr(), ws.data_ptr(), ws.numel(), _stream())
    return rc, int(out.cpu()[0])


@pytest.mark.parametrize("V", [640, 151936])
def test_sampler_matches_the_numpy_chain(lib, V):
    rng = np.random.default_rng(V)
    n_checked = 0
    for trial in range(60):
        logits = (rng.standard_normal(V) * 3).astype(np.float32)
        if trial % 3 == 0:   # ties: quantized logits
            logits = np.round(logits).astype(np.float32)
        hist = rng.integers(0, V, size=int(rng.integers(0, 65))).tolist()
        kw = dict(temperature=[0.0, 0.6, 1.0, 2.0][trial % 4], top_k=[1, 20, 40, 256][trial % 4],
                  top_p=[0.95, 0.5, 1.0, 0.8][(trial // 4) % 4], min_p=[0.0, 0.05][trial % 2], penalty=[1.1, 1.0][trial % 2],
                  u=float(np.float32(rng.random())))
        rc, got = _sample_dev(lib, logits, hist, **kw)
        assert rc == 0
        if kw["temperature"] > 0 and kw["min_p"] == 0 and sample_margin(logits, hist, **kw) < 1e-5:
            continue   # within float32 rounding of a CDF boundary
        assert got == sample(logits, hist, **kw), (trial, kw)
        n_checked += 1
    assert n_checked >= 40


def test_sampler_ties_take_the_lowest_id_and_top_p_keeps_the_crossing_token(lib):
    logits = np.zeros(640, np.float32)
    logits[[7, 3, 500]] = 5.0
    kw = dict(temperature=0.0, top_k=20, top_p=0.95, min_p=0.0, penalty=1.0, u=0.5)
    assert _sample_dev(lib, logits, [], **kw)[1] == 3
    kw.update(temperature=1.0, top_k=3, u=0.99)   # three equal candidates 3 < 7 < 500: u = 0.99 takes the last
    assert _sample_dev(lib, logits, [], **kw)[1] == 500
    # top-p 0.5 over {0.6, 0.3, 0.1}: the first token alone reaches 0.6 >= 0.5 -> only id 1 survives
    logits = np.full(640, -30.0, np.float32)
    logits[[1, 2, 4]] = np.log([0.6, 0.3, 0.1]).astype(np.float32)
    kw.update(top_p=0.5, top_k=20, u=0.99)
    assert _sample_dev(lib, logits, [], **kw)[1] == 1
    kw.update(top_p=0.7)   # 0.6 < 0.7 <= 0.9: the crossing token 2 is kept, u = 0.99 lands on it
    assert _sample_dev(lib, logits, [], **kw)[1] == 2
    # the penalty divides a positive logit: token 1 with history [1] drops below token 2 at penalty 10
    kw.update(temperature=0.0)
    assert _sample_dev(lib, logits, [1, 1], **dict(kw, penalty=10.0))[1] == 2


def test_refused_arguments_return_their_codes(lib):
    from raglite_b200._lib import LlmLinear

    dummy = torch.zeros(1024, dtype=torch.uint8, device="cuda").data_ptr()
    s = _stream()
    assert lib.rl_llm_sample(dummy, 640, dummy, 0, 0.6, 0, 0.9, 0.0, 1.1, 0.5, dummy, dummy, 4096, s) == -1     # top_k 0
    assert lib.rl_llm_sample(dummy, 640, dummy, 0, 0.6, 257, 0.9, 0.0, 1.1, 0.5, dummy, dummy, 4096, s) == -1   # top_k 257
    assert lib.rl_llm_sample(dummy, 640, dummy, 0, 0.6, 20, 0.9, 0.0, 1.1, 1.0, dummy, dummy, 4096, s) == -1    # u = 1
    assert lib.rl_llm_sample(dummy, 640, dummy, 0, 0.6, 20, 0.9, 0.0, 1.1, 0.5, dummy, dummy, 4, s) == -3       # workspace
    assert lib.rl_llm_attention(dummy, dummy, dummy, 1, 0, 6, 4, 0, dummy, dummy, 0, s) == -4   # 6 % 4 != 0
    assert lib.rl_llm_attention(dummy, dummy, dummy, 1, 0, 18, 2, 0, dummy, dummy, 0, s) == -4  # group 9
    assert lib.rl_llm_attention(dummy, dummy, dummy, 0, 0, 8, 2, 0, dummy, dummy, 0, s) == -1   # T 0
    assert lib.rl_llm_qk_norm_rope(dummy, 4, 254, 8, 2, dummy, dummy, 1e-6, 1e6, 256, dummy, dummy, dummy, s) == -1
    lin = LlmLinear()
    lin.n_parts, lin.N, lin.K = 1, 100, 256   # N % 32 != 0
    lin.parts[0] = dummy
    assert lib.rl_llm_qgemv(C.byref(lin), dummy, dummy, 1, dummy, 1 << 20, s) == -4
    lin.N, lin.n_parts = 8224, 1   # needs two parts
    assert lib.rl_llm_qgemv(C.byref(lin), dummy, dummy, 1, dummy, 1 << 20, s) == -4
    lin.N, lin.n_parts, lin.K = 128, 1, 200   # K % 128 != 0
    assert lib.rl_llm_qgemv(C.byref(lin), dummy, dummy, 1, dummy, 1 << 20, s) == -4
    assert lib.rl_llm_workspace_bytes(None, 16) == 0
