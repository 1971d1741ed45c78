"""GGUF embedders on the GPU: the quantized wgmma linear and the dequantized rows bit for bit against the NumPy
restatement of ggml's arithmetic, and whole engines loaded from F16 / Q8_0 / Q4_K_M-style files against ``from_hf`` on
the same (dequantized) weights."""

from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

from gguf_fixtures import Q4_K, Q6_K, Q8_0, dequant, random_blocks, write_xlmr_gguf

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():  # noqa: ANN201
    from raglite_b200 import _lib

    return _lib.load()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _fp16_image(lib, W: np.ndarray) -> torch.Tensor:  # noqa: ANN001
    N, K = W.shape
    Wd = torch.from_numpy(W).cuda()
    img = torch.empty(int(lib.rl_xenc_linear_image_bytes(N, K)), dtype=torch.uint8, device="cuda")
    assert lib.rl_xenc_pack_linear(Wd.data_ptr(), N, K, img.data_ptr(), _stream()) == 0
    return img


def _q_image(lib, parts: list[tuple[int, np.ndarray, int]], K: int) -> torch.Tensor:  # noqa: ANN001
    """Quantized image of (type, blocks, rows) parts: one pack per part, concatenated when there are several."""
    imgs = []
    for ty, raw, N in parts:
        blocks = torch.from_numpy(raw).cuda()
        img = torch.empty(int(lib.rl_xenc_qlinear_image_bytes(ty, N, K)), dtype=torch.uint8, device="cuda")
        assert img.numel() > 0
        assert lib.rl_xenc_pack_qlinear(ty, blocks.data_ptr(), N, K, img.data_ptr(), _stream()) == 0
        imgs.append(img)
    if len(imgs) == 1:
        return imgs[0]
    out = torch.empty(sum(i.numel() for i in imgs), dtype=torch.uint8, device="cuda")
    ptrs = (C.c_void_p * len(imgs))(*[i.data_ptr() for i in imgs])
    assert lib.rl_xenc_concat_qlinear(ptrs, len(imgs), out.data_ptr(), _stream()) == 0
    return out


def _run(lib, fn, X, img, bias, N, K, act):  # noqa: ANN001, ANN202
    Y = torch.empty((X.shape[0], N), dtype=torch.float16, device="cuda")
    assert fn(X.data_ptr(), img.data_ptr(), bias.data_ptr(), Y.data_ptr(), X.shape[0], N, K, act, _stream()) == 0, \
        lib.rl_last_error()
    return Y


SHAPES = [(1, 32, 256), (127, 96, 1024), (128, 1024, 1024), (129, 3072, 1024), (4097, 4096, 1024), (129, 1024, 4096),
          (4097, 1024, 4096), (1, 4096, 256), (128, 32, 4096), (127, 3072, 256), (65536, 4096, 1024), (65536, 1024, 4096)]


@pytest.mark.parametrize("ty", [Q8_0, Q4_K, Q6_K, "qkv"])
@pytest.mark.parametrize(("T", "N", "K"), SHAPES)
@pytest.mark.parametrize("act", [0, 1])
def test_linear_q_matches_fp16_image_of_dequantized_weights(lib, ty, T, N, K, act) -> None:  # noqa: ANN001
    rng = np.random.default_rng(hash((str(ty), T, N, K, act)) % 2**32)
    if ty == "qkv":   # Q4_K | Q4_K | Q6_K passes in one image (N rows each, N % 128 == 0 only)
        if N % 128:
            pytest.skip("mixed-type images concatenate whole passes")
        parts = [(t, random_blocks(t, N, K, rng), N) for t in (Q4_K, Q4_K, Q6_K)]
        N = 3 * N
        if N > 8192:
            pytest.skip("over the image's 64 passes")
    else:
        parts = [(ty, random_blocks(ty, N, K, rng), N)]
    W = np.concatenate([dequant(t, raw, n, K) for t, raw, n in parts])
    X = torch.from_numpy(rng.standard_normal((T, K)).astype(np.float16)).cuda()
    bias = torch.from_numpy(rng.standard_normal(N).astype(np.float32) * 0.1).cuda()
    want = _run(lib, lib.rl_xenc_linear, X, _fp16_image(lib, W), bias, N, K, act)
    img = _q_image(lib, parts, K)
    got = _run(lib, lib.rl_xenc_linear_q, X, img, bias, N, K, act)
    torch.cuda.synchronize()
    assert torch.isfinite(want.float()).all()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))
    gguf_bytes = sum(raw.nbytes for _, raw, _ in parts)
    assert img.numel() <= 1.07 * gguf_bytes + 2048 * len(parts)


@pytest.mark.parametrize("parts", [[(Q8_0, 8192)], [(Q4_K, 8192)], [(Q6_K, 8192)], [(Q4_K, 4096), (Q6_K, 4096)],
                                   [(Q4_K, 8064), (Q8_0, 96)], [(Q6_K, 128)] * 64])
@pytest.mark.parametrize("T", [1, 129])
def test_linear_q_at_64_passes(lib, parts, T) -> None:  # noqa: ANN001
    """N = 8192 (or just under): the image's last pass descriptors sit at the end of its header, packed alone or
    concatenated from parts of other types."""
    K = 1024
    rng = np.random.default_rng(len(parts) * 7 + T)
    parts = [(t, random_blocks(t, n, K, rng), n) for t, n in parts]
    N = sum(n for _, _, n in parts)
    W = np.concatenate([dequant(t, raw, n, K) for t, raw, n in parts])
    X = torch.from_numpy(rng.standard_normal((T, K)).astype(np.float16)).cuda()
    bias = torch.from_numpy(rng.standard_normal(N).astype(np.float32) * 0.1).cuda()
    want = _run(lib, lib.rl_xenc_linear, X, _fp16_image(lib, W), bias, N, K, 0)
    got = _run(lib, lib.rl_xenc_linear_q, X, _q_image(lib, parts, K), bias, N, K, 0)
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))


def test_qlinear_shape_limits(lib) -> None:  # noqa: ANN001
    assert lib.rl_xenc_qlinear_image_bytes(Q4_K, 8192, 1024) > 0
    assert lib.rl_xenc_qlinear_image_bytes(Q4_K, 8224, 1024) == 0   # 65 passes
    assert lib.rl_xenc_qlinear_image_bytes(Q8_0, 96, 96) == 0       # K % 128


@pytest.mark.parametrize("ty", [Q8_0, Q4_K, Q6_K])
def test_dequant_rows_matches_numpy(lib, ty) -> None:  # noqa: ANN001
    rng = np.random.default_rng(ty)
    for rows, K in ((1, 256), (3, 512), (1000, 1024)):
        raw = random_blocks(ty, rows, K, rng, scale=100.0)
        if ty == Q8_0:   # subnormal and extreme d
            raw.reshape(-1, 34)[:4, :2] = np.array([1, 0x8001, 0x03FF, 0x7BFF], np.uint16).view(np.uint8).reshape(4, 2)
        out = torch.empty((rows, K), dtype=torch.float16, device="cuda")
        assert lib.rl_dequant_rows_f16(ty, torch.from_numpy(raw).cuda().data_ptr(), rows, K, out.data_ptr(), _stream()) == 0
        with np.errstate(over="ignore"):   # d = 65504 times 127 rounds to inf, as on the device
            want = dequant(ty, raw, rows, K).astype(np.float16)
        assert np.array_equal(out.cpu().numpy().view(np.uint16), want.view(np.uint16))


# ---- whole engines ---------------------------------------------------------------------------------------------------
def _model():  # noqa: ANN202
    from oracle.embed import bge_m3_config, seeded_model

    return seeded_model(bge_m3_config(num_hidden_layers=2, vocab_size=5000, max_position_embeddings=514))


def _lengths() -> list[int]:
    base = [1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 200, 255, 256, 257, 383, 384, 385, 511, 512]
    return base + list(np.random.default_rng(5).integers(1, 513, 40))


@pytest.mark.parametrize(("mode", "fused"), [("F16", False), ("Q8_0", False), ("Q4_K_M", False), ("Q4_K_M", True)])
def test_engine_from_gguf_equals_from_hf(tmp_path, mode, fused) -> None:  # noqa: ANN001
    from oracle.embed import unigram_tokenizer
    from raglite_b200 import TokenEmbedderEngine

    model = _model()
    path = tmp_path / f"m-{mode}.gguf"
    sd = write_xlmr_gguf(path, model, unigram_tokenizer(), mode=mode, rng=np.random.default_rng(1), fused_qkv=fused)
    model.load_state_dict(sd)
    ref = TokenEmbedderEngine.from_hf(model, unigram_tokenizer())
    eng = TokenEmbedderEngine.from_gguf(path)
    assert eng.n_ctx() == 512 and eng.pos_offset == 0
    rng = np.random.default_rng(2)
    ids = [rng.integers(4, 5000, n).astype(np.int32) for n in _lengths()]
    a, oa = ref.embed_token_ids(ids)
    b, ob = eng.embed_token_ids(ids)
    assert np.array_equal(oa, ob)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_register_gguf_embedder_matches_from_hf(tmp_path, monkeypatch) -> None:  # noqa: ANN001
    import raglite_b200 as rl
    from oracle.embed import unigram_tokenizer
    from raglite_b200 import RAGLiteConfig, TokenEmbedderEngine

    model = _model()
    snap = tmp_path / "hub" / "models--lm-kit--bge-m3-gguf" / "snapshots" / "abc"
    snap.mkdir(parents=True)
    sd = write_xlmr_gguf(snap / "bge-m3-Q4_K_M.gguf", model, unigram_tokenizer(), mode="Q4_K_M",
                         rng=np.random.default_rng(3))
    model.load_state_dict(sd)
    monkeypatch.setenv("HF_HUB_CACHE", str(tmp_path / "hub"))
    cfg_g = RAGLiteConfig(embedder="llama-cpp-python/lm-kit/bge-m3-gguf/*Q4_K_M.gguf@512")
    cfg_h = RAGLiteConfig(embedder="llama-cpp-python/test/hf-reference/x.gguf@512")
    eng = rl.register_gguf_embedder(cfg_g)
    assert eng.n_ctx() == 512
    # the file says remove_extra_whitespaces: the reference tokenizer gets the same Replace(" {2,}", " ") normaliser
    from tokenizers import Regex, normalizers

    ref_tok = unigram_tokenizer()
    ref_tok.normalizer = normalizers.Replace(Regex(" {2,}"), " ")
    rl.register_token_embedder(cfg_h.embedder, TokenEmbedderEngine.from_hf(model, ref_tok))
    assert eng.tokenize(b"the   clock  of") == eng.tokenize(b"the clock of") == ref_tok.encode(
        "the clock of", add_special_tokens=False).ids
    sentences = ["What is the velocity of light? ", "The observer  in a   frame of time. ", "Alpha beta gamma delta. " * 30,
                 "A clock, a rod and an event.\n"]
    assert np.array_equal(rl.embed_strings(sentences, config=cfg_g).view(np.uint16),
                          rl.embed_strings(sentences, config=cfg_h).view(np.uint16))
    queries = ["what is time", "How does the observer see the clock?", "é light"]
    assert np.array_equal(rl.embed_queries(queries, config=cfg_g).view(np.uint16),
                          rl.embed_queries(queries, config=cfg_h).view(np.uint16))


def test_full_shape_q4_k_m_loads(tmp_path) -> None:  # noqa: ANN001
    """24 layers at bge-m3's full vocabulary: resident weights within 1.07x the file's quantized linear bytes, plus the
    fp16 embedding tables and the float32 biases and norms."""
    from oracle.embed import bge_m3_config, seeded_model, unigram_tokenizer
    from raglite_b200 import TokenEmbedderEngine
    from raglite_b200._gguf import QUANT_TYPES, GGUFFile

    model = seeded_model(bge_m3_config(max_position_embeddings=514), perturb=False)
    path = tmp_path / "bge-m3-Q4_K_M.gguf"
    write_xlmr_gguf(path, model, unigram_tokenizer(), mode="Q4_K_M", rng=np.random.default_rng(4), dequantize=False)
    del model
    f = GGUFFile(path)
    lin = sum(t.data.nbytes for n, t in f.tensors.items() if n.startswith("blk.") and t.ggml_type in QUANT_TYPES)
    emb = sum(np.prod(f.tensors[n].shape) * 2 for n in ("token_embd.weight", "position_embd.weight", "token_types.weight"))
    small = sum(t.data.nbytes for t in f.tensors.values() if len(t.shape) == 1)
    eng = TokenEmbedderEngine.from_gguf(path)
    resident = eng.weight_bytes()
    print(f"file tensors {f.tensor_bytes()} B, quantized linears {lin} B, resident {resident} B")
    assert resident <= 1.07 * lin + emb + small + 24 * 4 * 2048
    X, _ = eng.embed_token_ids([np.arange(4, 516, dtype=np.int32)])
    assert torch.isfinite(X).all()
