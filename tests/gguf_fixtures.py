"""GGUF test fixtures: a writer of the tests' own, ggml's Q8_0 / Q4_K / Q6_K dequantization restated in NumPy, seeded
quantized blocks, and XLM-RoBERTa models written the way llama.cpp's converter lays them out.

Dequantization follows ggml's C code (``dequantize_row_q8_0 / _q4_K / _q6_K``), in float32 with every product and
difference rounded on its own: Q8_0 ``d * q``; Q4_K ``d1 = d * sc``, ``m1 = dmin * m``, ``d1 * q - m1``; Q6_K
``d * sc * q`` evaluated left to right, ``(d * sc) * (q - 32)``.
"""

from __future__ import annotations

import struct
from pathlib import Path
from typing import Any

import numpy as np

F32, F16, Q8_0, Q4_K, Q6_K = 0, 1, 8, 12, 14
BLOCK = {F32: (1, 4), F16: (1, 2), Q8_0: (32, 34), Q4_K: (256, 144), Q6_K: (256, 210)}
# metadata value types
U8, I8, U16, I16, U32, I32, F32V, BOOL, STR, ARR, U64, I64, F64 = range(13)
_FMT = {U8: "<B", I8: "<b", U16: "<H", I16: "<h", U32: "<I", I32: "<i", F32V: "<f", BOOL: "<?", U64: "<Q", I64: "<q",
        F64: "<d"}


def _str(s: str | bytes) -> bytes:
    b = s.encode() if isinstance(s, str) else s
    return struct.pack("<Q", len(b)) + b


def _val(vtype: int, v: Any) -> bytes:
    if vtype in _FMT:
        return struct.pack(_FMT[vtype], v)
    if vtype == STR:
        return _str(v)
    sub, items = v
    out = struct.pack("<IQ", sub, len(items))
    return out + b"".join(_val(sub, x) for x in items)


def write_gguf(path: Path | str, metadata: list[tuple[str, int, Any]], tensors: list[tuple[str, int, tuple[int, ...], bytes]],
               *, alignment: int = 32, version: int = 3) -> None:
    """``metadata``: (key, value type, value; arrays as (sub type, items)).  ``tensors``: (name, GGML type, shape
    outermost first, raw bytes).  ``general.alignment`` is written when it is not 32."""
    meta = list(metadata)
    if alignment != 32:
        meta.append(("general.alignment", U32, alignment))
    head = b"GGUF" + struct.pack("<IQQ", version, len(tensors), len(meta))
    head += b"".join(_str(k) + struct.pack("<I", t) + _val(t, v) for k, t, v in meta)
    off, infos, datas = 0, b"", []
    for name, ty, shape, raw in tensors:
        infos += _str(name) + struct.pack("<I", len(shape)) + b"".join(struct.pack("<Q", n) for n in reversed(shape))
        infos += struct.pack("<IQ", ty, off)
        pad = (-len(raw)) % alignment
        datas.append(raw + b"\0" * pad)
        off += len(raw) + pad
    head += infos
    head += b"\0" * ((-len(head)) % alignment)
    Path(path).write_bytes(head + b"".join(datas))


# ---- dequantization ------------------------------------------------------------------------------------------------
def _h(b: np.ndarray) -> np.ndarray:
    return np.ascontiguousarray(b).view("<f2").astype(np.float32)


def dequant(ty: int, raw: np.ndarray, rows: int, K: int) -> np.ndarray:
    """float32 [rows, K] from GGUF block bytes (ggml's arithmetic, see the module docstring)."""
    be, bb = BLOCK[ty]
    b = np.asarray(raw, dtype=np.uint8).reshape(-1, bb)
    if ty == F32:
        return b.view("<f4").reshape(rows, K).astype(np.float32)
    if ty == F16:
        return _h(b).reshape(rows, K)
    if ty == Q8_0:
        d = _h(b[:, :2])
        q = b[:, 2:].view(np.int8).astype(np.float32)
        y = d * q
    elif ty == Q4_K:
        d, dmin, s, qs = _h(b[:, 0:2]), _h(b[:, 2:4]), b[:, 4:16].astype(np.int32), b[:, 16:]
        sc = np.empty((len(b), 8), np.int32)
        m = np.empty((len(b), 8), np.int32)
        for j in range(8):
            if j < 4:
                sc[:, j], m[:, j] = s[:, j] & 63, s[:, j + 4] & 63
            else:
                sc[:, j] = (s[:, j + 4] & 0xF) | ((s[:, j - 4] >> 6) << 4)
                m[:, j] = (s[:, j + 4] >> 4) | ((s[:, j] >> 6) << 4)
        y = np.empty((len(b), 256), np.float32)
        for j64 in range(4):
            q = qs[:, 32 * j64:32 * j64 + 32]
            for hi in range(2):
                sub = 2 * j64 + hi
                d1 = d * sc[:, sub:sub + 1].astype(np.float32)
                m1 = dmin * m[:, sub:sub + 1].astype(np.float32)
                y[:, 64 * j64 + 32 * hi:64 * j64 + 32 * hi + 32] = d1 * ((q >> (4 * hi)) & 0xF).astype(np.float32) - m1
    elif ty == Q6_K:
        ql, qh, sc, d = b[:, :128].astype(np.int32), b[:, 128:192].astype(np.int32), b[:, 192:208].view(np.int8), _h(b[:, 208:210])
        y = np.empty((len(b), 256), np.float32)
        for n in range(2):
            for g in range(4):
                l = np.arange(32)
                q = ((ql[:, 64 * n + l + 32 * (g & 1)] >> (4 * (g >> 1))) & 0xF) | (((qh[:, 32 * n + l] >> (2 * g)) & 3) << 4)
                s = sc[:, 8 * n + l // 16 + 2 * g].astype(np.float32)
                y[:, 128 * n + 32 * g + l] = (d * s) * (q - 32).astype(np.float32)
    else:
        raise ValueError(ty)
    return y.reshape(rows, K)


def random_blocks(ty: int, rows: int, K: int, rng: np.random.Generator, scale: float = 1.0) -> np.ndarray:
    """Seeded valid blocks of ``rows x K`` elements; fp16 scales small enough that nothing overflows fp16 downstream."""
    be, bb = BLOCK[ty]
    n = rows * K // be
    if ty in (F32, F16):
        w = (rng.standard_normal((rows, K)) * 0.05 * scale).astype(np.float16 if ty == F16 else np.float32)
        return w.view(np.uint8).reshape(-1)
    b = rng.integers(0, 256, (n, bb), dtype=np.uint8)

    def f16(lo: float, hi: float) -> np.ndarray:
        return (rng.uniform(lo, hi, (n, 1)) * scale).astype(np.float16).view(np.uint8)

    if ty == Q8_0:
        b[:, 0:2] = f16(2e-4, 8e-4)
    elif ty == Q4_K:
        b[:, 0:2] = f16(2e-5, 1e-4)
        b[:, 2:4] = f16(2e-5, 1e-4)
    else:
        b[:, 208:210] = f16(2e-6, 1e-5)
    return b.reshape(-1)


# ---- models as llama.cpp's converter writes them --------------------------------------------------------------------
def unigram_metadata(tok: Any, *, charsmap: bytes | None = None, remove_extra_ws: bool = True, bos: int = 0, eos: int = 2,
                     unk: int = 3, n_vocab: int | None = None) -> list[tuple[str, int, Any]]:
    """``tokenizer.ggml.*`` of a ``tokenizers`` Unigram tokenizer (tokens in id order with their scores), padded to
    ``n_vocab`` tokens with ``<unused{i}>`` pieces that no test text contains."""
    import json

    model = json.loads(tok.to_str())["model"]
    vocab = [tuple(v) for v in model["vocab"]]
    vocab += [(f"<unused{i}>", -100.0) for i in range((n_vocab or len(vocab)) - len(vocab))]
    md = [("tokenizer.ggml.model", STR, "t5"), ("tokenizer.ggml.tokens", ARR, (STR, [p for p, _ in vocab])),
          ("tokenizer.ggml.scores", ARR, (F32V, [float(s) for _, s in vocab])),
          ("tokenizer.ggml.token_type", ARR, (I32, [1] * len(vocab))),
          ("tokenizer.ggml.unknown_token_id", U32, unk), ("tokenizer.ggml.bos_token_id", U32, bos),
          ("tokenizer.ggml.eos_token_id", U32, eos), ("tokenizer.ggml.add_bos_token", BOOL, True),
          ("tokenizer.ggml.add_eos_token", BOOL, True), ("tokenizer.ggml.add_space_prefix", BOOL, True),
          ("tokenizer.ggml.remove_extra_whitespaces", BOOL, remove_extra_ws)]
    if charsmap is not None:
        md.append(("tokenizer.ggml.precompiled_charsmap", ARR, (U8, list(charsmap))))
    return md


# Q4_K_M as llama.cpp's quantizer mixes it for an encoder: attn_v and ffn_down of some layers in Q6_K, the rest Q4_K.
def q4_k_m_type(name: str, layer: int) -> int:
    if name in ("attn_v", "ffn_down") and layer % 2 == 0:
        return Q6_K
    return Q4_K


def write_xlmr_gguf(path: Path | str, model: Any, tok: Any, *, mode: str, rng: np.random.Generator | None = None,
                    fused_qkv: bool = False, alignment: int = 32, dequantize: bool = True) -> dict[str, Any]:
    """Write an ``XLMRobertaModel`` as a ``bert`` GGUF file.  ``mode`` "F16": its weights as fp16.  "Q8_0" / "Q4_K_M":
    seeded quantized blocks replace the 2-D weights (Q4_K_M: Q4_K / Q6_K by ``q4_k_m_type``, embeddings Q6_K), and the
    model's state dict is overwritten with their dequantized values (so ``from_hf`` on it is the reference; skipped when
    ``dequantize`` is false).  Returns the state dict."""
    import torch

    c = model.config
    H, L = c.hidden_size, c.num_hidden_layers
    sd = {k: v.detach().clone().float() for k, v in model.state_dict().items()}
    pad = c.pad_token_id + 1
    tensors: list[tuple[str, int, tuple[int, ...], bytes]] = []

    def put(name: str, hf: str, ty: int, rows: slice | None = None) -> None:
        w = sd[hf] if rows is None else sd[hf][rows]
        if w.dim() == 1 or ty == F32:
            tensors.append((name, F32, tuple(w.shape), w.numpy().astype("<f4").tobytes()))
        elif ty == F16:
            tensors.append((name, F16, tuple(w.shape), w.numpy().astype("<f2").tobytes()))
        else:
            N, K = w.shape
            raw = random_blocks(ty, N, K, rng)
            if dequantize:
                deq = torch.from_numpy(dequant(ty, raw, N, K))
                if rows is None:
                    sd[hf] = deq
                else:
                    sd[hf][rows] = deq
            tensors.append((name, ty, (N, K), raw.tobytes()))

    emb_ty = F16 if mode == "F16" else (Q8_0 if mode == "Q8_0" else Q6_K)
    e = "embeddings."
    put("token_embd.weight", e + "word_embeddings.weight", emb_ty)
    put("position_embd.weight", e + "position_embeddings.weight", emb_ty, slice(pad, None))
    put("token_types.weight", e + "token_type_embeddings.weight", F32)
    put("token_embd_norm.weight", e + "LayerNorm.weight", F32)
    put("token_embd_norm.bias", e + "LayerNorm.bias", F32)
    for i in range(L):
        p, b = f"encoder.layer.{i}.", f"blk.{i}."

        def ty(name: str, i: int = i) -> int:
            return {"F16": F16, "Q8_0": Q8_0}.get(mode) or q4_k_m_type(name, i)

        if fused_qkv:
            for part in ("weight", "bias"):
                names = [p + f"attention.self.{n}.{part}" for n in ("query", "key", "value")]
                sd[p + f"attention.self.qkv.{part}"] = torch.cat([sd[n] for n in names])
            put(b + "attn_qkv.weight", p + "attention.self.qkv.weight", ty("attn_qkv"))
            put(b + "attn_qkv.bias", p + "attention.self.qkv.bias", F32)
            for j, n in enumerate(("query", "key", "value")):
                for part in ("weight", "bias"):
                    sd[p + f"attention.self.{n}.{part}"] = sd[p + f"attention.self.qkv.{part}"][j * H:(j + 1) * H].clone()
            sd.pop(p + "attention.self.qkv.weight")
            sd.pop(p + "attention.self.qkv.bias")
        else:
            for n, g in (("query", "q"), ("key", "k"), ("value", "v")):
                put(b + f"attn_{g}.weight", p + f"attention.self.{n}.weight", ty(f"attn_{g}"))
                put(b + f"attn_{g}.bias", p + f"attention.self.{n}.bias", F32)
        for g, hf in (("attn_output", "attention.output.dense"), ("ffn_up", "intermediate.dense"), ("ffn_down", "output.dense")):
            put(b + f"{g}.weight", p + hf + ".weight", ty(g))
            put(b + f"{g}.bias", p + hf + ".bias", F32)
        for g, hf in (("attn_output_norm", "attention.output.LayerNorm"), ("layer_output_norm", "output.LayerNorm")):
            put(b + f"{g}.weight", p + hf + ".weight", F32)
            put(b + f"{g}.bias", p + hf + ".bias", F32)
    md = [("general.architecture", STR, "bert"), ("general.name", STR, "test"),
          ("bert.block_count", U32, L), ("bert.context_length", U32, c.max_position_embeddings - pad),
          ("bert.embedding_length", U32, H), ("bert.feed_forward_length", U32, c.intermediate_size),
          ("bert.attention.head_count", U32, c.num_attention_heads),
          ("bert.attention.layer_norm_epsilon", F32V, float(c.layer_norm_eps)), ("bert.attention.causal", BOOL, False),
          ("bert.pooling_type", U32, 2), *unigram_metadata(tok, n_vocab=c.vocab_size)]
    write_gguf(path, md, tensors, alignment=alignment)
    return sd
