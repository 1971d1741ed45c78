"""Qwen3 test fixtures: a tiny random ``transformers.Qwen3ForCausalLM`` written as a ``qwen3`` GGUF file the way
llama.cpp's converter lays Qwen3 out (Q / K unpermuted, names ``blk.{i}.attn_q`` ...), with seeded quantized blocks in
place of the 2-D weights and the model's state dict overwritten with their dequantized values, and a byte-level BPE
vocabulary trained offline."""

from __future__ import annotations

from pathlib import Path
from typing import Any

import numpy as np

from gguf_fixtures import ARR, BOOL, F32, F32V, I32, Q4_K, Q6_K, Q8_0, STR, U32, dequant, random_blocks, write_gguf

SPECIAL = ["<|endoftext|>", "<|im_start|>", "<|im_end|>"]
CORPUS = [
    "The quick brown fox jumps over the lazy dog. It's 2024, and we'll see 12345 results!",
    "Retrieval-augmented generation answers questions from documents: <context> holds them.",
    "日本語のテキストと中文文本。 Emoji 🎉🚀 and café naïve résumé.",
    "def f(x):\n    return x + 1\n\n\n  spaces   and\ttabs\r\n",
    "They're here, you've seen it, I'm sure, she'd go, we'll stay.",
] * 20


def train_bpe(vocab_size: int = 400) -> tuple[list[str], list[str]]:
    """Byte-level BPE tokens (special tokens last) and merges, trained on CORPUS with the Qwen2 split."""
    from tokenizers import Regex, Tokenizer, models, pre_tokenizers, trainers

    from raglite_b200._llm import QWEN2_SPLIT

    tok = Tokenizer(models.BPE())
    tok.pre_tokenizer = pre_tokenizers.Sequence([pre_tokenizers.Split(Regex(QWEN2_SPLIT), behavior="isolated"),
                                                 pre_tokenizers.ByteLevel(add_prefix_space=False, use_regex=False)])
    trainer = trainers.BpeTrainer(vocab_size=vocab_size, initial_alphabet=pre_tokenizers.ByteLevel.alphabet(),
                                  show_progress=False)
    tok.train_from_iterator(CORPUS, trainer)
    import json

    m = json.loads(tok.to_str())["model"]
    vocab = sorted(m["vocab"].items(), key=lambda kv: kv[1])
    tokens = [t for t, _ in vocab]
    merges = [" ".join(x) if isinstance(x, list) else x for x in m["merges"]]
    return tokens + SPECIAL, merges


def make_model(*, vocab: int = 640, hidden: int = 256, n_head: int = 4, n_kv: int = 2, ffn: int = 768, layers: int = 2,
               tied: bool = True, seed: int = 0, max_pos: int = 512) -> Any:
    import torch
    from transformers import Qwen3Config, Qwen3ForCausalLM

    torch.manual_seed(seed)
    cfg = Qwen3Config(vocab_size=vocab, hidden_size=hidden, intermediate_size=ffn, num_hidden_layers=layers,
                      num_attention_heads=n_head, num_key_value_heads=n_kv, head_dim=128, rope_theta=1e6,
                      rms_norm_eps=1e-6, max_position_embeddings=max_pos, tie_word_embeddings=tied, attention_bias=False)
    model = Qwen3ForCausalLM(cfg).eval()
    with torch.no_grad():   # norms away from 1 so that a skipped norm shows
        for n, p in model.named_parameters():
            if p.dim() == 1:
                p.copy_(1.0 + 0.2 * torch.randn_like(p))
    return model


def q4_k_m_type(name: str, layer: int) -> int:
    """Q4_K_M-style: attn_v and ffn_down Q6_K on even layers, the rest Q4_K."""
    return Q6_K if name in ("attn_v", "ffn_down") and layer % 2 == 0 else Q4_K


def write_qwen3_gguf(path: Path | str, model: Any, *, mode: str, seed: int = 1, tokens: list[str] | None = None,
                     merges: list[str] | None = None, context_length: int = 512,
                     drop: tuple[str, ...] = (), override: dict[str, Any] | None = None) -> dict[str, Any]:
    """Write ``model`` as a ``qwen3`` GGUF; ``mode`` "Q8_0" or "Q4_K_M".  The state dict is overwritten with the
    dequantized weights (returned).  ``drop`` omits tensors or keys, ``override`` replaces metadata values."""
    import torch

    rng = np.random.default_rng(seed)
    c = model.config
    sd = {k: v.detach().clone().float() for k, v in model.state_dict().items()}
    tensors: list[tuple[str, int, tuple[int, ...], bytes]] = []

    def put(name: str, hf: str, ty: int) -> None:
        if name in drop:
            return
        w = sd[hf]
        if w.dim() == 1:
            tensors.append((name, F32, tuple(w.shape), w.numpy().astype("<f4").tobytes()))
            return
        N, K = w.shape
        raw = random_blocks(ty, N, K, rng)
        sd[hf] = torch.from_numpy(dequant(ty, raw, N, K))
        tensors.append((name, ty, (N, K), raw.tobytes()))

    q = Q8_0 if mode == "Q8_0" else None
    # Q4_K_M as llama.cpp's quantizer types a tied embedding: with no output tensor, token_embd takes the output's Q6_K
    put("token_embd.weight", "model.embed_tokens.weight", q or (Q6_K if c.tie_word_embeddings else Q4_K))
    if c.tie_word_embeddings:
        sd["lm_head.weight"] = sd["model.embed_tokens.weight"]
    else:
        put("output.weight", "lm_head.weight", q or Q6_K)
    put("output_norm.weight", "model.norm.weight", F32)
    for i in range(c.num_hidden_layers):
        p, b = f"model.layers.{i}.", f"blk.{i}."
        for g, hf in (("attn_q", "self_attn.q_proj"), ("attn_k", "self_attn.k_proj"), ("attn_v", "self_attn.v_proj"),
                      ("attn_output", "self_attn.o_proj"), ("ffn_gate", "mlp.gate_proj"), ("ffn_up", "mlp.up_proj"),
                      ("ffn_down", "mlp.down_proj")):
            put(b + g + ".weight", p + hf + ".weight", q or q4_k_m_type(g, i))
        for g, hf in (("attn_norm", "input_layernorm"), ("attn_q_norm", "self_attn.q_norm"),
                      ("attn_k_norm", "self_attn.k_norm"), ("ffn_norm", "post_attention_layernorm")):
            put(b + g + ".weight", p + hf + ".weight", F32)
    if tokens is None:
        tokens, merges = train_bpe()
    toks = list(tokens) + [f"[PAD{i}]" for i in range(c.vocab_size - len(tokens))]
    types = [3 if t in SPECIAL else 1 for t in toks]
    md = {"general.architecture": (STR, "qwen3"), "general.name": (STR, "test"),
          "qwen3.block_count": (U32, c.num_hidden_layers), "qwen3.context_length": (U32, context_length),
          "qwen3.embedding_length": (U32, c.hidden_size), "qwen3.feed_forward_length": (U32, c.intermediate_size),
          "qwen3.attention.head_count": (U32, c.num_attention_heads),
          "qwen3.attention.head_count_kv": (U32, c.num_key_value_heads), "qwen3.attention.key_length": (U32, 128),
          "qwen3.attention.value_length": (U32, 128), "qwen3.rope.freq_base": (F32V, _rope_theta(c)),
          "qwen3.attention.layer_norm_rms_epsilon": (F32V, float(c.rms_norm_eps)),
          "tokenizer.ggml.model": (STR, "gpt2"), "tokenizer.ggml.pre": (STR, "qwen2"),
          "tokenizer.ggml.tokens": (ARR, (STR, toks)), "tokenizer.ggml.token_type": (ARR, (I32, types)),
          "tokenizer.ggml.merges": (ARR, (STR, list(merges))),
          "tokenizer.ggml.bos_token_id": (U32, toks.index("<|endoftext|>")),
          "tokenizer.ggml.eos_token_id": (U32, toks.index("<|im_end|>")), "tokenizer.ggml.add_bos_token": (BOOL, False)}
    for k, v in (override or {}).items():
        md[k] = v
    meta = [(k, t, v) for k, (t, v) in md.items() if k not in drop]
    write_gguf(path, meta, tensors)
    return sd


def _rope_theta(c: Any) -> float:
    rp = getattr(c, "rope_parameters", None) or {}
    return float(rp.get("rope_theta", getattr(c, "rope_theta", 1e6)) if isinstance(rp, dict) else c.rope_theta)


def hf_model_f64(model: Any, sd: dict[str, Any]) -> Any:
    """``model`` in float64 on the CPU with the dequantized state dict."""
    import copy

    import torch

    m = copy.deepcopy(model).double()
    m.load_state_dict({k: v.double() for k, v in sd.items()}, strict=False)
    if model.config.tie_word_embeddings:
        m.lm_head.weight = m.model.embed_tokens.weight
    return m.eval().to(torch.float64)
