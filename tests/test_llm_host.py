"""The decoder's host side without a GPU: the qwen3 plan's checks, the rebuilt byte-level BPE against transformers'
Qwen2TokenizerFast, byte-exact decoding and streaming hold-back, ChatML rendering, the context trimming, and the NumPy
sampler statement on hand cases."""

from __future__ import annotations

import json

import numpy as np
import pytest

from gguf_fixtures import F16, Q4_K, STR, U32
from llm_oracle import sample
from qwen3_fixtures import make_model, train_bpe, write_qwen3_gguf

TEXTS = ["It's 2024 and they'll've 12345 cats!", "日本語のテキストと中文文本。", "Emoji 🎉🚀 café", "a\n\n\nb  \n   c\t\td",
         "    spaces   everywhere   ", "<|im_start|>user\nhi<|im_end|>\n<|im_start|>assistant\n", "x<|im_end|>y 99"]


@pytest.fixture(scope="module")
def vocab():
    return train_bpe()


@pytest.fixture(scope="module")
def gguf_path(tmp_path_factory, vocab):
    path = tmp_path_factory.mktemp("q3") / "m.gguf"
    write_qwen3_gguf(path, make_model(layers=1), mode="Q8_0", tokens=vocab[0], merges=vocab[1])
    return path


def _plan(path):
    from raglite_b200._gguf import GGUFFile, qwen3_plan

    return qwen3_plan(GGUFFile(path))


def test_plan_reads_the_shapes(gguf_path):
    p = _plan(gguf_path)
    assert (p.n_layers, p.hidden, p.n_head, p.n_kv, p.ffn, p.vocab, p.tied) == (1, 256, 4, 2, 768, 640, True)
    assert p.tensors["output.weight"] is p.tensors["token_embd.weight"]


@pytest.mark.parametrize("kw,match", [
    (dict(override={"qwen3.attention.key_length": (U32, 64)}), "head_dim"),
    (dict(override={"qwen3.attention.head_count_kv": (U32, 3)}), "head_count"),
    (dict(override={"qwen3.attention.head_count": (U32, 18), "qwen3.attention.head_count_kv": (U32, 2)}), "group"),
    (dict(override={"qwen3.embedding_length": (U32, 384)}), "multiples of 256"),
    (dict(drop=("qwen3.rope.freq_base",)), "qwen3.rope.freq_base is missing"),
    (dict(drop=("blk.0.attn_k_norm.weight",)), "attn_k_norm.weight' is missing"),
    (dict(override={"general.architecture": (STR, "llama")}), "unsupported"),
])
def test_plan_refuses(tmp_path, vocab, kw, match):
    path = tmp_path / "bad.gguf"
    write_qwen3_gguf(path, make_model(layers=1), mode="Q8_0", tokens=vocab[0], merges=vocab[1], **kw)
    with pytest.raises(ValueError, match=match):
        _plan(path)


def test_plan_refuses_float_weights(tmp_path, vocab, monkeypatch):
    import qwen3_fixtures

    monkeypatch.setattr(qwen3_fixtures, "q4_k_m_type", lambda name, layer: F16 if name == "ffn_up" else Q4_K)
    path = tmp_path / "f16.gguf"
    write_qwen3_gguf(path, make_model(layers=1), mode="Q4_K_M", tokens=vocab[0], merges=vocab[1])
    with pytest.raises(ValueError, match="ffn_up.weight' is F16"):
        _plan(path)


def _tokenizers(gguf_path, vocab):
    from transformers import Qwen2TokenizerFast

    from raglite_b200._gguf import GGUFFile
    from raglite_b200._llm import QwenTokenizer

    tokens, merges = vocab
    hf = Qwen2TokenizerFast(vocab={t: i for i, t in enumerate(tokens)}, merges=[tuple(m.split(" ")) for m in merges],
                            unk_token=None, bos_token=None, eos_token="<|im_end|>", pad_token="<|endoftext|>",
                            additional_special_tokens=["<|im_start|>", "<|im_end|>"])
    return QwenTokenizer.from_gguf(GGUFFile(gguf_path)), hf


@pytest.mark.parametrize("text", TEXTS)
def test_tokenizer_equals_qwen2_tokenizer_fast(gguf_path, vocab, text):
    ours, hf = _tokenizers(gguf_path, vocab)
    assert ours.encode(text) == hf.encode(text, add_special_tokens=False)
    assert ours.decode_bytes(ours.encode(text)) == text.encode()


def test_tokenizer_refuses_other_vocabularies(tmp_path, vocab):
    from raglite_b200._gguf import GGUFFile
    from raglite_b200._llm import QwenTokenizer

    path = tmp_path / "t.gguf"
    write_qwen3_gguf(path, make_model(layers=1), mode="Q8_0", tokens=vocab[0], merges=vocab[1],
                     override={"tokenizer.ggml.pre": (STR, "llama-bpe")})
    with pytest.raises(ValueError, match="pre='llama-bpe'"):
        QwenTokenizer.from_gguf(GGUFFile(path))


class _FakeEngine:
    """generate()'s text layer over a fixed id stream (no device)."""

    def __init__(self, tok, ids):
        self.tokenizer, self._ids = tok, ids

    def generate_ids(self, prompt_ids, **kw):
        yield from self._ids


def test_streaming_holds_back_partial_utf8_and_stop_prefixes(gguf_path, vocab):
    from raglite_b200._llm import LlmEngine

    tok, _ = _tokenizers(gguf_path, vocab)
    text = "Emoji 🎉 done. STOP here"
    ids = tok.encode(text)
    fake = _FakeEngine(tok, ids)
    pieces = list(LlmEngine.generate(fake, [], stop=["STOP"]))
    assert "".join(pieces) == "Emoji 🎉 done. "
    assert all("�" not in p for p in pieces)
    whole = list(LlmEngine.generate(_FakeEngine(tok, ids), []))
    assert "".join(whole) == text


def test_chatml_rendering():
    from raglite_b200._rag import render_chatml

    msgs = [{"role": "system", "content": "S"}, {"role": "user", "content": "U"}, {"role": "assistant", "content": ""},
            {"role": "assistant", "content": "A"}, {"role": "tool", "content": "T"}]
    assert render_chatml(msgs) == ("<|im_start|>system\nS<|im_end|>\n<|im_start|>user\nU<|im_end|>\n"
                                   "<|im_start|>assistant\nA<|im_end|>\n<|im_start|>assistant\n")


def test_clip_and_limit_on_hand_cases(monkeypatch):
    import raglite_b200 as rl
    from raglite_b200 import _rag

    msgs = [{"role": "system", "content": "s" * 30}, {"role": "user", "content": "u" * 300},
            {"role": "assistant", "content": "a" * 300}, {"role": "user", "content": "q" * 30}]
    counts = [len(json.dumps(m)) // 3 for m in msgs]
    assert _rag._clip(msgs, sum(counts)) == msgs
    assert _rag._clip(msgs, counts[3] + counts[2]) == msgs[2:]
    assert _rag._clip(msgs, counts[3]) == msgs[3:]
    assert _rag._clip(msgs, counts[3] - 1) == []
    assert _rag._clip(msgs[:2], counts[0] + counts[1] - 1) == [msgs[1]]
    spans = [rl.ChunkSpan(chunks=[rl.Chunk(id=f"c{i}", document_id="d", index=i, body="b" * 300)]) for i in range(5)]
    per = len(spans[0].to_xml()) // 3
    monkeypatch.setattr(_rag, "get_context_size", lambda config: 3 * per + 10)
    kept = _rag._limit_chunkspans({"t": spans}, None)["t"]
    assert kept == spans[:3]
    msg = _rag.add_context("  Why?  ", spans[:1], None)
    assert msg["role"] == "user" and msg["content"].endswith("</context>\n\nWhy?")
    assert '<document index="1" id="d">' in msg["content"] and 'from_chunk_id="c0"' in msg["content"]


def test_numpy_sampler_ties_and_top_p_crossing():
    logits = np.zeros(10, np.float32)
    logits[[7, 3]] = 2.0
    kw = dict(top_k=5, top_p=1.0, min_p=0.0, penalty=1.0)
    assert sample(logits, [], temperature=0.0, u=0.5, **kw) == 3
    assert sample(logits, [], temperature=1.0, u=0.0, **kw) == 3
    logits = np.full(10, -30.0, np.float32)
    logits[[1, 2, 4]] = np.log([0.6, 0.3, 0.1]).astype(np.float32)
    assert sample(logits, [], temperature=1.0, u=0.99, top_k=5, top_p=0.5, min_p=0.0, penalty=1.0) == 1
    assert sample(logits, [], temperature=1.0, u=0.99, top_k=5, top_p=0.7, min_p=0.0, penalty=1.0) == 2
    assert sample(logits, [1], temperature=0.0, u=0.5, top_k=5, top_p=1.0, min_p=0.0, penalty=10.0) == 2
