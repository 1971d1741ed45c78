"""CPU tests of the token embedder's host side: the llama-like protocol over an in-memory tokenizer, sentinel detection and
token counting against the oracle, position ids of both model families, truncation, and the argument checks of
``rl_xenc_encode`` / ``rl_xenc_encode_attention`` (which refuse before any CUDA call)."""

from __future__ import annotations

import ctypes

import numpy as np
import pytest
from fake_llama import make_sentences

from oracle import embed as oe
from oracle import pool as opool

TOKENIZERS = {"unigram": oe.unigram_tokenizer, "wordpiece": oe.wordpiece_tokenizer}
SPECIALS = {"unigram": (0, 2), "wordpiece": (2, 3)}   # (first, last) special token of a sequence


class _NoModel:
    """The oracle wrapper's tokenizer side needs no model."""

    config = None

    def eval(self):  # noqa: ANN201
        return self


@pytest.mark.parametrize("kind", TOKENIZERS)
def test_protocol_methods(kind):
    from raglite_b200._xenc import EmbedderTokenizer

    tok = EmbedderTokenizer(TOKENIZERS[kind](), n_ctx=96)
    assert tok.n_ctx() == 96 and tok.n_batch == 96
    text = "The observer of the clock. What is time?\n"
    ids = tok.tokenize(text.encode(), add_bos=False)
    first, last = SPECIALS[kind]
    assert ids and first not in ids and last not in ids                      # no special tokens
    assert tok.detokenize(ids).decode().strip().lower() == text.strip().lower()
    [with_specials] = tok.token_ids_for_embedding([text])
    assert with_specials.dtype == np.int32
    assert with_specials.tolist() == [first, *ids, last]
    assert tok.token_ids_for_embedding([text, "a"])[1].tolist() == [first, *tok.tokenize(b"a"), last]


@pytest.mark.parametrize("kind", TOKENIZERS)
def test_sentinel_and_token_counts_match_the_oracle(kind):
    from raglite_b200 import _embed
    from raglite_b200._xenc import EmbedderTokenizer

    tokenizer = TOKENIZERS[kind]()
    tok = EmbedderTokenizer(tokenizer, n_ctx=64)
    ref = oe.HFEmbedder(_NoModel(), tokenizer, n_ctx=64)
    sentinels = _embed._sentinel_tokens(tok)
    assert sentinels == opool.find_sentinel_tokens(ref)
    assert all("⊕" in tok.detokenize([t]).decode() for t in sentinels)
    for seed in range(3):
        sentences = make_sentences(80, seed=seed)
        got = _embed.count_tokens(sentences, tok)
        want = opool.count_tokens(sentences, ref)
        np.testing.assert_array_equal(got, want)
        assert got.sum() > 0
        np.testing.assert_array_equal(_embed.plan_segments(got, tok.n_ctx(), tok.n_batch),
                                      opool.plan_segments(want, ref.n_ctx(), ref.n_batch))


def test_truncation_to_n_batch():
    from raglite_b200._xenc import EmbedderTokenizer

    tokenizer = oe.unigram_tokenizer()
    tok = EmbedderTokenizer(tokenizer, n_ctx=32)
    ref = oe.HFEmbedder(_NoModel(), tokenizer, n_ctx=32)
    long_text = "".join(make_sentences(40, seed=5))
    [ids] = tok.token_ids_for_embedding([long_text])
    assert len(ids) == 32 and ids[0] == 0 and ids[-1] != 2                   # <s> kept, </s> cut off with the tail
    assert ids.tolist() == ref.token_ids(long_text)
    short = "alpha beta."
    [ids] = tok.token_ids_for_embedding([short])
    assert ids.tolist() == ref.token_ids(short) and ids[-1] == 2


def test_position_ids_of_both_families():
    """XLM-RoBERTa counts positions from padding_idx + 1 (transformers' own rule), BERT from 0; type ids are 0."""
    from transformers.models.xlm_roberta.modeling_xlm_roberta import XLMRobertaEmbeddings

    from raglite_b200._xenc import _pack_inputs, _position_offset

    xlmr = oe.bge_m3_config(num_hidden_layers=1, vocab_size=1000)
    bert = oe.bert_config()
    assert _position_offset(xlmr) == 2 and _position_offset(bert) == 0
    rng = np.random.default_rng(0)
    lens = np.asarray([1, 2, 17, 512, 5], dtype=np.int64)
    ids = [rng.integers(3, 1000, size=int(n)).astype(np.int32) for n in lens]
    for offset in (2, 0):
        T = int(lens.sum())
        h = np.full(3 * T + len(ids) + 1, -7, dtype=np.int32)
        assert _pack_inputs(h, ids, None, lens, offset) == T
        np.testing.assert_array_equal(h[:T], np.concatenate(ids))
        assert (h[T:2 * T] == 0).all()
        np.testing.assert_array_equal(h[3 * T:], np.concatenate([[0], np.cumsum(lens)]))
        pos = h[2 * T:3 * T]
        for s, x in enumerate(ids):
            got = pos[int(lens[:s].sum()):int(lens[:s + 1].sum())]
            if offset:
                import torch

                want = XLMRobertaEmbeddings.create_position_ids_from_input_ids(torch.from_numpy(x.astype(np.int64))[None], padding_idx=1)[0].numpy()
            else:
                want = np.arange(len(x))
            np.testing.assert_array_equal(got, want)


def _weights(hidden=1024, heads=16, ffn=4096, max_pos=514, layers=2):
    from raglite_b200._lib import XencLayer, XencWeights

    w = XencWeights()
    w.n_layers, w.hidden, w.n_heads, w.ffn, w.vocab, w.max_pos, w.type_vocab, w.ln_eps = layers, hidden, heads, ffn, 1000, max_pos, 1, 1e-5
    w._layer_array = (XencLayer * layers)()
    w.layers = ctypes.cast(w._layer_array, ctypes.POINTER(XencLayer))
    for name in ("word_emb", "pos_emb", "type_emb", "emb_ln_g", "emb_ln_b"):
        setattr(w, name, 4096)
    return w


def test_encode_refuses_unsupported_arguments_before_any_cuda_call():
    """The pointers are placeholders: every call below is refused before anything is dereferenced or launched."""
    from raglite_b200 import _lib

    lib = _lib.load()
    ptr, ws = 4096, 8192

    def call(*, w=None, P=4, T=100, max_len=64, out=ptr, workspace=ws, ws_bytes=None, **shape):
        w = w or _weights(**shape)
        need = lib.rl_xenc_workspace_bytes(ctypes.byref(w), T)
        return lib.rl_xenc_encode(ctypes.byref(w), ptr, ptr, ptr, ptr, P, T, max_len, out, workspace,
                                  need if ws_bytes is None else ws_bytes, None)

    assert call(out=None) == -1
    assert call(hidden=384, heads=8) == -4                     # head_dim 48
    assert call(hidden=1024, heads=8) == -4                    # head_dim 128
    assert call(hidden=1056, heads=33) == -4                   # head_dim 32, but hidden > 1024
    assert call(hidden=1056, heads=16, ffn=4224) == -4         # hidden % heads
    assert call(ffn=4100) == -4                                # ffn % 32
    assert call(layers=0) == -4
    assert call(max_len=513, T=2000) == -4                     # longer than 512
    assert b"max_len=513" in lib.rl_last_error()
    assert call(max_len=100, max_pos=64) == -4                 # longer than the position table
    assert call(max_len=0) == -4
    assert call(P=101) == -1                                   # more sequences than tokens
    w = _weights()
    need = lib.rl_xenc_workspace_bytes(ctypes.byref(w), 100)
    assert call(w=w, ws_bytes=need - 1) == -3                  # short workspace
    assert call(w=w, workspace=ws + 8) == -3                   # misaligned workspace
    assert call(w=w, workspace=None) == -3
    assert lib.rl_xenc_encode(None, ptr, ptr, ptr, ptr, 4, 100, 64, ptr, ws, need, None) == -1


def test_encode_attention_hook_refuses_unsupported_arguments():
    from raglite_b200 import _lib

    lib = _lib.load()
    ptr, ws = 4096, 8192

    def call(*, qkv=ptr, P=4, T=100, max_len=64, hidden=1024, heads=16, workspace=ws, ws_bytes=16):
        return lib.rl_xenc_encode_attention(qkv, ptr, P, T, max_len, hidden, heads, ptr, workspace, ws_bytes, None)

    assert call(qkv=None) == -1
    assert call(hidden=384, heads=8) == -4                     # head_dim 48
    assert call(hidden=1024, heads=8) == -4                    # head_dim 128
    assert call(hidden=1056, heads=33) == -4                   # hidden > 1024
    assert call(hidden=48, heads=1) == -4                      # hidden % 32
    assert call(max_len=513, T=2000) == -4
    assert call(P=101) == -1                                   # more sequences than tokens
    assert call(max_len=0) == -1
    assert call(ws_bytes=15) == -3                             # 4 * P bytes
    assert call(workspace=ws + 4) == -3                        # 16-byte alignment
    assert call(workspace=None) == -3
    # the cross-encoder's hook keeps its own limits
    assert lib.rl_xenc_attention(ptr, ptr, 4, 100, 64, 1024, 16, ptr, ws, 16, None) == -4
