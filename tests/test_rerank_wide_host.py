"""CPU tests of the wide cross-encoder's host side: the ctypes mirror of ``rl_xenc_weights``, the argument checks of
``rl_xenc_score`` (which refuse before any CUDA call), the engine's ``ValueError`` for every model it cannot run (raised
before any device work), and the oracle's own conventions."""

from __future__ import annotations

import ctypes
import re
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]


def test_xenc_weights_fields_match_the_header():
    from raglite_b200._lib import XencWeights

    text = (ROOT / "include" / "raglite_b200.h").read_text()
    body = re.search(r"typedef struct rl_xenc_weights \{(.*?)\} rl_xenc_weights;", text, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = [n for decl in body.split(";") if decl.strip() for n in re.findall(r"(\w+)\s*(?:,|$)", decl.strip())]
    assert names == [f[0] for f in XencWeights._fields_]
    assert names[-3:] == ["cls_w", "cls_b", "n_labels"]


def _weights(hidden=768, heads=12, ffn=3072, max_pos=8194, layers=2, n_labels=2):
    from raglite_b200._lib import XencLayer, XencWeights

    w = XencWeights()
    w.n_layers, w.hidden, w.n_heads, w.ffn, w.vocab, w.max_pos, w.type_vocab, w.ln_eps = layers, hidden, heads, ffn, 1000, max_pos, 2, 1e-12
    w._layer_array = (XencLayer * layers)()
    w.layers = ctypes.cast(w._layer_array, ctypes.POINTER(XencLayer))
    for name in ("word_emb", "pos_emb", "type_emb", "emb_ln_g", "emb_ln_b", "pooler_w", "pooler_b", "cls_w", "cls_b"):
        setattr(w, name, 4096)
    w.n_labels = n_labels
    return w


def test_score_refuses_unsupported_arguments_before_any_cuda_call():
    """The pointers are placeholders: every call below is refused before anything is dereferenced or launched."""
    from raglite_b200 import _lib

    lib = _lib.load()
    ptr, ws = 4096, 8192

    def call(*, w=None, P=4, T=600, max_len=64, out=ptr, workspace=ws, ws_bytes=None, **shape):
        w = w or _weights(**shape)
        need = lib.rl_xenc_workspace_bytes(ctypes.byref(w), T)
        return lib.rl_xenc_score(ctypes.byref(w), ptr, ptr, ptr, ptr, P, T, max_len, out, ptr, workspace,
                                 need if ws_bytes is None else ws_bytes, None)

    def error() -> str:
        return lib.rl_last_error().decode()

    assert call(n_labels=3) == -4
    assert "n_labels=3" in error()
    assert call(n_labels=-1) == -4
    assert call(hidden=1024, heads=8) == -4                    # head_dim 128
    assert "hidden=1024 heads=8" in error()
    assert call(hidden=1056, heads=33, ffn=4224) == -4         # head_dim 32, but hidden > 1024
    assert "hidden=1056" in error()
    assert call(hidden=384, heads=8) == -4                     # head_dim 48
    assert call(max_len=513) == -4                             # head_dim 64: at most 512 tokens
    assert "max_len=513" in error()
    assert call(hidden=1024, heads=32, ffn=4096, max_len=513) == -4   # head_dim 32 above hidden 512: also 512
    assert call(hidden=384, heads=12, ffn=1536, max_len=1300, max_pos=2048) == -4   # head_dim 32 path: shared memory
    assert "max_len=1300" in error()
    assert call(max_len=100, max_pos=64) == -4                 # longer than the position table
    assert call(max_len=0) == -4
    assert call(layers=0) == -4                                # the wide envelope runs at least one layer
    assert call(ffn=3000) == -4                                # ffn % 32
    assert call(P=601) == -1                                   # more sequences than tokens
    assert call(out=None) == -1
    assert "null pointer" in error()
    w = _weights()
    need = lib.rl_xenc_workspace_bytes(ctypes.byref(w), 600)
    assert call(w=w, ws_bytes=need - 1) == -3
    assert call(w=w, workspace=None) == -3
    assert lib.rl_xenc_score(None, ptr, ptr, ptr, ptr, 4, 600, 64, ptr, ptr, ws, need, None) == -1
    assert lib.rl_xenc_score(ctypes.byref(w), None, ptr, ptr, ptr, 4, 600, 64, ptr, ptr, ws, need, None) == -1
    assert lib.rl_xenc_score(ctypes.byref(w), ptr, ptr, ptr, ptr, 4, 600, 64, ptr, None, ws, need, None) == -1


def _config(**over):
    c = dict(model_type="bert", num_labels=2, hidden_act="gelu", hidden_size=768, num_attention_heads=12,
             num_hidden_layers=2, intermediate_size=3072, max_position_embeddings=512, layer_norm_eps=1e-12, pad_token_id=0)
    c.update(over)
    return SimpleNamespace(**c)


class _Model:
    """A config without weights: the checks run before the state dict is read."""

    def __init__(self, config) -> None:  # noqa: ANN001
        self.config = config

    def state_dict(self):  # noqa: ANN201
        raise AssertionError("the state dict was read before the config was checked")


UNSUPPORTED = [
    (dict(model_type="deberta-v2"), "model_type"),
    (dict(num_labels=3), "num_labels=3"),
    (dict(num_labels=0), "num_labels=0"),
    (dict(hidden_act="relu"), "hidden_act"),
    (dict(hidden_act="gelu_new"), "hidden_act"),
    (dict(hidden_size=1024, num_attention_heads=8), "head_dim"),     # 128
    (dict(hidden_size=768, num_attention_heads=16), "head_dim"),     # 48
    (dict(hidden_size=1056, num_attention_heads=33), "at most 1024"),
    (dict(hidden_size=1280, num_attention_heads=20), "at most 1024"),
]


@pytest.mark.parametrize(("over", "names"), UNSUPPORTED, ids=[n for _, n in UNSUPPORTED])
def test_unsupported_models_raise_value_error_before_device_work(over, names):
    from raglite_b200._xenc import CrossEncoderEngine

    with pytest.raises(ValueError, match=re.escape(names)):
        CrossEncoderEngine.from_hf(_Model(_config(**over)))


def _state_dict(hidden=768, labels=2, model_type="bert"):
    import torch

    cls = "classifier." if model_type == "bert" else "classifier.out_proj."
    return {cls + "weight": torch.zeros(labels, hidden), cls + "bias": torch.zeros(labels)}


@pytest.mark.parametrize(("kw", "names"), [
    (dict(sd=_state_dict(labels=3)), "num_labels=3"),
    (dict(sd=_state_dict(labels=3, model_type="xlm-roberta"), model_type="xlm-roberta"), "num_labels=3"),
    (dict(sd=_state_dict(), model_type="electra"), "model_type"),
    (dict(sd=_state_dict(), hidden_act="silu"), "hidden_act"),
    (dict(sd=_state_dict(hidden=1024), hidden=1024, n_heads=8), "head_dim"),
    (dict(sd=_state_dict(hidden=1056), hidden=1056, n_heads=33), "at most 1024"),
    (dict(sd=_state_dict(hidden=384)), "[num_labels, 768]"),                 # classifier of another width
    (dict(sd=_state_dict(model_type="xlm-roberta")), "classifier.weight"),   # XLM-R head under a BERT model type
], ids=["labels3", "labels3_xlmr", "model_type", "hidden_act", "head_dim128", "hidden1056", "cls_width", "head_names"])
def test_constructor_raises_value_error_before_device_work(kw, names):
    from raglite_b200._xenc import CrossEncoderEngine

    kw = dict(kw)
    sd = kw.pop("sd")
    args = dict(n_layers=2, hidden=768, n_heads=12, ffn=3072, max_pos=512)
    args.update(kw)
    with pytest.raises(ValueError, match=re.escape(names)):
        CrossEncoderEngine(sd, **args)


def test_from_pretrained_checks_the_config_before_loading_weights(tmp_path):
    """A directory with only config.json: the refusal comes from the config, before any weights are looked for."""
    from transformers import BertConfig, XLMRobertaConfig

    from raglite_b200._xenc import CrossEncoderEngine

    BertConfig(num_labels=3).save_pretrained(tmp_path / "bert3")
    with pytest.raises(ValueError, match="num_labels=3"):
        CrossEncoderEngine.from_pretrained(tmp_path / "bert3")
    XLMRobertaConfig(hidden_size=1024, num_attention_heads=8, num_labels=1).save_pretrained(tmp_path / "xlmr128")
    with pytest.raises(ValueError, match="head_dim"):
        CrossEncoderEngine.from_pretrained(tmp_path / "xlmr128")


def test_missing_directory_message_names_both_families(tmp_path):
    from raglite_b200._rerank import B200CrossEncoderRanker

    with pytest.raises(FileNotFoundError) as e:
        B200CrossEncoderRanker("ms-marco-MultiBERT-L-12", cache_dir=tmp_path).rank(query="q", docs=["d"])
    msg = str(e.value)
    assert "bert" in msg and "xlm-roberta" in msg and "tokenizer.json" in msg and "config.json" in msg
    assert "cross-encoder/ms-marco-MultiBERT-L-12" not in msg and "<repo id>" in msg


def test_oracle_conventions():
    """FlashRank's two-label score is the stable sigmoid of l1 - l0; random XLM-R pairs hold no pad id, so
    transformers' positions are padding_idx + 1 + i, the offset the engine packs."""
    import torch
    from transformers.models.xlm_roberta.modeling_xlm_roberta import XLMRobertaEmbeddings

    import xenc_classifiers as xc

    lg = np.array([[0.3, -1.2], [5.0, 5.0], [-300.0, 300.0], [300.0, -300.0]], np.float32)
    s = xc.flashrank_scores(lg)
    np.testing.assert_allclose(s, 1.0 / (1.0 + np.exp(np.float64(lg[:, 0]) - lg[:, 1])), rtol=1e-12)
    assert s[1] == 0.5 and s[2] == 1.0 and 0.0 <= s[3] < 1e-200
    np.testing.assert_array_equal(xc.ranking_key(lg), np.float64(lg[:, 1]) - lg[:, 0])
    np.testing.assert_allclose(xc.flashrank_scores(lg[:1, :1]), 1.0 / (1.0 + np.exp(-0.3)), rtol=1e-6)
    rng = np.random.default_rng(0)
    ids, types = xc.random_pairs(20, 60, rng, "xlm-roberta", lo=1, hi=80, lengths=(1, 2, 5))
    for x, t in zip(ids, types, strict=True):
        assert 1 not in x and (t == 0).all()
        pos = XLMRobertaEmbeddings.create_position_ids_from_input_ids(torch.from_numpy(x.astype(np.int64))[None], padding_idx=1)
        np.testing.assert_array_equal(pos[0].numpy(), 2 + np.arange(len(x)))
    ids, types = xc.random_pairs(20, 5000, rng, "bert", lo=5, hi=80)
    assert all(x[0] == 101 and x[-1] == 102 and (x == 102).sum() >= 2 and t[-1] == 1 for x, t in zip(ids, types, strict=True))
