"""Host side of ``split_sentences``: the post-processing restatement against the reference's own outputs, the Markdown
boundaries, the block plan / hat weights / character targets against plain loops, ``SaTEngine``'s refusals and config
reading, and the public early exit and registration error.  No GPU."""

from __future__ import annotations

import json
from pathlib import Path

import numpy as np
import pytest
import sentences_oracle as so

from raglite_b200 import _sentences as S

GOLDEN = Path(__file__).parent / "golden" / "split_sentences.npz"
T_VALUES = (0, 1, 2, 253, 254, 255, 382, 383, 384, 5000)


def _cases():
    z = np.load(GOLDEN)
    return [(c, z[f"pred{i}"], z[f"md{i}"], z[f"known{i}"] if c["known"] else None)
            for i, c in enumerate(json.loads(z["cases"].tobytes()))]


CASES = _cases()


@pytest.mark.parametrize("i", range(len(CASES)), ids=[f"{c['name']}-{c['min_len']}-{c['max_len']}" for c, *_ in CASES])
def test_post_processing_matches_reference(i):
    c, pred, _md, known = CASES[i]
    if c["error"] is not None:
        with pytest.raises(ValueError, match="Sentence partition failed") as e:
            so.split_sentences_post(c["doc"], pred, min_len=c["min_len"], max_len=c["max_len"], known=known)
        assert str(e.value) == c["error"]
        return
    got = so.split_sentences_post(c["doc"], pred, min_len=c["min_len"], max_len=c["max_len"], known=known)
    assert got == c["sentences"]
    assert "".join(got) == c["doc"]


def test_golden_covers_the_issue_cases():
    names = {c["name"] for c, *_ in CASES}
    assert {"headings", "spaces", "multibyte", "len4", "len5", "len8", "infeasible"} <= names
    assert {8, 64, 2048, None} <= {c["max_len"] for c, *_ in CASES}
    assert any(c["error"] for c, *_ in CASES)
    assert any(c["max_len"] == 8 and c["sentences"] and max(map(len, c["sentences"])) <= 8 and len(c["doc"]) > 40
               for c, *_ in CASES)


@pytest.mark.parametrize("doc", sorted({c["doc"] for c, *_ in CASES}))
def test_markdown_boundaries_match_reference(doc):
    want = next(md for c, _p, md, _k in CASES if c["doc"] == doc)
    for got in (S.markdown_sentence_boundaries(doc), so.markdown_boundaries(doc)):
        assert got.dtype == want.dtype and got.shape == want.shape
        np.testing.assert_array_equal(got, want)   # NaN positions equal too


def test_markdown_headings_present():
    doc = next(c["doc"] for c, *_ in CASES if c["name"] == "headings")
    md = S.markdown_sentence_boundaries(doc)
    assert (md == 1).sum() >= 6 and (md == 0).sum() > 20 and np.isnan(md).sum() > 20


@pytest.mark.parametrize("T", T_VALUES)
def test_block_plan_matches_loop(T):
    B, starts = S.block_starts(T)
    wB, wstarts = so.plan_loop(T)
    assert B == wB and starts.tolist() == wstarts
    if T:
        assert starts[-1] + B == T and all(s + B < T for s in starts[:-1])
        covered = np.zeros(T, int)
        for s in starts:
            covered[s:s + B] += 1
        assert covered.min() >= 1 and covered.max() <= -(-B // S.SAT_STRIDE) + 1


def test_batch_plan_equals_per_document():
    T = np.array(T_VALUES + (0, 7, 1000), dtype=np.int64)
    B, off, start = S.plan_blocks(T)
    for d, t in enumerate(T):
        b, s = S.block_starts(int(t))
        assert (t == 0 or B[d] == b) and start[off[d]:off[d + 1]].tolist() == s.tolist()


@pytest.mark.parametrize("B", sorted({1, 2, 3, 127, 128, 253, 254} | {min(254, t) for t in T_VALUES if t}))
def test_hat_weights_match_loop(B):
    w = S.hat_weights(B)
    np.testing.assert_allclose(w, so.hat_loop(B), rtol=0, atol=2e-7)
    assert np.all(w > 0) and np.all(w <= 1) and np.allclose(w, w[::-1])
    table = S.hat_table()
    np.testing.assert_array_equal(table[B * (B - 1) // 2:B * (B + 1) // 2], w)


@pytest.mark.parametrize("T", T_VALUES)
def test_char_targets_match_loop(T):
    rng = np.random.default_rng(T)
    n = max(1, 2 * T)
    ends = np.sort(rng.integers(0, n + 1, size=T))
    skip = rng.random(T) < 0.2
    got = S.token_char_targets(ends, skip, n)
    assert got.tolist() == so.char_targets_loop(ends, skip, n)
    hit = got[got >= 0]
    assert len(np.unique(hit)) == len(hit)


def test_tokenizer_targets_on_multibyte_text():
    """Character offsets from ``tokenizers`` count Python characters: the target of each kept token is a character
    inside the document, and the multi-byte characters keep their own positions."""
    from oracle.embed import unigram_tokenizer

    tok = unigram_tokenizer()
    doc = "héllo  wörld　⊕ the  end.\n\nalpha 😀 x"
    e = tok.encode(doc, add_special_tokens=False)
    ends = np.array([o[1] for o in e.offsets])
    skip = np.isin(e.ids, [tok.token_to_id(p) for p in S.SAT_SKIP_PIECES if tok.token_to_id(p) is not None])
    tgt = S.token_char_targets(ends, skip, len(doc))
    assert tgt.max() < len(doc) and doc[tgt[np.array(e.tokens) == "."][0]] == "."


def test_whitespace_flags_are_str_isspace():
    every = "".join(chr(c) for c in range(0x110000) if not 0xD800 <= c < 0xE000)
    got = S.whitespace_flags(every)
    assert got.tolist() == [c.isspace() for c in every]
    assert S.code_points("a😀é").tolist() == [0x61, 0x1F600, 0xE9]


def _config(**over):
    c = {"model_type": "xlm-token", "architectures": ["SubwordXLMForTokenClassification"], "hidden_size": 768,
         "num_hidden_layers": 1, "num_attention_heads": 12, "intermediate_size": 3072, "max_position_embeddings": 514,
         "hidden_act": "gelu", "layer_norm_eps": 1e-5, "pad_token_id": 1, "vocab_size": 250002, "lookahead": None,
         "num_labels": 111}
    c.update(over)
    return c


def test_config_json_read_as_json(tmp_path):
    (tmp_path / "config.json").write_text(json.dumps(_config()))
    kw = S.read_sat_config(tmp_path)
    assert kw == dict(n_layers=1, hidden=768, n_heads=12, ffn=3072, max_pos=514, ln_eps=1e-5, pos_offset=2)


@pytest.mark.parametrize(("over", "match"), [
    ({"lookahead": 48}, "lookahead"),
    ({"hidden_act": "relu"}, "GELU"),
    ({"num_attention_heads": 6}, "head_dim"),
    ({"hidden_size": 1280, "num_attention_heads": 20}, "at most 1024"),
])
def test_config_refusals(tmp_path, over, match):
    (tmp_path / "config.json").write_text(json.dumps(_config(**over)))
    with pytest.raises(ValueError, match=match):
        S.read_sat_config(tmp_path)
    with pytest.raises(ValueError, match=match):
        S.SaTEngine.from_pretrained(tmp_path)


def test_missing_head_refused(tmp_path):
    import torch
    from safetensors.torch import save_file

    (tmp_path / "config.json").write_text(json.dumps(_config(hidden_size=64, num_attention_heads=1, intermediate_size=128)))
    save_file({"roberta.embeddings.word_embeddings.weight": torch.zeros(10, 64)}, str(tmp_path / "model.safetensors"))
    with pytest.raises(ValueError, match="token-classification head"):
        S.SaTEngine.from_pretrained(tmp_path)
    with pytest.raises(ValueError, match="token-classification head"):
        S.SaTEngine({"roberta.embeddings.word_embeddings.weight": torch.zeros(10, 64)}, n_layers=1, hidden=64,
                    n_heads=1, ffn=128, max_pos=514, tokenizer=None)


def test_early_exit_and_registration_error():
    saved = list(S._SPLITTER)
    S._SPLITTER.clear()
    try:
        for doc, min_len in (("", 4), ("abcd", 4), ("ab", 2), ("x", 1)):
            assert S.split_sentences(doc, min_len=min_len) == [doc]
        assert S.split_sentences_batch(["abc", "", "abcd"]) == [["abc"], [""], ["abcd"]]
        with pytest.raises(ModuleNotFoundError, match="register_sentence_splitter"):
            S.split_sentences("abcde")
        with pytest.raises(ModuleNotFoundError, match="register_sentence_splitter"):
            S.sentence_boundary_probas(["abc"])
    finally:
        S._SPLITTER[:] = saved
