"""``split_sentences`` on the GPU: SaT character probabilities against a float64 restatement, the partition bit for bit
against the reference's post-processing run on the device's probabilities, the reference's own outputs through the public
path, batch = single, and a 2 M-character document.

Tolerance of the probabilities.  The encoder's hidden states are within ``HIDDEN_MAX_ABS`` (``test_gpu_embedder.py``) of
the CPU model per element.  A logit is h . W_l + b_l, so its error is at most HIDDEN_MAX_ABS * sum|W_l| (plus float32
rounding of the head, far below).  Stitching is a convex combination of block logits and the fill is a minimum of
stitched logits, so neither widens the bound; the sigmoid's slope is at most 1/4.  A probability is therefore within
HIDDEN_MAX_ABS * max_l sum|W_l| / 4 of float64.  The measured maximum and mean go to ``sentence_errors.jsonl`` in the
temporary directory."""

from __future__ import annotations

import json
import tempfile
from pathlib import Path

import numpy as np
import pytest
import sentences_oracle as so

import raglite_b200 as rl
from raglite_b200 import _sentences as S

pytestmark = pytest.mark.gpu

HIDDEN_MAX_ABS = 1.4e-2
T_VALUES = (0, 1, 2, 253, 254, 255, 382, 383, 384, 5000)
WORDS = ("alpha", "beta", "gamma", "delta", "light", "clock", "rod", "frame", "event", "time", "of", "the",
         "observer", "velocity", "what", "is", "how", "does", "a", "an", "in", "to")
PAIRS = [(4, None), (4, 64), (1, 8), (10, 2048)]


def _record(payload: dict) -> None:
    with (Path(tempfile.gettempdir()) / "sentence_errors.jsonl").open("a") as f:
        f.write(json.dumps(payload) + "\n")


def _model(seed: int, *, layers: int, hidden: int, heads: int, labels: int, vocab: int):
    import torch
    from transformers import XLMRobertaConfig, XLMRobertaForTokenClassification

    from oracle.embed import _perturb

    cfg = XLMRobertaConfig(vocab_size=vocab, hidden_size=hidden, num_hidden_layers=layers, num_attention_heads=heads,
                           intermediate_size=4 * hidden, max_position_embeddings=514, type_vocab_size=1,
                           layer_norm_eps=1e-5, hidden_act="gelu", pad_token_id=1, bos_token_id=0, eos_token_id=2,
                           hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, num_labels=labels)
    cfg._attn_implementation = "eager"   # noqa: SLF001
    torch.manual_seed(seed)
    m = XLMRobertaForTokenClassification(cfg).eval()
    with torch.no_grad():
        _perturb(m)
        m.classifier.weight.normal_(0.0, 0.05)
    return m


@pytest.fixture(scope="module")
def tok():
    from oracle.embed import unigram_tokenizer

    return unigram_tokenizer()


@pytest.fixture(scope="module")
def sat1(tok):
    m = _model(1, layers=1, hidden=768, heads=12, labels=1, vocab=tok.get_vocab_size())
    return m, S.SaTEngine.from_hf(m, tok)


def _words_doc(rng, n_tokens: int) -> str:
    return " ".join(str(w) for w in rng.choice(WORDS, size=n_tokens)) if n_tokens else ""


def _prose(rng, n_chars: int) -> str:
    parts, n = [], 0
    while n < n_chars:
        w = str(rng.choice(WORDS))
        if rng.random() < 0.1:
            w = w.capitalize() + rng.choice([".", "!", "?", ".\n\n", ".  ", "é", "ï"])
        elif rng.random() < 0.03:
            w = rng.choice(["😀", "日本", "　", "\t\t", "ü"]) + w
        parts.append(w)
        n += len(w) + 1
    return " ".join(parts)


def _docs(tok, seed: int = 0) -> list[str]:
    rng = np.random.default_rng(seed)
    docs = []
    for T in T_VALUES:
        d = _words_doc(rng, T)
        assert len(tok.encode(d, add_special_tokens=False).ids) == T
        docs.append(d)
    docs += ["héllo  wörld　　⊕ the  end.\n\nalpha 😀 x", "# Heading\n\nBody.  More\t\ttext.   ", "   lead",
             _prose(rng, 3000)]
    return docs


@pytest.mark.parametrize(("name", "layers", "hidden", "heads", "labels"), [
    ("l1_h768_nl1", 1, 768, 12, 1), ("l1_h768_nl3", 1, 768, 12, 3), ("l3_h1024_nl1", 3, 1024, 16, 1)])
def test_char_probas_against_float64(tok, name, layers, hidden, heads, labels):
    m = _model(7 + layers + labels, layers=layers, hidden=hidden, heads=heads, labels=labels, vocab=tok.get_vocab_size())
    eng = S.SaTEngine.from_hf(m, tok)
    rl.register_sentence_splitter(eng)
    docs = _docs(tok, seed=layers * 10 + labels)
    got = rl.sentence_boundary_probas(docs)
    sumw = float(m.classifier.weight.detach().abs().sum(1).max())
    tol = HIDDEN_MAX_ABS * sumw / 4
    errs = []
    for d, g in zip(docs, got, strict=True):
        assert g.dtype == np.float32 and g.shape == (len(d),)
        want = so.sat_probas_f64(m, tok, d)
        errs.append(np.abs(g.astype(np.float64) - want))
        if not d:
            continue
        if len(tok.encode(d, add_special_tokens=False).ids) == 0:
            assert np.all(g == 0)
    err = np.concatenate(errs)
    _record({"case": name, "chars": int(err.size), "max_abs": float(err.max()), "mean_abs": float(err.mean()),
             "tol": tol})
    assert err.max() <= tol, (name, float(err.max()), tol)
    assert float(np.concatenate(got).std()) > 1e-3                  # the probabilities are not constant


def test_partition_bit_exact_against_reference_post_processing(tok, sat1):
    _m, eng = sat1
    rl.register_sentence_splitter(eng)
    rng = np.random.default_rng(5)
    docs = [_prose(rng, int(n)) for n in rng.integers(1, 900, size=200)]
    docs += ["# Title\n\nA b. C d.\n## Two\ntext here", "ab cd", "abcd", "abcde", "x" * 300]
    pred = rl.sentence_boundary_probas(docs)
    for min_len, max_len in PAIRS:
        batch = rl.split_sentences_batch(docs, min_len=min_len, max_len=max_len)
        for i, d in enumerate(docs):
            want = so.split_sentences_post(d, pred[i], min_len=min_len, max_len=max_len)
            assert batch[i] == want, (i, min_len, max_len)
            assert "".join(batch[i]) == d
        for i in range(0, len(docs), 20):
            assert rl.split_sentences(docs[i], min_len=min_len, max_len=max_len) == batch[i]
    with pytest.raises(ValueError, match="Sentence partition failed") as e:
        rl.split_sentences("abcdefghijklm", min_len=5, max_len=6, boundary_probas=np.zeros(13))
    assert str(e.value) == so.PARTITION_FAILED


def test_partition_ties_bit_exact(sat1):
    """Known probabilities from {0, 0.25, 0.5, 0.75, 1}: every score and every dp sum is exact, so the two options of a
    step and the deque's candidates tie often, and the strict comparisons and the eviction bound decide the result."""
    _m, eng = sat1
    rng = np.random.default_rng(13)
    docs = [_prose(rng, int(n)) for n in rng.integers(5, 700, size=150)]
    known = [rng.choice([0.0, 0.25, 0.5, 0.75, 1.0], size=len(d), p=[0.3, 0.2, 0.2, 0.2, 0.1]) for d in docs]
    zero = [np.zeros(len(d), np.float32) for d in docs]
    for min_len, max_len in [*PAIRS, (2, 5), (3, 16)]:
        try:
            got = eng.split(docs, known, min_len=min_len, max_len=max_len)
        except ValueError:
            got = None
        want = []
        for d, k, z in zip(docs, known, zero, strict=True):
            try:
                want.append(so.split_sentences_post(d, z, min_len=min_len, max_len=max_len, known=k))
            except ValueError:
                want = None
                break
        assert got == want, (min_len, max_len)


def test_golden_through_public_path(sat1):
    _m, eng = sat1
    rl.register_sentence_splitter(eng)
    z = np.load(Path(__file__).parent / "golden" / "split_sentences.npz")
    cases = json.loads(z["cases"].tobytes())
    n = 0
    for i, c in enumerate(cases):
        if not c["known"]:
            continue
        P = z[f"known{i}"]
        assert np.isfinite(P).all()
        if c["error"]:
            with pytest.raises(ValueError) as e:
                rl.split_sentences(c["doc"], min_len=c["min_len"], max_len=c["max_len"], boundary_probas=P)
            assert str(e.value) == c["error"]
        else:
            got = rl.split_sentences(c["doc"], min_len=c["min_len"], max_len=c["max_len"], boundary_probas=P)
            assert got == c["sentences"], c["name"]
        n += 1
    assert n >= 10


def test_batch_equals_single_across_calls_and_groups(tok, sat1):
    m, eng = sat1
    small = S.SaTEngine.from_hf(m, tok, max_tokens_per_call=600, group_chars=2500)   # ~2 blocks per call
    rng = np.random.default_rng(9)
    docs = [_prose(rng, int(n)) for n in (9000, 40, 1200, 7, 3000, 260)]
    a = eng.boundary_probas(docs)
    b = small.boundary_probas(docs)
    c = [eng.boundary_probas([d])[0] for d in docs]
    for x, y, z in zip(a, b, c, strict=True):
        np.testing.assert_array_equal(x.view(np.uint32), y.view(np.uint32))
        np.testing.assert_array_equal(x.view(np.uint32), z.view(np.uint32))
    known = [S.markdown_sentence_boundaries(d) for d in docs]
    for min_len, max_len in PAIRS:
        assert eng.split(docs, known, min_len=min_len, max_len=max_len) == small.split(docs, known, min_len=min_len,
                                                                                     max_len=max_len)


def test_two_million_character_document(tok, sat1):
    _m, eng = sat1
    rl.register_sentence_splitter(eng)
    rng = np.random.default_rng(11)
    doc = _prose(rng, 2_000_000)
    got = rl.split_sentences(doc, max_len=2048)
    assert "".join(got) == doc and max(map(len, got)) <= 2048 and min(map(len, got)) >= 4
    pred = rl.sentence_boundary_probas([doc])[0]
    assert got == so.split_sentences_post(doc, pred, min_len=4, max_len=2048)
