"""GPU parity of the cross-encoder engine at the multilingual rerankers' shapes against the float32 transformers oracle
(seeded weights, every bias and LayerNorm perturbed): BERT-base with two labels, XLM-R base and large with one, and the
two-label head on MiniLM's head_dim-32 path.  Then the default config end to end: ``rerank_chunks`` routed to the
``"other"`` reranker over seeded model directories."""

from __future__ import annotations

import json
import sys
import tempfile
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# lengths on either side of every 32 / 64 / 128 / 256 boundary, 1 and 512 included
BOUNDARY_LENGTHS = (1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 383, 384, 385, 511, 512)


def _record(name: str, payload: dict) -> None:
    """Append a line (case + measured error) to xenc_bounds.jsonl in the temporary directory."""
    with (Path(tempfile.gettempdir()) / "xenc_bounds.jsonl").open("a") as f:
        f.write(json.dumps({"test": name, **payload}) + "\n")


def _check(name, model, eng, ids, types):
    from scipy.stats import kendalltau

    import xenc_classifiers as xc

    got_logit, got_score = eng.score_tokens(ids, types)
    want = xc.classifier_logits(model, ids, types)
    n_labels = want.shape[1]
    assert got_logit.shape == ((len(ids), 2) if n_labels == 2 else (len(ids),))
    got2 = got_logit.reshape(len(ids), n_labels)
    err = np.abs(got2 - want)
    score_err = np.abs(got_score - xc.flashrank_scores(want))
    tau = kendalltau(xc.ranking_key(got2), xc.ranking_key(want))[0]
    worst = int(err.max(axis=1).argmax())
    _record(name, {"pairs": len(ids), "labels": n_labels, "max_len": max(len(x) for x in ids),
                   "max_abs_logit_err": float(err.max()), "worst_pair_len": len(ids[worst]),
                   "max_abs_score_err": float(score_err.max()), "kendall_tau": float(tau),
                   "logit_spread": float(xc.ranking_key(want).std())})
    assert err.max() < 4e-2, (name, float(err.max()), len(ids[worst]))
    assert score_err.max() < 1e-2, (name, float(score_err.max()))
    assert tau > 0.97, (name, tau)


CASES = [
    # name, shape, layers, labels, vocab (None: the shape's full vocabulary), random pairs
    ("multibert_l2_full_vocab", "multibert", 2, 2, None, 24),
    ("multibert_l12", "multibert", 12, 2, 5000, 16),
    ("xlmr_base_l2", "xlmr-base", 2, 1, 5000, 24),
    ("xlmr_large_l2", "xlmr-large", 2, 1, 5000, 24),
    ("xlmr_large_l24", "xlmr-large", 24, 1, 5000, 8),
    ("minilm_two_labels_l2", "minilm", 2, 2, 5000, 24),
]


@pytest.mark.parametrize(("name", "shape", "layers", "labels", "vocab", "n_random"), CASES, ids=[c[0] for c in CASES])
def test_wide_cross_encoder_matches_transformers_fp32(name, shape, layers, labels, vocab, n_random):
    """Several packed calls (a small ``max_tokens_per_call``) with long and short pairs mixed in each."""
    import xenc_classifiers as xc
    from raglite_b200._xenc import CrossEncoderEngine

    over = dict(num_hidden_layers=layers, num_labels=labels)
    if vocab is not None:
        over["vocab_size"] = vocab
    model = xc.seeded_classifier(shape, seed=layers + 7 * labels, **over)
    eng = CrossEncoderEngine.from_hf(model, max_tokens_per_call=3000)
    assert eng.n_labels == labels and eng.max_length == 512
    rng = np.random.default_rng(layers)
    ids, types = xc.random_pairs(n_random, model.config.vocab_size, rng, model.config.model_type, lo=3, hi=513,
                                 lengths=BOUNDARY_LENGTHS)
    order = rng.permutation(len(ids))
    ids, types = [ids[i] for i in order], [types[i] for i in order]
    _check(name, model, eng, ids, types)


def _wordpiece_tokenizer(n_words: int):
    from tokenizers import Tokenizer, models, pre_tokenizers, processors

    words = ["[PAD]", "[UNK]", "[CLS]", "[SEP]"] + [f"w{i}" for i in range(n_words)]
    tok = Tokenizer(models.WordPiece({w: i for i, w in enumerate(words)}, unk_token="[UNK]"))
    tok.pre_tokenizer = pre_tokenizers.Whitespace()
    tok.post_processor = processors.TemplateProcessing(single="[CLS] $A [SEP]", pair="[CLS] $A [SEP] $B:1 [SEP]:1",
                                                       special_tokens=[("[CLS]", 2), ("[SEP]", 3)])
    return tok, len(words)


def _roberta_tokenizer(n_words: int):
    from tokenizers import Tokenizer, models, pre_tokenizers, processors

    words = ["<s>", "<pad>", "</s>", "<unk>"] + [f"w{i}" for i in range(n_words)]
    tok = Tokenizer(models.WordLevel({w: i for i, w in enumerate(words)}, unk_token="<unk>"))
    tok.pre_tokenizer = pre_tokenizers.Whitespace()
    tok.post_processor = processors.RobertaProcessing(("</s>", 2), ("<s>", 0))
    return tok, len(words)


def _save(path: Path, model, tok) -> None:  # noqa: ANN001
    model.save_pretrained(path)
    tok.save(str(path / "tokenizer.json"))


def _chunks(n: int, n_words: int, seed: int):
    import raglite_b200 as rl

    rng = np.random.default_rng(seed)
    return [rl.Chunk(id=f"c{i}", body=" ".join(f"w{j}" for j in rng.integers(0, n_words, size=int(rng.integers(5, 120)))))
            for i in range(n)]


def _check_order(ranked, model, eng, query, chunks):
    import xenc_classifiers as xc

    ids, types = eng.encode_pairs([query] * len(chunks), [str(c) for c in chunks])
    ref_scores = xc.flashrank_scores(xc.classifier_logits(model, ids, types))
    want = np.argsort(-ref_scores, kind="stable")
    got = [int(c.id[1:]) for c in ranked]
    assert sorted(got) == list(range(len(chunks)))
    # identical order except where float32 scores are within fp16 noise of each other
    for a, b in zip(got, want.tolist(), strict=True):
        assert a == b or abs(ref_scores[a] - ref_scores[b]) < 2e-2
    return ids, types


def test_default_config_reranks_with_the_multilingual_reranker(tmp_path, monkeypatch):
    """``RAGLiteConfig()``'s two-entry reranker dict over a cache directory of seeded weights: without a language
    detector every call goes to ``"other"`` (the two-label MultiBERT-shaped model), and ``"en"`` is never loaded."""
    import raglite_b200 as rl
    import raglite_b200._config as rl_config
    import xenc_classifiers as xc
    from transformers import BertForSequenceClassification

    monkeypatch.setitem(sys.modules, "langdetect", None)   # the routing as without langdetect installed
    tok, n_vocab = _wordpiece_tokenizer(300)
    tok_en, n_vocab_en = _wordpiece_tokenizer(200)
    _save(tmp_path / "ms-marco-MiniLM-L-12-v2", xc.seeded_classifier("minilm", seed=3, num_hidden_layers=2,
                                                                      vocab_size=n_vocab_en), tok_en)
    _save(tmp_path / "ms-marco-MultiBERT-L-12", xc.seeded_classifier("multibert", seed=4, num_hidden_layers=2,
                                                                      vocab_size=n_vocab), tok)
    monkeypatch.setattr(rl_config, "cache_path", tmp_path)
    cfg = rl.RAGLiteConfig()
    assert set(cfg.reranker) == {"en", "other"}
    chunks = _chunks(24, 300, seed=0)
    query = "w1 w2 w3 w4 w5"
    ranked = rl.rerank_chunks(query, chunks, config=cfg)
    assert cfg.reranker["en"]._engine is None                     # noqa: SLF001
    eng = cfg.reranker["other"]._engine                           # noqa: SLF001
    assert eng is not None and eng.n_labels == 2 and eng.model_type == "bert"
    model = BertForSequenceClassification.from_pretrained(tmp_path / "ms-marco-MultiBERT-L-12", local_files_only=True).eval()
    _check_order(ranked, model, eng, query, chunks)


def test_xlm_roberta_ranker_directory(tmp_path, monkeypatch):
    """An XLM-R sequence classifier directory with a ``RobertaProcessing`` tokenizer as the ``"other"`` reranker."""
    import raglite_b200 as rl
    import xenc_classifiers as xc
    from raglite_b200._rerank import B200CrossEncoderRanker
    from transformers import XLMRobertaForSequenceClassification

    monkeypatch.setitem(sys.modules, "langdetect", None)
    tok, n_vocab = _roberta_tokenizer(300)
    _save(tmp_path / "xlmr-reranker", xc.seeded_classifier("xlmr-base", seed=5, num_hidden_layers=2, vocab_size=n_vocab), tok)
    rerankers = {"en": B200CrossEncoderRanker("absent-en-model", cache_dir=tmp_path),
                 "other": B200CrossEncoderRanker("xlmr-reranker", cache_dir=tmp_path)}
    cfg = rl.RAGLiteConfig(reranker=rerankers)
    chunks = _chunks(24, 300, seed=1)
    query = "w7 w8 w9"
    ranked = rl.rerank_chunks(query, chunks, config=cfg)
    assert rerankers["en"]._engine is None                        # noqa: SLF001
    eng = rerankers["other"]._engine                              # noqa: SLF001
    assert eng.model_type == "xlm-roberta" and eng.n_labels == 1 and eng.pos_offset == 2
    model = XLMRobertaForSequenceClassification.from_pretrained(tmp_path / "xlmr-reranker", local_files_only=True).eval()
    ids, types = _check_order(ranked, model, eng, query, chunks)
    assert all(int(t.max()) == 0 for t in types)                  # RobertaProcessing: zero type ids for pairs
    assert all(x[0] == 0 and x[-1] == 2 for x in ids)
