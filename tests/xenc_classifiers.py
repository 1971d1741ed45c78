"""Seeded BERT / XLM-RoBERTa sequence classifiers with one or two labels and their float32 ``transformers`` forward on
the CPU (TEST INFRASTRUCTURE): the oracle of the wide cross-encoder tests and of ``tools/bench_rerank.py``.

PARITY UNPINNED vs FlashRank, as for ``oracle.rerank``: no real reranker weights are available offline.  What is
restated: the two architectures (``BertForSequenceClassification``: pooler + classifier; ``XLMRobertaForSequence
Classification``: classifier.dense + tanh + out_proj on the first token, positions from ``padding_idx + 1``, zero type
ids) and FlashRank's post-processing as it is recalled (not verifiable offline): ``sigmoid(logit)`` for one label and
``softmax(logits)[:, 1]`` for two.  The shapes below are the ones recalled for the named checkpoints; they are test
shapes, not statements about those checkpoints.
"""

from __future__ import annotations

from collections.abc import Sequence

import numpy as np
import torch

# name -> (family, config overrides)
SHAPES = {
    # ms-marco-MiniLM-L-12-v2 (the "en" reranker of the default config)
    "minilm": ("bert", dict(vocab_size=30522, hidden_size=384, num_hidden_layers=12, num_attention_heads=12,
                            intermediate_size=1536, max_position_embeddings=512, num_labels=1)),
    # multilingual BERT-base passage reranker with two labels (the "other" reranker of the default config)
    "multibert": ("bert", dict(vocab_size=105879, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                               intermediate_size=3072, max_position_embeddings=512, num_labels=2)),
    # XLM-R base with one label (bge-reranker-base's recalled shape)
    "xlmr-base": ("xlm-roberta", dict(vocab_size=250002, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                                      intermediate_size=3072, max_position_embeddings=514, num_labels=1)),
    # XLM-R large with one label (bge-reranker-v2-m3's recalled shape)
    "xlmr-large": ("xlm-roberta", dict(vocab_size=250002, hidden_size=1024, num_hidden_layers=24, num_attention_heads=16,
                                       intermediate_size=4096, max_position_embeddings=8194, num_labels=1)),
}
# [CLS], [SEP], [PAD] of a BERT vocabulary; <s>, </s>, <pad> of XLM-R's
SPECIAL_IDS = {"bert": (101, 102, 0), "xlm-roberta": (0, 2, 1)}


def classifier_config(shape: str, **over):  # noqa: ANN003, ANN201
    from transformers import BertConfig, XLMRobertaConfig

    family, cfg = SHAPES[shape]
    cfg = dict(cfg, hidden_act="gelu", hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    if family == "bert":
        cfg.update(type_vocab_size=2, layer_norm_eps=1e-12, pad_token_id=0)
    else:
        cfg.update(type_vocab_size=1, layer_norm_eps=1e-5, pad_token_id=1, bos_token_id=0, eos_token_id=2)
    cfg.update(over)
    return BertConfig(**cfg) if family == "bert" else XLMRobertaConfig(**cfg)


def seeded_classifier(shape: str, seed: int = 0, *, perturb: bool = True, **over):  # noqa: ANN003, ANN201
    """Deterministic random sequence classifier of ``shape`` (float32, eval mode, eager attention); the output layer is
    scaled so that logits spread, and with ``perturb`` every bias and LayerNorm is drawn away from its init value
    (biases and betas from N(0, 0.1), gammas from 1 + N(0, 0.1)) so that a forward that dropped one would not match."""
    from transformers import BertForSequenceClassification, XLMRobertaForSequenceClassification

    config = classifier_config(shape, **over)
    config._attn_implementation = "eager"   # noqa: SLF001
    torch.manual_seed(seed)
    if config.model_type == "bert":
        model = BertForSequenceClassification(config).eval()
        out = model.classifier
    else:
        model = XLMRobertaForSequenceClassification(config).eval()
        out = model.classifier.out_proj
    with torch.no_grad():
        out.weight.mul_(8.0)
        if perturb:
            for m in model.modules():
                if isinstance(m, torch.nn.Linear) and m.bias is not None:
                    m.bias.normal_(0.0, 0.1)
                elif isinstance(m, torch.nn.LayerNorm):
                    m.weight.normal_(1.0, 0.1)
                    m.bias.normal_(0.0, 0.1)
    return model


def random_pairs(n: int, vocab: int, rng: np.random.Generator, family: str, *, lo: int = 6, hi: int = 180,
                 lengths: Sequence[int] = ()) -> tuple[list[np.ndarray], list[np.ndarray]]:
    """``lengths`` first, then ``n`` pairs of random length in [lo, hi): BERT's ``[CLS] q [SEP] d [SEP]`` with type ids
    0 / 1, XLM-R's ``<s> q </s></s> d </s>`` with zero type ids.  Ordinary tokens are drawn from [5, vocab) without
    the pad id: transformers derives XLM-R positions from ``input_ids != padding_idx``, so a pad id inside a sequence
    would shift the positions after it by design."""
    cls_id, sep_id, pad_id = SPECIAL_IDS[family]
    ids, types = [], []
    for L in [*lengths, *(int(rng.integers(lo, hi)) for _ in range(n))]:
        a = rng.integers(5, vocab, size=L).astype(np.int32)
        a[a == pad_id] = 5
        t = np.zeros(L, np.int32)
        a[0] = cls_id
        if L >= 2:
            a[-1] = sep_id
        if L >= 5:
            q = int(rng.integers(2, max(3, L // 3)))
            if family == "bert":
                a[q] = sep_id
                t[q + 1:] = 1
            else:
                a[q], a[q + 1] = sep_id, sep_id
        ids.append(a)
        types.append(t)
    return ids, types


@torch.no_grad()
def classifier_logits(model, ids: Sequence[np.ndarray], type_ids: Sequence[np.ndarray] | None = None,  # noqa: ANN001
                      batch: int = 16) -> np.ndarray:
    """Padded float32 forward with an attention mask: ``[P, num_labels]`` logits.  Batches are formed in length order so
    that little padding is computed; XLM-R gets zero type ids and the pad id as padding."""
    c = model.config
    P = len(ids)
    out = np.zeros((P, c.num_labels), np.float32)
    order = sorted(range(P), key=lambda i: len(ids[i]))
    for s in range(0, P, batch):
        rows = order[s:s + batch]
        L = max(len(ids[i]) for i in rows)
        inp = torch.full((len(rows), L), int(c.pad_token_id), dtype=torch.long)
        typ = torch.zeros_like(inp)
        msk = torch.zeros_like(inp)
        for r, i in enumerate(rows):
            n = len(ids[i])
            inp[r, :n] = torch.from_numpy(np.asarray(ids[i], np.int64))
            if type_ids is not None and c.model_type == "bert":
                typ[r, :n] = torch.from_numpy(np.asarray(type_ids[i], np.int64))
            msk[r, :n] = 1
        out[rows] = model(input_ids=inp, token_type_ids=typ, attention_mask=msk).logits.float().numpy()
    return out


def flashrank_scores(logits: np.ndarray) -> np.ndarray:
    """FlashRank's score in float64: ``sigmoid(logit)`` for ``[P]`` / ``[P, 1]`` logits, ``softmax(logits)[:, 1]`` for
    ``[P, 2]``."""
    lg = np.asarray(logits, np.float64)
    if lg.ndim == 1 or lg.shape[1] == 1:
        return 1.0 / (1.0 + np.exp(-lg.reshape(-1)))
    e = np.exp(lg - lg.max(axis=1, keepdims=True))
    return e[:, 1] / e.sum(axis=1)


def ranking_key(logits: np.ndarray) -> np.ndarray:
    """What the score sorts by: the logit, or ``l1 - l0`` for two labels."""
    lg = np.asarray(logits, np.float64)
    if lg.ndim == 1 or lg.shape[1] == 1:
        return lg.reshape(-1)
    return lg[:, 1] - lg[:, 0]
