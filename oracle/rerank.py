"""CPU restatement of the cross-encoder scoring behind ``rerank_chunks`` (TEST INFRASTRUCTURE).

PARITY UNPINNED vs the real FlashRank model: the reference scores with ``rerankers``'
FlashRankRanker -> flashrank -> onnxruntime on ms-marco-MiniLM-L-12-v2 (all un-vendored third-party
code, weights unavailable offline).  What is restated: the architecture (BERT encoder + pooler +
1-logit classifier), FlashRank's post-processing (``score = sigmoid(logit)``, sort descending,
``doc_id`` = index into ``docs``) and the reorder of ``rerank_chunks`` (``_search.py:395-396``).  The
forward is ``transformers.BertForSequenceClassification`` in float32 on the CPU.
"""

from __future__ import annotations

from collections.abc import Sequence

import numpy as np
import torch


def minilm_config(**over):  # noqa: ANN003, ANN201
    """ms-marco-MiniLM-L-12-v2's architecture (SURVEY.md 8a-5)."""
    from transformers import BertConfig

    cfg = dict(vocab_size=30522, hidden_size=384, num_hidden_layers=12, num_attention_heads=12, intermediate_size=1536,
               max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12, hidden_act="gelu", num_labels=1,
               hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    cfg.update(over)
    return BertConfig(**cfg)


def seeded_model(seed: int = 0, *, perturb: bool = False, **over):  # noqa: ANN003, ANN201
    """Deterministic random weights (real ones cannot be downloaded here); scaled so that logits spread.

    The transformers init leaves every Linear bias at 0 and every LayerNorm at gamma = 1, beta = 0, so a forward
    that dropped them would still match.  ``perturb`` draws them instead: biases (pooler and classifier included)
    and LayerNorm betas from N(0, 0.1), LayerNorm gammas from 1 + N(0, 0.1)."""
    from transformers import BertForSequenceClassification

    torch.manual_seed(seed)
    model = BertForSequenceClassification(minilm_config(**over)).eval()
    with torch.no_grad():
        model.classifier.weight.mul_(8.0)
        if perturb:
            for m in model.modules():
                if isinstance(m, torch.nn.Linear) and m.bias is not None:
                    m.bias.normal_(0.0, 0.1)
                elif isinstance(m, torch.nn.LayerNorm):
                    m.weight.normal_(1.0, 0.1)
                    m.bias.normal_(0.0, 0.1)
    return model


@torch.no_grad()
def hf_logits(model, ids: Sequence[np.ndarray], type_ids: Sequence[np.ndarray], batch: int = 32) -> np.ndarray:  # noqa: ANN001
    """Padded float32 forward with an attention mask; returns one logit per pair."""
    out = []
    for s in range(0, len(ids), batch):
        chunk_i, chunk_t = ids[s:s + batch], type_ids[s:s + batch]
        L = max(len(x) for x in chunk_i)
        inp = torch.zeros((len(chunk_i), L), dtype=torch.long)
        typ = torch.zeros_like(inp)
        msk = torch.zeros_like(inp)
        for r, (a, b) in enumerate(zip(chunk_i, chunk_t, strict=True)):
            inp[r, :len(a)] = torch.from_numpy(np.asarray(a, np.int64))
            typ[r, :len(a)] = torch.from_numpy(np.asarray(b, np.int64))
            msk[r, :len(a)] = 1
        out.append(model(input_ids=inp, token_type_ids=typ, attention_mask=msk).logits.reshape(-1).float().numpy())
    return np.concatenate(out) if out else np.zeros(0, np.float32)


def flashrank_scores(logits: np.ndarray) -> np.ndarray:
    """FlashRank: ``1 / (1 + exp(-logit))`` for single-logit models."""
    return 1.0 / (1.0 + np.exp(-logits.astype(np.float64)))


def rank_order(scores: np.ndarray) -> np.ndarray:
    """Descending by score, stable (doc order breaks ties)."""
    return np.argsort(-scores, kind="stable")
