"""CPU restatement of the embedding model behind ``embed_strings`` (TEST INFRASTRUCTURE).

PARITY UNPINNED vs llama.cpp: the reference embeds with llama-cpp-python on bge-m3's GGUF weights
(``README.md:114``, ``_config.py:58-64``) -- un-vendored third-party code, and no weights or vocabulary are
available offline.  What is restated: the architecture (``transformers`` ``XLMRobertaModel`` / ``BertModel`` in
float32, last hidden state of every token), llama-cpp-python's ``embed(truncate=True)`` (the tokenizer's special
tokens included, truncated to ``n_batch`` tokens) and the llama-like protocol ``raglite._embed`` calls, so that
``oracle.pool.embed_with_llama(sentences, HFEmbedder(...))`` is the reference's whole late-chunking flow.

Tokenizers are built in memory with ``tokenizers`` (a Unigram vocabulary in XLM-RoBERTa's layout and a WordPiece
one in BERT's); both contain the sentinel ``⊕``.
"""

from __future__ import annotations

from collections.abc import Sequence

import numpy as np
import torch

WORDS = ("alpha", "beta", "gamma", "delta", "light", "clock", "rod", "frame", "event", "time", "of", "the",
         "simultaneous", "observer", "velocity", "what", "is", "how", "does", "a", "an", "in", "to")
CHARS = list("abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789.,;:?!'\"()-éï\n") + ["⊕"]


def bge_m3_config(**over):  # noqa: ANN003, ANN201
    """BAAI/bge-m3's architecture: XLM-RoBERTa large, 24 layers, H = 1024, 16 heads x 64, FFN 4096."""
    from transformers import XLMRobertaConfig

    cfg = dict(vocab_size=250002, hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, intermediate_size=4096,
               max_position_embeddings=8194, type_vocab_size=1, layer_norm_eps=1e-5, hidden_act="gelu", pad_token_id=1,
               bos_token_id=0, eos_token_id=2, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    cfg.update(over)
    return XLMRobertaConfig(**cfg)


def bert_config(**over):  # noqa: ANN003, ANN201
    from transformers import BertConfig

    cfg = dict(vocab_size=30522, hidden_size=768, num_hidden_layers=2, num_attention_heads=12, intermediate_size=3072,
               max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12, hidden_act="gelu",
               hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    cfg.update(over)
    return BertConfig(**cfg)


def _perturb(model: torch.nn.Module) -> None:
    """Biases and LayerNorm beta from N(0, 0.1), LayerNorm gamma from 1 + N(0, 0.1) (as ``oracle.rerank.seeded_model``):
    the init's zeros and ones would let a forward that drops them still match."""
    for m in model.modules():
        if isinstance(m, torch.nn.Linear) and m.bias is not None:
            m.bias.normal_(0.0, 0.1)
        elif isinstance(m, torch.nn.LayerNorm):
            m.weight.normal_(1.0, 0.1)
            m.bias.normal_(0.0, 0.1)


def seeded_model(config, seed: int = 0, *, perturb: bool = True):  # noqa: ANN001, ANN201
    """Deterministic random ``XLMRobertaModel`` / ``BertModel`` for ``config`` (float32, eval mode, eager attention)."""
    from transformers import BertModel, XLMRobertaModel

    torch.manual_seed(seed)
    cls = XLMRobertaModel if config.model_type == "xlm-roberta" else BertModel
    config._attn_implementation = "eager"   # noqa: SLF001
    model = cls(config, add_pooling_layer=False).eval()
    if perturb:
        with torch.no_grad():
            _perturb(model)
    return model


def unigram_tokenizer():  # noqa: ANN201
    """XLM-RoBERTa-like SentencePiece Unigram tokenizer: <s>=0, <pad>=1, </s>=2, <unk>=3, ``<s> $A </s>``."""
    from tokenizers import Tokenizer, decoders, models, pre_tokenizers, processors

    specials = ["<s>", "<pad>", "</s>", "<unk>"]
    pieces = [(s, 0.0) for s in specials]
    pieces += [("▁" + w, -3.0) for w in WORDS] + [("▁" + w.capitalize(), -3.5) for w in WORDS]
    pieces += [("▁⊕", -4.0), ("▁", -5.0)] + [(c, -6.0) for c in CHARS]
    tok = Tokenizer(models.Unigram(pieces, unk_id=3))
    tok.pre_tokenizer = pre_tokenizers.Metaspace(replacement="▁", prepend_scheme="always")
    tok.decoder = decoders.Metaspace(replacement="▁", prepend_scheme="always")
    tok.post_processor = processors.TemplateProcessing(single="<s> $A </s>", special_tokens=[("<s>", 0), ("</s>", 2)])
    return tok


def wordpiece_tokenizer():  # noqa: ANN201
    """BERT-like WordPiece tokenizer: [PAD]=0, [UNK]=1, [CLS]=2, [SEP]=3, ``[CLS] $A [SEP]``."""
    from tokenizers import Tokenizer, decoders, models, normalizers, pre_tokenizers, processors

    vocab = {t: i for i, t in enumerate(["[PAD]", "[UNK]", "[CLS]", "[SEP]", "[MASK]"])}
    for t in [*WORDS, *[c for c in CHARS if not c.isupper()], *["##" + c for c in CHARS if not c.isupper()]]:
        vocab.setdefault(t, len(vocab))
    tok = Tokenizer(models.WordPiece(vocab, unk_token="[UNK]"))
    tok.normalizer = normalizers.BertNormalizer(lowercase=True)
    tok.pre_tokenizer = pre_tokenizers.BertPreTokenizer()
    tok.decoder = decoders.WordPiece()
    tok.post_processor = processors.TemplateProcessing(single="[CLS] $A [SEP]", special_tokens=[("[CLS]", 2), ("[SEP]", 3)])
    return tok


class HFEmbedder:
    """llama-like embedder (``n_ctx() / n_batch / n_embd() / tokenize / detokenize / embed``) over a float32
    ``transformers`` encoder on the CPU and a ``tokenizers.Tokenizer``."""

    def __init__(self, model, tokenizer, n_ctx: int = 512) -> None:  # noqa: ANN001
        self.model = model.eval()
        self.tokenizer = tokenizer
        self._n_ctx = n_ctx
        self.n_batch = n_ctx

    def n_ctx(self) -> int:
        return self._n_ctx

    def n_embd(self) -> int:
        return int(self.model.config.hidden_size)

    def tokenize(self, text: bytes, add_bos: bool = False, special: bool = False) -> list[int]:  # noqa: ARG002
        return list(self.tokenizer.encode(text.decode(), add_special_tokens=False).ids)

    def detokenize(self, tokens: Sequence[int]) -> bytes:
        return self.tokenizer.decode([int(t) for t in tokens], skip_special_tokens=False).encode()

    def token_ids(self, text: str) -> list[int]:
        """llama-cpp-python's ``embed(truncate=True)`` input: special tokens included, at most ``n_batch`` tokens."""
        return list(self.tokenizer.encode(text, add_special_tokens=True).ids[: self.n_batch])

    @torch.no_grad()
    def hidden_states(self, ids: Sequence[int]) -> np.ndarray:
        """Last hidden state ``[len(ids), H]`` (float32) of one sequence."""
        x = torch.as_tensor(np.asarray(ids, dtype=np.int64))[None]
        return self.model(input_ids=x, attention_mask=torch.ones_like(x)).last_hidden_state[0].float().numpy()

    def embed(self, text):  # noqa: ANN001, ANN201
        if isinstance(text, str):
            return self.hidden_states(self.token_ids(text))
        return [self.hidden_states(self.token_ids(t)) for t in text]
