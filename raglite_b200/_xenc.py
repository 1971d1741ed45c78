"""BERT / XLM-RoBERTa cross-encoder engine on the GPU -- the arithmetic behind ``rerank_chunks``.

The reference calls ``reranker.rank(query=, docs=)`` (``_search.py:395``) on a ``rerankers``
FlashRankRanker: tokenise (query, passage) pairs, run ms-marco-MiniLM-L-12-v2 (BERT, 12 layers, H=384,
12 heads, FFN=1536) with onnxruntime, sigmoid the logit, sort.  Here the forward runs in
``rl_xenc_score`` (hand-written CUDA: wgmma linear layers with fused bias/GELU, attention,
LayerNorm, pooler+classifier) on packed variable-length batches -- no padding tokens are computed.
The same engine scores wider multilingual rerankers: BERT-base and XLM-RoBERTa sequence classifiers
(head_dim 64, H <= 1024) with one logit, or two scored as ``softmax(logits)[1]``.

``TokenEmbedderEngine`` runs the same encoder without the head (``rl_xenc_encode``: head_dim 32 or 64, H <= 1024) and
returns per-token hidden states: the embedding model behind ``embed_strings`` (bge-m3 by default), which the reference
runs in llama.cpp.
"""

from __future__ import annotations

import ctypes as C
import threading
from collections.abc import Sequence
from pathlib import Path
from typing import Any

import numpy as np
import torch

from . import _lib
from ._gguf import QUANT_TYPES, GGUFTensor, tensor_to_f32
from ._lib import XencLayer, XencWeights, check


def _stream() -> int:
    return int(torch.cuda.current_stream().cuda_stream)


def random_minilm_state_dict(seed: int = 0, *, n_layers: int = 12, hidden: int = 384, ffn: int = 1536,
                             vocab: int = 30522, max_pos: int = 512) -> dict[str, torch.Tensor]:
    """Seeded random weights with the HF ``BertForSequenceClassification`` names/shapes of
    ms-marco-MiniLM-L-12-v2 (real weights cannot be downloaded offline); for benchmarks and smoke tests."""
    g = torch.Generator().manual_seed(seed)

    def w(*shape: int) -> torch.Tensor:
        return torch.randn(shape, generator=g) * 0.02

    sd = {
        "bert.embeddings.word_embeddings.weight": w(vocab, hidden),
        "bert.embeddings.position_embeddings.weight": w(max_pos, hidden),
        "bert.embeddings.token_type_embeddings.weight": w(2, hidden),
        "bert.embeddings.LayerNorm.weight": torch.ones(hidden), "bert.embeddings.LayerNorm.bias": torch.zeros(hidden),
        "bert.pooler.dense.weight": w(hidden, hidden), "bert.pooler.dense.bias": torch.zeros(hidden),
        "classifier.weight": w(1, hidden) * 8.0, "classifier.bias": torch.zeros(1),
    }
    for l in range(n_layers):
        p = f"bert.encoder.layer.{l}."
        for n in ("query", "key", "value"):
            sd[p + f"attention.self.{n}.weight"], sd[p + f"attention.self.{n}.bias"] = w(hidden, hidden), torch.zeros(hidden)
        sd[p + "attention.output.dense.weight"], sd[p + "attention.output.dense.bias"] = w(hidden, hidden), torch.zeros(hidden)
        sd[p + "attention.output.LayerNorm.weight"], sd[p + "attention.output.LayerNorm.bias"] = torch.ones(hidden), torch.zeros(hidden)
        sd[p + "intermediate.dense.weight"], sd[p + "intermediate.dense.bias"] = w(ffn, hidden), torch.zeros(ffn)
        sd[p + "output.dense.weight"], sd[p + "output.dense.bias"] = w(hidden, ffn), torch.zeros(hidden)
        sd[p + "output.LayerNorm.weight"], sd[p + "output.LayerNorm.bias"] = torch.ones(hidden), torch.zeros(hidden)
    return sd


def _pack_inputs(h: np.ndarray, ids: Sequence[np.ndarray], type_ids: Sequence[np.ndarray] | None, lens: np.ndarray,
                 pos_offset: int) -> int:
    """Lay one packed call out in the int32 array ``h``: ids [T] | type ids [T] | position ids [T] | cu_seqlens [P + 1].
    Position ids run ``pos_offset + i`` per sequence (0 for BERT; ``padding_idx + 1`` for XLM-RoBERTa, whose table
    keeps rows for the padding index and below); type ids are 0 when ``type_ids`` is None.  Returns T."""
    P, T = len(ids), int(lens.sum())
    if T:
        np.concatenate(ids, out=h[:T], casting="unsafe")
    if type_ids is None:
        h[T:2 * T] = 0
    elif T:
        np.concatenate(type_ids, out=h[T:2 * T], casting="unsafe")
    cu = h[3 * T:3 * T + P + 1]
    cu[0] = 0
    np.cumsum(lens, out=cu[1:])
    h[2 * T:3 * T] = np.arange(T, dtype=np.int32) - np.repeat(cu[:-1], lens) + pos_offset
    return T


class _EncoderEngine:
    """Device-resident packed encoder weights (embeddings + layers), the workspace and the pinned double-buffered call
    pipeline: what the cross-encoder and the token embedder share."""

    def __init__(self, state_dict: dict[str, torch.Tensor], *, n_layers: int, hidden: int, n_heads: int, ffn: int,
                 max_pos: int, ln_eps: float, device: Any | None, max_tokens_per_call: int, pos_offset: int = 0) -> None:
        if not torch.cuda.is_available():
            raise RuntimeError("raglite_b200 needs a CUDA device (there is no CPU fallback)")
        self.lib = _lib.load()
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.max_tokens_per_call = max_tokens_per_call
        self.hidden, self.n_layers = hidden, n_layers
        self.pos_offset = pos_offset
        self._keep: list[torch.Tensor] = []
        sd = {k.removeprefix("bert.").removeprefix("roberta."): v for k, v in state_dict.items()}
        self._sd = sd

        self._layers = (XencLayer * n_layers)()
        for l in range(n_layers):
            pre = f"encoder.layer.{l}."
            qkv_b = torch.cat([sd[pre + f"attention.self.{n}.bias"] for n in ("query", "key", "value")], dim=0)
            qkv_b = qkv_b.detach().to(device=self.device, dtype=torch.float32).contiguous()
            self._keep.append(qkv_b)
            L = self._layers[l]
            L.qkv_img, L.qkv_type = self._image([sd[pre + f"attention.self.{n}.weight"] for n in ("query", "key", "value")])
            L.qkv_bias = qkv_b.data_ptr()
            L.o_img, L.o_type = self._image([sd[pre + "attention.output.dense.weight"]])
            L.o_bias = self._f32(pre + "attention.output.dense.bias").data_ptr()
            L.ln1_g, L.ln1_b = self._f32(pre + "attention.output.LayerNorm.weight").data_ptr(), self._f32(pre + "attention.output.LayerNorm.bias").data_ptr()
            L.up_img, L.up_type = self._image([sd[pre + "intermediate.dense.weight"]])
            L.up_bias = self._f32(pre + "intermediate.dense.bias").data_ptr()
            L.down_img, L.down_type = self._image([sd[pre + "output.dense.weight"]])
            L.down_bias = self._f32(pre + "output.dense.bias").data_ptr()
            L.ln2_g, L.ln2_b = self._f32(pre + "output.LayerNorm.weight").data_ptr(), self._f32(pre + "output.LayerNorm.bias").data_ptr()
        w = XencWeights()
        w.n_layers, w.hidden, w.n_heads, w.ffn = n_layers, hidden, n_heads, ffn
        w.vocab, w.max_pos = int(sd["embeddings.word_embeddings.weight"].shape[0]), max_pos
        w.type_vocab, w.ln_eps = int(sd["embeddings.token_type_embeddings.weight"].shape[0]), ln_eps
        w.word_emb = self._f16("embeddings.word_embeddings.weight").data_ptr()
        w.pos_emb = self._f16("embeddings.position_embeddings.weight").data_ptr()
        w.type_emb = self._f16("embeddings.token_type_embeddings.weight").data_ptr()
        w.emb_ln_g, w.emb_ln_b = self._f32("embeddings.LayerNorm.weight").data_ptr(), self._f32("embeddings.LayerNorm.bias").data_ptr()
        w.layers = C.cast(self._layers, C.POINTER(XencLayer))
        self.weights = w
        self._ws: torch.Tensor | None = None
        self._host_bufs: dict[str, torch.Tensor] = {}   # pinned staging (double-buffered inputs / outputs)
        self._dev_bufs: dict[int, torch.Tensor] = {}
        self._lock = threading.RLock()   # reference callers rerank from thread pools (_rag.py:317)

    def _f32(self, name: str) -> torch.Tensor:
        t = self._sd[name].detach().to(device=self.device, dtype=torch.float32).contiguous()
        self._keep.append(t)
        return t

    def _f16(self, name: str) -> torch.Tensor:
        w = self._sd[name]
        if isinstance(w, GGUFTensor):   # an embedding table of a GGUF file: quantized ones are dequantized on the device
            if w.ggml_type not in QUANT_TYPES:
                w = torch.from_numpy(tensor_to_f32(w))
            else:
                blocks = torch.from_numpy(w.data.copy()).to(self.device)
                t = torch.empty(w.shape, dtype=torch.float16, device=self.device)
                with torch.cuda.device(self.device):
                    check(self.lib.rl_dequant_rows_f16(w.ggml_type, blocks.data_ptr(), w.shape[0], w.shape[1], t.data_ptr(),
                                                       _stream()), "rl_dequant_rows_f16")
                    torch.cuda.current_stream().synchronize()
                self._keep.append(t)
                return t
        t = w.detach().to(device=self.device, dtype=torch.float16).contiguous()
        self._keep.append(t)
        return t

    def _image(self, parts: list[Any]) -> tuple[int, int]:
        """The packed image of the row-wise concatenation of ``parts`` (torch float weights, or tensors of a GGUF file)
        and its ``RL_XENC_IMAGE_*`` type.  Quantized parts stay quantized: one image when they share a type, else one
        image per part concatenated pass by pass.  Quantized parts were checked by ``_gguf.bert_plan`` before any device
        work."""
        quant = [isinstance(p, GGUFTensor) and p.ggml_type in QUANT_TYPES for p in parts]
        if not any(quant):
            ws = [torch.from_numpy(tensor_to_f32(p)) if isinstance(p, GGUFTensor) else p for p in parts]
            return self._packed(torch.cat(ws, dim=0) if len(ws) > 1 else ws[0]).data_ptr(), _lib.RL_XENC_IMAGE_F16
        K = parts[0].shape[1]   # (bert_plan has checked the parts: all quantized, K % 128 == 0)
        groups = [list(parts)] if len({p.ggml_type for p in parts}) == 1 else [[p] for p in parts]
        imgs = []
        for g in groups:
            blocks = torch.from_numpy(np.concatenate([p.data for p in g])).to(self.device)
            N = sum(p.shape[0] for p in g)
            img = torch.empty(int(self.lib.rl_xenc_qlinear_image_bytes(g[0].ggml_type, N, K)), dtype=torch.uint8,
                              device=self.device)
            with torch.cuda.device(self.device):
                check(self.lib.rl_xenc_pack_qlinear(g[0].ggml_type, blocks.data_ptr(), N, K, img.data_ptr(), _stream()),
                      "rl_xenc_pack_qlinear")
                torch.cuda.current_stream().synchronize()
            imgs.append(img)
        if len(imgs) > 1:
            out = torch.empty(sum(i.numel() for i in imgs), dtype=torch.uint8, device=self.device)
            ptrs = (C.c_void_p * len(imgs))(*[i.data_ptr() for i in imgs])
            with torch.cuda.device(self.device):
                check(self.lib.rl_xenc_concat_qlinear(ptrs, len(imgs), out.data_ptr(), _stream()), "rl_xenc_concat_qlinear")
                torch.cuda.current_stream().synchronize()
            imgs = [out]
        self._keep.append(imgs[0])
        return imgs[0].data_ptr(), _lib.RL_XENC_IMAGE_QUANT

    def weight_bytes(self) -> int:
        """Device bytes this engine holds for its weights: images, embedding tables, biases and LayerNorms."""
        return sum(int(t.numel() * t.element_size()) for t in self._keep)

    def _packed(self, weight: torch.Tensor) -> torch.Tensor:
        W = weight.detach().to(device=self.device, dtype=torch.float32).contiguous()
        N, K = W.shape
        img = torch.empty(int(self.lib.rl_xenc_linear_image_bytes(N, K)), dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            check(self.lib.rl_xenc_pack_linear(W.data_ptr(), N, K, img.data_ptr(), _stream()), "rl_xenc_pack_linear")
            torch.cuda.current_stream().synchronize()
        self._keep.append(img)
        return img

    def _pipelined(self, lens: np.ndarray, launch: Any, collect: Any) -> None:
        """Cut the sequences into calls of at most ``max_tokens_per_call`` tokens and pipeline them: while the GPU runs
        call *i*, the host packs call *i+1* into the other half of a pinned double buffer and enqueues its upload and
        kernels; call *i* is only waited for (``collect(lo, hi, item)``) once the next call is in the queue.  A pinned
        half is refilled two calls later, after its call was collected.  ``launch(lo, hi, slot)`` returns ``item``."""
        P = len(lens)
        cuts = [0]
        tok = 0
        for i in range(P):
            if i > cuts[-1] and tok + lens[i] > self.max_tokens_per_call:
                cuts.append(i)
                tok = 0
            tok += int(lens[i])
        cuts.append(P)
        with self._lock, torch.cuda.device(self.device):
            pending: tuple[int, int, Any] | None = None
            for c in range(len(cuts) - 1):
                lo, hi = cuts[c], cuts[c + 1]
                if hi == lo:
                    continue
                item = launch(lo, hi, c & 1)
                if pending is not None:
                    collect(*pending)
                pending = (lo, hi, item)
            if pending is not None:
                collect(*pending)

    def _pinned(self, name: str, n: int, dtype: torch.dtype) -> torch.Tensor:
        buf = self._host_bufs.get(name)
        if buf is None or buf.numel() < n:
            buf = torch.empty(max(n, 1024), dtype=dtype, pin_memory=True)
            self._host_bufs[name] = buf
        return buf

    def _upload_packed(self, ids: Sequence[np.ndarray], type_ids: Sequence[np.ndarray] | None, lens: np.ndarray, *, slot: int
                       ) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
        """Pack one call into pinned buffer ``slot`` and enqueue its upload; returns the device ids, type ids, position
        ids and cu_seqlens, and makes sure the workspace holds the call.  Caller holds the lock."""
        P, T = len(ids), int(lens.sum())
        n_in = 3 * T + P + 1
        host_in = self._pinned(f"in{slot}", n_in, torch.int32)
        h = host_in.numpy()
        _pack_inputs(h, ids, type_ids, lens, self.pos_offset)
        # A tokenizer that does not match the weights would index past the embedding tables.
        w = self.weights
        if T and (int(h[:T].min()) < 0 or int(h[:T].max()) >= w.vocab):
            raise ValueError(f"token id outside the model's vocabulary [0, {w.vocab}) -- tokenizer / weights mismatch?")
        if T and (int(h[T:2 * T].min()) < 0 or int(h[T:2 * T].max()) >= w.type_vocab):
            raise ValueError(f"token type id outside [0, {w.type_vocab})")
        if P and int(lens.max()) + self.pos_offset > w.max_pos:
            raise ValueError(f"sequence longer than the model's {w.max_pos - self.pos_offset} positions")
        dev = self._dev_bufs.get(slot)
        if dev is None or dev.numel() < n_in:
            dev = torch.empty(max(n_in, 1024), dtype=torch.int32, device=self.device)
            self._dev_bufs[slot] = dev
        dev[:n_in].copy_(host_in[:n_in], non_blocking=True)
        need = int(self.lib.rl_xenc_workspace_bytes(C.byref(self.weights), T))
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        return dev[:T], dev[T:2 * T], dev[2 * T:3 * T], dev[3 * T:n_in]


# Tokens per forward call of CrossEncoderEngine.  The workspace takes T (12 H + 2 F) bytes: 2^18 tokens are 1.9 GB at
# MiniLM's shape (H = 384, F = 1536) but 4 GB at BERT-base's (H = 768, F = 3072) and 5.4 GB at XLM-R large's (H = 1024,
# F = 4096), so wider models take 2^16 (1.0 / 1.34 GB).
XENC_TOKENS_PER_CALL = 1 << 18
XENC_WIDE_TOKENS_PER_CALL = 1 << 16
# The families whose sequence classifiers load, and where their head lives in the state dict: (pooler dense, classifier)
# prefixes.  XLM-RoBERTa's classifier.dense -> tanh -> classifier.out_proj on the first token is BERT's pooler -> classifier.
_XENC_HEADS = {"bert": ("pooler.dense.", "classifier."), "xlm-roberta": ("classifier.dense.", "classifier.out_proj."),
               "roberta": ("classifier.dense.", "classifier.out_proj.")}
XENC_MAX_HIDDEN = 1024


def check_cross_encoder_shape(*, model_type: str, num_labels: int, hidden_act: str, hidden: int, n_heads: int) -> None:
    """Raise ``ValueError`` naming the limit when ``rl_xenc_score`` or the engine cannot run a model (no device work)."""
    if model_type not in _XENC_HEADS:
        raise ValueError(f"model_type={model_type!r} unsupported: the cross-encoder loads BERT or XLM-RoBERTa / RoBERTa "
                         "sequence classifiers")
    if num_labels not in (1, 2):
        raise ValueError(f"num_labels={num_labels} unsupported: the classification head computes 1 or 2 labels")
    if hidden_act != "gelu":
        raise ValueError(f"hidden_act={hidden_act!r} unsupported: the encoder's FFN computes GELU(erf) only")
    if n_heads <= 0 or hidden % n_heads or hidden // n_heads not in (32, 64):
        raise ValueError(f"hidden={hidden} heads={n_heads} unsupported: head_dim (hidden / heads) must be 32 or 64")
    if hidden % 32 or hidden > XENC_MAX_HIDDEN:
        raise ValueError(f"hidden={hidden} unsupported: hidden must be a multiple of 32 and at most {XENC_MAX_HIDDEN}")


class CrossEncoderEngine(_EncoderEngine):
    """Device-resident packed weights + tokenizer + batching for BERT and XLM-RoBERTa / RoBERTa sequence classifiers with
    one or two labels (head_dim 32 or 64, H <= 1024).  ``score_tokens`` returns logits ``[P]`` (one label) or ``[P, 2]``
    (two) and FlashRank's score ``[P]``: ``sigmoid(logit)``, or ``softmax(logits)[1]``."""

    def __init__(self, state_dict: dict[str, torch.Tensor], *, n_layers: int, hidden: int, n_heads: int, ffn: int,
                 max_pos: int, ln_eps: float = 1e-12, tokenizer: Any | None = None, max_length: int = 512,
                 device: Any | None = None, max_tokens_per_call: int | None = None, model_type: str = "bert",
                 pos_offset: int = 0, hidden_act: str = "gelu") -> None:
        head = _XENC_HEADS.get(model_type)
        cls_weight = state_dict.get(head[1] + "weight") if head else None
        n_labels = int(cls_weight.shape[0]) if cls_weight is not None and cls_weight.dim() == 2 else 1
        check_cross_encoder_shape(model_type=model_type, num_labels=n_labels, hidden_act=hidden_act, hidden=hidden,
                                  n_heads=n_heads)
        if cls_weight is None or tuple(cls_weight.shape[-1:]) != (hidden,):
            raise ValueError(f"no {head[1]}weight of shape [num_labels, {hidden}] in the state dict")
        # head_dim 32 at H <= 512 (MiniLM) keeps rl_xenc_score's own envelope: sequences up to the position table
        narrow = hidden <= 512 and hidden // n_heads == 32
        if max_tokens_per_call is None:
            max_tokens_per_call = XENC_TOKENS_PER_CALL if hidden <= 512 else XENC_WIDE_TOKENS_PER_CALL
        super().__init__(state_dict, n_layers=n_layers, hidden=hidden, n_heads=n_heads, ffn=ffn, max_pos=max_pos,
                         ln_eps=ln_eps, device=device, max_tokens_per_call=max_tokens_per_call, pos_offset=pos_offset)
        self.tokenizer = tokenizer
        self.model_type = model_type
        self.n_labels = n_labels
        self.max_length = min(max_length, max_pos - pos_offset) if narrow else min(max_length, max_pos - pos_offset, 512)
        w = self.weights
        pooler, classifier = head
        w.pooler_w, w.pooler_b = self._f32(pooler + "weight").data_ptr(), self._f32(pooler + "bias").data_ptr()
        w.cls_w, w.cls_b = self._f32(classifier + "weight").data_ptr(), self._f32(classifier + "bias").data_ptr()
        w.n_labels = n_labels

    # ---- constructors ------------------------------------------------------------------------------
    @classmethod
    def from_hf(cls, model: Any, tokenizer: Any | None = None, **kw: Any) -> "CrossEncoderEngine":
        """From a ``transformers`` ``BertForSequenceClassification`` or ``XLMRobertaForSequenceClassification`` /
        ``RobertaForSequenceClassification`` with one or two labels."""
        c = model.config
        check_cross_encoder_shape(model_type=c.model_type, num_labels=int(c.num_labels),
                                  hidden_act=getattr(c, "hidden_act", "gelu"), hidden=c.hidden_size,
                                  n_heads=c.num_attention_heads)
        return cls(model.state_dict(), n_layers=c.num_hidden_layers, hidden=c.hidden_size, n_heads=c.num_attention_heads,
                   ffn=c.intermediate_size, max_pos=c.max_position_embeddings, ln_eps=c.layer_norm_eps,
                   tokenizer=tokenizer, model_type=c.model_type, pos_offset=_position_offset(c),
                   hidden_act=getattr(c, "hidden_act", "gelu"), **kw)

    @classmethod
    def from_pretrained(cls, path: Path | str, **kw: Any) -> "CrossEncoderEngine":
        """Load HF weights + ``tokenizer.json`` from a local directory (no network access is attempted).  The class is
        chosen by ``config.json``'s ``model_type``: ``bert``, ``xlm-roberta`` or ``roberta``."""
        path = Path(path)
        if not (path / "config.json").exists():
            raise FileNotFoundError(f"No cross-encoder weights at {path} (expected an HF model directory)")
        from tokenizers import Tokenizer
        from transformers import (AutoConfig, BertForSequenceClassification, RobertaForSequenceClassification,
                                  XLMRobertaForSequenceClassification)

        config = AutoConfig.from_pretrained(path, local_files_only=True)
        check_cross_encoder_shape(model_type=config.model_type, num_labels=int(config.num_labels),
                                  hidden_act=getattr(config, "hidden_act", "gelu"), hidden=config.hidden_size,
                                  n_heads=config.num_attention_heads)
        model_cls = {"bert": BertForSequenceClassification, "xlm-roberta": XLMRobertaForSequenceClassification,
                     "roberta": RobertaForSequenceClassification}[config.model_type]
        model = model_cls.from_pretrained(path, config=config, local_files_only=True)
        tok = Tokenizer.from_file(str(path / "tokenizer.json")) if (path / "tokenizer.json").exists() else None
        return cls.from_hf(model, tok, **kw)

    # ---- scoring ---------------------------------------------------------------------------------------
    def score_tokens(self, ids: Sequence[np.ndarray], type_ids: Sequence[np.ndarray]) -> tuple[np.ndarray, np.ndarray]:
        """Logits (``[P]`` for one label, ``[P, 2]`` for two) and FlashRank's scores ``[P]`` for already-tokenised pairs
        (variable lengths, no padding).

        The pairs are cut into calls of at most ``max_tokens_per_call`` tokens.  Calls are pipelined: while
        the GPU runs call *i*, the host packs call *i+1* into the other half of a pinned double buffer and
        enqueues its upload and kernels; results come back through pinned memory and are only waited for
        once the next call is in the queue -- the host packing disappears behind the forward."""
        P, NL = len(ids), self.n_labels
        logits = np.empty((P, NL) if NL > 1 else P, np.float32)
        scores = np.empty(P, np.float32)
        lens = np.fromiter((len(x) for x in ids), dtype=np.int64, count=P)
        if P and lens.max() > self.max_length:
            raise ValueError(f"sequence longer than max_length={self.max_length}")

        def launch(lo: int, hi: int, slot: int) -> tuple[torch.Tensor, torch.cuda.Event]:
            return self._launch_packed(ids[lo:hi], type_ids[lo:hi], lens[lo:hi], slot=slot)

        def collect(lo: int, hi: int, item: tuple[torch.Tensor, torch.cuda.Event]) -> None:
            host, ev = item
            ev.synchronize()
            logits[lo:hi], scores[lo:hi] = self._split(host.numpy(), hi - lo)

        self._pipelined(lens, launch, collect)
        return logits, scores

    def _split(self, res: np.ndarray, P: int) -> tuple[np.ndarray, np.ndarray]:
        """The logits [P] / [P, 2] and scores [P] of one call's result buffer (logits [P, n_labels] | scores [P])."""
        NL = self.n_labels
        lg = res[: NL * P]
        return (lg.reshape(P, NL) if NL > 1 else lg), res[NL * P:(NL + 1) * P]

    def _launch_packed(self, ids: Sequence[np.ndarray], type_ids: Sequence[np.ndarray], lens: np.ndarray, *, slot: int
                       ) -> tuple[torch.Tensor, torch.cuda.Event]:
        """Pack one call into pinned buffer ``slot``, enqueue upload + forward + download; returns the pinned
        result buffer (logits [P, n_labels] then scores [P]) and the event that marks it complete.  Caller holds the
        lock."""
        P, n_out = len(ids), (self.n_labels + 1) * len(ids)
        d_ids, d_types, d_pos, d_cu = self._upload_packed(ids, type_ids, lens, slot=slot)
        out = torch.empty(n_out, dtype=torch.float32, device=self.device)
        check(self.lib.rl_xenc_score(C.byref(self.weights), d_ids.data_ptr(), d_types.data_ptr(), d_pos.data_ptr(),
                                     d_cu.data_ptr(), P, len(d_ids), int(lens.max()), out.data_ptr(),
                                     out[self.n_labels * P:].data_ptr(), self._ws.data_ptr(), self._ws.numel(), _stream()),
              "rl_xenc_score")
        host_out = self._pinned(f"out{slot}", n_out, torch.float32)
        host_out[:n_out].copy_(out, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        return host_out, ev

    def _score_packed(self, ids: Sequence[np.ndarray], type_ids: Sequence[np.ndarray], lens: np.ndarray
                      ) -> tuple[np.ndarray, np.ndarray]:
        """One synchronous call (kept for callers that time a single forward)."""
        with self._lock, torch.cuda.device(self.device):
            host, ev = self._launch_packed(ids, type_ids, np.asarray(lens, dtype=np.int64), slot=0)
            ev.synchronize()
            logits, scores = self._split(host.numpy(), len(ids))
        return logits.copy(), scores.copy()

    def encode_pairs(self, queries: Sequence[str], docs: Sequence[str]) -> tuple[list[np.ndarray], list[np.ndarray]]:
        """[CLS] query [SEP] passage [SEP] with truncation to ``max_length`` (FlashRank's tokenizer setup)."""
        if self.tokenizer is None:
            raise ValueError("this engine was built without a tokenizer; use score_tokens")
        self.tokenizer.enable_truncation(max_length=self.max_length)
        self.tokenizer.no_padding()
        enc = self.tokenizer.encode_batch(list(zip(queries, docs, strict=True)))
        return [np.asarray(e.ids, np.int32) for e in enc], [np.asarray(e.type_ids, np.int32) for e in enc]

    def score_pairs(self, queries: Sequence[str], docs: Sequence[str]) -> list[float]:
        ids, types = self.encode_pairs(queries, docs)
        return [float(s) for s in self.score_tokens(ids, types)[1]]


# ---- token embedder (late-chunking ingest, string queries) -------------------------------------------------------------
# Tokens per forward call of TokenEmbedderEngine: 65,536 tokens take about 1.34 GB of workspace and 0.27 GB of fp32
# output at bge-m3's shape (H = 1024, FFN = 4096: ~20 KB of workspace per token); the cross-encoder's 2^18 would take
# 5.4 GB + 1.1 GB.  A call of 2^16 tokens is already ~130 tokens per SM per linear layer pass.
EMBED_TOKENS_PER_CALL = 1 << 16


class EmbedderTokenizer:
    """The llama-like tokenizer side of ``TokenEmbedderEngine`` (host only): ``n_ctx() / n_batch / tokenize /
    detokenize`` as ``raglite_b200._embed`` calls them, over a ``tokenizers.Tokenizer`` (or a transformers fast
    tokenizer, whose backend is used).  ``token_ids_for_embedding`` adds the tokenizer's special tokens
    (``<s> ... </s>`` / ``[CLS] ... [SEP]``) and truncates to ``n_batch`` tokens, as llama-cpp-python's
    ``embed(truncate=True)`` does."""

    def __init__(self, tokenizer: Any, n_ctx: int) -> None:
        from tokenizers import Tokenizer

        tok = getattr(tokenizer, "backend_tokenizer", tokenizer)
        self.tokenizer = Tokenizer.from_str(tok.to_str())   # a private copy: truncation / padding are turned off here
        self.tokenizer.no_truncation()
        self.tokenizer.no_padding()
        self._n_ctx = int(n_ctx)
        self.n_batch = int(n_ctx)

    def n_ctx(self) -> int:
        return self._n_ctx

    def tokenize(self, text: bytes, add_bos: bool = False, special: bool = False) -> list[int]:  # noqa: ARG002
        """Token ids of ``text`` without special tokens (``add_bos`` / ``special`` only mirror llama.cpp's signature)."""
        return list(self.tokenizer.encode(text.decode(), add_special_tokens=False).ids)

    def detokenize(self, tokens: Sequence[int]) -> bytes:
        return self.tokenizer.decode([int(t) for t in tokens], skip_special_tokens=False).encode()

    def token_ids_for_embedding(self, texts: Sequence[str]) -> list[np.ndarray]:
        enc = self.tokenizer.encode_batch(list(texts), add_special_tokens=True)
        return [np.asarray(e.ids[: self.n_batch], dtype=np.int32) for e in enc]


def _position_offset(config: Any) -> int:
    """First position id of a sequence: XLM-RoBERTa counts from ``padding_idx + 1`` (its table keeps rows for the
    padding index and below), BERT from 0."""
    if config.model_type in ("xlm-roberta", "roberta"):
        return int(config.pad_token_id) + 1
    if config.model_type == "bert":
        return 0
    raise ValueError(f"unsupported encoder model type {config.model_type!r} (BERT or XLM-RoBERTa)")


class TokenEmbedderEngine(_EncoderEngine):
    """Per-token embeddings of a BERT / XLM-RoBERTa encoder (bge-m3: XLM-RoBERTa, 24 layers, H = 1024, 16 heads x 64,
    FFN 4096) on the GPU: the forward runs in ``rl_xenc_encode`` and returns the last layer's LayerNorm output of every
    token in float32.  It implements the llama-like protocol of ``raglite_b200._embed`` (``n_ctx() / n_batch /
    n_embd() / tokenize / detokenize / embed``) plus ``embed_token_ids``, a packed forward whose output stays on the
    device, which ``embed_strings`` uses to pool without a host round trip.  Register it with
    ``register_token_embedder(config.embedder, TokenEmbedderEngine.from_pretrained(local_dir))``."""

    def __init__(self, state_dict: dict[str, torch.Tensor], *, n_layers: int, hidden: int, n_heads: int, ffn: int,
                 max_pos: int, ln_eps: float = 1e-5, pos_offset: int = 0, tokenizer: Any | None = None, n_ctx: int = 512,
                 device: Any | None = None, max_tokens_per_call: int = EMBED_TOKENS_PER_CALL) -> None:
        super().__init__(state_dict, n_layers=n_layers, hidden=hidden, n_heads=n_heads, ffn=ffn, max_pos=max_pos,
                         ln_eps=ln_eps, device=device, max_tokens_per_call=max_tokens_per_call, pos_offset=pos_offset)
        n_ctx = min(int(n_ctx), max_pos - pos_offset, 512)
        self.tok = EmbedderTokenizer(tokenizer, n_ctx) if tokenizer is not None else None
        self._n_ctx = n_ctx
        self.n_batch = n_ctx

    # ---- constructors ------------------------------------------------------------------------------
    @classmethod
    def from_hf(cls, model: Any, tokenizer: Any | None = None, **kw: Any) -> "TokenEmbedderEngine":
        """From a ``transformers`` ``XLMRobertaModel`` or ``BertModel`` (or a model that wraps one under
        ``roberta.`` / ``bert.``) and its tokenizer."""
        c = model.config
        if getattr(c, "hidden_act", "gelu") != "gelu":
            raise ValueError(f"hidden_act={c.hidden_act!r}: the encoder's FFN computes GELU(erf) only")
        return cls(model.state_dict(), n_layers=c.num_hidden_layers, hidden=c.hidden_size, n_heads=c.num_attention_heads,
                   ffn=c.intermediate_size, max_pos=c.max_position_embeddings, ln_eps=c.layer_norm_eps,
                   pos_offset=_position_offset(c), tokenizer=tokenizer, **kw)

    @classmethod
    def from_pretrained(cls, path: Path | str, n_ctx: int = 512, **kw: Any) -> "TokenEmbedderEngine":
        """Load HF weights + ``tokenizer.json`` from a local directory (e.g. ``BAAI/bge-m3``); no network access is
        attempted."""
        path = Path(path)
        if not (path / "config.json").exists():
            raise FileNotFoundError(f"No embedder weights at {path} (expected an HF model directory)")
        from tokenizers import Tokenizer
        from transformers import AutoModel

        model = AutoModel.from_pretrained(path, local_files_only=True)
        if not (path / "tokenizer.json").exists():
            raise FileNotFoundError(f"No tokenizer.json in {path}")
        return cls.from_hf(model, Tokenizer.from_file(str(path / "tokenizer.json")), n_ctx=n_ctx, **kw)

    @classmethod
    def from_gguf(cls, path: Path | str, n_ctx: int = 512, tokenizer: Any | None = None, **kw: Any) -> "TokenEmbedderEngine":
        """Load a llama.cpp GGUF file of a BERT / XLM-RoBERTa embedder (``general.architecture == "bert"``, e.g.
        lm-kit/bge-m3-gguf) with F32 / F16 / Q8_0 / Q4_K / Q6_K weights.  Quantized linears stay quantized on the device
        and are expanded inside the linear kernel; embedding tables are dequantized to fp16 once.  The tokenizer is rebuilt
        from the file's SentencePiece Unigram metadata unless ``tokenizer`` (a ``tokenizers.Tokenizer``, or the path of a
        ``tokenizer.json``) is given.  ``n_ctx`` 0 means the file's context length; it is capped at 512.  Every check
        that can fail raises ``ValueError`` before any device work."""
        from ._gguf import GGUFFile, bert_plan, gguf_tokenizer

        f = GGUFFile(path)
        plan = bert_plan(f)
        if tokenizer is None:
            tokenizer = gguf_tokenizer(f)
        elif isinstance(tokenizer, (str, Path)):
            from tokenizers import Tokenizer

            tokenizer = Tokenizer.from_file(str(tokenizer))
        # 1-D tensors (biases, norms) as float32; 2-D weights stay GGUF tensors for _image / _f16.
        sd = {k: (torch.from_numpy(tensor_to_f32(t)) if len(t.shape) == 1 else t) for k, t in plan.state_dict.items()}
        max_pos = sd["embeddings.position_embeddings.weight"].shape[0]
        # the converter drops XLM-RoBERTa's first pad_token_id + 1 position rows: positions count from 0 here
        return cls(sd, n_layers=plan.n_layers, hidden=plan.hidden, n_heads=plan.n_heads, ffn=plan.ffn, max_pos=max_pos,
                   ln_eps=plan.ln_eps, pos_offset=0, tokenizer=tokenizer,
                   n_ctx=int(n_ctx) if n_ctx else plan.context_length, **kw)

    @classmethod
    def from_embedder_string(cls, embedder: str, hub_cache: Path | str | None = None, **kw: Any) -> "TokenEmbedderEngine":
        """The engine behind a RAGLite ``config.embedder`` such as ``llama-cpp-python/lm-kit/bge-m3-gguf/*F16.gguf@512``:
        the one GGUF file in the Hugging Face hub cache that matches it (``HF_HUB_CACHE``, else ``HF_HOME/hub``, else
        ``~/.cache/huggingface/hub``).  Nothing is downloaded."""
        from ._gguf import find_cached_gguf, parse_embedder

        repo_id, filename, n_ctx = parse_embedder(embedder)
        return cls.from_gguf(find_cached_gguf(repo_id, filename, hub_cache), n_ctx=n_ctx, **kw)

    # ---- llama-like protocol -----------------------------------------------------------------------
    def _tokenizer(self) -> EmbedderTokenizer:
        if self.tok is None:
            raise ValueError("this engine was built without a tokenizer; use embed_token_ids")
        return self.tok

    def n_ctx(self) -> int:
        return self._n_ctx

    def n_embd(self) -> int:
        return self.hidden

    def tokenize(self, text: bytes, add_bos: bool = False, special: bool = False) -> list[int]:
        return self._tokenizer().tokenize(text, add_bos=add_bos, special=special)

    def detokenize(self, tokens: Sequence[int]) -> bytes:
        return self._tokenizer().detokenize(tokens)

    def token_ids_for_embedding(self, texts: Sequence[str]) -> list[np.ndarray]:
        return self._tokenizer().token_ids_for_embedding(texts)

    def embed(self, text: str | Sequence[str]) -> np.ndarray | list[np.ndarray]:
        """float32 ``[tokens, H]`` per text, special tokens included, truncated to ``n_batch`` tokens."""
        texts = [text] if isinstance(text, str) else list(text)
        X, offs = self.embed_token_ids(self.token_ids_for_embedding(texts))
        host = X.cpu().numpy()
        rows = [host[offs[i]:offs[i + 1]] for i in range(len(texts))]
        return rows[0] if isinstance(text, str) else rows

    # ---- device path -------------------------------------------------------------------------------
    def embed_token_ids(self, ids: Sequence[np.ndarray]) -> tuple[torch.Tensor, np.ndarray]:
        """One packed forward over token-id sequences (1 to ``n_ctx`` tokens each), in calls of at most
        ``max_tokens_per_call`` tokens: float32 hidden states ``[T_total, H]`` on the device and the row offsets
        ``[P + 1]`` of the sequences in it."""
        P = len(ids)
        lens = np.fromiter((len(x) for x in ids), dtype=np.int64, count=P)
        if P and (lens.min() < 1 or lens.max() > self._n_ctx):
            raise ValueError(f"every sequence needs 1 to {self._n_ctx} tokens")
        offs = np.zeros(P + 1, dtype=np.int64)
        np.cumsum(lens, out=offs[1:])
        out = torch.empty((int(offs[-1]), self.hidden), dtype=torch.float32, device=self.device)

        def launch(lo: int, hi: int, slot: int) -> torch.cuda.Event:
            d_ids, d_types, d_pos, d_cu = self._upload_packed(ids[lo:hi], None, lens[lo:hi], slot=slot)
            check(self.lib.rl_xenc_encode(C.byref(self.weights), d_ids.data_ptr(), d_types.data_ptr(), d_pos.data_ptr(),
                                          d_cu.data_ptr(), hi - lo, len(d_ids), int(lens[lo:hi].max()),
                                          out[int(offs[lo]):].data_ptr(), self._ws.data_ptr(), self._ws.numel(), _stream()),
                  "rl_xenc_encode")
            ev = torch.cuda.Event()
            ev.record()
            return ev

        def collect(lo: int, hi: int, ev: torch.cuda.Event) -> None:   # noqa: ARG001  (the pinned half is free again)
            ev.synchronize()

        self._pipelined(lens, launch, collect)
        return out, offs
