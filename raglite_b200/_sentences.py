"""Sentence splitting on the GPU -- ``split_sentences`` as ``raglite/_split_sentences.py`` computes it.

The reference asks a SaT model (``sat-1l-sm``: a one-layer XLM-RoBERTa token classifier, run by wtpsplit-lite) for one
boundary probability per character, overrides it with the known probabilities of the document's Markdown headings,
propagates it over whitespace runs and solves a dynamic program for the sentence partition (``:146-219``).  Here:

* the host tokenizes every document of a batch at once, plans the overlapping 256-token blocks and decides which
  character each token writes (this module; the rules are the constants and functions below, in one place);
* ``SaTEngine`` runs the blocks through the encoder (``rl_xenc_encode``, packed and pipelined) and the classification
  head (``rl_sat_token_logits``) without the hidden states leaving the device;
* ``rl_sat_char_probas`` stitches the blocks, maps tokens to characters, applies the sigmoid, the override and the
  whitespace propagation; ``rl_sentence_partition`` runs both stages of the reference's dynamic program, one thread per
  document, bit for bit.

What wtpsplit's ``predict_proba`` does is recalled, not pinned against wtpsplit (DESIGN.md section 5):
``SAT_BLOCK_SIZE`` / ``SAT_STRIDE``, ``block_starts``, ``hat_weights``, ``SAT_SKIP_PIECES`` / ``token_char_targets`` and
the float32 sigmoid.  An integrator who can run wtpsplit-lite corrects them here.
"""

from __future__ import annotations

import ctypes as C
import json
from collections.abc import Callable, Sequence
from pathlib import Path
from typing import Any

import numpy as np
import torch

from ._lib import check
from ._xenc import XENC_MAX_HIDDEN, XENC_WIDE_TOKENS_PER_CALL, _EncoderEngine, _stream

# ---- what wtpsplit's predict_proba(doc, stride=128, block_size=256, weighting="hat") does (recalled) ------------------
SAT_BLOCK_SIZE = 256      # counts <s> and </s>: a block holds min(254, T) document tokens
SAT_STRIDE = 128
SAT_SKIP_PIECES = ("<s>", "</s>", "<pad>", "▁")   # tokens that write no character
SAT_MAX_LABELS = 16       # rl_sat_token_logits / rl_sat_char_probas
# Characters per device group: the probabilities, the partition's scratch and the planning arrays take about 40 bytes
# per character, so a group of 2^25 characters stays near 1.3 GB whatever the batch.
SAT_GROUP_CHARS = 1 << 25
PARTITION_FAILED = "Sentence partition failed: no valid split satisfies the constraints."


def hat_weights(B: int) -> np.ndarray:
    """Weight of in-block position k of a block of B tokens: 1 - |x_k|, x = linspace(-(1 - 1/B), 1 - 1/B, B)."""
    x = np.linspace(-(1 - 1 / B), 1 - 1 / B, B)
    return (1 - np.abs(x)).astype(np.float32)


def hat_table(max_block: int = SAT_BLOCK_SIZE - 2) -> np.ndarray:
    """``hat_weights(B)`` for B = 1 .. max_block, the one for B at offset B (B - 1) / 2 (``rl_sat_char_probas``)."""
    return np.concatenate([hat_weights(B) for B in range(1, max_block + 1)])


def block_starts(T: int, block_size: int = SAT_BLOCK_SIZE, stride: int = SAT_STRIDE) -> tuple[int, np.ndarray]:
    """(B, document-relative token starts) of one document of T tokens: blocks at 0, stride, 2 stride, ...; the first
    one whose end reaches T is moved back to end at T and is the last.  No blocks when T = 0."""
    if T == 0:
        return 0, np.zeros(0, np.int32)
    B = min(block_size - 2, T)
    n_reg = -(-(T - B) // stride)
    return B, np.r_[np.arange(n_reg, dtype=np.int64) * stride, T - B].astype(np.int32)


def plan_blocks(T: np.ndarray, block_size: int = SAT_BLOCK_SIZE, stride: int = SAT_STRIDE
                ) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """``block_starts`` for a whole batch at once: per-document B [D], block offsets [D + 1] and the concatenated
    document-relative starts."""
    T = np.asarray(T, dtype=np.int64)
    B = np.minimum(block_size - 2, T)
    n_blk = np.where(T > 0, -(-(T - B) // stride) + 1, 0)
    off = np.zeros(len(T) + 1, np.int64)
    np.cumsum(n_blk, out=off[1:])
    start = (np.arange(off[-1], dtype=np.int64) - np.repeat(off[:-1], n_blk)) * stride
    last = off[1:][n_blk > 0] - 1
    start[last] = (T - B)[n_blk > 0]
    return B.astype(np.int32), off, start.astype(np.int32)


def token_char_targets(ends: np.ndarray, skip: np.ndarray, n_chars: int) -> np.ndarray:
    """The character each token of one document writes its label-0 logit to: ``end - 1`` (as a NumPy index, so -1 is
    the last character), -1 (none) for a skipped token and for every token whose character a later token writes too."""
    tgt = np.asarray(ends, dtype=np.int64) - 1
    tgt = np.where(tgt < 0, tgt + n_chars, tgt)
    tgt[np.asarray(skip, dtype=bool)] = -1
    keep = np.full(len(tgt), -1, np.int64)
    rev = tgt[::-1]
    _, first = np.unique(rev, return_index=True)          # the last writer of each character
    idx = len(tgt) - 1 - first
    keep[idx] = tgt[idx]
    return np.where(keep >= 0, keep, -1)


# ---- code points and whitespace ----------------------------------------------------------------------------------------
_SPACE_CODEPOINTS = np.array([c for c in range(0x3001) if chr(c).isspace()], dtype=np.uint32)   # none above U+3000


def code_points(text: str) -> np.ndarray:
    return np.frombuffer(text.encode("utf-32-le", errors="surrogatepass"), dtype=np.uint32)


def whitespace_flags(text: str) -> np.ndarray:
    """``str.isspace`` of every character, from the code points."""
    return np.isin(code_points(text), _SPACE_CODEPOINTS)


def markdown_sentence_boundaries(doc: str, tokens: list[Any] | None = None) -> np.ndarray:
    """Known boundary probabilities from the Markdown headings (``_split_sentences.py:23-53``): for each heading the
    character before it gets 1, its body 0 and its last character 1 (its line span, counted over ``str.splitlines``);
    NaN elsewhere.  ``tokens`` is markdown-it's parse of ``doc`` when the caller already has it."""
    from markdown_it import MarkdownIt

    out = np.full(len(doc), np.nan)
    spans = [t.map for t in (MarkdownIt().parse(doc) if tokens is None else tokens) if t.type == "heading_open"]
    if not spans:
        return out
    line_start = np.zeros(1, np.int64)
    line_start = np.r_[line_start, np.cumsum([len(x) for x in doc.splitlines(keepends=True)], dtype=np.int64)]
    n = len(doc)
    for first_line, last_line in spans:
        a, e = int(line_start[first_line]), int(line_start[last_line]) + 1
        if 0 <= a - 1 < n:
            out[a - 1] = 1
        out[a:e - 1] = 0
        if 0 <= e - 1 < n:
            out[e - 1] = 1
    return out


# ---- the engine --------------------------------------------------------------------------------------------------------
def check_sat_shape(*, lookahead: Any, hidden_act: str, hidden: int, n_heads: int) -> None:
    """Raise ``ValueError`` naming the limit when the engine cannot run a SaT model (no device work)."""
    if lookahead is not None:
        raise ValueError(f"lookahead={lookahead!r} unsupported: a limited lookahead changes the attention mask, and the "
                         "encoder attends over the whole block")
    if hidden_act != "gelu":
        raise ValueError(f"hidden_act={hidden_act!r} unsupported: the encoder's FFN computes GELU(erf) only")
    if n_heads <= 0 or hidden % n_heads or hidden // n_heads not in (32, 64):
        raise ValueError(f"hidden={hidden} heads={n_heads} unsupported: head_dim (hidden / heads) must be 32 or 64")
    if hidden % 32 or hidden > XENC_MAX_HIDDEN:
        raise ValueError(f"hidden={hidden} unsupported: hidden must be a multiple of 32 and at most {XENC_MAX_HIDDEN}")


def _check_head(state_dict: dict[str, Any], hidden: int) -> int:
    w, b = state_dict.get("classifier.weight"), state_dict.get("classifier.bias")
    if w is None or b is None or w.dim() != 2 or int(w.shape[1]) != hidden or tuple(b.shape) != (int(w.shape[0]),):
        raise ValueError(f"no token-classification head: expected classifier.weight [num_labels, {hidden}] and "
                         "classifier.bias [num_labels] in the state dict")
    n = int(w.shape[0])
    if not 1 <= n <= SAT_MAX_LABELS:
        raise ValueError(f"num_labels={n} unsupported: the head computes 1 to {SAT_MAX_LABELS} labels")
    return n


def read_sat_config(path: Path | str) -> dict[str, Any]:
    """``config.json`` of a SaT model directory, read as JSON (its ``model_type`` is wtpsplit's ``"xlm-token"``, which
    ``AutoConfig`` does not know), checked by ``check_sat_shape``; returns the engine's keyword arguments."""
    c = json.loads(Path(path, "config.json").read_text())
    hidden, n_heads = int(c["hidden_size"]), int(c["num_attention_heads"])
    check_sat_shape(lookahead=c.get("lookahead"), hidden_act=c.get("hidden_act", "gelu"), hidden=hidden, n_heads=n_heads)
    return dict(n_layers=int(c["num_hidden_layers"]), hidden=hidden, n_heads=n_heads, ffn=int(c["intermediate_size"]),
                max_pos=int(c["max_position_embeddings"]), ln_eps=float(c.get("layer_norm_eps", 1e-5)),
                pos_offset=int(c.get("pad_token_id", 1)) + 1)


class SaTEngine(_EncoderEngine):
    """A SaT token classifier (XLM-RoBERTa encoder + ``classifier`` head, head_dim 32 or 64, H <= 1024, GELU) on the
    GPU with its tokenizer: ``boundary_probas`` is wtpsplit's ``predict_proba(doc, stride=128, block_size=256,
    weighting="hat")`` and ``split`` the reference's whole ``split_sentences`` for a batch of documents.  Register it
    with ``register_sentence_splitter(SaTEngine.from_pretrained(local_dir))``."""

    def __init__(self, state_dict: dict[str, torch.Tensor], *, n_layers: int, hidden: int, n_heads: int, ffn: int,
                 max_pos: int, tokenizer: Any, ln_eps: float = 1e-5, pos_offset: int = 2, hidden_act: str = "gelu",
                 lookahead: Any = None, device: Any | None = None,
                 max_tokens_per_call: int = XENC_WIDE_TOKENS_PER_CALL, group_chars: int = SAT_GROUP_CHARS) -> None:
        check_sat_shape(lookahead=lookahead, hidden_act=hidden_act, hidden=hidden, n_heads=n_heads)
        sd = {k.removeprefix("roberta."): v for k, v in state_dict.items()}
        n_labels = _check_head(sd, hidden)
        if max_pos - pos_offset < SAT_BLOCK_SIZE:
            raise ValueError(f"max_position_embeddings={max_pos} holds fewer than {SAT_BLOCK_SIZE} positions")
        super().__init__(sd, n_layers=n_layers, hidden=hidden, n_heads=n_heads, ffn=ffn, max_pos=max_pos, ln_eps=ln_eps,
                         device=device, max_tokens_per_call=max_tokens_per_call, pos_offset=pos_offset)
        from tokenizers import Tokenizer

        tok = getattr(tokenizer, "backend_tokenizer", tokenizer)
        self.tokenizer = Tokenizer.from_str(tok.to_str())    # a private copy with truncation and padding off
        self.tokenizer.no_truncation()
        self.tokenizer.no_padding()
        self.bos_id, self.eos_id = self.tokenizer.token_to_id("<s>"), self.tokenizer.token_to_id("</s>")
        if self.bos_id is None or self.eos_id is None:
            raise ValueError("the tokenizer has no <s> / </s> (SaT takes XLM-RoBERTa's tokenizer)")
        self._skip_ids = np.array(sorted({i for i in (self.tokenizer.token_to_id(p) for p in SAT_SKIP_PIECES)
                                          if i is not None}), dtype=np.int64)
        self.n_labels = n_labels
        self.group_chars = group_chars
        self._cls_w, self._cls_b = self._f32("classifier.weight"), self._f32("classifier.bias")
        self._hat = torch.from_numpy(hat_table()).to(self.device)
        self._hid: torch.Tensor | None = None

    @classmethod
    def from_hf(cls, model: Any, tokenizer: Any, **kw: Any) -> "SaTEngine":
        """From a ``transformers`` ``XLMRobertaForTokenClassification`` and its tokenizer (tests and benchmarks)."""
        c = model.config
        return cls(model.state_dict(), n_layers=c.num_hidden_layers, hidden=c.hidden_size, n_heads=c.num_attention_heads,
                   ffn=c.intermediate_size, max_pos=c.max_position_embeddings, ln_eps=c.layer_norm_eps,
                   pos_offset=int(c.pad_token_id) + 1, hidden_act=getattr(c, "hidden_act", "gelu"),
                   lookahead=getattr(c, "lookahead", None), tokenizer=tokenizer, **kw)

    @classmethod
    def from_pretrained(cls, path: Path | str, **kw: Any) -> "SaTEngine":
        """Load ``config.json``, ``model.safetensors`` (``roberta.*`` + ``classifier.weight`` / ``classifier.bias``) and
        ``tokenizer.json`` (xlm-roberta-base's) from a local directory; nothing is downloaded."""
        path = Path(path)
        if not (path / "config.json").exists():
            raise FileNotFoundError(f"No SaT model at {path} (expected config.json, model.safetensors, tokenizer.json)")
        shape = read_sat_config(path)
        from safetensors.torch import load_file
        from tokenizers import Tokenizer

        sd = load_file(str(path / "model.safetensors"))
        _check_head({k.removeprefix("roberta."): v for k, v in sd.items()}, shape["hidden"])
        if not (path / "tokenizer.json").exists():
            raise FileNotFoundError(f"No tokenizer.json in {path} (copy xlm-roberta-base's)")
        return cls(sd, tokenizer=Tokenizer.from_file(str(path / "tokenizer.json")), **shape, **kw)

    # ---- planning ----------------------------------------------------------------------------------------------------
    def _plan(self, docs: Sequence[str]) -> dict[str, np.ndarray]:
        """Tokens, blocks, block rows and character targets of one group of documents."""
        enc = self.tokenizer.encode_batch(list(docs), add_special_tokens=False)
        D = len(docs)
        n_chars = np.fromiter((len(d) for d in docs), dtype=np.int64, count=D)
        char_off = np.zeros(D + 1, np.int64)
        np.cumsum(n_chars, out=char_off[1:])
        ids = [np.asarray(e.ids, dtype=np.int64) for e in enc]
        T = np.fromiter((len(x) for x in ids), dtype=np.int64, count=D)
        tok_off = np.zeros(D + 1, np.int64)
        np.cumsum(T, out=tok_off[1:])
        flat = np.concatenate(ids) if tok_off[-1] else np.zeros(0, np.int64)
        targets = [np.zeros(0, np.int64)]
        for d, (e, x) in enumerate(zip(enc, ids, strict=True)):
            t = token_char_targets(np.asarray(e.offsets, dtype=np.int64).reshape(-1, 2)[:, 1], np.isin(x, self._skip_ids),
                                   int(n_chars[d]))
            targets.append(np.where(t >= 0, t + char_off[d], -1))
        tok_char = np.concatenate(targets)
        B, blk_off, blk_start = plan_blocks(T)
        blk_doc = np.repeat(np.arange(D), np.diff(blk_off))
        blk_B = B[blk_doc].astype(np.int64)
        seq_len = blk_B + 2                                          # <s> tokens </s>
        row_off = np.zeros(len(seq_len) + 1, np.int64)
        np.cumsum(seq_len, out=row_off[1:])
        rows = np.full(int(row_off[-1]), self.eos_id, np.int32)
        rows[row_off[:-1]] = self.bos_id
        inner = int(blk_B.sum())
        within = np.arange(inner, dtype=np.int64) - np.repeat(np.cumsum(blk_B) - blk_B, blk_B)
        rows[np.repeat(row_off[:-1] + 1, blk_B) + within] = flat[np.repeat(tok_off[blk_doc] + blk_start, blk_B) + within]
        return dict(char_off=char_off, tok_off=tok_off, tok_char=tok_char, B=B, blk_off=blk_off, blk_start=blk_start,
                    blk_row=row_off[:-1] + 1, seq_len=seq_len, row_off=row_off, rows=rows)

    # ---- device path ------------------------------------------------------------------------------------------------
    def _char_probas(self, docs: Sequence[str], known: np.ndarray | None, propagate: bool) -> tuple[torch.Tensor, np.ndarray]:
        """float32 probabilities of every character of one group on the device, and the character offsets [D + 1].
        ``known`` (float32, NaN = none, one per character) overrides them and ``propagate`` runs the whitespace step.
        Caller holds the lock."""
        p = self._plan(docs)
        dev = self.device
        NL, R = self.n_labels, int(p["row_off"][-1])
        logits = torch.empty((max(R, 1), NL), dtype=torch.float32, device=dev)
        seqs = np.split(p["rows"], p["row_off"][1:-1]) if R else []
        if R:
            need = min(R, self.max_tokens_per_call + SAT_BLOCK_SIZE)
            if self._hid is None or self._hid.shape[0] < need:
                self._hid = torch.empty((need, self.hidden), dtype=torch.float32, device=dev)
            row_off = p["row_off"]

            def launch(lo: int, hi: int, slot: int) -> torch.cuda.Event:
                d_ids, d_types, d_pos, d_cu = self._upload_packed(seqs[lo:hi], None, p["seq_len"][lo:hi], slot=slot)
                n = int(row_off[hi] - row_off[lo])
                check(self.lib.rl_xenc_encode(C.byref(self.weights), d_ids.data_ptr(), d_types.data_ptr(),
                                              d_pos.data_ptr(), d_cu.data_ptr(), hi - lo, n,
                                              int(p["seq_len"][lo:hi].max()), self._hid.data_ptr(), self._ws.data_ptr(),
                                              self._ws.numel(), _stream()), "rl_xenc_encode")
                check(self.lib.rl_sat_token_logits(self._hid.data_ptr(), n, self.hidden, self._cls_w.data_ptr(),
                                                   self._cls_b.data_ptr(), NL, logits[int(row_off[lo]):].data_ptr(),
                                                   _stream()), "rl_sat_token_logits")
                ev = torch.cuda.Event()
                ev.record()
                return ev

            def collect(lo: int, hi: int, ev: torch.cuda.Event) -> None:   # noqa: ARG001  (the pinned half is free again)
                ev.synchronize()

            self._pipelined(p["seq_len"], launch, collect)

        def up(a: np.ndarray) -> torch.Tensor:
            return torch.from_numpy(np.ascontiguousarray(a)).to(dev)

        D, N, T = len(docs), int(p["char_off"][-1]), int(p["tok_off"][-1])
        out = torch.empty(max(N, 1), dtype=torch.float32, device=dev)
        ws = torch.empty(int(self.lib.rl_sat_workspace_bytes(T, D, NL)), dtype=torch.uint8, device=dev)
        args = [up(p["tok_off"]), up(p["char_off"]), up(p["B"]), up(p["blk_off"]), up(p["blk_start"]), up(p["blk_row"]),
                up(p["tok_char"])]
        d_known = up(known) if known is not None else None
        d_space = up(whitespace_flags("".join(docs)).view(np.uint8)) if propagate else None
        check(self.lib.rl_sat_char_probas(logits.data_ptr(), NL, args[0].data_ptr(), args[1].data_ptr(), args[2].data_ptr(),
                                          D, T, N, args[3].data_ptr(), args[4].data_ptr(), args[5].data_ptr(),
                                          self._hat.data_ptr(), args[6].data_ptr(),
                                          d_known.data_ptr() if d_known is not None else None,
                                          d_space.data_ptr() if d_space is not None else None, out.data_ptr(),
                                          ws.data_ptr(), ws.numel(), _stream()), "rl_sat_char_probas")
        return out, p["char_off"]

    def _groups(self, docs: Sequence[str]) -> list[tuple[int, int]]:
        cuts, chars = [0], 0
        for i, d in enumerate(docs):
            if i > cuts[-1] and chars + len(d) > self.group_chars:
                cuts.append(i)
                chars = 0
            chars += len(d)
        cuts.append(len(docs))
        return [(a, b) for a, b in zip(cuts[:-1], cuts[1:], strict=True) if b > a]

    def boundary_probas(self, docs: Sequence[str]) -> list[np.ndarray]:
        """wtpsplit's ``predict_proba`` of every document: float32, one per character (0 for a document without
        tokens)."""
        res: list[np.ndarray] = []
        for a, b in self._groups(docs):
            with self._lock, torch.cuda.device(self.device):
                out, off = self._char_probas(docs[a:b], None, False)
                host = out.cpu().numpy()
            res.extend(host[off[i]:off[i + 1]].copy() for i in range(b - a))
        return res

    def split(self, docs: Sequence[str], known: Sequence[np.ndarray], *, min_len: int, max_len: int | None
              ) -> list[list[str]]:
        """The reference's ``split_sentences`` past its early exit for every document (each longer than ``min_len``),
        with ``known[i]`` the known probabilities of document i (float, NaN = none): one forward and one partition
        launch per group.  Raises the reference's ``ValueError`` when a document cannot be partitioned."""
        res: list[list[str]] = []
        for a, b in self._groups(docs):
            group = docs[a:b]
            k32 = np.concatenate([_known_f32(known[i], len(docs[i])) for i in range(a, b)])
            with self._lock, torch.cuda.device(self.device):
                probas, off = self._char_probas(group, k32, True)
                D, N = b - a, int(off[-1])
                dev = self.device
                lens = np.diff(off).astype(np.int32)
                d_off = torch.from_numpy(off[:-1].copy()).to(dev)
                d_len = torch.from_numpy(lens).to(dev)
                d_min = torch.full((D,), min_len, dtype=torch.int32, device=dev)
                d_max = torch.full((D,), max_len if max_len is not None else 0, dtype=torch.int32, device=dev)
                cuts = torch.empty(max(N, 1), dtype=torch.int32, device=dev)
                cs = torch.empty(2 * D, dtype=torch.int32, device=dev)
                ws = torch.empty(int(self.lib.rl_sentence_partition_workspace_bytes(N)), dtype=torch.uint8, device=dev)
                check(self.lib.rl_sentence_partition(probas.data_ptr(), d_off.data_ptr(), d_len.data_ptr(),
                                                     d_min.data_ptr(), d_max.data_ptr(), D, N, cuts.data_ptr(),
                                                     cs.data_ptr(), cs[D:].data_ptr(), ws.data_ptr(), ws.numel(),
                                                     _stream()), "rl_sentence_partition")
                counts_status = cs.cpu().numpy()
                h_cuts = cuts.cpu().numpy()
            counts, status = counts_status[:D], counts_status[D:]
            if status.any():
                raise ValueError(PARTITION_FAILED)
            for i, doc in enumerate(group):
                c = h_cuts[off[i]:off[i] + counts[i]].tolist()
                res.append([doc[x:y] for x, y in zip([0, *c], [*c, None], strict=True)])
        return res


def _known_f32(known: np.ndarray, n: int) -> np.ndarray:
    """Known probabilities as ``rl_sat_char_probas`` takes them: float32, NaN where the caller's value is not finite
    (so a finite value that overflows float32 still overrides, as the reference's assignment does)."""
    k = np.asarray(known)
    if k.shape != (n,):
        raise ValueError(f"boundary_probas has shape {k.shape}, expected ({n},): one value per character")
    fin = np.isfinite(k)
    return np.where(fin, k.astype(np.float32), np.float32(np.nan)).astype(np.float32)


# ---- public surface ----------------------------------------------------------------------------------------------------
_SPLITTER: list[Any] = []


def register_sentence_splitter(engine: Any) -> None:
    """Provide the SaT model behind ``split_sentences`` (a ``SaTEngine``; the reference loads ``sat-1l-sm`` through
    wtpsplit-lite, ``_split_sentences.py:15-20``)."""
    _SPLITTER[:] = [engine]


def _splitter() -> Any:
    if _SPLITTER:
        return _SPLITTER[0]
    raise ModuleNotFoundError(
        "No sentence splitter registered: the SaT model runs on the GPU through raglite_b200.SaTEngine; call "
        "raglite_b200.register_sentence_splitter(raglite_b200.SaTEngine.from_pretrained(local_sat_dir)).")


FloatVector = np.ndarray
BoundaryProbas = FloatVector | Callable[[str], FloatVector]


def split_sentences_batch(docs: Sequence[str], *, min_len: int = 4, max_len: int | None = None,
                          boundary_probas: BoundaryProbas = markdown_sentence_boundaries) -> list[list[str]]:
    """``split_sentences`` of every document, with one forward and one partition launch per group of documents.
    ``boundary_probas`` is a callable applied to each document, or one array used for every document."""
    docs = list(docs)
    out: list[list[str] | None] = [[d] if len(d) <= min_len else None for d in docs]
    todo = [i for i, o in enumerate(out) if o is None]
    if not todo:
        return out  # type: ignore[return-value]
    if min_len < 1 or (max_len is not None and max_len < 1):
        raise ValueError(f"min_len={min_len}, max_len={max_len}: both must be at least 1")
    engine = _splitter()
    known = [boundary_probas(docs[i]) if callable(boundary_probas) else boundary_probas for i in todo]
    for i, s in zip(todo, engine.split([docs[i] for i in todo], known, min_len=min_len, max_len=max_len), strict=True):
        out[i] = s
    return out  # type: ignore[return-value]


def split_sentences(doc: str, min_len: int = 4, max_len: int | None = None,
                    boundary_probas: BoundaryProbas = markdown_sentence_boundaries) -> list[str]:
    """Split a document into sentences (``raglite._split_sentences.split_sentences``): at least ``min_len`` and, when
    given, at most ``max_len`` characters each, maximising the sum of SaT's boundary probabilities above 0.25.
    ``boundary_probas`` (an array, or a callable of the document) overrides the model wherever it is finite."""
    return split_sentences_batch([doc], min_len=min_len, max_len=max_len, boundary_probas=boundary_probas)[0]


def sentence_boundary_probas(docs: Sequence[str]) -> list[np.ndarray]:
    """What ``sat.predict_proba(doc, stride=128, block_size=256, weighting="hat")`` returns for every document: float32,
    one probability per character, from the registered engine."""
    return _splitter().boundary_probas(list(docs))
