"""Qwen3 GGUF decoder on the GPU: the LLM behind ``rag()``, which the reference runs in llama.cpp through litellm.

``LlmEngine`` holds every 2-D weight once as a quantized image (``rl_xenc_pack_qlinear``; weights of more than 8192 rows
as parts of 8192), an fp16 KV cache of ``n_ctx`` positions and one workspace.  A prompt is prefilled in chunks through
the wgmma quantized linear (``rl_llm_forward`` with T > 1), then each token is one decode step (T = 1: every linear a
GEMV) and one ``rl_llm_sample`` on the device.  The sampled id feeds the next step on the device; one copy per step
brings it to the host for the text.

Under a grammar (``generate(..., grammar=...)``) the step samples with ``rl_llm_sample_masked`` instead: the engine
keeps, per grammar text, its DFA and the token index ``rl_grammar_token_index`` built over ``QwenTokenizer.token_bytes``
(control tokens as their text), and the DFA state stays on the device between steps.
"""

from __future__ import annotations

import codecs
import ctypes as C
import secrets
from collections import OrderedDict
from collections.abc import Iterator, Sequence
from pathlib import Path
from typing import Any

import numpy as np
import torch

from . import _lib
from ._gguf import GGUFFile, GGUFTensor, Qwen3Plan, find_cached_gguf, parse_embedder, qwen3_plan
from ._grammar import Grammar, compile_gbnf
from ._lib import LlmLayer, LlmLinear, LlmWeights, check

PART_ROWS = 8192
MAX_TOP_K = 256
PENALTY_LAST_N = 64
# Token indexes an engine keeps (least recently used dropped first): each is S x vocab int16 of device memory, 40 MB
# at 130 states and Qwen3's vocabulary, 311 MB at the 1024-state cap.  rag() uses three grammars per tool.
MAX_GRAMMARS = 8
# The Qwen2 pre-tokenizer's split (llama.cpp's LLAMA_VOCAB_PRE_TYPE_QWEN2, transformers' Qwen2TokenizerFast)
QWEN2_SPLIT = (r"(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+|"
               r"\s+(?!\S)|\s+")
TOKEN_CONTROL, TOKEN_USER_DEFINED = 3, 4


def _stream() -> int:
    return int(torch.cuda.current_stream().cuda_stream)


# ---- tokenizer -----------------------------------------------------------------------------------------------------
def _byte_decoder() -> dict[str, int]:
    """GPT-2's byte-level alphabet, inverted: the printable character standing for each byte -> the byte."""
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    cs = bs[:]
    n = 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return {chr(c): b for b, c in zip(bs, cs, strict=True)}


class QwenTokenizer:
    """The byte-level BPE of a ``gpt2`` / ``qwen2`` GGUF vocabulary, rebuilt with ``tokenizers``: BPE over
    ``tokenizer.ggml.tokens`` / ``merges``, the Qwen2 split then ByteLevel pre-tokenisation, control (type 3) and
    user-defined (type 4) tokens as special tokens.  ``token_bytes`` gives each id's exact bytes."""

    def __init__(self, tokens: Sequence[str], merges: Sequence[str], token_types: Sequence[int] | None, *,
                 add_bos: bool = False, bos_id: int | None = None) -> None:
        from tokenizers import AddedToken, Regex, Tokenizer, decoders, models, pre_tokenizers

        types = list(token_types) if token_types is not None else [1] * len(tokens)
        special = [i for i, t in enumerate(types) if t in (TOKEN_CONTROL, TOKEN_USER_DEFINED)]
        vocab = {t: i for i, t in enumerate(tokens)}
        pairs = [tuple(m.split(" ", 1)) for m in merges]
        tok = Tokenizer(models.BPE(vocab=vocab, merges=pairs, fuse_unk=False, byte_fallback=False))
        tok.pre_tokenizer = pre_tokenizers.Sequence([
            pre_tokenizers.Split(Regex(QWEN2_SPLIT), behavior="isolated", invert=False),
            pre_tokenizers.ByteLevel(add_prefix_space=False, use_regex=False)])
        tok.decoder = decoders.ByteLevel()
        tok.add_special_tokens([AddedToken(tokens[i], special=True, normalized=False) for i in special])
        self.tokenizer = tok
        self.add_bos, self.bos_id = add_bos, bos_id
        dec = _byte_decoder()
        sp = set(special)
        self.token_bytes = [t.encode() if i in sp else bytes(dec[c] for c in t) if all(c in dec for c in t) else t.encode()
                            for i, t in enumerate(tokens)]
        self.ids = vocab

    @classmethod
    def from_gguf(cls, f: GGUFFile) -> "QwenTokenizer":
        model, pre = f.get("tokenizer.ggml.model"), f.get("tokenizer.ggml.pre")
        if model != "gpt2" or pre != "qwen2":
            raise ValueError(f"{f.path}: tokenizer.ggml.model={model!r} pre={pre!r} unsupported: the decoder rebuilds "
                             "byte-level BPE vocabularies ('gpt2' with the 'qwen2' pre-tokenizer)")
        tokens, merges = f.get("tokenizer.ggml.tokens"), f.get("tokenizer.ggml.merges")
        if tokens is None or merges is None:
            raise ValueError(f"{f.path}: tokenizer.ggml.tokens / merges missing")
        bos = f.get("tokenizer.ggml.bos_token_id")
        return cls(tokens, merges, f.get("tokenizer.ggml.token_type"), add_bos=bool(f.get("tokenizer.ggml.add_bos_token", False)),
                   bos_id=None if bos is None else int(bos))

    def encode(self, text: str) -> list[int]:
        """Token ids of ``text`` with the special tokens' texts parsed as those tokens, as ``create_completion``
        tokenizes a prompt (BOS first when the file asks for it)."""
        ids = self.tokenizer.encode(text, add_special_tokens=False).ids
        return ([self.bos_id] if self.add_bos and self.bos_id is not None else []) + ids

    def decode_bytes(self, ids: Sequence[int]) -> bytes:
        return b"".join(self.token_bytes[int(i)] for i in ids)


# ---- weights --------------------------------------------------------------------------------------------------------
def _tensor_parts(t: GGUFTensor) -> list[tuple[int, np.ndarray]]:
    """(rows, raw block bytes) of each part of at most PART_ROWS rows."""
    N = t.shape[0]
    row_bytes = t.data.nbytes // N
    return [(min(PART_ROWS, N - r0), t.data[r0 * row_bytes:(r0 + min(PART_ROWS, N - r0)) * row_bytes])
            for r0 in range(0, N, PART_ROWS)]


class LlmEngine:
    """A Qwen3 decoder on one GPU: resident quantized weights, an fp16 KV cache of ``n_ctx`` positions
    (``kv_cache_bytes``, allocated once) and the prefill / decode / sampling steps."""

    def __init__(self, plan: Qwen3Plan, tokenizer: QwenTokenizer | None, *, n_ctx: int = 0, device: Any | None = None,
                 prefill_chunk: int = 512) -> None:
        if not torch.cuda.is_available():
            raise RuntimeError("raglite_b200 needs a CUDA device (there is no CPU fallback)")
        if n_ctx < 0:
            raise ValueError(f"n_ctx={n_ctx} must be >= 0 (0: the file's context_length)")
        self.lib = _lib.load()
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        self.plan, self.tokenizer = plan, tokenizer
        self.n_ctx = int(n_ctx or plan.context_length)
        self.prefill_chunk = int(prefill_chunk)
        self._keep: list[torch.Tensor] = []
        with torch.cuda.device(self.device):
            self._build(plan)
            n_kv_elems = plan.n_layers * self.n_ctx * plan.n_kv * 128
            self.kv_cache_bytes = 2 * n_kv_elems * 2
            self.k_cache = torch.empty(n_kv_elems, dtype=torch.float16, device=self.device)
            self.v_cache = torch.empty(n_kv_elems, dtype=torch.float16, device=self.device)
            ws = int(self.lib.rl_llm_workspace_bytes(C.byref(self.weights), self.prefill_chunk))
            if ws == 0:
                raise ValueError("the decoder refused these weights: " + self.lib.rl_last_error().decode(errors="replace"))
            self._ws = torch.empty(ws, dtype=torch.uint8, device=self.device)
            self.logits = torch.empty(plan.vocab, dtype=torch.float32, device=self.device)
            self._sample_ws = torch.empty(int(self.lib.rl_llm_sample_workspace_bytes(plan.vocab)), dtype=torch.uint8,
                                          device=self.device)
            self._ids = torch.empty(self.n_ctx, dtype=torch.int32, device=self.device)   # prompt ids by position
            self._tok = torch.empty(1, dtype=torch.int32, device=self.device)
            self._hist = torch.empty(PENALTY_LAST_N, dtype=torch.int32, device=self.device)
        self._tok_host = torch.empty(1, dtype=torch.int32, pin_memory=True)
        self._ids_host = torch.empty(self.n_ctx, dtype=torch.int32, pin_memory=True)
        self._ids_copied: torch.cuda.Event | None = None   # the last copy out of _ids_host
        self._hist_host = torch.empty(PENALTY_LAST_N, dtype=torch.int32, pin_memory=True)
        self.n_past = 0
        self._grammars: OrderedDict[str, GrammarIndex] = OrderedDict()
        self._vocab_dev: tuple[torch.Tensor, torch.Tensor] | None = None
        with torch.cuda.device(self.device):
            self.grammar_state = torch.zeros(1, dtype=torch.int32, device=self.device)

    # -- construction --
    @classmethod
    def from_gguf(cls, path: Path | str, n_ctx: int = 0, **kw: Any) -> "LlmEngine":
        """Load a ``qwen3`` GGUF file (2-D weights Q8_0 / Q4_K / Q6_K).  ``n_ctx`` 0 means the file's
        ``context_length``, as llama-cpp-python reads ``n_ctx=0``."""
        f = GGUFFile(path)
        plan = qwen3_plan(f)
        return cls(plan, QwenTokenizer.from_gguf(f), n_ctx=n_ctx, **kw)

    @classmethod
    def from_llm_string(cls, llm: str, hub_cache: Path | str | None = None, **kw: Any) -> "LlmEngine":
        """The config's ``llama-cpp-python/{org}/{repo}/{file glob}@{n_ctx}`` from the Hugging Face hub cache (never
        downloads)."""
        repo_id, glob, n_ctx = parse_embedder(llm)
        return cls.from_gguf(find_cached_gguf(repo_id, glob, hub_cache), n_ctx=n_ctx, **kw)

    def _linear(self, t: GGUFTensor) -> LlmLinear:
        lin = LlmLinear()
        parts = _tensor_parts(t)
        K = t.shape[1]
        for i, (n, raw) in enumerate(parts):
            blocks = torch.from_numpy(np.array(raw)).to(self.device)   # a writable copy of the mapped bytes
            img = torch.empty(int(self.lib.rl_xenc_qlinear_image_bytes(t.ggml_type, n, K)), dtype=torch.uint8,
                              device=self.device)
            check(self.lib.rl_xenc_pack_qlinear(t.ggml_type, blocks.data_ptr(), n, K, img.data_ptr(), _stream()),
                  "rl_xenc_pack_qlinear")
            torch.cuda.current_stream().synchronize()
            self._keep.append(img)
            lin.parts[i] = img.data_ptr()
        lin.n_parts, lin.N, lin.K = len(parts), t.shape[0], K
        return lin

    def _f32(self, t: GGUFTensor) -> int:
        x = torch.from_numpy(t.data.view("<f4").astype(np.float32)).to(self.device)
        self._keep.append(x)
        return x.data_ptr()

    def _build(self, p: Qwen3Plan) -> None:
        ts = p.tensors
        self._layers = (LlmLayer * p.n_layers)()
        for i in range(p.n_layers):
            L, b = self._layers[i], f"blk.{i}."
            for field, name in (("q", "attn_q"), ("k", "attn_k"), ("v", "attn_v"), ("o", "attn_output"),
                                ("gate", "ffn_gate"), ("up", "ffn_up"), ("down", "ffn_down")):
                setattr(L, field, self._linear(ts[b + name + ".weight"]))
            for field, name in (("attn_norm", "attn_norm"), ("q_norm", "attn_q_norm"), ("k_norm", "attn_k_norm"),
                                ("ffn_norm", "ffn_norm")):
                setattr(L, field, self._f32(ts[b + name + ".weight"]))
        w = LlmWeights()
        w.n_layers, w.hidden, w.n_head, w.n_kv, w.ffn, w.vocab = p.n_layers, p.hidden, p.n_head, p.n_kv, p.ffn, p.vocab
        w.n_ctx, w.eps, w.rope_base = self.n_ctx, p.eps, p.rope_base
        w.token_embd = self._linear(ts["token_embd.weight"])
        w.output = w.token_embd if p.tied else self._linear(ts["output.weight"])
        w.output_norm = self._f32(ts["output_norm.weight"])
        w.layers = C.cast(self._layers, C.POINTER(LlmLayer))
        self.weights = w

    def weight_bytes(self) -> int:
        return sum(int(t.numel() * t.element_size()) for t in self._keep)

    # -- steps --
    def reset(self) -> None:
        self.n_past = 0

    def _forward_dev(self, ids_ptr: int, T: int) -> None:
        check(self.lib.rl_llm_forward(C.byref(self.weights), ids_ptr, T, self.n_past, self.k_cache.data_ptr(),
                                      self.v_cache.data_ptr(), self.logits.data_ptr(), self._ws.data_ptr(),
                                      self._ws.numel(), _stream()), "rl_llm_forward")
        self.n_past += T

    def prefill(self, ids: Sequence[int], *, chunk: int | None = None) -> torch.Tensor:
        """Append ``ids`` at positions n_past ...; returns the last row's logits (device fp32 [vocab])."""
        ids = np.asarray(ids, dtype=np.int32)
        if ids.ndim != 1 or len(ids) == 0:
            raise ValueError("prefill needs a non-empty 1-D list of token ids")
        if np.any(ids < 0) or np.any(ids >= self.plan.vocab):
            raise ValueError(f"token ids must be in [0, {self.plan.vocab})")
        if self.n_past + len(ids) > self.n_ctx:
            raise ValueError(f"Requested tokens ({self.n_past + len(ids)}) exceed context window of {self.n_ctx}")
        step = min(int(chunk or self.prefill_chunk), self.prefill_chunk)
        p0, n = self.n_past, len(ids)
        if self._ids_copied is not None:   # the pinned buffer is free once its previous copy has run
            self._ids_copied.synchronize()
        self._ids_host[:n] = torch.from_numpy(ids)
        with torch.cuda.device(self.device):
            # one asynchronous copy of the whole prompt, so the host enqueues the chunks while the device runs them
            self._ids[p0:p0 + n].copy_(self._ids_host[:n], non_blocking=True)
            self._ids_copied = torch.cuda.Event()
            self._ids_copied.record()
            for lo in range(0, n, step):
                self._forward_dev(self._ids[p0 + lo:].data_ptr(), min(step, n - lo))
        return self.logits

    def grammar_index(self, grammar: "str | Grammar") -> "GrammarIndex":
        """The DFA and device token index of a grammar (GBNF text or compiled), built once per grammar text and kept
        for the ``MAX_GRAMMARS`` most recently used."""
        text = grammar if isinstance(grammar, str) else grammar.text
        if text in self._grammars:
            self._grammars.move_to_end(text)
        else:
            g = grammar if isinstance(grammar, Grammar) else compile_gbnf(grammar)
            if self.tokenizer is None:
                raise ValueError("grammar-constrained generation needs the engine's tokenizer")
            with torch.cuda.device(self.device):
                if self._vocab_dev is None:
                    pieces = list(self.tokenizer.token_bytes[:self.plan.vocab])
                    pieces += [b""] * (self.plan.vocab - len(pieces))   # ids past the vocabulary: empty, never allowed
                    offs = np.zeros(len(pieces) + 1, dtype=np.int64)
                    offs[1:] = np.cumsum([len(p) for p in pieces])
                    flat = np.frombuffer(b"".join(pieces) or b"\0", dtype=np.uint8)
                    self._vocab_dev = (torch.from_numpy(flat.copy()).to(self.device), torch.from_numpy(offs).to(self.device))
                trans = torch.from_numpy(np.ascontiguousarray(g.trans, dtype=np.int16)).to(self.device)
                index = torch.empty((g.n_states, self.plan.vocab), dtype=torch.int16, device=self.device)
                check(self.lib.rl_grammar_token_index(trans.data_ptr(), g.n_states, self._vocab_dev[0].data_ptr(),
                                                      self._vocab_dev[1].data_ptr(), self.plan.vocab, index.data_ptr(),
                                                      _stream()), "rl_grammar_token_index")
                accept = torch.from_numpy(g.accept.astype(np.uint8)).to(self.device)
            self._grammars[text] = GrammarIndex(g, index, accept)
            while len(self._grammars) > MAX_GRAMMARS:
                self._grammars.popitem(last=False)
        return self._grammars[text]

    def sample(self, history: Sequence[int], *, temperature: float, top_k: int, top_p: float, min_p: float,
               repeat_penalty: float, u: float, grammar: "GrammarIndex | None" = None) -> torch.Tensor:
        """Sample from ``self.logits`` into the device id ``self._tok`` (see ``rl_llm_sample``); under ``grammar``,
        among the ids its state ``self.grammar_state`` allows, advancing that state (see ``rl_llm_sample_masked``)."""
        hist = np.asarray(history[-PENALTY_LAST_N:], dtype=np.int32)
        self._hist_host[:len(hist)] = torch.from_numpy(hist)
        with torch.cuda.device(self.device):
            self._hist[:len(hist)].copy_(self._hist_host[:len(hist)], non_blocking=True)
            if grammar is None:
                check(self.lib.rl_llm_sample(self.logits.data_ptr(), self.plan.vocab, self._hist.data_ptr(), len(hist),
                                             float(temperature), int(top_k), float(top_p), float(min_p),
                                             float(repeat_penalty), float(u), self._tok.data_ptr(),
                                             self._sample_ws.data_ptr(), self._sample_ws.numel(), _stream()),
                      "rl_llm_sample")
            else:
                eog = sorted(self.stop_ids())
                check(self.lib.rl_llm_sample_masked(
                    self.logits.data_ptr(), self.plan.vocab, self._hist.data_ptr(), len(hist), float(temperature),
                    int(top_k), float(top_p), float(min_p), float(repeat_penalty), float(u), grammar.index.data_ptr(),
                    grammar.dfa.n_states, grammar.accept.data_ptr(), (C.c_int32 * max(1, len(eog)))(*eog), len(eog),
                    self.grammar_state.data_ptr(), self._tok.data_ptr(), self._sample_ws.data_ptr(),
                    self._sample_ws.numel(), _stream()), "rl_llm_sample_masked")
        return self._tok

    def stop_ids(self) -> set[int]:
        ids = set()
        if self.tokenizer is not None:
            for t in ("<|im_end|>", "<|endoftext|>"):
                if t in self.tokenizer.ids:
                    ids.add(self.tokenizer.ids[t])
        return ids

    def generate_ids(self, prompt_ids: Sequence[int], *, max_tokens: int | None = None, temperature: float = 0.6,
                     top_k: int = 20, top_p: float = 0.95, min_p: float = 0.0, repeat_penalty: float = 1.1,
                     seed: int | None = None, grammar: "str | Grammar | None" = None) -> Iterator[int]:
        """Token ids after ``prompt_ids`` (a fresh sequence), stop tokens excluded: until a stop token, ``max_tokens``
        (None: until ``n_ctx``) or the context is full.  Under ``grammar`` (GBNF text or compiled) every id keeps the
        text a prefix of the grammar's language, and a stop token is allowed only where the text is complete; where it
        is complete and cannot continue, a stop token is the only choice."""
        gi = None if grammar is None else self.grammar_index(grammar)
        if not (1 <= top_k <= MAX_TOP_K):
            raise ValueError(f"top_k={top_k} unsupported (1 .. {MAX_TOP_K})")
        if temperature < 0:
            raise ValueError(f"temperature={temperature} must be >= 0")
        prompt = [int(i) for i in prompt_ids]
        if len(prompt) > self.n_ctx:
            raise ValueError(f"Requested tokens ({len(prompt)}) exceed context window of {self.n_ctx}")
        rng = np.random.default_rng(secrets.randbits(32) if seed is None else seed)
        self.reset()
        self.prefill(prompt)
        history, stops = list(prompt), self.stop_ids()
        if gi is not None:
            self.grammar_state.zero_()
        n = 0
        while max_tokens is None or n < max_tokens:
            u = min(float(np.float32(rng.random())), float(np.nextafter(np.float32(1), np.float32(0))))
            tok = self.sample(history, temperature=temperature, top_k=top_k, top_p=top_p, min_p=min_p,
                              repeat_penalty=repeat_penalty, u=u, grammar=gi)
            self._tok_host.copy_(tok, non_blocking=True)
            torch.cuda.current_stream(self.device).synchronize()
            t = int(self._tok_host[0])
            if t == _lib.RL_LLM_NO_TOKEN:
                raise RuntimeError("the grammar allows no token of this vocabulary here (and no end-of-generation "
                                   "token unless the text is complete)")
            if t in stops:
                return
            yield t
            n += 1
            history.append(t)
            if self.n_past >= self.n_ctx:
                return
            if max_tokens is not None and n >= max_tokens:
                return
            with torch.cuda.device(self.device):
                self._forward_dev(tok.data_ptr(), 1)

    def generate(self, prompt_ids: Sequence[int], *, stop: Sequence[str] = (), **kw: Any) -> Iterator[str]:
        """Text pieces of ``generate_ids``: UTF-8 held back until a character is complete, generation ended at the
        first stop string (excluded), and text that could still begin one held back."""
        if self.tokenizer is None:
            raise ValueError("this engine has no tokenizer")
        dec = codecs.getincrementaldecoder("utf-8")(errors="replace")
        stop = [s for s in stop if s]
        pending = ""
        for t in self.generate_ids(prompt_ids, **kw):
            pending += dec.decode(self.tokenizer.token_bytes[t])
            hit = min((i for i in (pending.find(s) for s in stop) if i >= 0), default=-1)
            if hit >= 0:
                if pending[:hit]:
                    yield pending[:hit]
                return
            hold = max((k for s in stop for k in range(min(len(s) - 1, len(pending)), 0, -1) if pending.endswith(s[:k])),
                       default=0)
            if len(pending) > hold:
                yield pending[:len(pending) - hold]
                pending = pending[len(pending) - hold:]
        pending += dec.decode(b"", final=True)
        if pending:
            yield pending


class GrammarIndex:
    """A grammar on one engine: its DFA, the device token index int16 [S, vocab] and accepting states uint8 [S]."""

    def __init__(self, dfa: Grammar, index: torch.Tensor, accept: torch.Tensor) -> None:
        self.dfa, self.index, self.accept = dfa, index, accept


# ---- registry ----------------------------------------------------------------------------------------------------
_LLMS: dict[str, LlmEngine] = {}


def _llm_key(config_or_llm: Any) -> str:
    return config_or_llm if isinstance(config_or_llm, str) else str(config_or_llm.llm)


def register_llm(config_or_llm_string: Any, engine: LlmEngine) -> None:
    """Use ``engine`` for ``rag()`` under a config whose ``llm`` is this string."""
    _LLMS[_llm_key(config_or_llm_string)] = engine


def register_gguf_llm(config: Any, hub_cache: Path | str | None = None, **kw: Any) -> LlmEngine:
    """Load ``config.llm``'s GGUF file from the hub cache and register it."""
    engine = LlmEngine.from_llm_string(config.llm, hub_cache=hub_cache, **kw)
    register_llm(config, engine)
    return engine


def find_llm(config: Any) -> LlmEngine | None:
    """The engine registered for ``config.llm``, or None."""
    return _LLMS.get(_llm_key(config))


def get_llm(config: Any) -> LlmEngine:
    key = _llm_key(config)
    if key not in _LLMS:
        raise NotImplementedError(f"no LLM is registered for llm={key!r}: load its GGUF file with register_gguf_llm(config) "
                                  "(or register_llm(config, LlmEngine.from_gguf(path)))")
    return _LLMS[key]
