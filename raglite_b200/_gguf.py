"""GGUF reader (host only, no dependency beyond NumPy): the file format llama.cpp's converter writes.

A file is: magic ``GGUF``, a little-endian uint32 version (2 or 3), the tensor and metadata counts (uint64), the metadata
key / value pairs, the tensor infos (name, dimensions innermost first, GGML type, offset into the data section), padding
to ``general.alignment`` (32 when absent) and the data section.  Tensors are returned as views of a memory map: a 2-D
tensor of ``ne = (K, N)`` is ``[N, K]`` (row-major, K innermost) and keeps its raw block bytes.
"""

from __future__ import annotations

import mmap
import struct
from dataclasses import dataclass
from pathlib import Path
from typing import Any

import numpy as np

GGUF_MAGIC = b"GGUF"
# GGML type ids read here: (name, elements per block, bytes per block)
GGML_TYPES = {0: ("F32", 1, 4), 1: ("F16", 1, 2), 8: ("Q8_0", 32, 34), 12: ("Q4_K", 256, 144), 14: ("Q6_K", 256, 210)}
F32, F16, Q8_0, Q4_K, Q6_K = 0, 1, 8, 12, 14
QUANT_TYPES = (Q8_0, Q4_K, Q6_K)

# metadata value types: id -> struct format (scalars), 8 = string, 9 = array
_SCALARS = {0: "<B", 1: "<b", 2: "<H", 3: "<h", 4: "<I", 5: "<i", 6: "<f", 7: "<?", 10: "<Q", 11: "<q", 12: "<d"}
_NUMPY = {0: np.uint8, 1: np.int8, 2: np.uint16, 3: np.int16, 4: np.uint32, 5: np.int32, 6: np.float32, 7: np.bool_,
          10: np.uint64, 11: np.int64, 12: np.float64}
_STRING, _ARRAY = 8, 9


@dataclass(frozen=True)
class GGUFTensor:
    name: str
    ggml_type: int
    shape: tuple[int, ...]     # outermost first: [N, K] for a 2-D weight whose ne0 is K
    data: np.ndarray           # raw bytes (uint8), a view of the file

    @property
    def type_name(self) -> str:
        return GGML_TYPES[self.ggml_type][0]

    @property
    def n_elements(self) -> int:
        return int(np.prod(self.shape, dtype=np.int64))


class _Cursor:
    def __init__(self, buf: memoryview, path: Path) -> None:
        self.buf, self.pos, self.path = buf, 0, path

    def take(self, n: int) -> memoryview:
        if n < 0 or self.pos + n > len(self.buf):
            raise ValueError(f"{self.path}: truncated GGUF file (needs {n} bytes at offset {self.pos}, has {len(self.buf)})")
        out = self.buf[self.pos:self.pos + n]
        self.pos += n
        return out

    def scalar(self, fmt: str) -> Any:
        return struct.unpack(fmt, self.take(struct.calcsize(fmt)))[0]

    def string(self) -> str:
        return bytes(self.take(self.scalar("<Q"))).decode("utf-8", errors="replace")

    def value(self, vtype: int) -> Any:
        if vtype in _SCALARS:
            return self.scalar(_SCALARS[vtype])
        if vtype == _STRING:
            return self.string()
        if vtype == _ARRAY:
            sub, n = self.scalar("<I"), self.scalar("<Q")
            if sub in _NUMPY:
                dt = np.dtype(_NUMPY[sub]).newbyteorder("<")
                return np.frombuffer(self.take(n * dt.itemsize), dtype=dt).copy()
            return [self.value(sub) for _ in range(n)]
        raise ValueError(f"{self.path}: unknown GGUF metadata value type {vtype} at offset {self.pos}")


class GGUFFile:
    """Metadata (``dict``) and tensors (``dict`` of ``GGUFTensor``) of one GGUF v2 / v3 file."""

    def __init__(self, path: Path | str) -> None:
        self.path = Path(path)
        with open(self.path, "rb") as f:
            size = f.seek(0, 2)
            self._mm = mmap.mmap(f.fileno(), 0, access=mmap.ACCESS_READ) if size else None
        buf = memoryview(self._mm) if self._mm is not None else memoryview(b"")
        cur = _Cursor(buf, self.path)
        if bytes(cur.take(4)) != GGUF_MAGIC:
            raise ValueError(f"{self.path}: not a GGUF file (bad magic)")
        self.version = cur.scalar("<I")
        if self.version not in (2, 3):
            raise ValueError(f"{self.path}: GGUF version {self.version} unsupported (2 or 3)")
        n_tensors, n_kv = cur.scalar("<Q"), cur.scalar("<Q")
        self.metadata: dict[str, Any] = {}
        for _ in range(n_kv):
            key = cur.string()
            self.metadata[key] = cur.value(cur.scalar("<I"))
        infos = []
        for _ in range(n_tensors):
            name = cur.string()
            n_dims = cur.scalar("<I")
            ne = [cur.scalar("<Q") for _ in range(n_dims)]
            infos.append((name, ne, cur.scalar("<I"), cur.scalar("<Q")))
        align = int(self.metadata.get("general.alignment", 32))
        if align <= 0 or align & (align - 1):
            raise ValueError(f"{self.path}: general.alignment={align} is not a power of two")
        data_start = (cur.pos + align - 1) // align * align
        self.alignment = align
        self.tensors: dict[str, GGUFTensor] = {}
        for name, ne, ty, off in infos:
            if ty not in GGML_TYPES:
                raise ValueError(f"{self.path}: tensor {name!r} has GGML type {ty}, unsupported (F32, F16, Q8_0, Q4_K, Q6_K)")
            _, be, bb = GGML_TYPES[ty]
            if not ne or ne[0] % be:
                raise ValueError(f"{self.path}: tensor {name!r}: ne0={ne[0] if ne else None} is not a whole number of "
                                 f"{GGML_TYPES[ty][0]} blocks")
            n = int(np.prod(ne, dtype=np.int64))
            nbytes = n // be * bb
            begin = data_start + off
            if begin + nbytes > len(buf):
                raise ValueError(f"{self.path}: tensor {name!r} runs past the end of the file")
            data = np.frombuffer(buf, dtype=np.uint8, count=nbytes, offset=begin)
            self.tensors[name] = GGUFTensor(name, ty, tuple(int(x) for x in reversed(ne)), data)

    def get(self, key: str, default: Any = None) -> Any:
        return self.metadata.get(key, default)

    def tensor_bytes(self) -> int:
        return sum(int(t.data.nbytes) for t in self.tensors.values())


def tensor_to_f32(t: GGUFTensor) -> np.ndarray:
    """F32 / F16 tensor as a float32 copy of its shape (quantized types are dequantized on the device)."""
    if t.ggml_type == F32:
        return t.data.view("<f4").astype(np.float32).reshape(t.shape)
    if t.ggml_type == F16:
        return t.data.view("<f2").astype(np.float32).reshape(t.shape)
    raise ValueError(f"tensor {t.name!r} is {t.type_name}: not a float tensor")


# ---- BERT / XLM-RoBERTa embedders (llama.cpp's "bert" architecture) -----------------------------------------------------
# GGUF tensor name -> the state-dict name _EncoderEngine reads ({i}: block index).  Names from gguf.constants
# (TENSOR_NAMES of MODEL_TENSORS[MODEL_ARCH.BERT]).
_BERT_GLOBAL = {"token_embd.weight": "embeddings.word_embeddings.weight",
                "position_embd.weight": "embeddings.position_embeddings.weight",
                "token_types.weight": "embeddings.token_type_embeddings.weight",
                "token_embd_norm.weight": "embeddings.LayerNorm.weight", "token_embd_norm.bias": "embeddings.LayerNorm.bias"}
_BERT_BLOCK = {"attn_output.weight": "attention.output.dense.weight", "attn_output.bias": "attention.output.dense.bias",
               "attn_output_norm.weight": "attention.output.LayerNorm.weight",
               "attn_output_norm.bias": "attention.output.LayerNorm.bias",
               "ffn_up.weight": "intermediate.dense.weight", "ffn_up.bias": "intermediate.dense.bias",
               "ffn_down.weight": "output.dense.weight", "ffn_down.bias": "output.dense.bias",
               "layer_output_norm.weight": "output.LayerNorm.weight", "layer_output_norm.bias": "output.LayerNorm.bias"}
GGUF_MAX_HIDDEN = 1024


@dataclass(frozen=True)
class BertPlan:
    n_layers: int
    hidden: int
    n_heads: int
    ffn: int
    ln_eps: float
    context_length: int
    state_dict: dict[str, Any]   # state-dict name -> GGUFTensor (projections' q / k / v split when the file fuses them)


def bert_plan(f: GGUFFile) -> BertPlan:
    """Check a GGUF file against what the token encoder runs and map its tensors to state-dict names.  Raises
    ``ValueError`` (nothing touches a device)."""
    arch = f.get("general.architecture")
    if arch != "bert":
        raise ValueError(f"{f.path}: general.architecture={arch!r} unsupported: the token encoder loads 'bert' "
                         "(BERT and XLM-RoBERTa models such as bge-m3)")

    def key(k: str) -> int:
        v = f.get(f"bert.{k}")
        if v is None:
            raise ValueError(f"{f.path}: metadata key bert.{k} is missing")
        return v

    n_layers, hidden, ffn = int(key("block_count")), int(key("embedding_length")), int(key("feed_forward_length"))
    n_heads, eps, ctx = int(key("attention.head_count")), float(key("attention.layer_norm_epsilon")), int(key("context_length"))
    if n_heads <= 0 or hidden % n_heads or hidden // n_heads not in (32, 64):
        raise ValueError(f"{f.path}: hidden={hidden} heads={n_heads}: head_dim must be 32 or 64")
    if hidden % 32 or hidden > GGUF_MAX_HIDDEN or ffn % 32 or n_layers < 1:
        raise ValueError(f"{f.path}: hidden={hidden} ffn={ffn} layers={n_layers} unsupported (hidden and ffn multiples of "
                         f"32, hidden <= {GGUF_MAX_HIDDEN}, at least one layer)")

    def tensor(name: str, shape: tuple[int, ...] | None = None) -> GGUFTensor:
        t = f.tensors.get(name)
        if t is None:
            raise ValueError(f"{f.path}: tensor {name!r} is missing")
        if shape is not None and t.shape != shape:
            raise ValueError(f"{f.path}: tensor {name!r} has shape {list(t.shape)}, expected {list(shape)}")
        return t

    vocab = tensor("token_embd.weight").shape[0]
    tokens = f.get("tokenizer.ggml.tokens")
    if tokens is not None and len(tokens) != vocab:
        raise ValueError(f"{f.path}: the vocabulary has {len(tokens)} tokens but token_embd has {vocab} rows")
    sd: dict[str, Any] = {v: tensor(k) for k, v in _BERT_GLOBAL.items()}
    for v in ("embeddings.word_embeddings.weight", "embeddings.position_embeddings.weight",
              "embeddings.token_type_embeddings.weight"):
        if len(sd[v].shape) != 2 or sd[v].shape[1] != hidden:
            raise ValueError(f"{f.path}: {v} has shape {list(sd[v].shape)}, expected [rows, {hidden}]")
    shapes = {"attn_output.weight": (hidden, hidden), "ffn_up.weight": (ffn, hidden), "ffn_down.weight": (hidden, ffn),
              "attn_output.bias": (hidden,), "ffn_up.bias": (ffn,), "ffn_down.bias": (hidden,)}
    for i in range(n_layers):
        b, pre = f"blk.{i}.", f"encoder.layer.{i}."
        for k, v in _BERT_BLOCK.items():
            sd[pre + v] = tensor(b + k, shapes.get(k, (hidden,)))
        if b + "attn_qkv.weight" in f.tensors:   # fused Q | K | V: split into row views
            w, bias = tensor(b + "attn_qkv.weight", (3 * hidden, hidden)), tensor(b + "attn_qkv.bias", (3 * hidden,))
            for j, n in enumerate(("query", "key", "value")):
                sd[pre + f"attention.self.{n}.weight"] = _rows(w, j * hidden, hidden)
                sd[pre + f"attention.self.{n}.bias"] = _rows(bias, j * hidden, hidden)
        else:
            for n, g in (("query", "q"), ("key", "k"), ("value", "v")):
                sd[pre + f"attention.self.{n}.weight"] = tensor(b + f"attn_{g}.weight", (hidden, hidden))
                sd[pre + f"attention.self.{n}.bias"] = tensor(b + f"attn_{g}.bias", (hidden,))
    for name, t in sd.items():
        if len(t.shape) == 1 and t.ggml_type not in (F32, F16):
            raise ValueError(f"{f.path}: 1-D tensor {name} is {t.type_name}; biases and norms must be F32 or F16")
    for i in range(n_layers):   # each linear (Q | K | V fused) as the engine packs it
        pre = f"encoder.layer.{i}."
        for names in (("attention.self.query", "attention.self.key", "attention.self.value"), ("attention.output.dense",),
                      ("intermediate.dense",), ("output.dense",)):
            parts = [sd[pre + n + ".weight"] for n in names]
            if any(p.ggml_type in QUANT_TYPES for p in parts):
                check_quantized_linear(parts)
    return BertPlan(n_layers, hidden, n_heads, ffn, eps, ctx, sd)


def _rows(t: GGUFTensor, r0: int, n: int) -> GGUFTensor:
    """Rows [r0, r0 + n) of a tensor (its first dimension), as a view of the same bytes."""
    row_bytes = t.data.nbytes // t.shape[0]
    return GGUFTensor(t.name, t.ggml_type, (n, *t.shape[1:]), t.data[r0 * row_bytes:(r0 + n) * row_bytes])


def check_quantized_linear(parts: list[GGUFTensor]) -> None:
    """Raise ``ValueError`` when quantized weights cannot form one quantized linear image."""
    if not all(p.ggml_type in QUANT_TYPES for p in parts):
        raise ValueError(f"{[p.name for p in parts]}: quantized and float tensors in one fused projection are unsupported")
    K = parts[0].shape[1]
    if any(p.shape[1] != K for p in parts) or K % 128:
        raise ValueError(f"{[p.name for p in parts]}: quantized linears need one K, a multiple of 128 (got {K})")
    # Parts of different types concatenate whole 128-row passes.  Q | K | V is the only fused linear and its rows per
    # part equal its K, so K % 128 == 0 already gives this; it stays a check of the concatenation's own condition.
    if len({p.ggml_type for p in parts}) > 1 and any(p.shape[0] % 128 for p in parts[:-1]):
        raise ValueError(f"{[p.name for p in parts]}: projections of different types fuse only when each has a "
                         "multiple of 128 rows")


# ---- tokenizer from the file's metadata ---------------------------------------------------------------------------------
def gguf_tokenizer(f: GGUFFile) -> Any:
    """A ``tokenizers.Tokenizer`` rebuilt from ``tokenizer.ggml.*`` for SentencePiece Unigram vocabularies (llama.cpp's
    ``t5`` model, which bge-m3 uses), as ``transformers`` builds it from the SentencePiece model: Unigram over the tokens
    and scores, ``Precompiled`` charsmap normaliser then ``Replace(" {2,}", " ")``, ``Metaspace`` pre-tokeniser and
    ``<s> $A </s>`` post-processor."""
    from tokenizers import Regex, Tokenizer, decoders, models, normalizers, pre_tokenizers, processors

    model = f.get("tokenizer.ggml.model")
    if model != "t5":
        raise ValueError(f"{f.path}: tokenizer.ggml.model={model!r}: only SentencePiece Unigram ('t5') vocabularies are "
                         "rebuilt; pass tokenizer= with the path of the model's tokenizer.json")
    tokens, scores = f.get("tokenizer.ggml.tokens"), f.get("tokenizer.ggml.scores")
    if tokens is None or scores is None or len(tokens) != len(scores):
        raise ValueError(f"{f.path}: tokenizer.ggml.tokens / scores missing or of different lengths")
    unk = f.get("tokenizer.ggml.unknown_token_id")
    tok = Tokenizer(models.Unigram([(t, float(s)) for t, s in zip(tokens, scores, strict=True)],
                                   unk_id=None if unk is None else int(unk)))
    norm = []
    charsmap = f.get("tokenizer.ggml.precompiled_charsmap")
    if charsmap is not None and len(charsmap):
        norm.append(normalizers.Precompiled(bytes(np.asarray(charsmap, dtype=np.uint8))))
    if f.get("tokenizer.ggml.remove_extra_whitespaces", False):
        norm.append(normalizers.Replace(Regex(" {2,}"), " "))
    if norm:
        tok.normalizer = normalizers.Sequence(norm)
    if f.get("tokenizer.ggml.add_space_prefix", True):
        tok.pre_tokenizer = pre_tokenizers.Metaspace(replacement="▁", prepend_scheme="always")
        tok.decoder = decoders.Metaspace(replacement="▁", prepend_scheme="always")
    else:
        tok.pre_tokenizer = pre_tokenizers.Metaspace(replacement="▁", prepend_scheme="never")
        tok.decoder = decoders.Metaspace(replacement="▁", prepend_scheme="never")
    single, special = "$A", []
    for flag, key, where in (("tokenizer.ggml.add_bos_token", "tokenizer.ggml.bos_token_id", "pre"),
                             ("tokenizer.ggml.add_eos_token", "tokenizer.ggml.eos_token_id", "post")):
        tid = f.get(key)
        if f.get(flag, True) and tid is not None:
            name = tokens[int(tid)]
            single = f"{name} {single}" if where == "pre" else f"{single} {name}"
            special.append((name, int(tid)))
    tok.post_processor = processors.TemplateProcessing(single=single, special_tokens=special)
    return tok


# ---- resolving the config's embedder string ----------------------------------------------------------------------------
def parse_embedder(embedder: str) -> tuple[str, str, int]:
    """``llama-cpp-python/{org}/{repo}/{filename glob}@{n_ctx}`` -> (repo_id, filename glob, n_ctx), with the behaviour of
    RAGLite's LiteLLM adapter (``_litellm.py:100-106``): every ``llama-cpp-python/`` is removed, the last ``/`` separates
    the repository from the file name, and a last ``@`` in the file name starts ``n_ctx`` (0 when there is none)."""
    repo_id, sep, name = embedder.replace("llama-cpp-python/", "").rpartition("/")
    if not sep:
        raise ValueError(f"{embedder!r} is not 'llama-cpp-python/<repo_id>/<filename>[@n_ctx]'")
    glob, at, ctx = name.rpartition("@")
    return (repo_id, glob, int(ctx)) if at else (repo_id, name, 0)


def hub_cache_dir() -> Path:
    import os

    if os.environ.get("HF_HUB_CACHE"):
        return Path(os.environ["HF_HUB_CACHE"])
    if os.environ.get("HF_HOME"):
        return Path(os.environ["HF_HOME"]) / "hub"
    return Path.home() / ".cache" / "huggingface" / "hub"


def find_cached_gguf(repo_id: str, filename: str, hub_cache: Path | str | None = None) -> Path:
    """The one file under the hub cache's ``models--{org}--{name}/snapshots/*/`` matching the glob ``filename`` (files
    of several snapshots that resolve to one blob count once).  Never downloads; raises ``FileNotFoundError`` listing
    the directory searched and the candidates when zero or several distinct files match."""
    root = (Path(hub_cache) if hub_cache is not None else hub_cache_dir()) / ("models--" + repo_id.replace("/", "--"))
    snaps = root / "snapshots"
    matches = sorted(snaps.glob(f"*/{filename}")) if snaps.is_dir() else []
    distinct = {p.resolve(): p for p in matches if p.is_file()}
    if len(distinct) != 1:
        cands = sorted(str(p.relative_to(snaps)) for p in snaps.glob("*/*")) if snaps.is_dir() else []
        what = "no file" if not distinct else f"{len(distinct)} files"
        raise FileNotFoundError(f"{what} matching {filename!r} in {snaps}/*/ (candidates: {cands}); download the GGUF "
                                "file with llama-cpp-python or huggingface_hub first")
    return next(iter(distinct.values()))
