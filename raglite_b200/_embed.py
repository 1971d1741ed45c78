"""Late-chunking sentence embedding: host planning + the CUDA pool kernel.

Mirrors ``raglite/_embed.py``: ``embed_strings`` dispatches on the embedder string (``:193-200``);
the late-chunking path (``:16-141``) counts tokens with the sentinel trick, cuts the document into
preamble+content segments, asks the token embedder (llama.cpp in the reference; here any object with
``n_ctx() / n_batch / tokenize / detokenize / embed``, e.g. ``TokenEmbedderEngine``, which runs the encoder
on the GPU) for per-token embeddings, and then pools.  An embedder that also offers the packed device path
(``token_ids_for_embedding`` + ``embed_token_ids``, as ``TokenEmbedderEngine`` does) runs every segment
of a call in one packed forward, and the pool reads its output where it lies on the device.  The pool itself -- largest-remainder split, per-sentence mean, L2 normalise, fp16 cast
(``:122-140``) -- is what this package accelerates: sizes are computed on the host with the same
NumPy calls as the reference, the arithmetic runs in ``rl_segment_mean_pool``.
"""

from __future__ import annotations

from collections.abc import Sequence
from typing import Any

import numpy as np
import torch

from . import _lib
from ._config import RAGLiteConfig
from ._lib import check
from ._typing import FloatMatrix

SENTINEL_CHAR = "⊕"  # _embed.py:69
_TOKEN_EMBEDDERS: dict[str, Any] = {}


def register_token_embedder(embedder: str, model: Any) -> None:
    """Provide the llama.cpp-like model object behind ``config.embedder`` (the reference loads it
    through ``LlamaCppPythonLLM.llm``, ``_embed.py:64-66``)."""
    _TOKEN_EMBEDDERS[embedder] = model


def register_gguf_embedder(config: RAGLiteConfig, hub_cache: Any | None = None, **kw: Any) -> Any:
    """Load the GGUF file ``config.embedder`` names from the Hugging Face hub cache onto the GPU
    (``TokenEmbedderEngine.from_embedder_string``) and register it for that string; returns the engine."""
    from ._xenc import TokenEmbedderEngine

    engine = TokenEmbedderEngine.from_embedder_string(config.embedder, hub_cache=hub_cache, **kw)
    register_token_embedder(config.embedder, engine)
    return engine


def _token_embedder(config: RAGLiteConfig) -> Any:
    if config.embedder in _TOKEN_EMBEDDERS:
        return _TOKEN_EMBEDDERS[config.embedder]
    raise ModuleNotFoundError(
        f"No token embedder registered for {config.embedder!r}: the transformer forward stays in "
        "llama.cpp; call raglite_b200.register_token_embedder(config.embedder, llama_model)."
    )


def _sentinel_tokens(model: Any) -> list[int]:
    probe = f"A{SENTINEL_CHAR}B {SENTINEL_CHAR} C.\n{SENTINEL_CHAR}D"
    toks = [t for t in model.tokenize(probe.encode(), add_bos=False)
            if SENTINEL_CHAR in model.detokenize([t]).decode()]
    if not toks:
        raise AssertionError(f"Sentinel `{SENTINEL_CHAR}` not supported by embedder")
    return toks


def count_tokens(sentences: Sequence[str], model: Any) -> np.ndarray:
    """Tokens per sentence via sentinel-joined batches (``_embed.py:21-36, 77-93``)."""
    sentinels = np.asarray(_sentinel_tokens(model), dtype=np.intp)
    half_ctx = model.n_ctx() // 2
    counts: list[int] = []
    start, chars = 0, 0
    for i, sentence in enumerate(sentences):
        chars += len(sentence)
        if i == len(sentences) - 1 or chars > half_ctx:
            batch = sentences[start : i + 1]
            toks = np.asarray(model.tokenize(SENTINEL_CHAR.join(batch).encode(), add_bos=False), dtype=np.intp)
            marks = np.flatnonzero(np.isin(toks, sentinels))
            gaps = np.diff(marks, prepend=0, append=len(toks))
            if len(gaps) != len(batch):
                raise AssertionError(f"Sentinel `{SENTINEL_CHAR}` appears in document")
            counts.extend(gaps.tolist())
            start, chars = i + 1, 0
    return np.asarray(counts, dtype=np.intp)


def plan_segments(num_tokens: np.ndarray, n_ctx: int, n_batch: int) -> list[tuple[int, int, int]]:
    """``(segment_start, content_start, segment_end)`` sentence triples (``_embed.py:38-58, 99-110``):
    each segment holds up to ``round(0.382 * max_tokens)`` tokens of preceding sentences as preamble;
    preamble budget that goes unused is handed to the content."""
    max_tokens = min(n_ctx, n_batch) - 16
    max_pre = round(0.382 * max_tokens)
    max_content = max_tokens - max_pre
    n = len(num_tokens)
    csum = np.concatenate([[0], np.cumsum(num_tokens)])
    segments = []
    c = 0
    while c < n:
        # furthest-back start with tokens(start..c) <= max_pre
        s = int(np.searchsorted(csum, csum[c] - max_pre, side="left"))
        budget = max_content + (max_pre - int(csum[c] - csum[s]))
        e = int(np.searchsorted(csum, csum[c] + budget, side="right")) - 1
        e = max(e, c + 1)  # the reference never terminates on a sentence longer than the budget
        segments.append((s, c, min(e, n)))
        c = min(e, n)
    return segments


def largest_remainder_sizes(num_rows: int, segment_tokens: np.ndarray) -> np.ndarray:
    """Token rows per sentence (``_embed.py:122-128``), same NumPy ops as the reference so that the
    tie-breaking of ``argsort`` is identical."""
    frac = num_rows * (segment_tokens / np.sum(segment_tokens))
    size = np.floor(frac).astype(np.intp)
    remainder = num_rows - np.sum(size)
    if remainder > 0:
        size[np.argsort(frac - size)[-remainder:]] += 1
    return size


def segment_mean_pool(X: torch.Tensor, row_begin: np.ndarray, row_end: np.ndarray, *, normalize: int) -> torch.Tensor:
    """``rl_segment_mean_pool``: fp16 ``[S, d]`` device tensor from float32 token rows ``X [T, d]``."""
    lib = _lib.load()
    if X.dtype != torch.float32 or X.ndim != 2 or not X.is_cuda or X.stride(1) != 1:
        raise ValueError("X must be a CUDA float32 [T, d] tensor with unit inner stride")
    S, d = len(row_begin), int(X.shape[1])
    rb = torch.from_numpy(np.ascontiguousarray(row_begin, dtype=np.int32)).to(X.device)
    re = torch.from_numpy(np.ascontiguousarray(row_end, dtype=np.int32)).to(X.device)
    out = torch.empty((S, d), dtype=torch.float16, device=X.device)
    with torch.cuda.device(X.device):
        check(lib.rl_segment_mean_pool(X.data_ptr(), X.stride(0), d, rb.data_ptr(), re.data_ptr(), S, normalize,
                                       out.data_ptr(), torch.cuda.current_stream().cuda_stream),
              "rl_segment_mean_pool")
    return out


def _device_path(model: Any) -> bool:
    """Whether the embedder runs packed forwards whose token rows stay on the device."""
    return hasattr(model, "embed_token_ids") and hasattr(model, "token_ids_for_embedding")


def pool_segments(  # noqa: PLR0913
    segment_embeddings: Sequence[np.ndarray | torch.Tensor] | torch.Tensor, num_tokens: np.ndarray,
    segments: Sequence[tuple[int, int, int]], *, normalize: bool = True, device: Any | None = None,
    row_offsets: np.ndarray | None = None,
) -> torch.Tensor:
    """Pool all segments of a document in ONE kernel launch: stack the token matrices, list the
    content sentences' row ranges (preamble sentences are skipped, ``_embed.py:133``).  With ``row_offsets``
    (``[n_segments + 1]``), ``segment_embeddings`` is already the packed float32 ``[T, d]`` device matrix and
    segment i owns its rows ``row_offsets[i] : row_offsets[i + 1]``."""
    if row_offsets is None:
        device = torch.device(device if device is not None else "cuda")
        mats = [torch.as_tensor(np.asarray(x, dtype=np.float32) if not isinstance(x, torch.Tensor) else x)
                for x in segment_embeddings]
        X = torch.cat([m.to(device=device, dtype=torch.float32, non_blocking=True) for m in mats], dim=0)
        rows = [int(m.shape[0]) for m in mats]
    else:
        X = segment_embeddings
        rows = np.diff(np.asarray(row_offsets)).tolist()
    begins, ends = [], []
    base = 0
    for n, (s, c, e) in zip(rows, segments, strict=True):
        sizes = largest_remainder_sizes(n, np.asarray(num_tokens[s:e]))
        cuts = np.concatenate([[0], np.cumsum(sizes)]) + base
        begins.append(cuts[c - s : -1])
        ends.append(cuts[c - s + 1 :])
        base += n
    return segment_mean_pool(X.contiguous(), np.concatenate(begins), np.concatenate(ends), normalize=1 if normalize else 0)


def _pool_planned(model: Any, texts: list[str], num_tokens: np.ndarray, segments: list[tuple[int, int, int]], *,
                  normalize: bool) -> torch.Tensor:
    """Embed the planned segments (``texts[i]`` is the text of ``segments[i]``) and pool them."""
    if _device_path(model):
        X, offs = model.embed_token_ids(model.token_ids_for_embedding(texts))
        return pool_segments(X, num_tokens, segments, normalize=normalize, row_offsets=offs)
    seg_emb = [np.asarray(model.embed(t), dtype=np.float32) for t in texts]
    return pool_segments(seg_emb, num_tokens, segments, normalize=normalize)


def embed_strings_with_late_chunking(sentences: list[str], *, config: RAGLiteConfig | None = None) -> FloatMatrix:
    """Embed a document's sentences with late chunking (``_embed.py:16-141``); fp16 ``[n, d]``."""
    config = config or RAGLiteConfig()
    assert config.embedder.startswith("llama-cpp-python")
    model = _token_embedder(config)
    num_tokens = count_tokens(sentences, model)
    segments = plan_segments(num_tokens, model.n_ctx(), model.n_batch)
    texts = ["".join(sentences[s:e]) for (s, _, e) in segments]
    return _pool_planned(model, texts, num_tokens, segments, normalize=config.embedder_normalize).cpu().numpy()


def _mean_pool_device(strings: Sequence[str], config: RAGLiteConfig) -> torch.Tensor:
    """fp16 ``[n, d]`` device rows of ``embed_strings_without_late_chunking``: on the device path every string runs in
    one packed forward and one pool launch (a string's row does not depend on the others in the call)."""
    model = _token_embedder(config)
    if _device_path(model):
        X, offs = model.embed_token_ids(model.token_ids_for_embedding(list(strings)))
        return segment_mean_pool(X, offs[:-1], offs[1:], normalize=2 if config.embedder_normalize else 0)
    outs = []
    for i in range(0, len(strings), 96):  # batch size 96 (_embed.py:173)
        mats = [np.asarray(m, dtype=np.float32) for m in model.embed(list(strings[i : i + 96]))]
        X = torch.from_numpy(np.concatenate(mats, axis=0)).cuda()
        cuts = np.concatenate([[0], np.cumsum([len(m) for m in mats])])
        outs.append(segment_mean_pool(X, cuts[:-1], cuts[1:], normalize=2 if config.embedder_normalize else 0))
    return torch.cat(outs, dim=0)


def embed_strings_without_late_chunking(strings: list[str], *, config: RAGLiteConfig | None = None) -> FloatMatrix:
    """Plain per-string mean pool (``_embed.py:144-184``) for llama-like embedders; API embedders
    (LiteLLM) are outside the accelerated path."""
    return _mean_pool_device(strings, config or RAGLiteConfig()).cpu().numpy()


def embed_queries(queries: Sequence[str], *, config: RAGLiteConfig | None = None) -> FloatMatrix:
    """fp16 ``[B, d]`` embeddings of a batch of query strings; row b equals ``embed_strings([queries[b]])[0]`` bit for
    bit.  Each query is planned as a one-sentence document, exactly as ``embed_strings`` plans it, and all of their
    segments run in one packed forward and one pool launch, ready for ``vector_search_batch(...,
    queries_are_fp16=True)``.  An embedder without the device path embeds the queries one by one."""
    config = config or RAGLiteConfig()
    queries = list(queries)
    model = _token_embedder(config)
    if not queries or not _device_path(model):
        rows = [embed_strings([q], config=config)[0] for q in queries]
        return np.stack(rows) if rows else np.zeros((0, model.n_embd()), dtype=np.float16)
    if embedding_type(config=config) != "late_chunking":
        return embed_strings_without_late_chunking(queries, config=config)
    texts, all_tokens, all_segments = [], [], []
    base = 0
    for q in queries:
        num_tokens = count_tokens([q], model)
        for s, c, e in plan_segments(num_tokens, model.n_ctx(), model.n_batch):
            texts.append(q)   # ("".join of the query's single sentence)
            all_segments.append((s + base, c + base, e + base))
        all_tokens.append(num_tokens)
        base += len(num_tokens)
    return _pool_planned(model, texts, np.concatenate(all_tokens), all_segments,
                         normalize=config.embedder_normalize).cpu().numpy()


def embedding_type(*, config: RAGLiteConfig | None = None) -> str:
    """``_embed.py:187-190``."""
    config = config or RAGLiteConfig()
    return "late_chunking" if config.embedder.startswith("llama-cpp-python") else "standard"


def embed_strings(strings: list[str], *, config: RAGLiteConfig | None = None) -> FloatMatrix:
    """``_embed.py:193-200``."""
    config = config or RAGLiteConfig()
    if embedding_type(config=config) == "late_chunking":
        return embed_strings_with_late_chunking(strings, config=config)
    return embed_strings_without_late_chunking(strings, config=config)
