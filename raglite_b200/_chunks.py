"""Chunklets and chunks on the GPU -- ``split_chunklets`` and ``split_chunks`` as ``raglite/_split_chunklets.py`` and
``raglite/_split_chunks.py`` compute them, and ``split_documents``, steps 1-4 of the reference's
``_create_chunk_records`` (``_insert.py:93-101``) for many documents.

* ``split_chunklets``: the Markdown boundary probabilities and the statement counts stay on the host (NumPy, as the
  reference computes them); ``rl_chunklet_partition`` runs the reference's dynamic program, one warp per document, bit
  for bit but for the square (DESIGN.md section 5).
* ``split_chunks``: the input checks, the early exit, the size quantiles and the heading flags stay on the host;
  ``rl_chunk_similarities`` computes the cut costs in float32 and ``rl_chunk_partition`` the exact optimum of the
  reference's integer program, which is a windowed dynamic program over those costs.
"""

from __future__ import annotations

import re
from collections.abc import Callable, Sequence
from typing import Any

import numpy as np
import torch

from . import _lib
from ._config import RAGLiteConfig
from ._embed import (
    _device_path,
    _pool_planned,
    _token_embedder,
    count_tokens,
    embed_strings,
    embedding_type,
    plan_segments,
)
from ._lib import check
from ._sentences import markdown_sentence_boundaries, split_sentences_batch

# token type -> chunklet boundary probability of the sentence holding its first line (_split_chunklets.py:29-35)
CHUNKLET_BOUNDARY_PROBA = {"blockquote_open": 0.75, "bullet_list_open": 0.25, "heading_open": 1.0,
                           "paragraph_open": 0.5, "ordered_list_open": 0.25}
EMPTY_DOCUMENT = "attempt to get argmax of an empty sequence"   # what the reference's empty list raises
CHUNKLET_TOO_LARGE = "Chunklet larger than chunk max_size detected."
ZERO_NORM = "Chunklet embeddings with zero norm detected."
_HEADING = re.compile(r"^#+\s")


def _parse(doc: str) -> list[Any]:
    from markdown_it import MarkdownIt

    return MarkdownIt().parse(doc)


def markdown_chunklet_boundaries(sentences: Sequence[str], tokens: list[Any] | None = None) -> np.ndarray:
    """Chunklet boundary probability of each sentence (``_split_chunklets.py:11-55``): a block token's probability goes
    to the sentence holding its first line unless the previous such token went to the same sentence; within each run of
    nonzero probabilities only the first maximum stays.  ``tokens`` is markdown-it's parse of ``"".join(sentences)``
    when the caller already has it."""
    doc = "".join(sentences)
    if tokens is None:
        tokens = _parse(doc)
    line_len = np.fromiter((len(x) for x in doc.splitlines(keepends=True)), dtype=np.int64)
    line_start = np.r_[np.int64(0), np.cumsum(line_len)[:-1]]
    sent_start = np.r_[np.int64(0), np.cumsum(np.fromiter((len(s) for s in sentences), dtype=np.int64))]
    line_sentence = np.searchsorted(sent_start, line_start, side="right") - 1
    out = np.zeros(len(sentences))
    last = -1
    for t in tokens:
        p = CHUNKLET_BOUNDARY_PROBA.get(t.type)
        if p is not None and (i := int(line_sentence[t.map[0]])) != last:
            out[i] = p
            last = i
    if len(out) == 0:
        raise ValueError(EMPTY_DOCUMENT)
    nz = out != 0.0
    edges = np.r_[0, np.flatnonzero(nz[1:] != nz[:-1]) + 1, len(out)]
    for a, e in zip(edges[:-1], edges[1:], strict=True):
        if nz[a]:
            k = a + int(np.argmax(out[a:e]))
            v = out[k]
            out[a:e] = 0.0
            out[k] = v
    return out


def num_statements(sentences: Sequence[str]) -> np.ndarray:
    """Approximate statements per sentence (``_split_chunklets.py:58-71``): 0.75 at the first quartile of the word
    counts, rising linearly below it from 0 and above it by 0.5 per interquartile range."""
    words = np.asarray([len(s.split()) for s in sentences], dtype=np.float64)
    q25, q75 = np.quantile(words, [0.25, 0.75])
    tiny = np.sqrt(np.finfo(np.float64).eps)
    q25 = max(q25, tiny)
    q75 = max(q75, q25 + tiny)
    return np.where(words <= q25, 0.75 * words / q25, 0.75 + 0.5 * (words - q25) / (q75 - q25))


def _up(a: np.ndarray, dev: Any) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _offsets(counts: Sequence[int]) -> np.ndarray:
    off = np.zeros(len(counts) + 1, np.int64)
    np.cumsum(np.asarray(counts, dtype=np.int64), out=off[1:])
    return off


def _join_pieces(items: Sequence[str], cuts: Sequence[int]) -> list[str]:
    return ["".join(items[a:b]) for a, b in zip([0, *cuts], [*cuts, len(items)], strict=True)]


def _check_max_size(max_size: int) -> None:
    if not 0 <= max_size < 2**31:
        raise ValueError(f"max_size={max_size} unsupported: the device takes 0 <= max_size < 2^31")


# ---- chunklets -----------------------------------------------------------------------------------------------------------
def _chunklet_cuts(docs_sentences: Sequence[Sequence[str]], max_size: int,
                   tokens: Sequence[list[Any] | None] | None = None) -> list[list[int]]:
    """The partition indices of every document, one ``rl_chunklet_partition`` launch."""
    _check_max_size(max_size)
    D = len(docs_sentences)
    if D == 0:
        return []
    p = [markdown_chunklet_boundaries(s, None if tokens is None else tokens[i]) for i, s in enumerate(docs_sentences)]
    st = [num_statements(s) for s in docs_sentences]
    lens = np.fromiter((len(x) for s in docs_sentences for x in s), dtype=np.int64)
    if lens.size and lens.max() >= 2**31:
        raise ValueError("a sentence of 2^31 or more characters is unsupported")
    off = _offsets([len(s) for s in docs_sentences])
    N = int(off[-1])
    lib, dev = _lib.load(), torch.device("cuda", torch.cuda.current_device())
    d_p, d_s = _up(np.concatenate(p), dev), _up(np.concatenate(st), dev)
    d_len, d_off = _up(lens.astype(np.int32), dev), _up(off, dev)
    d_max = torch.full((D,), max_size, dtype=torch.int32, device=dev)
    cuts = torch.empty(max(N, 1), dtype=torch.int32, device=dev)
    cs = torch.empty(2 * D, dtype=torch.int32, device=dev)
    ws = torch.empty(int(lib.rl_chunklet_partition_workspace_bytes(N, D)), dtype=torch.uint8, device=dev)
    check(lib.rl_chunklet_partition(d_p.data_ptr(), d_s.data_ptr(), d_len.data_ptr(), d_off.data_ptr(),
                                    d_max.data_ptr(), D, N, cuts.data_ptr(), cs.data_ptr(), cs[D:].data_ptr(),
                                    ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream),
          "rl_chunklet_partition")
    h_cuts, h_cs = cuts.cpu().numpy(), cs.cpu().numpy()
    return [h_cuts[off[i]:off[i] + h_cs[i]].tolist() for i in range(D)]


def split_chunklets_batch(docs_sentences: Sequence[Sequence[str]], *, max_size: int = 2048) -> list[list[str]]:
    """``split_chunklets`` of every document with its default costs, one partition launch for the whole batch."""
    docs_sentences = [list(s) for s in docs_sentences]
    return [_join_pieces(s, c) for s, c in zip(docs_sentences, _chunklet_cuts(docs_sentences, max_size), strict=True)]


def split_chunklets(sentences: list[str], boundary_cost: Callable[[np.ndarray], float] | None = None,
                    statement_cost: Callable[[float], float] | None = None, max_size: int = 2048) -> list[str]:
    """Split a document's sentences into chunklets (``raglite._split_chunklets.split_chunklets``): the partition into
    pieces of at most ``max_size`` characters (a longer sentence stays whole, as in the reference) minimising the sum of
    (1 - p_first) + sum(p_rest) + (s - 3)^2 / sqrt(s) / 2 over the pieces.  Only the default costs run on the GPU."""
    if boundary_cost is not None or statement_cost is not None:
        raise NotImplementedError("custom boundary_cost / statement_cost are unsupported: the chunklet partition runs "
                                  "the default costs on the GPU (the reference's O(1) cost path)")
    return split_chunklets_batch([sentences], max_size=max_size)[0]


# ---- chunks --------------------------------------------------------------------------------------------------------------
def is_heading(chunklet: str) -> bool:
    """Whether the chunklet starts a Markdown heading (``_split_chunks.py:76``)."""
    return _HEADING.match(chunklet.replace("\n", "").strip()) is not None


def _check_chunks(chunklets: Sequence[str], emb: np.ndarray, max_size: int) -> np.ndarray:
    """The reference's input checks, in its order; returns the chunklet sizes."""
    size = np.asarray([len(c) for c in chunklets])
    if not np.all(size <= max_size):
        raise ValueError(CHUNKLET_TOO_LARGE)
    if not np.all(np.linalg.norm(emb, axis=1) > 0.0):
        raise ValueError(ZERO_NORM)
    return size


def _nonoutlying(size: np.ndarray) -> np.ndarray:
    q15, q85 = np.quantile(size, [0.15, 0.85])
    return (q15 <= size) & (size <= q85)


def chunk_cut_costs(X: torch.Tensor, row_off: np.ndarray, sizes: Sequence[np.ndarray],
                    headings: Sequence[Sequence[bool]]) -> tuple[torch.Tensor, np.ndarray]:
    """``rl_chunk_similarities`` of every document: float32 cut costs on the device (document d's at
    ``row_off[d] .. row_off[d + 1] - 1``) and the per-document status (1: a zero-norm row)."""
    lib, dev = _lib.load(), X.device
    if X.dtype not in (torch.float16, torch.float32) or X.ndim != 2 or X.stride(1) != 1:
        raise ValueError("X must be a float16 or float32 [n, d] tensor with unit inner stride")
    D, N = len(sizes), int(row_off[-1])
    nonout = np.concatenate([_nonoutlying(s) for s in sizes]) if N else np.zeros(0, bool)
    head = np.fromiter((h for hs in headings for h in hs), dtype=bool, count=N)
    costs = torch.empty(max(N, 1), dtype=torch.float32, device=dev)
    status = torch.empty(max(D, 1), dtype=torch.int32, device=dev)
    ws = torch.empty(int(lib.rl_chunk_similarities_workspace_bytes(N)), dtype=torch.uint8, device=dev)
    d_off, d_non, d_head = _up(row_off.astype(np.int64), dev), _up(nonout.view(np.uint8), dev), _up(head.view(np.uint8), dev)
    check(lib.rl_chunk_similarities(X.data_ptr(), 1 if X.dtype == torch.float16 else 0, X.stride(0), int(X.shape[1]),
                                    d_off.data_ptr(), D, N, d_non.data_ptr(), d_head.data_ptr(), costs.data_ptr(),
                                    status.data_ptr(), ws.data_ptr(), ws.numel(),
                                    torch.cuda.current_stream().cuda_stream), "rl_chunk_similarities")
    return costs, status[:D].cpu().numpy()


def chunk_partition(costs: torch.Tensor, row_off: np.ndarray, sizes: Sequence[np.ndarray], max_size: int
                    ) -> list[list[int]]:
    """``rl_chunk_partition`` of every document: its partition indices (chunklets that start a chunk, but the first)."""
    _check_max_size(max_size)
    lib, dev = _lib.load(), costs.device
    D, N = len(sizes), int(row_off[-1])
    lens = np.concatenate([np.asarray(s, dtype=np.int32) for s in sizes]) if N else np.zeros(0, np.int32)
    d_len, d_off = _up(lens, dev), _up(row_off.astype(np.int64), dev)
    d_max = torch.full((D,), max_size, dtype=torch.int32, device=dev)
    cuts = torch.empty(max(N, 1), dtype=torch.int32, device=dev)
    cs = torch.empty(2 * D, dtype=torch.int32, device=dev)
    ws = torch.empty(int(lib.rl_chunk_partition_workspace_bytes(N, D)), dtype=torch.uint8, device=dev)
    check(lib.rl_chunk_partition(costs.data_ptr(), d_len.data_ptr(), d_off.data_ptr(), d_max.data_ptr(), D, N,
                                 cuts.data_ptr(), cs.data_ptr(), cs[D:].data_ptr(), ws.data_ptr(), ws.numel(),
                                 torch.cuda.current_stream().cuda_stream), "rl_chunk_partition")
    h_cuts, h_cs = cuts.cpu().numpy(), cs.cpu().numpy()
    if h_cs[D:].any():
        raise ValueError(CHUNKLET_TOO_LARGE)
    return [h_cuts[row_off[i]:row_off[i] + h_cs[i]].tolist() for i in range(D)]


def _split_chunks_all(docs_chunklets: Sequence[Sequence[str]], docs_embeddings: Sequence[np.ndarray], max_size: int,
                      device_rows: tuple[torch.Tensor, np.ndarray] | None = None
                      ) -> list[tuple[list[str], list[np.ndarray]]]:
    """``split_chunks`` of every document: checks and early exits on the host, one similarity and one partition launch
    per embedding width for the rest.  ``device_rows`` = (X, row offsets) when the rows already lie on the device."""
    _check_max_size(max_size)
    out: list[Any] = []
    todo: list[int] = []
    for i, (chunklets, emb) in enumerate(zip(docs_chunklets, docs_embeddings, strict=True)):
        size = _check_chunks(chunklets, emb, max_size)
        if len(chunklets) <= 1 or sum(size) <= max_size:
            out.append((["".join(chunklets)] if chunklets else list(chunklets), [emb]))
        else:
            out.append(None)
            todo.append(i)
    if not todo:
        return out
    if device_rows is not None:
        groups = [todo]
    else:                                  # one launch per embedding width: each document is its own problem
        widths = sorted({int(docs_embeddings[i].shape[1]) for i in todo})
        groups = [[i for i in todo if docs_embeddings[i].shape[1] == w] for w in widths]
    for group in groups:
        for i, c in zip(group, _chunk_cuts(docs_chunklets, docs_embeddings, group, max_size, device_rows), strict=True):
            out[i] = (_join_pieces(docs_chunklets[i], c), np.split(docs_embeddings[i], c))
    return out


def _chunk_cuts(docs_chunklets: Sequence[Sequence[str]], docs_embeddings: Sequence[np.ndarray], todo: list[int],
                max_size: int, device_rows: tuple[torch.Tensor, np.ndarray] | None) -> list[list[int]]:
    """The partitions of documents ``todo`` (rows of one width): one similarity and one partition launch."""
    sizes = [np.asarray([len(c) for c in docs_chunklets[i]]) for i in todo]
    row_off = _offsets([len(docs_chunklets[i]) for i in todo])
    if device_rows is not None:
        X_all, all_off = device_rows
        idx = np.concatenate([np.arange(all_off[i], all_off[i + 1]) for i in todo])
        X = X_all if len(idx) == len(X_all) else X_all[torch.from_numpy(idx).to(X_all.device)]
    else:
        embs = [docs_embeddings[i] for i in todo]
        dt = np.float16 if all(e.dtype == np.float16 for e in embs) else np.float32
        X = _up(np.concatenate([np.asarray(e, dtype=dt) for e in embs]), torch.device("cuda", torch.cuda.current_device()))
    costs, status = chunk_cut_costs(X, row_off, sizes, [[is_heading(c) for c in docs_chunklets[i]] for i in todo])
    if status.any():
        raise ValueError(ZERO_NORM)
    return chunk_partition(costs, row_off, sizes, max_size)


def split_chunks_batch(docs_chunklets: Sequence[Sequence[str]], docs_embeddings: Sequence[np.ndarray], *,
                       max_size: int = 2048) -> list[tuple[list[str], list[np.ndarray]]]:
    """``split_chunks`` of every document; the documents past the early exit whose rows have the same width share one
    launch of each kernel."""
    return _split_chunks_all([list(c) for c in docs_chunklets], list(docs_embeddings), max_size)


def split_chunks(chunklets: list[str], chunklet_embeddings: np.ndarray, max_size: int = 2048
                 ) -> tuple[list[str], list[np.ndarray]]:
    """Split chunklets into chunks (``raglite._split_chunks.split_chunks``): the partition into chunks of at most
    ``max_size`` characters with the least total cost of its cuts, a cut costing the similarity of its two neighbouring
    chunklets after the discourse vector is removed.  Returns the chunks and ``np.split`` of the caller's rows."""
    return split_chunks_batch([chunklets], [chunklet_embeddings], max_size=max_size)[0]


# ---- embeddings and whole documents --------------------------------------------------------------------------------------
def _embed_batch_device(docs_strings: Sequence[Sequence[str]], config: RAGLiteConfig
                        ) -> tuple[torch.Tensor, np.ndarray]:
    """fp16 ``[sum n_b, d]`` device rows of every document's ``embed_strings`` and the row offsets.  With a
    late-chunking embedder on the device path, every document is planned as ``embed_strings`` plans it and all of their
    segments run in packed forwards and one pool launch (as ``embed_queries`` does); otherwise document by document."""
    model = _token_embedder(config)
    off = _offsets([len(s) for s in docs_strings])
    dev = torch.device("cuda", torch.cuda.current_device())
    if not _device_path(model) or embedding_type(config=config) != "late_chunking":
        mats = [torch.from_numpy(np.asarray(embed_strings(list(s), config=config))).to(dev) for s in docs_strings if s]
        return (torch.cat(mats) if mats else torch.zeros((0, 1), dtype=torch.float16, device=dev)), off
    texts, all_tokens, all_segments = [], [], []
    for b, strings in enumerate(docs_strings):
        strings = list(strings)
        if not strings:
            continue
        num_tokens = count_tokens(strings, model)
        for s, c, e in plan_segments(num_tokens, model.n_ctx(), model.n_batch):
            texts.append("".join(strings[s:e]))
            all_segments.append((s + int(off[b]), c + int(off[b]), e + int(off[b])))
        all_tokens.append(num_tokens)
    if not texts:
        return torch.zeros((0, model.n_embd()), dtype=torch.float16, device=dev), off
    return _pool_planned(model, texts, np.concatenate(all_tokens), all_segments,
                         normalize=config.embedder_normalize), off


def embed_strings_batch(docs_strings: Sequence[Sequence[str]], *, config: RAGLiteConfig | None = None
                        ) -> list[np.ndarray]:
    """``embed_strings(docs_strings[b], config=config)`` for every document b, bit for bit: with a late-chunking
    embedder on the device path, all documents' segments run in packed forwards and one pool launch."""
    config = config or RAGLiteConfig()
    X, off = _embed_batch_device(docs_strings, config)
    host = X.cpu().numpy()
    return [host[off[b]:off[b + 1]] for b in range(len(docs_strings))]


def split_documents(docs: Sequence[str], *, config: RAGLiteConfig | None = None
                    ) -> list[tuple[list[str], list[np.ndarray]]]:
    """Steps 1-4 of the reference's ``_create_chunk_records`` for every document: ``split_sentences`` (``max_len`` =
    ``config.chunk_max_size``), ``split_chunklets``, ``embed_strings`` and ``split_chunks`` (``max_size`` the same).
    Returns what ``split_chunks`` returns, per document.  Each document is parsed by markdown-it once; the chunklet
    embeddings stay on the device from the pool to the similarity kernel."""
    config = config or RAGLiteConfig()
    docs = list(docs)
    _token_embedder(config)                       # the embedder's error before any device work
    max_size = int(config.chunk_max_size)
    parsed = {d: _parse(d) for d in docs}
    sentences = split_sentences_batch(docs, max_len=max_size,
                                      boundary_probas=lambda d: markdown_sentence_boundaries(d, tokens=parsed[d]))
    cuts = _chunklet_cuts(sentences, max_size, [parsed[d] for d in docs])
    chunklets = [_join_pieces(s, c) for s, c in zip(sentences, cuts, strict=True)]
    X, off = _embed_batch_device(chunklets, config)
    host = X.cpu().numpy()
    return _split_chunks_all(chunklets, [host[off[b]:off[b + 1]] for b in range(len(docs))], max_size,
                             device_rows=(X, off))
