"""Ingest on the GPU: drop-in ``insert_documents``, ``delete_documents`` and ``delete_documents_by_metadata``
(``raglite/_insert.py``, ``raglite/_delete.py``) over the index registered for ``config.db_url``, and the reference's
document and chunk records (``Document``, ``Chunk.from_body`` and its heading rules, ``_database.py:151-277``).

``insert_documents`` runs ``_create_chunk_records`` (``_insert.py:88-155``) for every new document with the rows on the
device: sentences, chunklets, chunklet embeddings and chunks come from ``_split_documents_device`` (the steps behind
``split_documents``); the chunk records are built on the host; the rows of a chunk are its chunklets' rows
(``late_chunking``), or with the ``standard`` embedding type the α-blend ``rl_chunk_embedding_blend`` computes from the
chunklet rows and one packed forward over every chunk's ``content``.  All documents are processed before the index is
touched, and the rows enter it in one ``CorpusIndex.append``: a failure leaves the index as it was, as the reference's
rollback leaves the database.

The index keeps the ``Document`` records ``insert_documents`` saw (``CorpusIndex.documents``), which is the table
``delete_documents_by_metadata`` matches against.  Documents whose chunks reached the index another way (``append``,
``from_table_rows``) have no record there and never match it; ``delete_documents`` finds them by their chunks.
"""

from __future__ import annotations

from collections.abc import Sequence
from dataclasses import dataclass, field
from hashlib import sha256
from pathlib import Path
from typing import Any

import numpy as np
import torch

from . import _lib
from ._chunks import _join_pieces, _offsets, _parse, _split_documents_device
from ._config import RAGLiteConfig
from ._embed import _mean_pool_device, _token_embedder, embedding_type
from ._index import Chunk, CorpusIndex, fp16_rows_unit_scale_device, get_index, register_index
from ._lib import check
from ._typing import DocumentId

ALPHA = 0.15                 # weight of the chunklet row in the standard embedding type's blend (_insert.py:132)
_GROUP_TOKEN_BYTES = 4 << 30  # float32 token rows one group of documents may hold on the device at once
EMPTY_FILTER = "metadata_filter cannot be empty to prevent accidental deletion of all documents"


def adapt_metadata(metadata: dict[str, Any] | None) -> dict[str, list[Any]]:
    """Every metadata value made a list (``_database.py:51-55``)."""
    return {k: v if isinstance(v, list) else [v] for k, v in (metadata or {}).items()}


def hash_bytes(data: bytes) -> str:
    """The first 16 hex digits of the SHA-256 of ``data``: document and chunk ids."""
    return sha256(data, usedforsecurity=False).hexdigest()[:16]


@dataclass
class Document:
    """Stand-in for ``raglite._database.Document``: the record ``insert_documents`` takes, with its ``content``."""

    id: DocumentId
    filename: str
    url: str | None = None
    metadata_: dict[str, Any] = field(default_factory=dict)
    content: str | None = None

    @staticmethod
    def from_text(content: str, *, id: DocumentId | None = None, url: str | None = None,  # noqa: A002
                  filename: str | None = None, **kwargs: Any) -> "Document":
        """A document from Markdown or plain text: the id hashes the content, the filename defaults to the first
        non-blank line cut to 80 characters (plus ``...``), and the metadata holds ``filename``, ``uri`` (the given
        id), ``url``, ``size`` (UTF-8 bytes) and ``kwargs``, every value a list."""
        first_line = content.strip().split("\n", 1)[0].strip()
        if len(first_line) > 80:  # noqa: PLR2004
            first_line = first_line[:80] + "..."
        name = filename or first_line
        metadata = {"filename": name, "uri": id, "url": url, "size": len(content.encode()), **kwargs}
        return Document(id=id if id is not None else hash_bytes(content.encode()), filename=name, url=url,
                        metadata_=adapt_metadata(metadata), content=content)

    @staticmethod
    def from_path(doc_path: Path | str, *, id: DocumentId | None = None, url: str | None = None,  # noqa: A002
                  **kwargs: Any) -> "Document":
        """A document from a ``.md`` or ``.txt`` file, read as text: the id hashes the file's bytes, and the metadata
        holds ``filename``, ``uri``, ``url``, ``size``, ``created``, ``modified`` and ``kwargs``.  Other formats need a
        Markdown conversion this package does not do: ``ValueError``."""
        doc_path = Path(doc_path)
        if doc_path.suffix not in (".md", ".txt"):
            raise ValueError(f"{doc_path.name}: only .md and .txt files are read; convert other formats to Markdown "
                             "and use Document.from_text")
        st = doc_path.stat()
        metadata = {"filename": doc_path.name, "uri": id, "url": url, "size": st.st_size, "created": st.st_ctime,
                    "modified": st.st_mtime, **kwargs}
        return Document(id=id if id is not None else hash_bytes(doc_path.read_bytes()), filename=doc_path.name, url=url,
                        metadata_=adapt_metadata(metadata), content=doc_path.read_text())


# ---- chunk records (_database.py:227-277) ---------------------------------------------------------------------------------
def extract_heading_lines(doc: str, leading_only: bool = False) -> list[str]:  # noqa: FBT001, FBT002
    """The Markdown heading state after ``doc``: six slots, slot L - 1 holding ``"#" * L + " " + text`` of the last
    level-L heading (newlines in it become spaces) and "" where unset; a heading clears every deeper slot.  With
    ``leading_only`` the scan stops at the first token outside a heading that has non-blank content."""
    slots = [""] * 6
    level = 0
    for tok in _parse(doc):
        if tok.type == "heading_open":
            level = int(tok.tag[1])
        elif tok.type == "heading_close":
            level = 0
        elif level:
            slots[level - 1:] = ["#" * level + " " + tok.content.strip().replace("\n", " ")] + [""] * (6 - level)
        elif leading_only and tok.content and not tok.content.isspace():
            break
    return slots


def truncate_headings(headings: str, body: str) -> str:
    """The contextual headings ``headings`` leaves for a chunk whose ``body`` opens with a heading of level L: the
    slots of level L and deeper are dropped."""
    slots = extract_heading_lines(headings)
    lead = extract_heading_lines(body, leading_only=True)
    first = next((i for i, s in enumerate(lead) if s), None)
    if first is not None:
        slots[first:] = [""] * (6 - first)
    return "\n".join(s for s in slots if s)


def extract_headings(chunk: Chunk) -> str:
    """The headings in force after ``chunk``, starting from its contextual headings."""
    return "\n".join(s for s in extract_heading_lines(chunk.headings + "\n\n" + chunk.body) if s)


def chunk_from_body(document: Document, index: int, body: str, headings: str = "", **kwargs: Any) -> Chunk:
    """Chunk ``index`` of ``document`` (``Chunk.from_body``): id = the hash of ``"{document.id}-{index}"``."""
    return Chunk(id=hash_bytes(f"{document.id}-{index}".encode()), document_id=document.id, index=index,
                 headings=truncate_headings(headings, body), body=body,
                 metadata_=adapt_metadata({"filename": document.filename, "url": document.url, **kwargs}))


def chunk_records(document: Document, bodies: Sequence[str]) -> list[Chunk]:
    """The ``Chunk`` records of a document's chunks, the headings carried from each chunk to the next."""
    records: list[Chunk] = []
    headings = ""
    for i, body in enumerate(bodies):
        records.append(chunk_from_body(document, i, body, headings, **document.metadata_))
        headings = extract_headings(records[-1])
    return records


# ---- rows ---------------------------------------------------------------------------------------------------------------
def chunk_embedding_blend(X: torch.Tensor, F: torch.Tensor, chunk_off: np.ndarray | Sequence[int],
                          alpha: float = ALPHA) -> torch.Tensor:
    """``rl_chunk_embedding_blend``: fp16 ``[N, d]`` device rows ``alpha * X[r] + (1 - alpha) * F[chunk(r)]`` as NumPy
    evaluates that expression on float16 rows with Python float weights (each weight rounded to float16, each product
    and the sum rounded to float16).  ``X`` fp16 ``[N, d]`` chunklet rows, ``F`` fp16 ``[C, d]`` full-chunk rows,
    ``chunk_off`` the ``[C + 1]`` CSR of the chunks' rows."""
    if (X.dtype != torch.float16 or F.dtype != torch.float16 or X.ndim != 2 or F.ndim != 2 or not X.is_cuda
            or X.stride(1) != 1 or X.shape[1] != F.shape[1] or F.device != X.device):
        raise ValueError("X and F must be float16 [N, d] / [C, d] tensors on one CUDA device, X with unit inner stride")
    F = F.contiguous()
    N, d, C = int(X.shape[0]), int(X.shape[1]), int(F.shape[0])
    off = np.ascontiguousarray(np.asarray(chunk_off, dtype=np.int64))
    if len(off) != C + 1 or off[0] != 0 or off[-1] != N or np.any(np.diff(off) < 0):
        raise ValueError("chunk_off must be a CSR offset array of F's chunks over X's rows")
    a, b = (int(np.float16(w).view(np.uint16)) for w in (alpha, 1 - alpha))
    out = torch.empty((N, d), dtype=torch.float16, device=X.device)
    with torch.cuda.device(X.device):
        d_off = torch.from_numpy(off).to(X.device)
        check(_lib.load().rl_chunk_embedding_blend(X.data_ptr(), X.stride(0), F.data_ptr(), d_off.data_ptr(), C, N, d,
                                                   a, b, out.data_ptr(), torch.cuda.current_stream().cuda_stream),
              "rl_chunk_embedding_blend")
    return out


def _document_rows(docs: Sequence[Document], config: RAGLiteConfig
                   ) -> tuple[list[Chunk], torch.Tensor, np.ndarray]:
    """``(chunk records, fp16 device rows, rows per chunk)`` of a group of documents, in document order."""
    chunklets, X, _, cuts = _split_documents_device([doc.content for doc in docs], config)
    records: list[Chunk] = []
    counts: list[np.ndarray] = []
    for doc, c, cut in zip(docs, chunklets, cuts, strict=True):
        records += chunk_records(doc, _join_pieces(c, cut))
        counts.append(np.diff([0, *cut, len(c)]))
    rows_per_chunk = np.concatenate(counts).astype(np.int64)
    if embedding_type(config=config) == "late_chunking":
        return records, X, rows_per_chunk
    F = _mean_pool_device([r.content for r in records], config)
    if not config.vector_search_multivector:
        return records, F, np.ones(len(records), dtype=np.int64)
    return records, chunk_embedding_blend(X, F, _offsets(rows_per_chunk)), rows_per_chunk


def _document_groups(docs: Sequence[Document], config: RAGLiteConfig) -> list[list[Document]]:
    """Consecutive runs of documents whose float32 token rows stay under ``_GROUP_TOKEN_BYTES``, counting a token per
    character (a token covers at least one) and late chunking's preamble (at most 0.382 / 0.618 of a segment's
    content is repeated)."""
    model = _token_embedder(config)
    width = int(model.n_embd()) if hasattr(model, "n_embd") else 1024
    groups: list[list[Document]] = []
    used = _GROUP_TOKEN_BYTES
    for doc in docs:
        need = int((len(doc.content) / 0.618 + 64) * 4 * width)
        if groups and used + need <= _GROUP_TOKEN_BYTES:
            groups[-1].append(doc)
            used += need
        else:
            groups.append([doc])
            used = need
    return groups


# ---- the public surface ---------------------------------------------------------------------------------------------------
def _corpus_index(config: RAGLiteConfig) -> CorpusIndex | None:
    index = get_index(config)
    if index is not None and not isinstance(index, CorpusIndex):
        raise NotImplementedError(f"a {type(index).__name__} is registered for db_url={config.db_url!r}: inserting "
                                  "and deleting documents is supported on a CorpusIndex only")
    return index


def _live_document_ids(index: CorpusIndex) -> set[DocumentId]:
    return {c.document_id for c in index.live_chunks}


def insert_documents(documents: list[Document], *, max_workers: int | None = None,  # noqa: ARG001
                     config: RAGLiteConfig | None = None) -> None:
    """Insert documents into the index registered for ``config.db_url`` (``raglite.insert_documents``); with no index
    registered, the first insert builds one (``storage`` chosen as ``from_table_rows(storage="auto")`` chooses it,
    tracking chunk ids, ``Chunk`` records and chunk metadata) and registers it.

    Duplicate ids collapse to the last document given, blank documents are dropped, and documents whose id already has
    live chunks in the index are skipped; the rest are appended in input order.  A document without ``content``
    raises ``ValueError`` up front; a failure while processing any document raises ``ValueError("Error processing
    document: ...")`` and leaves the index unchanged.  ``max_workers`` is accepted for signature parity: every
    document of a call is processed in the same batched device passes.

    On a ``postgresql`` config, ``ts_rank`` keyword search reads the database's tsvectors: inserted chunks have none
    until they are given with ``CorpusIndex.add_tsvector_rows``."""
    if not all(isinstance(doc.content, str) for doc in documents):
        raise ValueError("Some or all documents have missing `document.content`.")
    docs = [doc for doc in {doc.id: doc for doc in documents}.values() if doc.content.strip()]  # type: ignore[union-attr]
    if not docs:
        return
    config = config or RAGLiteConfig()
    index = _corpus_index(config)
    if index is not None:
        if index.n_chunks and (index.chunk_ids is None or index.chunks is None or index.chunk_metadata is None):
            raise ValueError(f"the index registered for db_url={config.db_url!r} does not hold chunk ids, Chunk records "
                             "and chunk metadata, which insert_documents appends")
        present = _live_document_ids(index)
        docs = [doc for doc in docs if doc.id not in present]
        if not docs:
            return
    try:
        records: list[Chunk] = []
        rows: list[torch.Tensor] = []
        counts: list[np.ndarray] = []
        for group in _document_groups(docs, config):
            r, X, n = _document_rows(group, config)
            records += r
            rows.append(X)
            counts.append(n)
        X = rows[0] if len(rows) == 1 else torch.cat(rows)
    except Exception as e:
        raise ValueError(f"Error processing document: {e}") from e
    off = _offsets(np.concatenate(counts))
    kw = dict(chunk_ids=[c.id for c in records], chunks=records, chunk_metadata=[c.metadata_ for c in records])
    if index is None:
        index = CorpusIndex(X, off, storage=_auto_storage(X), **kw)
        register_index(config, index)
    else:
        index.append(X, off, **kw)
    index.documents.update({doc.id: doc for doc in docs})


def _auto_storage(X: torch.Tensor) -> str:
    """``CorpusIndex._pick_storage(rows, "auto")`` for fp16 device rows: float16 unless d % 8 != 0 or the rows fail
    the fp16 cosine fast path's gate as ``rl_row_stats_f16`` decides it (a zero row, a norm below 0.5, a value's
    magnitude above 1024)."""
    if X.shape[1] % 8 or X.numel() == 0:
        return "fp32"
    return "fp16" if fp16_rows_unit_scale_device(X.contiguous()) else "fp32"


def delete_documents(document_ids: list[DocumentId], *, config: RAGLiteConfig | None = None,
                     invalidate_query_adapter: bool = False) -> int:
    """Delete documents from the index registered for ``config.db_url`` (``raglite.delete_documents``): every chunk of
    the given documents is tombstoned (``CorpusIndex.delete_documents``; ``compact`` drops them).  Returns how many of
    the given documents had live chunks.  With ``invalidate_query_adapter`` (and at least one document deleted) the
    index's query adapter is cleared."""
    if not document_ids:
        return 0
    config = config or RAGLiteConfig()
    index = _corpus_index(config)
    if index is None:
        return 0
    present = _live_document_ids(index) & set(document_ids)
    if not present:
        return 0
    index.delete_documents(sorted(present))
    for doc_id in present:
        index.documents.pop(doc_id, None)
    if invalidate_query_adapter:
        index.set_query_adapter(None)
    return len(present)


def metadata_contains(metadata: dict[str, Any], metadata_filter: dict[str, list[Any]]) -> bool:
    """Whether ``metadata`` holds every requested value (JSON containment on list-valued metadata, as
    ``CorpusIndex.filter_chunks`` matches chunks)."""
    for key, wanted in metadata_filter.items():
        if key not in metadata:
            return False
        have = metadata[key] if isinstance(metadata[key], (list, tuple)) else [metadata[key]]
        if not all(w in have for w in wanted):
            return False
    return True


def delete_documents_by_metadata(metadata_filter: dict[str, Any], *, config: RAGLiteConfig | None = None,
                                 invalidate_query_adapter: bool = False) -> int:
    """Delete the documents whose ``Document.metadata_`` contains every value of ``metadata_filter``
    (``raglite.delete_documents_by_metadata``).  Only documents ``insert_documents`` inserted have a record to match:
    chunks that reached the index through ``append`` or ``from_table_rows`` are never selected.  An empty filter
    raises ``ValueError``."""
    if not metadata_filter:
        raise ValueError(EMPTY_FILTER)
    config = config or RAGLiteConfig()
    index = _corpus_index(config)
    if index is None:
        return 0
    wanted = adapt_metadata(metadata_filter)
    ids = [doc.id for doc in index.documents.values() if metadata_contains(doc.metadata_, wanted)]
    return delete_documents(ids, config=config, invalidate_query_adapter=invalidate_query_adapter)
