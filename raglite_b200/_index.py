"""Device-resident corpus index: the hot-path view of RAGLite's ``chunk_embedding`` table.

Layout in HBM (one shard per GPU, rows of a chunk contiguous as the reference inserts them,
``_insert.py:247-251``; variable vectors per chunk, ``_split_chunks.py:121``):

    E          float32 [N, d] row-major      -- ``chunk_embedding.embedding`` (DuckDB FLOAT[d], _typing.py:187-198)
    inv_norm   float32 [N]                   -- 1 / |e_j|   (rl_row_stats)
    sq_norm    float32 [N]                   -- |e_j|^2
    row_chunk  int32   [N]                   -- owner chunk of each row (``chunk_embedding.chunk_id``)
    chunk_off  int64   [C + 1] (host)        -- CSR offsets
    chunk_ids  list[str] (host)              -- ``chunk.id`` strings handed back to the caller

The index follows the table as the reference mutates it: ``append_chunk_embedding_rows`` mirrors the
flushes of ``insert_documents`` (``_insert.py:247-255``), ``delete_chunks`` / ``delete_documents`` the cascade of
``delete_documents`` (``_delete.py:146-152``).  Deletes are tombstones (a per-row byte the scan already
reads for metadata filters); ``compact`` drops them physically, in place.

The registry maps ``RAGLiteConfig.db_url`` to an index, which is how the drop-in ``vector_search``
finds its corpus given only a config (the reference opens the database named by ``db_url``).
"""

from __future__ import annotations

import ctypes as C
import threading
from collections.abc import Callable, Sequence
from dataclasses import dataclass, field
from typing import Any

import numpy as np
import torch
import torch.distributed as dist

from . import _lib
from ._lib import (RL_ALGO, RL_FLAG_COUNT_UNFILTERED, RL_FLAG_REUSE_THRESHOLDS, RL_METRIC, RL_STATUS_CAND_OVERFLOW,
                   RL_STATUS_QUERY_NONFINITE, ScanParams, ScanStats, check)
from ._typing import ChunkId


def _stream() -> int:
    return int(torch.cuda.current_stream().cuda_stream)


def _ptr(t: torch.Tensor | None) -> int | None:
    return None if t is None else int(t.data_ptr())


def csr_from_row_chunk_ids(ids: Sequence[ChunkId], known: set[ChunkId] | None = None) -> tuple[np.ndarray, list[ChunkId]]:
    """Consecutive equal ``chunk_id`` values form one CSR segment (a chunk's vectors are inserted
    contiguously, ``_insert.py:247-251``).  A chunk id that re-appears after another chunk, or that is
    already ``known`` to the index, is a layout error."""
    ids = list(ids)
    offsets, chunk_ids, seen = [0], [], set()
    for i, cid in enumerate(ids):
        if i == 0 or cid != ids[i - 1]:
            if cid in seen or (known is not None and cid in known):
                raise ValueError(f"chunk_id {cid!r} is not contiguous in the chunk_embedding rows")
            seen.add(cid)
            chunk_ids.append(cid)
            if i:
                offsets.append(i)
    offsets.append(len(ids))
    if not ids:
        offsets = [0]
    return np.asarray(offsets, dtype=np.int64), chunk_ids


def stats_unit_scale(stats: np.ndarray) -> bool:
    """The gate of the fp16 scan's unscaled fast path on ``rl_row_stats`` statistics ``{max |e|, max |x|, max 1/|e|,
    zero row}``: every row has 1/|e| <= 2 (norm >= 0.5), no value exceeds 1024 and no row is zero."""
    return bool(0.0 < stats[2] <= 2.0 and stats[1] <= 1024.0 and stats[3] == 0.0)


def fp16_rows_unit_scale(h: np.ndarray) -> bool:
    """``stats_unit_scale`` of float16 rows ``h [n, d]`` as ``rl_row_stats_f16`` computes the statistics: per row the
    float64 sum of squares s, then float32(1 / sqrt(s)).  The float64 sum is the kernel's in any order wherever the gate
    can go either way: float16 squares are multiples of 2^-48, so a sum below 16 holds every partial sum exactly, and
    a larger one gives 1/sqrt(s) < 0.25."""
    if h.size == 0:
        return False
    h64 = h.astype(np.float64)
    s = np.einsum("ij,ij->i", h64, h64)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = (1.0 / np.sqrt(s)).astype(np.float32)
    return bool((s > 0).all() and (inv <= 2.0).all() and np.abs(h).max() <= 1024)


def fp16_rows_unit_scale_device(X: torch.Tensor) -> bool:
    """``stats_unit_scale`` of contiguous float16 device rows ``X [n, d]`` (d % 8 == 0), from ``rl_row_stats_f16``
    itself.  Synchronises."""
    n, d = int(X.shape[0]), int(X.shape[1])
    if n == 0:
        return False
    dev = X.device
    inv, sq = torch.empty(n, dtype=torch.float32, device=dev), torch.empty(n, dtype=torch.float32, device=dev)
    st = torch.zeros(4, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        check(_lib.load().rl_row_stats_f16(_ptr(X), n, d, d, _ptr(inv), _ptr(sq), _ptr(st), _stream()), "rl_row_stats_f16")
    return stats_unit_scale(st.cpu().numpy())


@dataclass
class Chunk:
    """Minimal stand-in for ``raglite._database.Chunk`` (``_database.py:196-324``): what
    ``rerank_chunks`` needs -- an id and the ``str(chunk)`` text the cross-encoder scores."""

    id: ChunkId
    document_id: str = ""
    index: int = 0
    headings: str = ""
    body: str = ""
    metadata_: dict[str, Any] = field(default_factory=dict)

    @property
    def front_matter(self) -> str:
        meta = "\n".join(f"{k}: {self.metadata_.get(k)}" for k in ("filename", "url", "uri") if self.metadata_.get(k))
        return f"---\n{meta}\n---" if meta else ""

    @property
    def content(self) -> str:
        """Front matter, contextual headings and body (``_database.py:317-324``)."""
        return f"{self.front_matter}\n\n{self.headings.strip()}\n\n{self.body.strip()}".strip()

    def __str__(self) -> str:
        return self.content

    def __hash__(self) -> int:
        return hash(self.id)


@dataclass
class ScanResult:
    """Device-side output of one shard scan (inputs of ``rl_topk_merge``)."""

    hit_sim: torch.Tensor    # [B, H] float32
    hit_chunk: torch.Tensor  # [B, H] int64 (global chunk index)
    hit_count: torch.Tensor  # [B] int32
    status: torch.Tensor     # [B] int32
    num_hits: int
    k: int
    packed: torch.Tensor | None = None   # the uint8 buffer the four tensors above are views of (hits_views); every scan sets it


def hits_views(packed: torch.Tensor, R: int, B: int, H: int
               ) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """``(chunk [R, B, H] int64, sim [R, B, H] float32, count [R, B] int32, status [R, B] int32)``: views of ``R``
    packed hit lists laid end to end in the uint8 buffer ``packed``, ``rl_hits_packed_bytes(B, H, 1)`` bytes each
    (at least 16).  The scan writes one such list, the sharded search all-gathers R of them, and
    ``rl_topk_merge_packed`` reads them in place."""
    per = max(int(_lib.load().rl_hits_packed_bytes(B, H, 1)), 16)
    lists = packed[: R * per].view(R, per)
    n8, n4 = B * H * 8, B * H * 4
    return (lists[:, :n8].view(torch.int64).view(R, B, H), lists[:, n8:n8 + n4].view(torch.float32).view(R, B, H),
            lists[:, n8 + n4:n8 + n4 + B * 4].view(torch.int32), lists[:, n8 + n4 + B * 4:n8 + n4 + B * 8].view(torch.int32))


def new_scan_result(B: int, H: int, num_hits: int, k: int, device: Any) -> ScanResult:
    """Scan outputs laid out as ONE packed hit list: the all-gather of the sharded path sends it as is."""
    buf = torch.empty(max(int(_lib.load().rl_hits_packed_bytes(B, H, 1)), 16), dtype=torch.uint8, device=device)
    chunk, sim, count, status = hits_views(buf, 1, B, H)
    return ScanResult(sim[0], chunk[0], count[0], status[0], num_hits, k, buf)


class CorpusIndex:
    """One shard of the corpus, resident on one GPU."""

    def __init__(  # noqa: PLR0913
        self,
        embeddings: torch.Tensor | np.ndarray,
        chunk_offsets: np.ndarray | Sequence[int] | None = None,
        *,
        vecs_per_chunk: int | None = None,
        chunk_ids: Sequence[ChunkId] | None = None,
        chunk_base: int = 0,
        chunks: Sequence[Chunk] | None = None,
        chunk_metadata: Sequence[dict[str, Any]] | None = None,
        device: torch.device | str | None = None,
        storage: str = "fp32",
    ) -> None:
        if not torch.cuda.is_available():
            raise RuntimeError("raglite_b200 needs a CUDA device (there is no CPU fallback)")
        self.lib = _lib.load()
        self.device = torch.device(device if device is not None else f"cuda:{torch.cuda.current_device()}")
        E = torch.as_tensor(embeddings)
        if E.ndim != 2:
            raise ValueError("embeddings must be [n_rows, d]")
        if storage not in ("fp32", "fp16"):
            raise ValueError("storage must be 'fp32' or 'fp16'")
        self.storage = storage
        self.E = self._to_storage(E)
        self.n_rows, self.d = int(self.E.shape[0]), int(self.E.shape[1])
        if storage == "fp16" and self.d % 8:
            raise ValueError("storage='fp16' needs d % 8 == 0")
        if chunk_offsets is None:
            v = 1 if vecs_per_chunk is None else int(vecs_per_chunk)
            if self.n_rows % v:
                raise ValueError("n_rows is not a multiple of vecs_per_chunk")
            chunk_offsets = np.arange(0, self.n_rows + 1, v, dtype=np.int64)
        self.chunk_off = np.ascontiguousarray(np.asarray(chunk_offsets, dtype=np.int64))
        if self.chunk_off[0] != 0 or self.chunk_off[-1] != self.n_rows or np.any(np.diff(self.chunk_off) < 0):
            raise ValueError("chunk_offsets must be a CSR offset array covering all rows")
        self.n_chunks = len(self.chunk_off) - 1
        counts = np.diff(self.chunk_off)
        self.max_vecs = int(counts.max()) if self.n_chunks else 1
        self.chunk_base = int(chunk_base)
        self.chunk_ids = list(chunk_ids) if chunk_ids is not None else None
        if self.chunk_ids is not None and len(self.chunk_ids) != self.n_chunks:
            raise ValueError("chunk_ids must have one entry per chunk")
        self.chunks = list(chunks) if chunks is not None else None
        self.chunk_metadata = list(chunk_metadata) if chunk_metadata is not None else None
        self.documents: dict[str, Any] = {}   # Document records of insert_documents, by id (delete_documents_by_metadata)
        self._alive: torch.Tensor | None = None        # uint8 [n_rows]; None = no tombstones
        self._alive_buf: torch.Tensor | None = None    # capacity buffer behind _alive
        self._bufs: dict[str, torch.Tensor] | None = None  # owned capacity buffers once the index has grown
        self._chunk_alive = np.ones(self.n_chunks, dtype=bool)
        self._chunk_pos: dict[ChunkId, int] | None = None
        self.query_adapter: np.ndarray | None = None  # IndexMetadata["default"]["query_adapter"]
        self._adapter_dev: torch.Tensor | None = None
        # One workspace per CUDA stream: a scan is asynchronous, so two host threads driving two streams
        # must never share the thresholds / candidate lists a retry reads back (reference callers search
        # from thread pools, _rag.py:317).  The lock is re-entrant: scan_checked / search_to_host hold it
        # across the status read-back and the retries.
        self._ws: dict[int, torch.Tensor] = {}
        self._lock = threading.RLock()
        self._shard_guard: Any | None = None           # the ShardedIndex this shard belongs to, if any
        self._meta_inv: dict[tuple[str, Any], np.ndarray] | None = None   # (key, value) -> chunk indices
        self._meta_inv_chunks = 0                      # chunks covered by _meta_inv
        self._filter_cache: dict[Any, tuple[torch.Tensor, int]] = {}      # filter -> (chunk_ok uint8 [C], matching live rows)
        self._keyword: Any | None = None               # BM25 postings of the chunk bodies (keyword_index), built on demand
        self._tsrank: Any | None = None                # ts_rank postings of PostgreSQL tsvectors (add_tsvector_rows)
        self._pinned: dict[Any, torch.Tensor] = {}     # result staging buffers (pinned host memory) by (size, stream)
        self._slots: list[Any] = []                    # streams + pinned buffers of the asynchronous searches (search_async)
        self.last_params: ScanParams | None = None
        self.last_ws: torch.Tensor | None = None
        with torch.cuda.device(self.device):
            self.inv_norm = torch.empty(self.n_rows, dtype=torch.float32, device=self.device)
            self.sq_norm = torch.empty(self.n_rows, dtype=torch.float32, device=self.device)
            self.stats = torch.zeros(4, dtype=torch.float32, device=self.device)
            self.row_chunk = torch.empty(self.n_rows, dtype=torch.int32, device=self.device)
            off_dev = torch.from_numpy(self.chunk_off).to(self.device)
            self._row_stats(self.E, self.inv_norm, self.sq_norm)
            check(self.lib.rl_chunk_row_map(_ptr(off_dev), self.n_chunks, _ptr(self.row_chunk), _stream()),
                  "rl_chunk_row_map")
            torch.cuda.current_stream().synchronize()
            self._refresh_fp16_flag()

    @classmethod
    def from_chunk_embedding_rows(cls, row_chunk_ids: Sequence[ChunkId], embeddings: torch.Tensor | np.ndarray,
                                  **kw: Any) -> "CorpusIndex":
        """Build the index from the rows of RAGLite's ``chunk_embedding`` table read in insertion order
        (``SELECT chunk_id, embedding FROM chunk_embedding ORDER BY id``; ``_database.py:403-430``): a
        chunk's vectors are contiguous (``_insert.py:247-251``), so consecutive equal ``chunk_id`` values
        form one CSR segment.  A chunk id that re-appears after another chunk is a layout error."""
        ids = list(row_chunk_ids)
        E = torch.as_tensor(embeddings)
        if len(ids) != int(E.shape[0]):
            raise ValueError("one chunk_id per embedding row is required")
        offsets, chunk_ids = csr_from_row_chunk_ids(ids)
        return cls(E, offsets, chunk_ids=chunk_ids, **kw)

    @classmethod
    def from_table_rows(cls, rows: Any, dialect: str, *, storage: str = "auto", **kw: Any) -> "CorpusIndex":
        """Build the index from a ``chunk_embedding`` result set as the database driver returns it:
        ``(chunk_id, embedding)`` tuples of ``SELECT chunk_id, embedding FROM chunk_embedding ORDER BY id``
        with DuckDB ``FLOAT[d]`` lists (``dialect="duckdb"``, ``_typing.py:178-208``), PostgreSQL ``halfvec``
        text (``"postgresql"``, ``_typing.py:145-175``) or ``np.save`` blobs (``"numpy"``, ``_typing.py:57-78``).
        ``storage="auto"`` picks the lossless float16 layout when every value is float16-representable
        -- always the case for rows RAGLite wrote (``_embed.py:140``) -- and float32 otherwise."""
        from . import _rows

        ids, E = _rows.table_rows(rows, dialect)
        E, storage = cls._pick_storage(E, storage)
        return cls.from_chunk_embedding_rows(ids, E, storage=storage, **kw)

    def append_table_rows(self, rows: Any, dialect: str, **kw: Any) -> None:
        """``append_chunk_embedding_rows`` for driver-shaped rows (one flush of ``insert_documents``,
        ``_insert.py:247-255``)."""
        from . import _rows

        ids, E = _rows.table_rows(rows, dialect)
        self.append_chunk_embedding_rows(ids, E, **kw)

    @staticmethod
    def _pick_storage(E: np.ndarray, storage: str) -> tuple[np.ndarray, str]:
        from . import _rows

        if storage != "auto":
            return E, storage
        d = int(E.shape[1]) if E.ndim == 2 else 0
        h = _rows.lossless_float16(E) if d % 8 == 0 and E.size else None
        if h is None or not fp16_rows_unit_scale(h):   # the cosine fast path of the float16 layout needs unit-scale rows
            return E.astype(np.float32, copy=False), "fp32"
        return h, "fp16"

    def _to_storage(self, E: torch.Tensor) -> torch.Tensor:
        """Rows in the index's storage dtype on its device.  ``fp16`` storage is lossless only: RAGLite's
        embeddings are fp16-rounded already (``_embed.py:140``) and DuckDB merely widens them to FLOAT[d];
        anything else must stay float32."""
        if self.storage == "fp32":
            return E.to(device=self.device, dtype=torch.float32).contiguous()
        Eh = self._lossless_fp16(E)
        if Eh is None:
            raise ValueError("storage='fp16' needs embeddings that are exactly representable in float16")
        return Eh

    def _lossless_fp16(self, E: torch.Tensor) -> torch.Tensor | None:
        """``E`` as float16 rows on the device, or None when a value is not exactly representable in float16."""
        Eh = E.to(device=self.device, dtype=torch.float16).contiguous()
        if E.dtype != torch.float16:
            step = 1 << 20
            for r0 in range(0, int(E.shape[0]), step):
                blk = E[r0:r0 + step].to(self.device, dtype=torch.float32)
                if not torch.equal(Eh[r0:r0 + step].float(), blk):
                    return None
        return Eh

    # ---- mutation: the index follows the chunk_embedding table --------------------------------------
    @property
    def n_live_chunks(self) -> int:
        return int(self._chunk_alive.sum())

    @property
    def live_chunks(self) -> list[Chunk]:
        """``Chunk`` records that have not been deleted."""
        if self.chunks is None:
            return []
        return [c for c, ok in zip(self.chunks, self._chunk_alive, strict=True) if ok]

    def _row_stats(self, E: torch.Tensor, inv_norm: torch.Tensor, sq_norm: torch.Tensor) -> None:
        stats_fn = self.lib.rl_row_stats_f16 if self.storage == "fp16" else self.lib.rl_row_stats
        check(stats_fn(_ptr(E), int(E.shape[0]), self.d, self.d, _ptr(inv_norm), _ptr(sq_norm), _ptr(self.stats),
                       _stream()), "rl_row_stats")

    def _refresh_fp16_flag(self) -> None:
        """Host copy of the decision the scan otherwise takes on the device: can rows enter the fp16 tensor-core
        scan unscaled (norms >= 0.5, |x| <= 1024, no zero row -- normalised embeddings)?  Read once per index
        change (build / append / compact synchronise anyway), passed as ``rl_scan_params.rows_unit_scale``."""
        self._rows_unit_scale = bool(self.n_rows) and stats_unit_scale(self.stats.cpu().numpy())
        if self.storage == "fp16":   # an empty shard holds no row too small for the cosine fast path
            self._fp16_cosine_ok = self._rows_unit_scale or self.n_rows == 0

    def _widen_to_fp32(self) -> None:
        """Move the rows to float32 storage (same values; the capacity buffer keeps its size).  ``append`` does this
        before it adds rows that the float16 layout cannot hold losslessly, or that would take its cosine fast path
        away: a search never starts failing because of an earlier append.  The row statistics stay valid."""
        cap = int(self._bufs["E"].shape[0]) if self._bufs is not None else self.n_rows
        E32 = torch.empty((cap, self.d), dtype=torch.float32, device=self.device)
        E32[: self.n_rows] = self.E
        if self._bufs is not None:
            self._bufs["E"] = E32
        self.E, self.storage = E32[: self.n_rows], "fp32"

    @property
    def rows_unit_scale(self) -> bool:
        """True when every row can enter the fp16 scan unscaled (normalised embeddings): ``rl_scan_params.rows_unit_scale``."""
        return bool(getattr(self, "_rows_unit_scale", False))

    def reserve(self, n_rows: int) -> None:
        """Pre-size the row buffers (size HBM for the final corpus once instead of re-growing per flush)."""
        with self._lock, torch.cuda.device(self.device):
            self._reserve(int(n_rows))

    _ROW_ARRAYS = ("E", "inv_norm", "sq_norm", "row_chunk")

    def _reserve(self, n_rows: int) -> None:
        """Make the owned capacity buffers hold ``n_rows`` rows; the public arrays stay views of their
        first ``self.n_rows`` rows.  (The constructor adopts the caller's tensor without a copy, so the
        first growth is also the point where the index starts owning its storage.)"""
        cap = int(self._bufs["E"].shape[0]) if self._bufs is not None else -1
        if n_rows <= cap:
            return
        new_cap = max(n_rows, self.n_rows + self.n_rows // 2 + 1024)
        bufs = {}
        for name in self._ROW_ARRAYS:
            t = getattr(self, name)
            bufs[name] = torch.empty((new_cap, *t.shape[1:]), dtype=t.dtype, device=self.device)
            bufs[name][: self.n_rows] = t
            setattr(self, name, bufs[name][: self.n_rows])
        self._bufs = bufs

    def append(  # noqa: PLR0913
        self, embeddings: torch.Tensor | np.ndarray, chunk_offsets: np.ndarray | Sequence[int] | None = None, *,
        vecs_per_chunk: int | None = None, chunk_ids: Sequence[ChunkId] | None = None,
        chunks: Sequence[Chunk] | None = None, chunk_metadata: Sequence[dict[str, Any]] | None = None,
    ) -> None:
        """Append whole chunks (rows of a chunk contiguous) behind the resident rows: one flush of
        ``insert_documents`` (``_insert.py:247-255``).  Only the new rows are read: their norms are
        computed by ``rl_row_stats``, which folds their maxima into the shard statistics.  A float16 index moves to
        float32 storage first when a new row is not exactly representable in float16, or when the index passes the
        cosine fast path's gate (``fp16_rows_unit_scale``) and a new row does not."""
        E = torch.as_tensor(embeddings)
        if E.ndim != 2 or int(E.shape[1]) != self.d:
            raise ValueError(f"embeddings must be [n_rows, {self.d}]")
        m = int(E.shape[0])
        if chunk_offsets is None:
            v = 1 if vecs_per_chunk is None else int(vecs_per_chunk)
            if m % v:
                raise ValueError("n_rows is not a multiple of vecs_per_chunk")
            chunk_offsets = np.arange(0, m + 1, v, dtype=np.int64)
        off = np.ascontiguousarray(np.asarray(chunk_offsets, dtype=np.int64))
        if off[0] != 0 or off[-1] != m or np.any(np.diff(off) < 0):
            raise ValueError("chunk_offsets must be a CSR offset array covering all rows")
        c_new = len(off) - 1
        for name, given in (("chunk_ids", chunk_ids), ("chunks", chunks), ("chunk_metadata", chunk_metadata)):
            tracked = getattr(self, name) is not None
            if tracked and given is None:
                raise ValueError(f"the index tracks {name}: pass one per appended chunk")
            if given is not None and not tracked and self.n_chunks:
                raise ValueError(f"the index holds no {name}; it cannot start tracking them on append")
            if given is not None and len(given) != c_new:
                raise ValueError(f"{name} must have one entry per appended chunk")
        if chunk_ids is not None:
            known = self._positions()
            for cid in chunk_ids:   # a deleted chunk may come back (re-inserting a document re-creates its ids)
                if cid in known and self._chunk_alive[known[cid]]:
                    raise ValueError(f"chunk_id {cid!r} is already in the index")
        if m == 0:
            return
        if self._shard_guard is not None:
            self._shard_guard.check_local_growth(self.n_chunks + c_new)
        with self._lock, torch.cuda.device(self.device):
            self._invalidate_filters()
            rows = self._lossless_fp16(E) if self.storage == "fp16" else None
            if self.storage == "fp16" and (rows is None or (self._fp16_cosine_ok and not fp16_rows_unit_scale_device(rows))):
                self._widen_to_fp32()
                rows = None
            if rows is None:
                rows = self._to_storage(E)
            n0 = self.n_rows
            self._reserve(n0 + m)
            for name in self._ROW_ARRAYS:
                setattr(self, name, self._bufs[name][: n0 + m])
            self.E[n0:] = rows
            self._row_stats(self.E[n0:], self.inv_norm[n0:], self.sq_norm[n0:])
            counts = torch.from_numpy(np.diff(off)).to(self.device)
            owners = torch.arange(self.n_chunks, self.n_chunks + c_new, dtype=torch.int32, device=self.device)
            self.row_chunk[n0:] = torch.repeat_interleave(owners, counts)
            if self._alive is not None:
                self._alive = torch.cat([self._alive, torch.ones(m, dtype=torch.uint8, device=self.device)])
            self.chunk_off = np.concatenate([self.chunk_off, off[1:] + n0])
            self._chunk_alive = np.concatenate([self._chunk_alive, np.ones(c_new, dtype=bool)])
            for name, given in (("chunk_ids", chunk_ids), ("chunks", chunks), ("chunk_metadata", chunk_metadata)):
                if given is not None:
                    setattr(self, name, (getattr(self, name) or []) + list(given))
            if chunk_ids is not None and self._chunk_pos is not None:
                self._chunk_pos.update({cid: self.n_chunks + i for i, cid in enumerate(chunk_ids)})
            self.n_rows, self.n_chunks = n0 + m, self.n_chunks + c_new
            self.max_vecs = max(self.max_vecs, int(np.diff(off).max()))
            torch.cuda.current_stream().synchronize()
            self._refresh_fp16_flag()

    def append_chunk_embedding_rows(self, row_chunk_ids: Sequence[ChunkId], embeddings: torch.Tensor | np.ndarray,
                                    **kw: Any) -> None:
        """``append`` for rows spelled like the table: one ``chunk_id`` per embedding row."""
        ids = list(row_chunk_ids)
        if len(ids) != int(torch.as_tensor(embeddings).shape[0]):
            raise ValueError("one chunk_id per embedding row is required")
        offsets, chunk_ids = csr_from_row_chunk_ids(ids)
        self.append(embeddings, offsets, chunk_ids=chunk_ids, **kw)

    def _positions(self) -> dict[ChunkId, int]:
        if self._chunk_pos is None:
            self._chunk_pos = {cid: i for i, cid in enumerate(self.chunk_ids or [])}
        return self._chunk_pos

    def delete_chunks(self, chunk_ids: Sequence[ChunkId]) -> int:
        """Tombstone the rows of the given chunks (``DELETE FROM chunk_embedding WHERE chunk_id IN ...``,
        the cascade of ``_delete.py:146-152``); unknown or already deleted ids are ignored.  Returns the
        number of chunks removed.  Chunk indices stay stable until ``compact``."""
        if self.chunk_ids is None:
            raise ValueError("the index holds no chunk ids")
        pos = self._positions()
        local = sorted({pos[c] for c in chunk_ids if c in pos and self._chunk_alive[pos[c]]})
        return self._delete_local(np.asarray(local, dtype=np.int64))

    def delete_documents(self, document_ids: Sequence[str]) -> int:
        """Tombstone every chunk of the given documents (``_delete.py:146-152``)."""
        if self.chunks is None:
            raise ValueError("the index holds no Chunk records (document ids unknown)")
        wanted = set(document_ids)
        local = [i for i, c in enumerate(self.chunks) if c.document_id in wanted and self._chunk_alive[i]]
        return self._delete_local(np.asarray(local, dtype=np.int64))

    def _delete_local(self, local: np.ndarray) -> int:
        if len(local) == 0:
            return 0
        lo, hi = self.chunk_off[local], self.chunk_off[local + 1]
        rows = np.concatenate([np.arange(a, b, dtype=np.int64) for a, b in zip(lo, hi, strict=True)]) if len(local) else lo
        with self._lock, torch.cuda.device(self.device):
            self._invalidate_filters()
            if self._alive is None:
                self._alive = torch.ones(self.n_rows, dtype=torch.uint8, device=self.device)
            if len(rows):
                self._alive.index_fill_(0, torch.from_numpy(rows).to(self.device), 0)
            self._chunk_alive[local] = False
        return int(len(local))

    def compact(self, block_rows: int = 1 << 20) -> None:
        """Drop tombstoned rows physically: surviving rows slide down in place, block by block (a staged
        block is at most ``block_rows`` rows, so the corpus never needs a second copy in HBM).  Chunk
        indices are renumbered inside this shard's range; ``chunk_base`` does not move, so the other shards of
        a ``ShardedIndex`` are unaffected (call ``ShardedIndex.refresh`` afterwards: it re-gathers the shard
        ranges and the chunk-id tables)."""
        if self._alive is None:
            return
        with self._lock, torch.cuda.device(self.device):
            self._invalidate_filters()
            self._meta_inv = None
            dst = 0
            for r0 in range(0, self.n_rows, block_rows):
                r1 = min(self.n_rows, r0 + block_rows)
                idx = torch.nonzero(self._alive[r0:r1], as_tuple=False).flatten()
                n_keep = int(idx.numel())
                if n_keep and not (dst == r0 and n_keep == r1 - r0):
                    self.E[dst:dst + n_keep] = self.E[r0:r1].index_select(0, idx)   # staged copy; lands below r0 + n_keep
                dst += n_keep
            keep = self._chunk_alive
            counts = np.diff(self.chunk_off)[keep]
            self.chunk_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
            assert int(self.chunk_off[-1]) == dst
            for name in ("chunk_ids", "chunks", "chunk_metadata"):
                have = getattr(self, name)
                if have is not None:
                    setattr(self, name, [x for x, ok in zip(have, keep, strict=True) if ok])
            self.n_rows, self.n_chunks = dst, int(keep.sum())
            self.max_vecs = int(counts.max()) if len(counts) else 1
            if self._keyword is not None:
                self._keyword.compact(keep)
            if self._tsrank is not None:
                self._tsrank.compact(keep)
            self._chunk_alive = np.ones(self.n_chunks, dtype=bool)
            self._chunk_pos, self._alive = None, None
            for name in self._ROW_ARRAYS:
                setattr(self, name, getattr(self, name)[:dst])
            self.stats.zero_()
            self._row_stats(self.E, self.inv_norm, self.sq_norm)
            off_dev = torch.from_numpy(self.chunk_off).to(self.device)
            check(self.lib.rl_chunk_row_map(_ptr(off_dev), self.n_chunks, _ptr(self.row_chunk), _stream()),
                  "rl_chunk_row_map")
            torch.cuda.current_stream().synchronize()
            self._refresh_fp16_flag()

    # ---- query adapter (IndexMetadata.get("default")["query_adapter"], _search.py:60) ------------
    def set_query_adapter(self, A: np.ndarray | None) -> None:
        if A is None:
            self.query_adapter, self._adapter_dev = None, None
            return
        A = np.asarray(A, dtype=np.float64)
        if A.shape != (self.d, self.d):
            raise ValueError(f"query adapter must be [{self.d}, {self.d}]")
        self.query_adapter = A
        self._adapter_dev = torch.from_numpy(np.ascontiguousarray(A)).to(self.device)

    def apply_adapter(self, Q: torch.Tensor, *, round_fp16: bool) -> torch.Tensor:
        """``(A @ q).astype(q.dtype)`` for a batch (``_search.py:62``), float64 accumulate on device."""
        if self._adapter_dev is None:
            return Q
        out = torch.empty_like(Q)
        with torch.cuda.device(self.device):
            check(self.lib.rl_adapter_apply(_ptr(self._adapter_dev), _ptr(Q), _ptr(out), Q.shape[0], self.d,
                                            1 if round_fp16 else 0, _stream()), "rl_adapter_apply")
        return out

    # ---- metadata filters resolved on the device (_search.py:82-95) -------------------------------------
    def _metadata_index(self) -> dict[tuple[str, Any], np.ndarray]:
        """Inverted index ``(key, value) -> chunk indices`` over ``chunk_metadata``, built in one pass (and
        extended over appended chunks): a search then never walks the chunk table on the host."""
        if self.chunk_metadata is None:
            raise ValueError("metadata_filter given but the index holds no chunk metadata")
        if self._meta_inv is None or self._meta_inv_chunks > self.n_chunks:
            self._meta_inv, self._meta_inv_chunks = {}, 0
        if self._meta_inv_chunks < self.n_chunks:
            fresh: dict[tuple[str, Any], list[int]] = {}
            for c in range(self._meta_inv_chunks, self.n_chunks):
                for key, have in self.chunk_metadata[c].items():
                    for v in (have if isinstance(have, (list, tuple)) else [have]):
                        try:
                            fresh.setdefault((key, v), []).append(c)
                        except TypeError:   # unhashable metadata value: cannot be asked for by a MetadataFilter
                            continue
            for kv, lst in fresh.items():
                arr = np.asarray(lst, dtype=np.int64)
                old = self._meta_inv.get(kv)
                self._meta_inv[kv] = arr if old is None else np.concatenate([old, arr])
            self._meta_inv_chunks = self.n_chunks
        return self._meta_inv

    def filter_chunks(self, metadata_filter: dict[str, list[Any]]) -> tuple[torch.Tensor, int]:
        """``(chunk_ok uint8 [n_chunks] on the device, number of matching live rows)`` for a normalised
        filter ``{key: [values...]}``: a chunk matches when its metadata contains every requested value
        (JSON containment on list-valued metadata, ``_search.py:82-95``).  Cached per filter until the
        index changes."""
        key = tuple(sorted((k, tuple(v)) for k, v in metadata_filter.items()))
        with self._lock:
            hit = self._filter_cache.get(key)
            if hit is not None:
                return hit
            inv = self._metadata_index()
            ok: np.ndarray | None = None
            for k, wanted in metadata_filter.items():
                for w in wanted:
                    ids = inv.get((k, w), np.zeros(0, np.int64))
                    ok = ids if ok is None else np.intersect1d(ok, ids, assume_unique=False)
            ok = np.zeros(0, np.int64) if ok is None else np.unique(ok)
            ok = ok[self._chunk_alive[ok]] if len(ok) else ok
            n_rows = int((self.chunk_off[ok + 1] - self.chunk_off[ok]).sum()) if len(ok) else 0
            with torch.cuda.device(self.device):
                chunk_ok = torch.zeros(max(self.n_chunks, 1), dtype=torch.uint8, device=self.device)
                if len(ok):
                    chunk_ok.index_fill_(0, torch.from_numpy(ok).to(self.device), 1)
            if len(self._filter_cache) >= 32:
                self._filter_cache.pop(next(iter(self._filter_cache)))
            self._filter_cache[key] = (chunk_ok, n_rows)
            return chunk_ok, n_rows

    def row_mask(self, chunk_ok: torch.Tensor | None) -> torch.Tensor | None:
        """``rl_row_mask``: the per-row byte mask of a per-chunk filter, ANDed with the tombstones."""
        if chunk_ok is None:
            return self._alive
        out = torch.empty(self.n_rows + 16, dtype=torch.uint8, device=self.device)[: self.n_rows]
        with torch.cuda.device(self.device):
            check(self.lib.rl_row_mask(_ptr(chunk_ok), _ptr(self.row_chunk), _ptr(self._alive), self.n_rows, _ptr(out),
                                       _stream()), "rl_row_mask")
        return out

    def _invalidate_filters(self) -> None:
        self._filter_cache.clear()
        self._n_live_rows = None
        self._span_tables = None
        if self._keyword is not None:
            self._keyword.stale = True
        if self._tsrank is not None:
            self._tsrank.stale = True

    def keyword_index(self) -> Any:
        """The BM25 index over ``chunks[i].body`` (``_keyword.KeywordIndex``), brought up to date with the table:
        built on the first call, appended chunks analysed, statistics recomputed over the live chunks after any
        change.  Needs the ``Chunk`` records (``ValueError`` otherwise, as ``retrieve_chunks``)."""
        if self.chunks is None:
            raise ValueError("The registered index holds no chunk texts")
        from ._keyword import KeywordIndex

        with self._lock, torch.cuda.device(self.device):
            if self._keyword is None:
                self._keyword = KeywordIndex(self.device)
            kw = self._keyword
            if kw.n_chunks < self.n_chunks:
                kw.extend([c.body for c in self.chunks[kw.n_chunks:]])
            if kw.stale:
                kw.refresh(self._chunk_alive)
            return kw

    def add_tsvector_rows(self, rows: Any) -> int:
        """Index the tsvectors PostgreSQL computes for a ``postgresql`` keyword search (``ts_rank``, ``_search.py:176-201``):
        ``(chunk_id, text)`` rows of ``SELECT id, to_tsvector('simple', body)::text FROM chunk``, in any order.  Call it
        once after building the index and again after each ``append`` for the new chunks.  A chunk id the index does not
        hold, a chunk given a second time, or a tsvector that ``to_tsvector`` does not print (weights, more than 256
        positions per lexeme, malformed text) raises ``ValueError`` and leaves the index unchanged.  Returns the number
        of rows indexed."""
        return self._add_tsvector_rows(rows, others_ok=False)

    def _add_tsvector_rows(self, rows: Any, *, others_ok: bool) -> int:
        """``add_tsvector_rows``; ``others_ok``: skip the rows of chunk ids this index does not hold (a shard's share)."""
        import time

        from . import _pgfts
        from ._keyword import TsRankIndex

        if self.chunk_ids is None:
            raise ValueError("the index holds no chunk ids: tsvector rows cannot be matched to chunks")
        t0 = time.perf_counter()
        with self._lock:
            pos = self._positions()
            have = self._tsrank.has_tsvector if self._tsrank is not None else np.zeros(0, dtype=bool)
            chunks: list[int] = []
            parsed = []
            seen: set[int] = set()
            for cid, text in rows:
                p = pos.get(cid)
                if p is None:
                    if others_ok:
                        continue
                    raise ValueError(f"chunk_id {cid!r} is not in the index")
                if p in seen or (p < len(have) and have[p]):
                    raise ValueError(f"chunk_id {cid!r} already has a tsvector (a chunk's body never changes)")
                seen.add(p)
                chunks.append(p)
                parsed.append(_pgfts.parse_tsvector(text, cid))
            with torch.cuda.device(self.device):
                if self._tsrank is None:
                    self._tsrank = TsRankIndex(self.device)
                self._tsrank.add(np.asarray(chunks, dtype=np.int64), parsed, time.perf_counter() - t0)
        return len(chunks)

    def span_tables(self) -> dict[str, torch.Tensor]:
        """Device tables ``rl_span_collate`` needs (built once per index change from the ``Chunk`` records):
        ``chunk_doc`` = ordinal of each chunk's document in ascending ``document_id`` order (the order
        ``retrieve_chunk_spans`` sorts by, ``_search.py:343``), ``chunk_pos`` = ``Chunk.index``, ``chunk_alive``, and the
        lookup ``(doc << 32 | pos) -> chunk`` sorted by key.  The lookup holds every chunk, deleted ones included: its
        length is also the range the kernel accepts retrieved chunk indices from, and a deleted chunk is turned away
        there through ``chunk_alive``.  Among equal keys the live chunk comes first, which is the one found."""
        if self.chunks is None:
            raise ValueError("The registered index holds no Chunk records (document ids / positions unknown)")
        with self._lock:
            if getattr(self, "_span_tables", None) is None:
                docs = sorted({c.document_id for c in self.chunks})
                ordinal = {d: i for i, d in enumerate(docs)}
                doc = np.fromiter((ordinal[c.document_id] for c in self.chunks), dtype=np.int32, count=len(self.chunks))
                pos = np.fromiter((c.index for c in self.chunks), dtype=np.int32, count=len(self.chunks))
                key = (doc.astype(np.uint64) << np.uint64(32)) | pos.astype(np.uint32).astype(np.uint64)
                order = np.lexsort((~self._chunk_alive.astype(bool), key))   # by key, then live first
                dev = self.device
                self._span_tables = {
                    "chunk_doc": torch.from_numpy(doc).to(dev), "chunk_pos": torch.from_numpy(pos).to(dev),
                    "chunk_alive": torch.from_numpy(self._chunk_alive.astype(np.uint8)).to(dev),
                    "sorted_key": torch.from_numpy(key[order].view(np.int64)).to(dev),
                    "sorted_chunk": torch.from_numpy(order.astype(np.int64)).to(dev)}
            return self._span_tables

    @property
    def n_live_rows(self) -> int:
        """Rows that are not tombstoned (cached until the index changes)."""
        if getattr(self, "_n_live_rows", None) is None:
            self._n_live_rows = int(np.diff(self.chunk_off)[self._chunk_alive].sum()) if self.n_chunks else 0
        return self._n_live_rows

    # ---- scan ---------------------------------------------------------------------------------------
    def _params(self, Q: torch.Tensor, k: int, num_hits: int, metric: str, algo: str,
                row_allowed: torch.Tensor | None, flags: int, sample_stride: int, cand_cap: int) -> ScanParams:
        p = ScanParams()
        p.E, p.inv_norm, p.sq_norm = _ptr(self.E), _ptr(self.inv_norm), _ptr(self.sq_norm)
        p.row_chunk, p.row_stats, p.row_allowed = _ptr(self.row_chunk), _ptr(self.stats), _ptr(row_allowed)
        p.n_rows, p.ld, p.chunk_base = self.n_rows, self.d, self.chunk_base
        p.d, p.max_vecs_per_chunk = self.d, max(1, self.max_vecs)
        p.Q, p.B = _ptr(Q), int(Q.shape[0])
        p.metric, p.k, p.num_hits, p.algo = RL_METRIC[metric], int(k), int(num_hits), RL_ALGO[algo]
        p.flags, p.sample_stride, p.cand_cap = flags, sample_stride, cand_cap
        p.e_dtype = 1 if self.storage == "fp16" else 0
        p.rows_unit_scale = 1 if getattr(self, "_rows_unit_scale", False) else 0
        if self.storage == "fp16" and metric == "cosine" and not getattr(self, "_fp16_cosine_ok", True):
            raise ValueError("storage='fp16' with the cosine metric needs rows with norm >= 0.5 (normalised embeddings)")
        return p

    def _workspace(self, need: int) -> torch.Tensor:
        """The workspace of the CURRENT stream, grown on demand (caller holds the lock)."""
        key = _stream()
        ws = self._ws.get(key)
        if ws is None or ws.numel() < need:
            if ws is not None:
                self.lib.rl_maxsim_release(_ptr(ws))
                del self._ws[key]
                ws = None  # free before the larger allocation
            ws = torch.empty(max(need, 256), dtype=torch.uint8, device=self.device)
            self._ws[key] = ws
        return ws

    def close(self) -> None:
        """Release the per-stream workspaces (and the timing events the library keeps per workspace pointer)."""
        with self._lock:
            for ws in self._ws.values():
                self.lib.rl_maxsim_release(_ptr(ws))
            self._ws.clear()
            self.last_ws = None

    def __del__(self) -> None:
        try:
            self.close()
        except Exception:  # noqa: BLE001, S110  (interpreter shutdown: the library may be gone)
            pass

    def scan(  # noqa: PLR0913
        self, Q: torch.Tensor, *, k: int, num_hits: int, metric: str = "cosine", algo: str = "auto",
        row_allowed: torch.Tensor | None = None, flags: int = 0, sample_stride: int = 0, cand_cap: int = 0,
        out: ScanResult | None = None, mask_has_tombstones: bool = False,
    ) -> ScanResult:
        """Asynchronous shard scan on the current stream: Q is float32 ``[B, d]`` on this device.
        ``row_allowed`` is the optional per-row byte mask (``row_mask`` builds it from a metadata filter;
        ``mask_has_tombstones`` says the tombstones are already folded in)."""
        if Q.dtype != torch.float32 or Q.ndim != 2 or Q.shape[1] != self.d or not Q.is_contiguous():
            raise ValueError(f"Q must be a contiguous float32 [B, {self.d}] tensor")
        if metric not in RL_METRIC:
            raise ValueError(f"Unsupported metric: {metric}")
        B = int(Q.shape[0])
        H = num_hits if num_hits > 0 else k
        with self._lock, torch.cuda.device(self.device):
            if self._alive is not None and not mask_has_tombstones:  # tombstoned rows are masked like a metadata filter
                row_allowed = self._alive if row_allowed is None else (row_allowed & self._alive)
            p = self._params(Q, k, num_hits, metric, algo, row_allowed, flags, sample_stride, cand_cap)
            if flags & RL_FLAG_COUNT_UNFILTERED:
                p.row_alive = _ptr(self._alive)
            need = int(self.lib.rl_maxsim_workspace_bytes(C.byref(p)))
            if need == 0 and B > 0:
                raise _lib.RagliteB200Error("rl_maxsim_workspace_bytes: " + self.lib.rl_last_error().decode())
            ws = self._workspace(need)
            if out is None:
                out = new_scan_result(B, H, num_hits, k, self.device)
            check(self.lib.rl_maxsim_topk(C.byref(p), _ptr(out.hit_sim), _ptr(out.hit_chunk), _ptr(out.hit_count),
                                          _ptr(out.status), _ptr(ws), ws.numel(), _stream()),
                  "rl_maxsim_topk")
            self.last_params, self.last_ws = p, ws
        return out

    def count_at_least(  # noqa: PLR0913
        self, Q: torch.Tensor, sim_floor: torch.Tensor, *, k: int, num_hits: int, metric: str = "cosine",
        algo: str = "auto", bound: int = 1,
    ) -> torch.Tensor:
        """``rl_maxsim_count_at_least``: per query, how many live rows of the shard have a similarity of at
        least ``sim_floor[b]`` (``bound=+1``: upper bound of the exact count, ``-1``: lower bound, ``0``:
        raw approximate keys).  One pass over the corpus on the current stream; int32 ``[B]`` on device."""
        if Q.dtype != torch.float32 or Q.ndim != 2 or Q.shape[1] != self.d or not Q.is_contiguous():
            raise ValueError(f"Q must be a contiguous float32 [B, {self.d}] tensor")
        B = int(Q.shape[0])
        floor = sim_floor.to(device=self.device, dtype=torch.float32).contiguous()
        if floor.shape != (B,):
            raise ValueError("sim_floor must be [B]")
        counts = torch.zeros(B, dtype=torch.int32, device=self.device)
        with self._lock, torch.cuda.device(self.device):
            p = self._params(Q, k, num_hits, metric, algo, self._alive, 0, 0, 0)
            need = int(self.lib.rl_maxsim_workspace_bytes(C.byref(p)))
            if need == 0 and B > 0:
                raise _lib.RagliteB200Error("rl_maxsim_workspace_bytes: " + self.lib.rl_last_error().decode())
            ws = self._workspace(need)
            check(self.lib.rl_maxsim_count_at_least(C.byref(p), _ptr(floor), int(bound), _ptr(counts), _ptr(ws),
                                                    ws.numel(), _stream()), "rl_maxsim_count_at_least")
        return counts

    def unfiltered_bound(self) -> torch.Tensor:
        """``rl_maxsim_unfiltered_bound`` of the last scan (made with ``RL_FLAG_COUNT_UNFILTERED``): per query an
        upper bound of the live rows of this shard at least as near as the worst filtered hit; -1 where the
        scan did not count (float32 kernel).  int64 ``[B]`` on the device, no synchronisation."""
        p = self.last_params
        out = torch.empty(int(p.B), dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            check(self.lib.rl_maxsim_unfiltered_bound(C.byref(p), _ptr(self.last_ws), _ptr(out), _stream()),
                  "rl_maxsim_unfiltered_bound")
        return out

    def sum_over_shards(self, x: torch.Tensor) -> torch.Tensor:
        """A single shard is the whole corpus (``ShardedIndex`` all-reduces)."""
        return x

    def max_over_shards(self, x: torch.Tensor) -> torch.Tensor:
        return x

    def scan_stats(self) -> dict[str, int]:
        """Counters of the last scan (synchronises)."""
        if self.last_params is None or self.last_ws is None:
            return {}
        st = ScanStats()
        with torch.cuda.device(self.device):
            check(self.lib.rl_maxsim_stats(C.byref(self.last_params), _ptr(self.last_ws), C.byref(st), _stream()),
                  "rl_maxsim_stats")
        return {name: int(getattr(st, name)) for name, _ in ScanStats._fields_}

    def debug_dump(self) -> torch.Tensor:
        """Sampled approximate keys ``[B, n_sample_rows]`` of the last scan (test hook)."""
        n = C.c_int64(0)
        p = self.last_params
        check(self.lib.rl_maxsim_copy_dump(C.byref(p), _ptr(self.last_ws), None, C.byref(n), _stream()), "rl_maxsim_copy_dump")
        out = torch.empty((int(p.B), int(n.value)), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            check(self.lib.rl_maxsim_copy_dump(C.byref(p), _ptr(self.last_ws), _ptr(out), C.byref(n), _stream()),
                  "rl_maxsim_copy_dump")
        return out

    def debug_eps(self) -> torch.Tensor:
        """Per-query error bound ``eps [B]`` of the approximate keys of the last scan, as the kernels computed it (test hook)."""
        p = self.last_params
        out = torch.empty(int(p.B), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            check(self.lib.rl_maxsim_copy_eps(C.byref(p), _ptr(self.last_ws), _ptr(out), _stream()), "rl_maxsim_copy_eps")
        return out

    def debug_candidates(self) -> dict[str, torch.Tensor]:
        """Candidate list of the last scan (test hook): ``key`` float32 and ``row`` int32 ``[B, cap]`` (the first
        ``min(cand_cnt[b], cap)`` entries of row b are valid), ``cand_cnt`` int32 ``[B]``, the select kernel's emission
        threshold ``thr`` and the refinement histogram's ``hist_inv_w`` (float32 ``[B]``)."""
        p = self.last_params
        B, cap = int(p.B), self.scan_stats()["cand_cap"]
        dev = self.device
        out = {"key": torch.empty((B, cap), dtype=torch.float32, device=dev),
               "row": torch.empty((B, cap), dtype=torch.int32, device=dev),
               "cand_cnt": torch.empty(B, dtype=torch.int32, device=dev),
               "thr": torch.empty(B, dtype=torch.float32, device=dev),
               "hist_inv_w": torch.empty(B, dtype=torch.float32, device=dev)}
        with torch.cuda.device(dev):
            check(self.lib.rl_maxsim_copy_candidates(C.byref(p), _ptr(self.last_ws), *(_ptr(out[n]) for n in out), _stream()),
                  "rl_maxsim_copy_candidates")
        return out

    def kernel_times_ms(self) -> dict[str, float]:
        """Stage times of the last scan made with ``flags=RL_FLAG_TIME_KERNELS`` (synchronises)."""
        ms = (C.c_float * 5)()
        check(self.lib.rl_maxsim_kernel_times(_ptr(self.last_ws), ms), "rl_maxsim_kernel_times")
        return dict(zip(("prep", "sample_scan", "select", "main_scan", "finalize"), (float(x) for x in ms), strict=True))

    def scan_checked(self, Q: torch.Tensor, **kw: Any) -> ScanResult:
        """Scan, read the status back and resolve a candidate-list overflow with ``run_until_no_overflow``.
        The index lock is held throughout: the retry reads thresholds that live in this stream's workspace.

        More than ``RL_MAX_SURVIVORS`` vectors inside the coarse scan's error band of the cut (tight
        clusters, thousands of near-duplicates) need no retry: ``finalize`` streams them."""
        kw = dict(kw)
        res = kw.pop("out", None)
        flags0, cap0 = kw.pop("flags", 0), int(kw.pop("cand_cap", 0))

        def run(flags: int, cand_cap: int) -> torch.Tensor:
            nonlocal res
            res = self.scan(Q, **kw, flags=flags, cand_cap=cand_cap, out=res)
            return res.status

        with self._lock:
            run_until_no_overflow(self, run, flags=flags0, cand_cap=cap0)
        return res

    def search_pipeline(self, Q: torch.Tensor, **kw: Any) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
        """``scan_gather_merge`` over this shard alone."""
        return scan_gather_merge(self, Q, **kw)

    def chunk_id_of(self, global_chunk: int) -> ChunkId:
        local = int(global_chunk) - self.chunk_base
        return self.chunk_ids[local] if self.chunk_ids is not None else str(int(global_chunk))

    # ---- results to the host in one copy ------------------------------------------------------------------
    @staticmethod
    def _pack_result(sim: torch.Tensor, chunk: torch.Tensor, count: torch.Tensor, status: torch.Tensor,
                     extra: torch.Tensor | None = None) -> torch.Tensor:
        """[extra int64 [B]] | chunk int64 [B, k] | sim float32 [B, k] | count int32 [B] | OR of the status words."""
        st_any = status.reshape(-1).to(torch.int32)
        st_any = st_any.max().reshape(1) if st_any.numel() else torch.zeros(1, dtype=torch.int32, device=sim.device)
        parts = [chunk.contiguous().view(torch.uint8).reshape(-1), sim.contiguous().view(torch.uint8).reshape(-1),
                 count.to(torch.int32).contiguous().view(torch.uint8).reshape(-1), st_any.view(torch.uint8).reshape(-1)]
        if extra is not None:   # an int64 [B] vector rides along (e.g. the rank-then-filter bound)
            parts.insert(0, extra.to(torch.int64).contiguous().view(torch.uint8).reshape(-1))
        return torch.cat(parts)

    @staticmethod
    def _parse_result(raw: np.ndarray, B: int, k: int, n_extra: int = 0) -> tuple:
        ext = None
        if n_extra:
            ext = raw[: n_extra * 8].view(np.int64).copy()
            raw = raw[n_extra * 8:]
        n8, n4 = B * k * 8, B * k * 4
        ids = raw[:n8].view(np.int64).reshape(B, k).copy()
        sims = raw[n8:n8 + n4].view(np.float32).reshape(B, k).copy()
        counts = raw[n8 + n4:n8 + n4 + B * 4].view(np.int32).copy()
        st = int(raw[n8 + n4 + B * 4:].view(np.int32)[0])
        return (ids, sims, counts, st) if ext is None else (ids, sims, counts, st, ext)

    @staticmethod
    def _enqueue_download(host: torch.Tensor | None, sim: torch.Tensor, chunk: torch.Tensor, count: torch.Tensor,
                          status: torch.Tensor, extra: torch.Tensor | None = None) -> torch.Tensor:
        """Enqueue ONE device->host copy of a merged result (``_pack_result`` layout) into the pinned buffer
        ``host`` -- a new one when ``host`` is missing or of another size -- and return that buffer.  Its contents
        are valid once the current stream has passed this point; ``_parse_result`` reads them."""
        dev = CorpusIndex._pack_result(sim, chunk, count, status, extra)
        if host is None or host.numel() != dev.numel():
            host = torch.empty(int(dev.numel()), dtype=torch.uint8, pin_memory=True)
        host.copy_(dev, non_blocking=True)
        return host

    def to_host(self, sim: torch.Tensor, chunk: torch.Tensor, count: torch.Tensor, status: torch.Tensor,
                extra: torch.Tensor | None = None) -> tuple[np.ndarray, np.ndarray, np.ndarray, int] | tuple:
        """One device->host copy (pinned staging buffer) of a merged result plus the OR of the status words,
        then ONE stream synchronisation -- the only host sync of a search."""
        B, k = int(sim.shape[0]), int(sim.shape[1])
        n_extra = 0 if extra is None else int(extra.numel())
        key = (B, k, n_extra, _stream())   # one staging buffer per (shape, stream): concurrent searches never share one
        if key not in self._pinned and len(self._pinned) >= 16:
            self._pinned.pop(next(iter(self._pinned)))
        host = self._pinned[key] = self._enqueue_download(self._pinned.get(key), sim, chunk, count, status, extra)
        torch.cuda.current_stream().synchronize()
        return self._parse_result(host.numpy(), B, k, n_extra)


MAX_SCAN_RUNS = 16


def raise_if_query_nonfinite(status: Any) -> None:
    """``RL_STATUS_QUERY_NONFINITE`` in any status word (an int or an int tensor) -> ``ValueError``: an ``l1`` query
    with an infinite or NaN element, which pgvector refuses as a ``halfvec``."""
    bad = status & RL_STATUS_QUERY_NONFINITE
    if bool(bad.any()) if isinstance(bad, torch.Tensor) else bad:
        raise ValueError("a query element is not finite in float16: pgvector refuses such a halfvec")


def run_until_no_overflow(local: "CorpusIndex", run: Callable[[int, int], Any], *, flags: int = 0,
                          cand_cap: int = 0) -> None:
    """The candidate-overflow policy of every search.  ``run(flags, cand_cap)`` enqueues one search and returns its
    status words (an int or an int tensor; on a sharded index the gathered words of every shard).  A candidate list
    overflows on adversarial corpus order, or when more near-ties sit at the cut than the list holds; then odd
    re-runs re-use the thresholds the failed pass wrote (``RL_FLAG_REUSE_THRESHOLDS``, same list size) and even
    re-runs start over with a list four times as large (a larger workspace: thresholds are not carried over).  Each
    shard grows its own list up to ``n_rows + 1024`` entries, which holds every row of the shard.  The loop ends on
    the status alone or after ``MAX_SCAN_RUNS`` runs, so the ranks of a sharded index, which all see the same
    gathered status, stop together; running out of runs raises ``RagliteB200Error``."""
    cap, fl = cand_cap, flags
    for n_run in range(1, MAX_SCAN_RUNS + 1):
        st = run(fl, cap)
        raise_if_query_nonfinite(st)   # (a non-finite l1 query can overflow every list: never retried)
        overflow = st & RL_STATUS_CAND_OVERFLOW
        if not (bool(overflow.any()) if isinstance(overflow, torch.Tensor) else overflow):   # (a tensor synchronises)
            return
        if n_run % 2 == 1:
            fl = flags | RL_FLAG_REUSE_THRESHOLDS
        else:
            if cap <= 0:
                cap = int(local.scan_stats().get("cand_cap", 1024))
            cap, fl = min(cap * 4, local.n_rows + 1024), flags & ~RL_FLAG_REUSE_THRESHOLDS
    raise _lib.RagliteB200Error(f"candidate lists still overflow after {MAX_SCAN_RUNS} runs")


def scan_gather_merge(  # noqa: PLR0913
    index: Any, Q: torch.Tensor, *, k: int, num_hits: int, metric: str = "cosine", algo: str = "auto",
    row_allowed: torch.Tensor | None = None, mask_has_tombstones: bool = False, flags: int = 0, cand_cap: int = 0,
    sample_stride: int = 0, rank_first_limit: int | None = None,
) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """The search pipeline of a ``CorpusIndex`` (one shard) or a ``ShardedIndex``: scan the local shard into one
    packed hit list, all-gather the lists of the R shards (none when R = 1), [rank-then-filter cut], merge the
    gathered lists in place.  Everything is enqueued on the current stream, nothing synchronises.  Returns
    ``(sim [B, k], chunk [B, k], count [B], status [R, B])``; every rank holds the same four tensors, and the
    status words of every shard ride along in the one collective."""
    local: CorpusIndex = getattr(index, "local", index)
    R = getattr(index, "world", 1)
    res = local.scan(Q, k=k, num_hits=num_hits, metric=metric, algo=algo, row_allowed=row_allowed,
                     mask_has_tombstones=mask_has_tombstones, flags=flags, cand_cap=cand_cap, sample_stride=sample_stride)
    B, H = int(res.hit_sim.shape[0]), int(res.hit_sim.shape[1])
    allb = res.packed
    if R > 1:
        allb = torch.empty(R * res.packed.numel(), dtype=torch.uint8, device=res.packed.device)
        dist.all_gather_into_tensor(allb, res.packed, group=index.group)
    _, sim, count, status = hits_views(allb, R, B, H)
    if rank_first_limit is not None:
        count.copy_(limit_hits_to_nearest(index, Q, sim, count, k=k, num_hits=num_hits, metric=metric, algo=algo,
                                          limit=rank_first_limit))
    return (*merge_packed(allb, R, B, H, num_hits=num_hits, k=k), status)


def search_to_host(  # noqa: PLR0913
    index: Any, Q: torch.Tensor, *, k: int, num_hits: int, metric: str, algo: str = "auto",
    chunk_ok: torch.Tensor | None = None, rank_first_limit: int | None = None,
) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """The whole search for a (sharded or single) index with ONE host synchronisation: scan ->
    [all-gather] -> merge are enqueued back to back, results and status come back in one pinned copy,
    and only then is the (rare) candidate overflow looked at.  On a sharded corpus the status words
    travel with the gathered hit lists, so every rank takes the same retry decision without a second
    collective.  Holds the index lock from the first launch to the verified result."""
    local: CorpusIndex = getattr(index, "local", index)
    with local._lock, torch.cuda.device(local.device):
        mask = local.row_mask(chunk_ok)
        kw = dict(k=k, num_hits=num_hits, metric=metric, algo=algo, row_allowed=mask, mask_has_tombstones=True)
        # Rank-then-filter branch (_search.py:122-143): first try to PROVE, from counters the filtered scan keeps
        # anyway, that fewer than `limit` rows of the whole corpus are as near as the worst filtered hit -- then
        # the filter-first answer is the answer and no second pass over the corpus is needed.
        fused = rank_first_limit is not None and mask is not None
        out = None

        def run(flags: int, cand_cap: int) -> int:
            nonlocal fused, out
            if fused:
                sim, chunk, count, status = index.search_pipeline(Q, **kw, flags=flags | RL_FLAG_COUNT_UNFILTERED,
                                                                  cand_cap=cand_cap)
                bound = index.sum_over_shards(local.unfiltered_bound().clamp(min=-1))
                neg = index.sum_over_shards((local.unfiltered_bound() < 0).to(torch.int64))   # any shard that did not count
                ids, sims, counts, st, ub = local.to_host(sim, chunk, count, status, torch.where(neg > 0, -1, bound))
                out = ids, sims, counts
                if st & (RL_STATUS_CAND_OVERFLOW | RL_STATUS_QUERY_NONFINITE) or (ub.min() >= 0 and ub.max() <= rank_first_limit):
                    return st   # (a non-finite query raises in the caller; it never reaches the counting passes)
                fused = False       # not provable from the counters: run the explicit rank probe
            ids, sims, counts, st = local.to_host(*index.search_pipeline(Q, **kw, flags=flags, cand_cap=cand_cap,
                                                                         rank_first_limit=rank_first_limit))
            out = ids, sims, counts
            return st

        run_until_no_overflow(local, run)
        return out


class _SearchSlot:
    """A CUDA stream with its own pinned result buffer: one search in flight."""

    def __init__(self, device: Any):
        self.stream = torch.cuda.Stream(device=device)
        self.host: torch.Tensor | None = None
        self.busy = False


class PendingSearch:
    """A search that has been enqueued on its own stream (queries up, kernels, results down to a private pinned
    buffer) but not waited for.  ``result()`` waits for THAT stream only; a candidate-list overflow (rare: adversarial
    row order, masses of near-ties) is then resolved by re-running the search synchronously on the same stream."""

    def __init__(self, index: Any, Q: torch.Tensor, kw: dict[str, Any], slot: _SearchSlot | None, event: Any, B: int, k: int,
                 ready: tuple | None = None):
        self._index, self._Q, self._kw, self._slot, self._event, self._B, self._k, self._ready = index, Q, kw, slot, event, B, k, ready

    def done(self) -> bool:
        return self._ready is not None or bool(self._event.query())

    def result(self) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
        if self._ready is None:
            slot = self._slot
            self._event.synchronize()
            ids, sims, counts, st = CorpusIndex._parse_result(slot.host.numpy(), self._B, self._k)
            if st & RL_STATUS_QUERY_NONFINITE:
                slot.busy = False
                raise_if_query_nonfinite(st)
            if st & RL_STATUS_CAND_OVERFLOW:
                with torch.cuda.stream(slot.stream):
                    ids, sims, counts = search_to_host(self._index, self._Q, **self._kw)
            slot.busy = False
            self._ready = (ids, sims, counts)
            self._Q = None
        return self._ready


def search_async(  # noqa: PLR0913
    index: Any, queries: Any, *, k: int, num_hits: int, metric: str, algo: str = "auto", chunk_ok: torch.Tensor | None = None,
    rank_first_limit: int | None = None, prepare: Any | None = None, max_in_flight: int = 8,
) -> PendingSearch:
    """``search_to_host`` without the wait: picks a free (stream, pinned buffer) slot of the index, and on that stream
    uploads the queries, runs ``prepare`` (e.g. the query adapter), enqueues scan -> [all-gather] -> merge and the
    device->host copy of the result.  Several calls overlap on the GPU -- the tail of one batch's scan with the
    sampling pass and selection of the next, the copies and the host-side launch work with everything -- which is
    how a server keeps the device busy.  The calling thread issues all launches (and, on a sharded index, all
    collectives) in program order, so every rank sees the same order.  Searches that may need a second corpus pass
    on the host's decision (the rank-then-filter branch) run synchronously on the slot's stream."""
    local: CorpusIndex = getattr(index, "local", index)
    with local._lock:
        slot = next((sl for sl in local._slots if not sl.busy), None)
        if slot is None:
            if len(local._slots) >= max_in_flight:
                raise RuntimeError(f"{max_in_flight} searches are already in flight on this index; collect a result() first")
            slot = _SearchSlot(local.device)
            local._slots.append(slot)
        slot.busy = True
    kw = dict(k=k, num_hits=num_hits, metric=metric, algo=algo, chunk_ok=chunk_ok, rank_first_limit=rank_first_limit)
    try:
        slot.stream.wait_stream(torch.cuda.current_stream(local.device))   # inputs produced on the caller's stream
        with torch.cuda.device(local.device), torch.cuda.stream(slot.stream):
            Q = torch.as_tensor(queries).to(device=local.device, dtype=torch.float32, non_blocking=True).contiguous()
            if prepare is not None:
                Q = prepare(Q)
            B = int(Q.shape[0])
            if rank_first_limit is not None:
                out = search_to_host(index, Q, **kw)
                slot.busy = False
                return PendingSearch(index, Q, kw, None, None, B, k, ready=out)
            with local._lock:
                mask = local.row_mask(chunk_ok)
                out = index.search_pipeline(Q, k=k, num_hits=num_hits, metric=metric, algo=algo, row_allowed=mask,
                                            mask_has_tombstones=True)
                slot.host = local._enqueue_download(slot.host, *out)
            event = torch.cuda.Event()
            event.record(slot.stream)
        return PendingSearch(index, Q, kw, slot, event, B, k)
    except Exception:
        slot.busy = False
        raise


def merge_hits(  # noqa: PLR0913
    hit_sim: torch.Tensor, hit_chunk: torch.Tensor, hit_count: torch.Tensor, *, num_hits: int, k: int
) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """``rl_topk_merge`` over ``[R, B, H]`` gathered shard outputs -> ``(sim[B,k], chunk[B,k], count[B])``."""
    lib = _lib.load()
    if hit_sim.ndim == 2:
        hit_sim, hit_chunk, hit_count = hit_sim[None], hit_chunk[None], hit_count[None]
    R, B, H = (int(x) for x in hit_sim.shape)
    dev = hit_sim.device
    out_sim = torch.empty((B, k), dtype=torch.float32, device=dev)
    out_chunk = torch.empty((B, k), dtype=torch.int64, device=dev)
    out_count = torch.empty((B,), dtype=torch.int32, device=dev)
    hs, hc, hn = hit_sim.contiguous(), hit_chunk.contiguous(), hit_count.contiguous()
    with torch.cuda.device(dev):
        check(lib.rl_topk_merge(_ptr(hs), _ptr(hc), _ptr(hn), R, B, H, num_hits, k, _ptr(out_sim), _ptr(out_chunk),
                                _ptr(out_count), _stream()), "rl_topk_merge")
    return out_sim, out_chunk, out_count


def merge_packed(packed: torch.Tensor, R: int, B: int, H: int, *, num_hits: int, k: int
                 ) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """``rl_topk_merge_packed`` over ``R`` gathered packed hit lists (``packed`` is the all-gather output)."""
    lib = _lib.load()
    dev = packed.device
    out_sim = torch.empty((B, k), dtype=torch.float32, device=dev)
    out_chunk = torch.empty((B, k), dtype=torch.int64, device=dev)
    out_count = torch.empty((B,), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        check(lib.rl_topk_merge_packed(_ptr(packed), packed.numel() // R, R, B, H, num_hits, k, _ptr(out_sim), _ptr(out_chunk),
                                       _ptr(out_count), _stream()), "rl_topk_merge_packed")
    return out_sim, out_chunk, out_count


def limit_hits_to_nearest(  # noqa: PLR0913
    index: Any, Q: torch.Tensor, hit_sim: torch.Tensor, hit_count: torch.Tensor, *, k: int, num_hits: int, metric: str,
    algo: str = "auto", limit: int = 1_000_000, bisect_steps: int = 26,
) -> torch.Tensor:
    """The rank-then-filter metadata branch (``_search.py:122-143``): of the filtered hits only those among
    the ``limit`` nearest vectors of the WHOLE corpus count.  ``hit_sim`` / ``hit_count`` are the gathered
    filter-first hit lists ``[R, B, H]`` / ``[R, B]`` (descending per list); returns the counts to keep.

    One counting pass proves the common case: if at most ``limit`` rows can be as near as the worst of
    the ``num_hits`` best filtered hits, the filter-first answer already is the answer.  Otherwise the
    similarity of the ``limit``-th nearest row is located by bisection over counting passes (raw
    approximate keys: rows within the key error of that similarity may land on either side -- the
    reference's HNSW scan is approximate at the same place)."""
    local: CorpusIndex = getattr(index, "local", index)
    R, B, H = (int(x) for x in hit_sim.shape)
    valid = torch.arange(H, device=hit_sim.device)[None, None, :] < hit_count[:, :, None]
    flat = torch.where(valid, hit_sim, hit_sim.new_full((), float("-inf"))).permute(1, 0, 2).reshape(B, R * H)
    top = flat.topk(min(num_hits, R * H), dim=1).values
    n_valid = hit_count.sum(0).clamp(max=top.shape[1]).to(torch.int64)
    floor = top.gather(1, (n_valid - 1).clamp(min=0)[:, None])[:, 0]
    floor = torch.where(n_valid > 0, floor, floor.new_full((), float("inf")))
    kw = {"k": k, "num_hits": num_hits, "metric": metric}
    ub = index.sum_over_shards(local.count_at_least(Q, floor, algo=algo, bound=1, **kw).to(torch.int64))
    need = torch.nonzero(ub > limit).flatten()
    if need.numel() == 0:
        return hit_count
    # bisection on the similarity of the limit-th nearest row, for the queries that need it
    Qn = Q[need].contiguous()
    lo = floor[need].clone()
    qn = Qn.double().norm(dim=1)
    # The bracket must be identical on every rank (the counts are summed over shards against one `mid`):
    # the largest row norm is taken over all shards, not this rank's own.
    max_norm = index.max_over_shards(local.stats[0:1].to(torch.float32).clone()).double()
    hi = (1.0 + qn * max_norm * 1.001 + 1e-3).float() if metric == "dot" else torch.full_like(lo, 1.0 + 1e-3)
    exact_algo = "fp32" if local.storage == "fp32" else algo   # tightest keys this storage allows
    for _ in range(bisect_steps):
        mid = (lo + hi) * 0.5
        c = index.sum_over_shards(local.count_at_least(Qn, mid, algo=exact_algo, bound=0, **kw).to(torch.int64))
        ge = c >= limit
        lo = torch.where(ge, mid, lo)
        hi = torch.where(ge, hi, mid)
    tau = torch.full((B,), float("-inf"), device=hit_sim.device)
    tau[need] = lo
    keep = (valid & (hit_sim >= tau[None, :, None])).sum(-1).to(hit_count.dtype)
    return torch.minimum(hit_count, keep)


# ---- registry: RAGLiteConfig.db_url -> index ---------------------------------------------------------
_REGISTRY: dict[str, Any] = {}


def register_index(config_or_url: Any, index: Any) -> None:
    """Attach a device-resident index to a ``RAGLiteConfig`` (keyed by ``db_url``)."""
    _REGISTRY[str(getattr(config_or_url, "db_url", config_or_url))] = index


def unregister_index(config_or_url: Any) -> None:
    _REGISTRY.pop(str(getattr(config_or_url, "db_url", config_or_url)), None)


def get_index(config: Any) -> Any | None:
    return _REGISTRY.get(str(config.db_url))
