"""Device-resident inverted index over the chunk bodies: the counterpart of DuckDB's FTS tables (``fts_main_chunk.dict``,
``docs``, ``terms``, ``stats``) that ``create_fts_index`` builds for the reference's ``keyword_search``
(``_database.py:618``, rebuilt after every insert and delete: ``_insert.py:268``, ``_delete.py:173``).

Layout on the device (``rl_bm25_stats`` / ``rl_bm25_topk_global``, include/raglite_b200.h):

    term_off  int64   [V + 1]   term-major postings CSR
    doc, tf   int32   [P]       postings sorted by chunk within each term (tf = occurrences of the term in the chunk)
    doc_len   int32   [C]       terms of each chunk after stop-word removal
    df        int32   [V]       live chunks holding each term       (rl_bm25_stats, recomputed after every change)
    corpus    float64 [3]       N, sum of doc_len, avgdl over the live chunks

The bodies are analysed on the device (``_fts.analyze_on_device``); the host keeps the ``stem -> term id`` dictionary
(``_fts.Analyzer``, which the device analysis grows exactly as the host analysis would) and, from each refresh, ``df``,
``N`` and the sum of ``doc_len`` as integers: a search looks up the statistics of its query terms there and uploads them
with its plan.
A ``CorpusIndex`` owns one of these and builds it on its first keyword search; appended chunks are analysed on the next
search, deletes only make the statistics stale (tombstoned chunks keep their postings and are masked), ``compact``
remaps the postings.

``TsRankIndex`` is the counterpart for a PostgreSQL database: ``ts_rank`` over ``to_tsvector('simple', body)``
(``_search.py:176-201``), built from the tsvectors the database computes (``CorpusIndex.add_tsvector_rows``) and searched
by ``rl_tsrank_topk_global`` with the same select, packed layout and shard merge.
"""

from __future__ import annotations

import time
from collections.abc import Sequence
from typing import Any

import numpy as np
import torch

from . import _lib, _pgfts
from ._fts import Analyzer, analyze_on_device

K1, B_PARAM = 1.2, 0.75          # match_bm25 defaults
MAX_RESULTS = 4096               # RL_MAX_SURVIVORS, the num_hits cap of the vector path
WORKSPACE_BYTES = 1 << 30        # dense score keys of one query group: 8 bytes per (query, chunk)


def _ptr(t: torch.Tensor | None) -> int | None:
    return None if t is None else int(t.data_ptr())


def _stream() -> int:
    return int(torch.cuda.current_stream().cuda_stream)


class _Postings:
    """A term-major postings CSR on one device (``term_off`` int64 [V + 1], ``doc`` int32 [P] sorted by chunk within each
    term; the subclass keeps one int32 value per posting) and what a top-k search over it reuses: a workspace per
    stream, pinned staging for the download, the shard merge."""

    def __init__(self, device: torch.device) -> None:
        self.lib = _lib.load()
        self.device = device
        with torch.cuda.device(device):
            self.term_off = torch.zeros(1, dtype=torch.int64, device=device)
            self.doc = torch.zeros(0, dtype=torch.int32, device=device)
        self._ws: dict[int, torch.Tensor] = {}
        self._pinned: dict[Any, torch.Tensor] = {}

    @property
    def n_terms(self) -> int:
        return int(self.term_off.numel()) - 1

    def _term_of_postings(self) -> torch.Tensor:
        return torch.repeat_interleave(torch.arange(self.n_terms, dtype=torch.int64, device=self.device),
                                       torch.diff(self.term_off))

    def _set_csr(self, term: torch.Tensor, doc: torch.Tensor, n_terms: int) -> None:
        """Postings given sorted by (term, doc)."""
        counts = torch.bincount(term, minlength=n_terms)
        self.term_off = torch.cat([torch.zeros(1, dtype=torch.int64, device=self.device), torch.cumsum(counts, 0)])
        self.doc = doc.to(torch.int32).contiguous()

    def _merge_postings(self, key: torch.Tensor, value: torch.Tensor, old_value: torch.Tensor, n_terms: int) -> torch.Tensor:
        """New postings -- packed ``term << 32 | chunk`` keys, sorted, none already held -- merged into the CSR with one
        sort on the device.  Returns the merged values (int32)."""
        if self.doc.numel():
            old = (self._term_of_postings() << 32) | self.doc.to(torch.int64)
            key, order = torch.sort(torch.cat([old, key]))
            value = torch.cat([old_value.to(torch.int64), value])[order]
        self._set_csr(key >> 32, key & 0xFFFFFFFF, n_terms)
        return value.to(torch.int32).contiguous()

    def _compact_postings(self, keep: np.ndarray, value: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        """Drop the postings of the chunks with ``keep[c] == False`` and renumber the rest (a monotone map, so every
        term's postings stay sorted).  Returns the kept values and ``keep`` on the device."""
        keep_d = torch.from_numpy(keep).to(self.device)
        new_index = torch.cumsum(keep_d.to(torch.int64), 0) - 1
        doc = self.doc.to(torch.int64)
        sel = keep_d[doc]
        term = self._term_of_postings()[sel]
        self._set_csr(term, new_index[doc][sel], self.n_terms)
        return value[sel].to(torch.int32).contiguous(), keep_d

    def _workspace(self, need: int) -> torch.Tensor:
        key = _stream()
        ws = self._ws.get(key)
        if ws is None or ws.numel() < need:
            self._ws.pop(key, None)
            ws = self._ws[key] = torch.empty(need, dtype=torch.uint8, device=self.device)
        return ws

    def _merge_shards(self, index: Any, packed: torch.Tensor, B: int, k: int) -> torch.Tensor:
        """On a ``ShardedIndex`` of R > 1 shards: ONE all-gather of the packed per-shard top k and ``rl_bm25_merge_packed``
        into a new packed buffer; ``packed`` itself otherwise."""
        if not hasattr(index, "group") or index.world <= 1:
            return packed
        gathered = index.gather_shards(packed)
        packed = torch.empty(packed.numel(), dtype=torch.uint8, device=self.device)
        _lib.check(self.lib.rl_bm25_merge_packed(_ptr(gathered), index.world, B, int(k), _ptr(packed), _ptr(packed) + B * k * 8,
                                                 _ptr(packed) + B * k * 16, _stream()), "rl_bm25_merge_packed")
        return packed

    def _download(self, out: torch.Tensor, B: int, k: int) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
        """One pinned copy of ``chunk int64 [B, k] | score float64 [B, k] | count int32 [B]`` and one synchronisation."""
        pkey = (out.numel(), _stream())
        host = self._pinned.get(pkey)
        if host is None:
            if len(self._pinned) >= 8:
                self._pinned.pop(next(iter(self._pinned)))
            host = self._pinned[pkey] = torch.empty(out.numel(), dtype=torch.uint8, pin_memory=True)
        host.copy_(out, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        raw = host.numpy()
        return (raw[: B * k * 8].view(np.int64).reshape(B, k).copy(), raw[B * k * 8: B * k * 16].view(np.float64).reshape(B, k).copy(),
                raw[B * k * 16: B * k * 16 + B * 4].view(np.int32).copy())


class KeywordIndex(_Postings):
    """BM25 postings of one ``CorpusIndex`` shard.  Every method is called under the owning index's lock."""

    def __init__(self, device: torch.device) -> None:
        super().__init__(device)
        self.analyzer = Analyzer()
        self.n_chunks = 0
        with torch.cuda.device(device):
            self.tf = torch.zeros(0, dtype=torch.int32, device=device)
            self.doc_len = torch.zeros(0, dtype=torch.int32, device=device)
            self.df = torch.zeros(0, dtype=torch.int32, device=device)
            self.corpus = torch.zeros(3, dtype=torch.float64, device=device)
        self.df_host = np.zeros(1, dtype=np.int64)   # df of every term, then a 0 that an entry of -1 looks up
        self.n_live, self.sum_len = 0, 0
        self.alive: torch.Tensor | None = None   # uint8 [C] of the last refresh; None = no tombstones
        self.stale = True
        self.build_seconds = {"analysis": 0.0, "postings": 0.0}
        self.analysis_seconds = {"encode": 0.0, "device": 0.0, "dictionary": 0.0}   # the split of build_seconds["analysis"]

    def extend(self, bodies: Sequence[str]) -> None:
        """Index the bodies of the chunks ``n_chunks, n_chunks + 1, ...`` (new terms get new ids).  The bodies are
        analysed on the device (``_fts.analyze_on_device``: the packed ``term << 32 | chunk`` key of every kept token),
        and the new (term, chunk) pairs are counted and merged into the postings there: one sort of the keys."""
        t0 = time.perf_counter()
        dev = self.device
        key, lens = analyze_on_device(self.analyzer, bodies, dev, chunk_base=self.n_chunks, seconds=self.analysis_seconds)
        t1 = time.perf_counter()
        with torch.cuda.device(dev):
            key, tf = torch.unique(key, sorted=True, return_counts=True)
            self.tf = self._merge_postings(key, tf, self.tf, len(self.analyzer.term_ids))
            self.doc_len = torch.cat([self.doc_len, lens])
            torch.cuda.current_stream().synchronize()
        self.n_chunks += len(bodies)
        self.stale = True
        self.build_seconds["analysis"] += t1 - t0
        self.build_seconds["postings"] += time.perf_counter() - t1

    def compact(self, keep: np.ndarray) -> None:
        """``CorpusIndex.compact``: drop the postings of the chunks with ``keep[c] == False`` and renumber the rest
        (a monotone map, so every term's postings stay sorted)."""
        keep = np.asarray(keep[: self.n_chunks], dtype=bool)
        dev = self.device
        with torch.cuda.device(dev):
            self.tf, keep_d = self._compact_postings(keep, self.tf)
            self.doc_len = self.doc_len[keep_d].contiguous()
            torch.cuda.current_stream().synchronize()
        self.n_chunks = int(keep.sum())
        self.alive, self.stale = None, True

    def refresh(self, chunk_alive: np.ndarray) -> None:
        """``rl_bm25_stats`` over the live chunks (``chunk_alive[:n_chunks]``), then host copies of ``df``, ``N`` and the
        sum of ``doc_len``; the copies synchronise, so that searches on other streams see the new statistics."""
        alive = np.asarray(chunk_alive[: self.n_chunks], dtype=bool)
        with torch.cuda.device(self.device):
            self.alive = None if alive.all() else torch.from_numpy(alive.astype(np.uint8)).to(self.device)
            V = self.n_terms
            self.df = torch.empty(V, dtype=torch.int32, device=self.device)
            _lib.check(self.lib.rl_bm25_stats(_ptr(self.term_off), _ptr(self.doc), _ptr(self.doc_len), _ptr(self.alive), V,
                                              self.n_chunks, _ptr(self.df), _ptr(self.corpus), _stream()), "rl_bm25_stats")
            self.df_host = np.append(self.df.cpu().numpy().astype(np.int64), 0)
            corpus = self.corpus.cpu().numpy()
        self.n_live, self.sum_len = int(corpus[0]), int(corpus[1])   # integer counts, exact in float64
        self.stale = False

    def stats(self) -> dict[str, Any]:
        """``N``, ``avgdl``, and ``df`` by stem (host copies; test and diagnostics hook)."""
        corpus = self.corpus.cpu().numpy()
        df = self.df.cpu().numpy()
        return {"N": float(corpus[0]), "sum_len": float(corpus[1]), "avgdl": float(corpus[2]),
                "df": {t: int(df[i]) for t, i in self.analyzer.term_ids.items()}}

    def topk_to_host(self, queries: Sequence[str], *, k: int, chunk_mask: torch.Tensor | None, max_group: int | None = None,
                     index: Any | None = None) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
        """The BM25 top k over ``index``: ``None`` or the ``CorpusIndex`` that owns these postings (one shard), or a
        ``ShardedIndex`` around it (a collective then: every rank calls it with the same queries and ``k``).  The query plan and its entries'
        statistics (``int64 [2 + J]`` = N, sum of doc_len, df of each entry) from the host, ONE upload of both, on more
        than one shard ONE all-reduce of the statistics (``index.sum_over_shards``), ``rl_bm25_topk_global`` into a
        packed buffer, on more than one shard ONE all-gather of the buffers (``index.gather_shards``) and
        ``rl_bm25_merge_packed``, then one pinned download and one synchronisation.  ``chunk_mask``: uint8 [C]
        (tombstones AND metadata filter), ``None`` = every chunk; ``max_group`` caps the queries scored at once.
        Returns host ``(chunk int64 [B, k] (-1 padded), score float64 [B, k] (-inf padded), count int32 [B])``, local
        chunk indices on a ``CorpusIndex`` and global ones (``chunk_base`` + local) on a ``ShardedIndex``."""
        B, C = len(queries), self.n_chunks
        sharded = hasattr(index, "group")
        if sharded:   # sorted stems, -1 kept: every shard sums the same entries in the same order
            q_off, _, ids = self.analyzer.query_plan(queries)
        else:         # the known term ids, ascending
            per = [self.analyzer.query_ids(q) for q in queries]
            q_off = np.zeros(B + 1, dtype=np.int32)
            np.cumsum([len(x) for x in per], out=q_off[1:])
            ids = np.concatenate([np.zeros(0, np.int32), *per])
        J = len(ids)
        stats = np.concatenate([[self.n_live, self.sum_len], self.df_host[ids]]).astype(np.int64)
        R = index.world if sharded else 1
        chunk_base = int(index.local.chunk_base) if sharded else 0
        group = max(1, min(B, int(max_group) if max_group else WORKSPACE_BYTES // max(8 * C, 1)))
        dev, lib = self.device, self.lib
        with torch.cuda.device(dev):
            plan = np.concatenate([stats.view(np.int32), q_off, ids])   # stats int64 [2 + J] | q_off [B + 1] | ids [J]
            plan = torch.from_numpy(plan).to(dev, non_blocking=True)
            stats_d, q_off_d = plan[: 2 * (2 + J)].view(torch.int64), _ptr(plan) + 8 * (2 + J)
            if R > 1:
                stats_d = index.sum_over_shards(stats_d)
            nbytes = int(lib.rl_bm25_packed_bytes(B, k))
            packed = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            need = int(lib.rl_bm25_workspace_bytes(C, group))
            ws = self._workspace(need) if need else None
            _lib.check(lib.rl_bm25_topk_global(
                _ptr(self.term_off), _ptr(self.doc), _ptr(self.tf), _ptr(self.doc_len), _ptr(stats_d), self.n_terms, C,
                _ptr(chunk_mask), q_off_d, q_off_d + 4 * (B + 1), B, int(k), K1, B_PARAM, chunk_base, _ptr(packed), _ptr(ws),
                need, _stream()), "rl_bm25_topk_global")
            return self._download(self._merge_shards(index, packed, B, k), B, k)


def tsrank_plan(queries: Sequence[str], lexeme_ids: dict[str, int]) -> tuple[np.ndarray, np.ndarray]:
    """The query plan of ``rl_tsrank_topk_global``: ``(q_off int32 [B + 1], q_terms int32 [J])``, each query's distinct
    lexemes in UTF-8 byte order (``_pgfts.query_lexemes``) as ids of ``lexeme_ids``, ``-1`` for a lexeme it does not hold.
    The entries and their order are the same on every shard.  Raises ``NotImplementedError`` for a phrase operand."""
    per = [[lexeme_ids.get(x, -1) for x in _pgfts.query_lexemes(q)] for q in queries]
    q_off = np.zeros(len(per) + 1, dtype=np.int32)
    np.cumsum([len(x) for x in per], out=q_off[1:])
    return q_off, np.asarray([i for x in per for i in x], dtype=np.int32)


class TsRankIndex(_Postings):
    """ts_rank postings of one ``CorpusIndex`` shard, built from PostgreSQL's ``to_tsvector('simple', body)::text``
    (``CorpusIndex.add_tsvector_rows``).  Layout (``rl_tsrank_topk_global``, include/raglite_b200.h):

        term_off  int64  [V + 1]   lexeme-major postings CSR
        doc, npos int32  [P]       postings sorted by chunk within each lexeme; npos = positions the tsvector lists (>= 1)

    The host keeps the ``lexeme -> id`` dictionary (ids in order of first appearance) and which chunks have a tsvector.
    ts_rank uses no corpus statistics: deletes only mask chunks, ``compact`` drops and renumbers their postings.  Every
    method is called under the owning index's lock."""

    def __init__(self, device: torch.device) -> None:
        super().__init__(device)
        self.lexeme_ids: dict[str, int] = {}
        self.has_tsvector = np.zeros(0, dtype=bool)   # per chunk of the owning index (chunks beyond it: none)
        with torch.cuda.device(device):
            self.npos = torch.zeros(0, dtype=torch.int32, device=device)
        self.alive: torch.Tensor | None = None   # uint8 tombstone mask of the chunks; None = every chunk live
        self.stale = True                         # the mask is rebuilt after the owning index changed
        self.build_seconds = {"parse": 0.0, "postings": 0.0}

    def add(self, chunks: np.ndarray, parsed: Sequence[tuple[Sequence[str], Sequence[int]]], parse_seconds: float = 0.0) -> None:
        """The postings of ``parsed[i] = (lexemes, npos)``, the tsvector of chunk ``chunks[i]`` (chunks without one so
        far), merged into the CSR with one device sort."""
        t0 = time.perf_counter()
        chunks = np.asarray(chunks, dtype=np.int64)
        ids = self.lexeme_ids
        term = np.fromiter((ids.setdefault(x, len(ids)) for lex, _ in parsed for x in lex), dtype=np.int64)
        owner = np.repeat(chunks, [len(lex) for lex, _ in parsed])
        npos = np.fromiter((n for _, ns in parsed for n in ns), dtype=np.int64, count=len(term))
        dev = self.device
        with torch.cuda.device(dev):
            key = torch.from_numpy((term << 32) | owner).to(dev)
            key, order = torch.sort(key)
            self.npos = self._merge_postings(key, torch.from_numpy(npos).to(dev)[order], self.npos, len(ids))
            torch.cuda.current_stream().synchronize()
        n = max(len(self.has_tsvector), int(chunks.max(initial=-1)) + 1)
        self.has_tsvector = np.concatenate([self.has_tsvector, np.zeros(n - len(self.has_tsvector), dtype=bool)])
        self.has_tsvector[chunks] = True
        self.build_seconds["parse"] += parse_seconds
        self.build_seconds["postings"] += time.perf_counter() - t0

    def missing(self, chunk_alive: np.ndarray) -> int:
        """Live chunks (``chunk_alive``) without a tsvector."""
        have = np.zeros(len(chunk_alive), dtype=bool)
        n = min(len(have), len(self.has_tsvector))
        have[:n] = self.has_tsvector[:n]
        return int((np.asarray(chunk_alive, dtype=bool) & ~have).sum())

    def compact(self, keep: np.ndarray) -> None:
        """``CorpusIndex.compact``: drop the postings of the chunks with ``keep[c] == False`` and renumber the rest."""
        keep = np.asarray(keep, dtype=bool)
        have = np.zeros(len(keep), dtype=bool)
        n = min(len(keep), len(self.has_tsvector))
        have[:n] = self.has_tsvector[:n]
        with torch.cuda.device(self.device):
            self.npos, _ = self._compact_postings(keep, self.npos)
            torch.cuda.current_stream().synchronize()
        self.has_tsvector = have[keep]
        self.alive, self.stale = None, True

    def alive_mask(self, chunk_alive: np.ndarray) -> torch.Tensor | None:
        """The tombstones as a uint8 device mask (``None`` when every chunk is live), uploaded once per index change."""
        if self.stale:
            alive = np.asarray(chunk_alive, dtype=bool)
            with torch.cuda.device(self.device):
                self.alive = None if alive.all() else torch.from_numpy(alive.astype(np.uint8)).to(self.device)
            self.stale = False
        return self.alive

    def topk_to_host(self, q_off: np.ndarray, q_terms: np.ndarray, *, k: int, n_chunks: int, chunk_mask: torch.Tensor | None,
                     index: Any | None = None, max_group: int | None = None) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
        """The ts_rank top k of a ``tsrank_plan`` over the ``n_chunks`` chunks of ``index`` (``None`` or the owning
        ``CorpusIndex``, or a ``ShardedIndex`` around it: a collective then).  ONE upload of the plan,
        ``rl_tsrank_topk_global`` into a packed buffer, on more than one shard ONE all-gather and
        ``rl_bm25_merge_packed``, one pinned download and one synchronisation.  ``chunk_mask``: uint8 [C] (tombstones AND
        metadata filter) or ``None``; ``max_group`` caps the queries scored at once.  Returns host ``(chunk int64 [B, k],
        score float64 [B, k] (the float32 ts_rank widened), count int32 [B])``, as ``KeywordIndex.topk_to_host``."""
        B, C = len(q_off) - 1, int(n_chunks)
        sharded = hasattr(index, "group")
        chunk_base = int(index.local.chunk_base) if sharded else 0
        group = max(1, min(B, int(max_group) if max_group else WORKSPACE_BYTES // max(8 * C, 1)))
        dev, lib = self.device, self.lib
        with torch.cuda.device(dev):
            plan = torch.from_numpy(np.concatenate([q_off, q_terms]).astype(np.int32)).to(dev, non_blocking=True)
            nbytes = int(lib.rl_bm25_packed_bytes(B, k))
            packed = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            need = int(lib.rl_bm25_workspace_bytes(C, group))
            ws = self._workspace(need) if need else None
            _lib.check(lib.rl_tsrank_topk_global(
                _ptr(self.term_off), _ptr(self.doc), _ptr(self.npos), self.n_terms, C, _ptr(chunk_mask), _ptr(plan),
                _ptr(plan) + 4 * (B + 1), B, int(k), chunk_base, _ptr(packed), _ptr(ws), need, _stream()),
                "rl_tsrank_topk_global")
            return self._download(self._merge_shards(index, packed, B, k), B, k)
