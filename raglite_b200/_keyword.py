"""Device-resident inverted index over the chunk bodies: the counterpart of DuckDB's FTS tables (``fts_main_chunk.dict``,
``docs``, ``terms``, ``stats``) that ``create_fts_index`` builds for the reference's ``keyword_search``
(``_database.py:618``, rebuilt after every insert and delete: ``_insert.py:268``, ``_delete.py:173``).

Layout on the device (``rl_bm25_stats`` / ``rl_bm25_topk_global``, include/raglite_b200.h):

    term_off  int64   [V + 1]   term-major postings CSR
    doc, tf   int32   [P]       postings sorted by chunk within each term (tf = occurrences of the term in the chunk)
    doc_len   int32   [C]       terms of each chunk after stop-word removal
    df        int32   [V]       live chunks holding each term       (rl_bm25_stats, recomputed after every change)
    corpus    float64 [3]       N, sum of doc_len, avgdl over the live chunks

The host keeps the ``stem -> term id`` dictionary (``_fts.Analyzer``) and, from each refresh, ``df``, ``N`` and the sum
of ``doc_len`` as integers: a search looks up the statistics of its query terms there and uploads them with its plan.
A ``CorpusIndex`` owns one of these and builds it on its first keyword search; appended chunks are analysed on the next
search, deletes only make the statistics stale (tombstoned chunks keep their postings and are masked), ``compact``
remaps the postings.
"""

from __future__ import annotations

import time
from collections.abc import Sequence
from typing import Any

import numpy as np
import torch

from . import _lib
from ._fts import Analyzer

K1, B_PARAM = 1.2, 0.75          # match_bm25 defaults
MAX_RESULTS = 4096               # RL_MAX_SURVIVORS, the num_hits cap of the vector path
WORKSPACE_BYTES = 1 << 30        # dense score keys of one query group: 8 bytes per (query, chunk)


def _ptr(t: torch.Tensor | None) -> int | None:
    return None if t is None else int(t.data_ptr())


def _stream() -> int:
    return int(torch.cuda.current_stream().cuda_stream)


class KeywordIndex:
    """BM25 postings of one ``CorpusIndex`` shard.  Every method is called under the owning index's lock."""

    def __init__(self, device: torch.device) -> None:
        self.lib = _lib.load()
        self.device = device
        self.analyzer = Analyzer()
        self.n_chunks = 0
        with torch.cuda.device(device):
            self.term_off = torch.zeros(1, dtype=torch.int64, device=device)
            self.doc = torch.zeros(0, dtype=torch.int32, device=device)
            self.tf = torch.zeros(0, dtype=torch.int32, device=device)
            self.doc_len = torch.zeros(0, dtype=torch.int32, device=device)
            self.df = torch.zeros(0, dtype=torch.int32, device=device)
            self.corpus = torch.zeros(3, dtype=torch.float64, device=device)
        self.df_host = np.zeros(1, dtype=np.int64)   # df of every term, then a 0 that an entry of -1 looks up
        self.n_live, self.sum_len = 0, 0
        self.alive: torch.Tensor | None = None   # uint8 [C] of the last refresh; None = no tombstones
        self.stale = True
        self.build_seconds = {"analysis": 0.0, "postings": 0.0}
        self._ws: dict[int, torch.Tensor] = {}
        self._pinned: dict[Any, torch.Tensor] = {}

    @property
    def n_terms(self) -> int:
        return int(self.term_off.numel()) - 1

    def _term_of_postings(self) -> torch.Tensor:
        return torch.repeat_interleave(torch.arange(self.n_terms, dtype=torch.int64, device=self.device),
                                       torch.diff(self.term_off))

    def _set_postings(self, term: torch.Tensor, doc: torch.Tensor, tf: torch.Tensor) -> None:
        """Postings given sorted by (term, doc); term ids index the analyzer's dictionary."""
        V = len(self.analyzer.term_ids)
        counts = torch.bincount(term, minlength=V)
        self.term_off = torch.cat([torch.zeros(1, dtype=torch.int64, device=self.device), torch.cumsum(counts, 0)])
        self.doc, self.tf = doc.to(torch.int32).contiguous(), tf.to(torch.int32).contiguous()

    def extend(self, bodies: Sequence[str]) -> None:
        """Index the bodies of the chunks ``n_chunks, n_chunks + 1, ...`` (new terms get new ids).  The new (term, chunk)
        pairs are counted and merged into the postings on the device: one sort of the packed ``term << 32 | chunk``
        keys."""
        t0 = time.perf_counter()
        terms, owners, lens = self.analyzer.analyze(bodies)
        t1 = time.perf_counter()
        dev = self.device
        with torch.cuda.device(dev):
            owners = torch.from_numpy(owners).to(dev, dtype=torch.int64) + self.n_chunks
            key = (torch.from_numpy(terms).to(dev, dtype=torch.int64) << 32) | owners
            key, tf = torch.unique(key, sorted=True, return_counts=True)
            if self.doc.numel():
                old = (self._term_of_postings() << 32) | self.doc.to(torch.int64)
                key, order = torch.sort(torch.cat([old, key]))
                tf = torch.cat([self.tf.to(torch.int64), tf])[order]
            self._set_postings(key >> 32, key & 0xFFFFFFFF, tf)
            self.doc_len = torch.cat([self.doc_len, torch.from_numpy(lens).to(dev)])
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
            keep_d = torch.from_numpy(keep).to(dev)
            new_index = torch.cumsum(keep_d.to(torch.int64), 0) - 1
            doc = self.doc.to(torch.int64)
            sel = keep_d[doc]
            term = self._term_of_postings()[sel]
            self._set_postings(term, new_index[doc][sel], self.tf[sel])
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

    def _workspace(self, need: int) -> torch.Tensor:
        key = _stream()
        ws = self._ws.get(key)
        if ws is None or ws.numel() < need:
            self._ws.pop(key, None)
            ws = self._ws[key] = torch.empty(need, dtype=torch.uint8, device=self.device)
        return ws

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
            if R > 1:
                gathered = index.gather_shards(packed)
                packed = torch.empty(nbytes, dtype=torch.uint8, device=dev)
                _lib.check(lib.rl_bm25_merge_packed(_ptr(gathered), R, B, int(k), _ptr(packed), _ptr(packed) + B * k * 8,
                                                    _ptr(packed) + B * k * 16, _stream()), "rl_bm25_merge_packed")
            return self._download(packed, B, k)

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
