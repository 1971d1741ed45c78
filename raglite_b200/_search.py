"""Drop-in ``vector_search`` / ``keyword_search`` / ``rerank_chunks`` over the device-resident index.

Signatures follow the reference (``raglite/_search.py:36-43``, ``:156-162`` and ``:364-366``); the arithmetic that
the reference delegates to DuckDB SQL runs in the CUDA library instead.  ``vector_search_batch`` /
``keyword_search_batch`` are the batched entries (the reference API is single-query, ``_search.py:54-56``).
"""

from __future__ import annotations

import contextlib
from collections.abc import Sequence
from dataclasses import dataclass
from typing import Any

import numpy as np
import torch

from ._config import RAGLiteConfig
from ._index import Chunk, CorpusIndex, PendingSearch, get_index, search_async, search_to_host
from ._typing import ChunkId, FloatVector, MetadataFilter

REFERENCE_CHUNK_MAX_SIZE = 2048  # RAGLiteConfig.chunk_max_size class default (_config.py:67)


def num_hits_rule(num_results: int, oversample: int, chunk_max_size: int) -> int:
    """``_search.py:66-67``."""
    corrected_oversample = oversample * chunk_max_size / REFERENCE_CHUNK_MAX_SIZE
    return round(corrected_oversample) * max(num_results, 10)


def _adapt_metadata(metadata_filter: MetadataFilter | None) -> dict[str, list[Any]] | None:
    """Normalise filter values to lists (``_database.py:51-55``)."""
    if not metadata_filter:
        return None
    return {k: (list(v) if isinstance(v, (list, tuple)) else [v]) for k, v in metadata_filter.items()}


FILTER_FIRST_MAX_ROWS = 100_000   # metadata_count <= 100_000: filter, then rank (_search.py:105)
RANK_FIRST_LIMIT = 1_000_000      # otherwise: the 1_000_000 nearest vectors, then the filter (_search.py:126)


def _filter_on_device(index: Any, metadata_filter: dict[str, list[Any]] | None) -> tuple[torch.Tensor | None, int]:
    """The metadata filter as a per-chunk byte mask on the device plus the number of live rows it
    matches on this shard (``CorpusIndex.filter_chunks``: an inverted index over the chunk metadata,
    built once and cached per filter -- a search never walks the chunk table on the host)."""
    if not metadata_filter:
        return None, 0
    local: CorpusIndex = getattr(index, "local", index)
    return local.filter_chunks(metadata_filter)


def halfvec_round(Q: torch.Tensor) -> torch.Tensor:
    """The query as pgvector's ``halfvec`` holds it, as float32.  ``PostgresHalfVec.bind_processor``
    (``_typing.py:157-163``) binds each element as the text ``str(x)``; pgvector parses it with ``strtof`` and rounds it to
    binary16, to nearest even.  float32 and float16 elements are therefore rounded once (float16: not at all); float64
    elements twice, to float32 and then to binary16.  An element beyond the binary16 range becomes +-inf here; pgvector
    refuses it."""
    return Q.to(torch.float32).to(torch.float16).to(torch.float32)


def _check_metric(config: RAGLiteConfig) -> None:
    """``l1`` exists on PostgreSQL only (pgvector's ``<+>``); the reference's DuckDB branch has no L1 function
    (``_typing.py:125-129``)."""
    if config.vector_search_distance_metric == "l1" and not str(config.db_url).startswith("postgresql"):
        raise ValueError(f"vector_search_distance_metric='l1' needs a PostgreSQL db_url (pgvector's <+> operator); "
                         f"db_url={config.db_url!r} has no L1 distance")


def _plan_search(  # noqa: PLR0913
    queries: Any, *, num_results: int, oversample: int, metadata_filter: MetadataFilter | None, config: RAGLiteConfig | None,
    index: Any | None, exact_maxsim: bool, queries_are_fp16: bool,
) -> tuple[Any, torch.Tensor, tuple | None, dict[str, Any], Any]:
    """Argument handling shared by the synchronous and the asynchronous batched search: returns
    ``(index, Q (as given, not yet on the device), empty result or None, search kwargs, prepare(Q_device))``.
    Under ``l1`` (PostgreSQL only) ``prepare`` rounds the adapted query to ``halfvec`` (``halfvec_round``).  A host
    query that no adapter changes is range-checked here; any other query reports a non-finite element through the
    result status (``RL_STATUS_QUERY_NONFINITE``) and the search raises after its one download."""
    config = config or RAGLiteConfig()
    _check_metric(config)
    index = index if index is not None else get_index(config)
    if index is None:
        raise ValueError(f"No index registered for db_url={config.db_url!r}; use raglite_b200.register_index")
    local: CorpusIndex = getattr(index, "local", index)
    Q = torch.as_tensor(queries)
    queries_are_fp16 = queries_are_fp16 or Q.dtype == torch.float16
    if Q.ndim != 2:
        raise ValueError("queries must be [B, d]")
    halfvec = config.vector_search_distance_metric == "l1"
    adapt = config.vector_search_query_adapter and local.query_adapter is not None
    if halfvec and not adapt and Q.device.type == "cpu" and not bool(torch.isfinite(halfvec_round(Q)).all()):
        raise ValueError("a query element is not finite in float16: pgvector refuses such a halfvec")
    k = int(num_results)
    B = int(Q.shape[0])
    sharded = hasattr(index, "group")
    empty = (np.full((B, k), -1, np.int64), np.full((B, k), -np.inf, np.float32), np.zeros(B, np.int32))
    if local.n_live_chunks == 0 and not sharded:
        return index, Q, empty, {}, None
    num_hits = 0 if exact_maxsim else num_hits_rule(k, oversample, config.chunk_max_size)
    if not exact_maxsim and num_hits == 0:  # round(oversample * size / 2048) == 0 -> LIMIT 0
        return index, Q, empty, {}, None
    prepare = None
    if adapt and not halfvec:
        def prepare(Qd: torch.Tensor) -> torch.Tensor:  # (A @ q).astype(q.dtype), _search.py:58-62
            return local.apply_adapter(Qd, round_fp16=queries_are_fp16)
    elif halfvec:
        def prepare(Qd: torch.Tensor) -> torch.Tensor:  # [adapter], then the query is bound as a halfvec
            return halfvec_round(local.apply_adapter(Qd, round_fp16=queries_are_fp16) if adapt else Qd)
    chunk_ok, n_match = _filter_on_device(index, _adapt_metadata(metadata_filter))
    metric = config.vector_search_distance_metric
    # Which metadata branch the reference would take (_search.py:96-143): many matching rows in a corpus
    # of more than 1M vectors -> only filtered hits among the 1M nearest vectors overall count.
    rank_first_limit = None
    if chunk_ok is not None and num_hits > 0:
        totals = [n_match, local.n_live_rows]
        if sharded:
            totals = index.sum_over_shards(torch.tensor(totals, dtype=torch.int64, device=local.device)).tolist()
        if totals[0] > FILTER_FIRST_MAX_ROWS and totals[1] > RANK_FIRST_LIMIT:
            rank_first_limit = RANK_FIRST_LIMIT
    return index, Q, None, dict(k=k, num_hits=num_hits, metric=metric, chunk_ok=chunk_ok, rank_first_limit=rank_first_limit), prepare


def vector_search_batch(  # noqa: PLR0913
    queries: np.ndarray | torch.Tensor,
    *,
    num_results: int = 3,
    oversample: int = 4,
    metadata_filter: MetadataFilter | None = None,
    config: RAGLiteConfig | None = None,
    index: Any | None = None,
    exact_maxsim: bool = False,
    algo: str = "auto",
    queries_are_fp16: bool = False,
) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Batched ``vector_search``: ``queries`` is ``[B, d]`` (host or device).

    Returns host arrays ``(chunk_index[B, k] int64 (-1 padded), sim[B, k] float32, count[B])``.
    ``exact_maxsim=True`` ranks by exact per-chunk MaxSim instead of the reference's
    top-``num_hits``-vectors semantics.  Host work per call is O(B): the query upload, kernel launches,
    one pinned device->host copy of the results and one stream synchronisation.
    """
    index, Q, empty, kw, prepare = _plan_search(queries, num_results=num_results, oversample=oversample,
                                                metadata_filter=metadata_filter, config=config, index=index,
                                                exact_maxsim=exact_maxsim, queries_are_fp16=queries_are_fp16)
    if empty is not None:
        return empty
    local: CorpusIndex = getattr(index, "local", index)
    Q = Q.to(device=local.device, dtype=torch.float32, non_blocking=True).contiguous()
    if prepare is not None:
        Q = prepare(Q)
    return search_to_host(index, Q, algo=algo, **kw)


def vector_search_batch_async(  # noqa: PLR0913
    queries: np.ndarray | torch.Tensor,
    *,
    num_results: int = 3,
    oversample: int = 4,
    metadata_filter: MetadataFilter | None = None,
    config: RAGLiteConfig | None = None,
    index: Any | None = None,
    exact_maxsim: bool = False,
    algo: str = "auto",
    queries_are_fp16: bool = False,
) -> PendingSearch:
    """``vector_search_batch`` that returns at once with a :class:`PendingSearch`; ``.result()`` gives the same three
    host arrays.  Each call runs on a stream of its own (query upload, kernels, result download into a private
    pinned buffer), so a caller that keeps two or three batches in flight -- what a retrieval server does -- never
    leaves the GPU idle between batches: the host-side work of batch i + 1 and the copies of batch i hide under the
    corpus scan, and the small kernels at either end of a search fill the scan's tail.  (The reference reaches the same
    concurrency with its thread pool, _rag.py:317; here one thread suffices.)"""
    index, Q, empty, kw, prepare = _plan_search(queries, num_results=num_results, oversample=oversample,
                                                metadata_filter=metadata_filter, config=config, index=index,
                                                exact_maxsim=exact_maxsim, queries_are_fp16=queries_are_fp16)
    if empty is not None:
        return PendingSearch(index, Q, {}, None, None, int(Q.shape[0]), int(num_results), ready=empty)
    return search_async(index, Q, algo=algo, prepare=prepare, **kw)


def vector_search(
    query: str | FloatVector,
    *,
    num_results: int = 3,
    oversample: int = 4,
    metadata_filter: MetadataFilter | None = None,
    config: RAGLiteConfig | None = None,
) -> tuple[list[ChunkId], list[float]]:
    """Search chunks by multi-vector similarity -- drop-in for ``raglite.vector_search``
    (``_search.py:36-153``): embed / ravel the query, apply the query adapter, keep the
    ``num_hits`` nearest vectors, group by chunk with ``max(sim)``, return the best ``num_results``."""
    config = config or RAGLiteConfig()
    _check_metric(config)
    index = get_index(config)
    if index is None:
        raise ValueError(f"No index registered for db_url={config.db_url!r}; use raglite_b200.register_index")
    if config.self_query and isinstance(query, str):
        raise NotImplementedError("self_query needs an LLM and is outside the accelerated hot path")
    if isinstance(query, str):
        from ._embed import embed_strings

        q = embed_strings([query], config=config)[0, :]
    else:
        q = np.ravel(query)
    local: CorpusIndex = getattr(index, "local", index)
    ids, sims, counts = vector_search_batch(
        q[None, :], num_results=num_results, oversample=oversample, metadata_filter=metadata_filter,
        config=config, index=index, queries_are_fp16=(q.dtype == np.float16),
    )
    n = int(counts[0])
    owner = index if hasattr(index, "chunk_id_of") else local
    return [owner.chunk_id_of(int(c)) for c in ids[0, :n]], [float(s) for s in sims[0, :n]]


def retrieve_chunks(chunk_ids: Sequence[ChunkId], *, config: RAGLiteConfig | None = None) -> list[Chunk]:
    """``_search.py:283-299`` over the registered index's chunk table (order follows ``chunk_ids``)."""
    config = config or RAGLiteConfig()
    if not chunk_ids:
        return []
    index = get_index(config)
    local = getattr(index, "local", index) if index is not None else None
    if local is None or local.chunks is None:
        raise ValueError("The registered index holds no chunk texts")
    by_id = {c.id: c for c in local.live_chunks}
    return [by_id[cid] for cid in chunk_ids if cid in by_id]


def rerank_chunks(
    query: str, chunk_ids: list[ChunkId] | list[Chunk], *, config: RAGLiteConfig | None = None
) -> list[Chunk]:
    """Rerank chunks by cross-encoder relevance -- drop-in for ``raglite.rerank_chunks``
    (``_search.py:364-397``): same early exits, language routing and ``.rank(query=, docs=)`` contract."""
    config = config or RAGLiteConfig()
    chunks: list[Chunk] = (
        retrieve_chunks(chunk_ids, config=config)  # type: ignore[arg-type]
        if all(isinstance(c, ChunkId) for c in chunk_ids)
        else list(chunk_ids)  # type: ignore[arg-type]
    )
    if not config.reranker or not chunks:
        return chunks
    if isinstance(config.reranker, dict):
        langs: set[str] = set()
        try:  # the reference detects languages with langdetect (_search.py:381-383); optional here
            from langdetect import LangDetectException, detect  # type: ignore[import-not-found]

            with contextlib.suppress(LangDetectException):
                langs = {detect(str(chunk)) for chunk in chunks}
                langs.add(detect(query))
        except ModuleNotFoundError:
            langs = set()
        rerankers = config.reranker
        if len(langs) == 1 and (lang := next(iter(langs))) in rerankers:
            reranker = rerankers[lang]
        else:
            reranker = rerankers.get("other")
    else:
        reranker = config.reranker
    if reranker:
        results = reranker.rank(query=query, docs=[str(chunk) for chunk in chunks])
        chunks = [chunks[result.doc_id] for result in results.results]
    return chunks


# ---- keyword search: BM25 (the DuckDB branch of _search.py:156-230) and ts_rank (its PostgreSQL branch) -----------
def keyword_search_batch(
    queries: Sequence[str],
    *,
    num_results: int = 3,
    metadata_filter: MetadataFilter | None = None,
    config: RAGLiteConfig | None = None,
    index: Any | None = None,
) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Batched ``keyword_search``.  With a DuckDB (or any non-PostgreSQL) ``db_url``: BM25 as DuckDB's
    ``fts_main_chunk.match_bm25(id, query)`` computes it at its defaults, over the ``Chunk`` bodies of the index
    (``CorpusIndex.keyword_index``; ``_fts`` has the text analysis).  With a ``postgresql`` ``db_url``: PostgreSQL's
    ``ts_rank(to_tsvector('simple', body), to_tsquery('simple', q))`` over the tsvectors given to
    ``CorpusIndex.add_tsvector_rows`` / ``ShardedIndex.add_tsvector_rows`` (``_pgfts`` has the query analysis); scores
    are the float32 ``ts_rank`` widened to float64, ties by ascending chunk index (PostgreSQL leaves their order
    unspecified).  It raises ``NotImplementedError`` when no index is registered or no shard has received tsvectors, and
    for a query operand PostgreSQL would make a phrase; ``ValueError`` when a live chunk has no tsvector.

    Returns host arrays ``(chunk_index [B, k] int64 (-1 padded), score [B, k] float64 (-inf padded), count [B])``,
    ordered by descending score, ties by ascending chunk index.  The metadata filter only decides which chunks can be
    results: ``N``, ``avgdl`` and ``df`` always cover every live chunk, as the reference's ``WHERE`` around the macro
    does.  Host work per call: analysing the queries, one upload, the kernel launches, one pinned download and one
    stream synchronisation.

    On a ``ShardedIndex`` the call is a collective, as the sharded ``vector_search_batch`` is: every rank passes the same
    queries, ``num_results`` and filter.  ``N``, ``avgdl`` and each query term's ``df`` are then summed over the shards
    (one all-reduce), each shard ranks its own chunks with those corpus-wide statistics, and the per-shard top k are
    merged after one all-gather; the returned chunk indices are GLOBAL (``chunk_base`` of the owning shard + local
    index), identical on every rank and for every shard layout of the same corpus (DESIGN.md section 3.7).  The
    metadata filter is applied by each rank to its own chunks.  ``ts_rank`` needs no statistics; its collectives are one
    all-reduce of each shard's count of live chunks without a tsvector, then the all-gather and merge (section 3.9)."""
    from ._keyword import MAX_RESULTS

    config = config or RAGLiteConfig()
    if str(config.db_url).startswith("postgresql"):
        return _ts_rank_search_batch(queries, num_results=num_results, metadata_filter=metadata_filter, config=config,
                                     index=index)
    index = index if index is not None else get_index(config)
    if index is None:
        raise ValueError(f"No index registered for db_url={config.db_url!r}; use raglite_b200.register_index")
    sharded = hasattr(index, "group")
    local: CorpusIndex = getattr(index, "local", index)
    queries = list(queries)
    k = int(num_results)
    if k < 0 or k > MAX_RESULTS:
        raise ValueError(f"num_results={k} is outside [0, {MAX_RESULTS}]")
    B = len(queries)
    empty = (np.full((B, k), -1, np.int64), np.full((B, k), -np.inf, np.float64), np.zeros(B, np.int32))
    if B == 0 or k == 0 or (local.n_live_chunks == 0 and not sharded):   # a shard takes part in the collectives even empty
        return empty
    with local._lock:
        kw = local.keyword_index()
        chunk_ok, _ = _filter_on_device(local, _adapt_metadata(metadata_filter))
        return kw.topk_to_host(queries, k=k, chunk_mask=chunk_ok if chunk_ok is not None else kw.alive, index=index)


_TS_RANK_NEEDS_TSVECTORS = ("keyword_search on PostgreSQL ranks with ts_rank over the database's own to_tsvector('simple', "
                            "body); give the index those tsvectors with add_tsvector_rows(rows), rows = {select}")


def _ts_rank_search_batch(
    queries: Sequence[str], *, num_results: int, metadata_filter: MetadataFilter | None, config: RAGLiteConfig,
    index: Any | None,
) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """The PostgreSQL branch of ``keyword_search_batch`` (``_search.py:176-201``): ``ts_rank`` on the device over the
    tsvectors given to ``add_tsvector_rows`` (``_keyword.TsRankIndex``).  Whether the search can run depends on every
    shard (no tsvectors anywhere: ``NotImplementedError``; a live chunk without one: ``ValueError``), so on a
    ``ShardedIndex`` both are decided after one all-reduce of each shard's count, and every rank raises alike."""
    from . import _pgfts
    from ._keyword import MAX_RESULTS, TsRankIndex, tsrank_plan

    hint = _TS_RANK_NEEDS_TSVECTORS.format(select=_pgfts.TSVECTOR_SELECT)
    index = index if index is not None else get_index(config)
    if index is None:
        raise NotImplementedError(f"No index registered for db_url={config.db_url!r}. {hint}")
    sharded = hasattr(index, "group")
    local: CorpusIndex = getattr(index, "local", index)
    queries = list(queries)
    k = int(num_results)
    if k < 0 or k > MAX_RESULTS:
        raise ValueError(f"num_results={k} is outside [0, {MAX_RESULTS}]")
    B = len(queries)
    empty = (np.full((B, k), -1, np.int64), np.full((B, k), -np.inf, np.float64), np.zeros(B, np.int32))
    if B == 0 or k == 0:
        return empty
    with local._lock:
        ts = local._tsrank
        q_off, q_terms = tsrank_plan(queries, ts.lexeme_ids if ts is not None else {})
        chunk_ok, _ = _filter_on_device(local, _adapt_metadata(metadata_filter))
        state = [ts.missing(local._chunk_alive) if ts is not None else local.n_live_chunks, int(ts is None)]
        if sharded:
            state = index.sum_over_shards(torch.tensor(state, dtype=torch.int64, device=local.device)).tolist()
        missing, without = state
        if without == (index.world if sharded else 1):
            raise NotImplementedError(f"The index has no tsvectors. {hint}")
        if missing:
            raise ValueError(f"{missing} live chunks have no tsvector: ts_rank cannot score them; pass their rows of "
                             f"{_pgfts.TSVECTOR_SELECT} to add_tsvector_rows")
        if local.n_live_chunks == 0 and not sharded:
            return empty
        if ts is None:   # a shard that never received tsvectors and holds no live chunk: it matches nothing
            ts = TsRankIndex(local.device)
        mask = chunk_ok if chunk_ok is not None else ts.alive_mask(local._chunk_alive)
        return ts.topk_to_host(q_off, q_terms, k=k, n_chunks=local.n_chunks, chunk_mask=mask, index=index)


def keyword_search(
    query: str,
    *,
    num_results: int = 3,
    metadata_filter: MetadataFilter | None = None,
    config: RAGLiteConfig | None = None,
) -> tuple[list[ChunkId], list[float]]:
    """Search chunks with keyword search -- drop-in for ``raglite.keyword_search`` (``_search.py:156-230``): the chunks
    that contain at least one query term, best ``num_results`` first, ranked by BM25 (DuckDB ``db_url``) or by
    ``ts_rank`` (``postgresql`` ``db_url``; the score as pg8000 hands a ``float4`` over, its shortest round-trip digits:
    see ``keyword_search_batch``).  On a registered ``ShardedIndex`` a collective (see ``keyword_search_batch``) that
    returns the ids of chunks owned by every rank."""
    config = config or RAGLiteConfig()
    if config.self_query and isinstance(query, str):
        raise NotImplementedError("self_query needs an LLM and is outside the accelerated hot path")
    index = get_index(config)
    ids, scores, counts = keyword_search_batch([query], num_results=num_results, metadata_filter=metadata_filter,
                                               config=config, index=index)
    n = int(counts[0])
    base = 0 if hasattr(index, "group") else index.chunk_base   # a ShardedIndex returns global indices
    if str(config.db_url).startswith("postgresql"):   # pg8000 reads a float4 as its shortest round-trip text
        values = [float(str(np.float32(s))) for s in scores[0, :n]]
    else:
        values = [float(s) for s in scores[0, :n]]
    return [index.chunk_id_of(base + int(c)) for c in ids[0, :n]], values


# ---- the steps right after the hot path (SURVEY.md section 8f-3) ------------------------------------------
@dataclass
class ChunkSpan:
    """A run of consecutive chunks of one document (reference ``_database.py:326-398``)."""

    chunks: list[Chunk]

    @property
    def document_id(self) -> str:
        return self.chunks[0].document_id if self.chunks else ""

    @property
    def content(self) -> str:
        """Front matter and heading of the first chunk, then all bodies (``_database.py:389-394``)."""
        if not self.chunks:
            return ""
        bodies = "".join(chunk.body for chunk in self.chunks)
        return f"{self.chunks[0].front_matter}\n\n{self.chunks[0].headings.strip()}\n\n{bodies}".strip()

    def __str__(self) -> str:
        return self.content


# ---- fusion and span collation batched on device chunk indices -----------------------------------------------
_KEYWORD_SEARCH: dict[str, Any] = {}


def register_keyword_search(config_or_url: Any, fn: Any) -> None:
    """Replace the keyword search ``hybrid_search`` uses for a database (by default the device ``keyword_search``):
    any callable with ``keyword_search``'s signature ``(query, *, num_results, metadata_filter, config) ->
    (chunk_ids, scores)`` -- e.g. one that queries the database itself.  Both of the reference's branches run on the
    device without one: BM25 for DuckDB, ``ts_rank`` for PostgreSQL once the index holds the database's tsvectors
    (``CorpusIndex.add_tsvector_rows``)."""
    _KEYWORD_SEARCH[str(getattr(config_or_url, "db_url", config_or_url))] = fn


def rrf_fuse_device(rankings: torch.Tensor, weights: Sequence[float], *, k: float = 60.0, num_results: int | None = None
                    ) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """``rl_rrf_fuse``: Reciprocal Rank Fusion (``_search.py:233-254``) of ``rankings`` -- int64 ``[B, R, L]`` chunk
    indices on the device, ``-1`` padded -- for a whole batch in one launch.  Returns device tensors
    ``(ids [B, K], score float64 [B, K], count [B])``, best first, ties in first-appearance order."""
    from . import _lib

    if rankings.dtype != torch.int64 or rankings.ndim != 3 or not rankings.is_cuda:
        raise ValueError("rankings must be a CUDA int64 [B, R, L] tensor")
    B, R, L = (int(x) for x in rankings.shape)
    if len(weights) != R:
        raise ValueError("The number of weights must match the number of rankings.")
    K = int(num_results) if num_results is not None else R * L
    dev = rankings.device
    w = torch.tensor(list(weights), dtype=torch.float64, device=dev)
    out_ids = torch.empty((B, K), dtype=torch.int64, device=dev)
    out_score = torch.empty((B, K), dtype=torch.float64, device=dev)
    out_count = torch.empty((B,), dtype=torch.int32, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        _lib.check(lib.rl_rrf_fuse(rankings.contiguous().data_ptr(), w.data_ptr(), B, R, L, float(k), K, out_ids.data_ptr(),
                                   out_score.data_ptr(), out_count.data_ptr(), torch.cuda.current_stream().cuda_stream),
                   "rl_rrf_fuse")
    return out_ids, out_score, out_count


def reciprocal_rank_fusion(rankings: Sequence[Sequence[ChunkId]], *, k: int = 60, weights: Sequence[float] | None = None
                           ) -> tuple[list[ChunkId], list[float]]:
    """Drop-in ``reciprocal_rank_fusion`` (``_search.py:233-254``): the ids are interned to integers, fused by
    ``rl_rrf_fuse`` on the device (float64, the reference's summation order) and mapped back."""
    weights = [1.0] * len(rankings) if weights is None else list(weights)
    if len(weights) != len(rankings):
        raise ValueError("The number of weights must match the number of rankings.")
    L = max((len(r) for r in rankings), default=0)
    if L == 0:
        return [], []
    intern: dict[ChunkId, int] = {}
    names: list[ChunkId] = []
    table = np.full((1, len(rankings), L), -1, dtype=np.int64)
    for r, ranking in enumerate(rankings):
        for i, cid in enumerate(ranking):
            j = intern.get(cid)
            if j is None:
                j = intern[cid] = len(names)
                names.append(cid)
            table[0, r, i] = j
    ids, score, count = rrf_fuse_device(torch.from_numpy(table).cuda(), weights, k=float(k))
    n = int(count[0])
    return [names[int(j)] for j in ids[0, :n].tolist()], [float(x) for x in score[0, :n].tolist()]


def hybrid_search(  # noqa: PLR0913
    query: str, *, num_results: int = 3, oversample: int = 2, vector_search_weight: float = 0.75,
    keyword_search_weight: float = 0.25, metadata_filter: MetadataFilter | None = None, config: RAGLiteConfig | None = None,
) -> tuple[list[ChunkId], list[float]]:
    """Drop-in ``hybrid_search`` (``_search.py:257-280``): vector search on the device index, keyword search -- the
    callable registered with ``register_keyword_search`` if there is one, the device ``keyword_search`` otherwise (BM25
    or, for a ``postgresql`` ``db_url``, ``ts_rank``) -- and Reciprocal Rank Fusion of the two rankings on the device."""
    config = config or RAGLiteConfig()
    ks = _KEYWORD_SEARCH.get(str(config.db_url), keyword_search)
    vs_ids, _ = vector_search(query, num_results=oversample * num_results, metadata_filter=metadata_filter, config=config)
    ks_ids, _ = ks(query, num_results=oversample * num_results, metadata_filter=metadata_filter, config=config)
    ids, score = reciprocal_rank_fusion([vs_ids, list(ks_ids)], weights=[vector_search_weight, keyword_search_weight])
    return ids[:num_results], score[:num_results]


def collate_spans_device(index: Any, ranked: torch.Tensor, *, neighbors: tuple[int, ...] | None = (-1, 1)
                         ) -> dict[str, torch.Tensor]:
    """``rl_span_collate`` for a batch of ranked chunk-index lists (int64 ``[B, M]`` on the device, ``-1`` padded,
    LOCAL chunk indices of the index): the neighbour join, dedup, run cutting and span ranking of
    ``retrieve_chunk_spans`` (``_search.py:323-360``) in one launch.  Returns device tensors ``member [B, cap]``,
    ``span_start`` / ``span_len`` / ``span_score [B, cap]``, ``n_span [B]``, ``n_member [B]``."""
    from . import _lib

    local: CorpusIndex = getattr(index, "local", index)
    tabs = local.span_tables()
    B, M = (int(x) for x in ranked.shape)
    nb = torch.tensor(list(neighbors or ()), dtype=torch.int32, device=local.device)
    cap = M * (1 + int(nb.numel()))
    dev = local.device
    out = {"member": torch.empty((B, cap), dtype=torch.int64, device=dev),
           "span_start": torch.empty((B, cap), dtype=torch.int32, device=dev),
           "span_len": torch.empty((B, cap), dtype=torch.int32, device=dev),
           "span_score": torch.empty((B, cap), dtype=torch.float64, device=dev),
           "n_span": torch.empty((B,), dtype=torch.int32, device=dev), "n_member": torch.empty((B,), dtype=torch.int32, device=dev)}
    lib = _lib.load()
    with torch.cuda.device(dev):
        _lib.check(lib.rl_span_collate(
            ranked.contiguous().data_ptr(), B, M, tabs["chunk_doc"].data_ptr(), tabs["chunk_pos"].data_ptr(),
            tabs["chunk_alive"].data_ptr(), tabs["sorted_key"].data_ptr(), tabs["sorted_chunk"].data_ptr(),
            int(tabs["sorted_chunk"].numel()), nb.data_ptr() if nb.numel() else None, int(nb.numel()), out["member"].data_ptr(),
            out["span_start"].data_ptr(), out["span_len"].data_ptr(), out["span_score"].data_ptr(), out["n_span"].data_ptr(),
            out["n_member"].data_ptr(), torch.cuda.current_stream().cuda_stream), "rl_span_collate")
    return out


def retrieve_chunk_spans(
    chunk_ids: list[ChunkId] | list[Chunk], *, neighbors: tuple[int, ...] | None = (-1, 1),
    config: RAGLiteConfig | None = None,
) -> list[ChunkSpan]:
    """Group chunks (plus their ``neighbors`` in the same document) into contiguous spans, ordered by the summed
    reciprocal rank ``1 / (i + 1)`` of the chunks they contain (``_search.py:302-361``).  With a registered index
    that holds the ``Chunk`` records the whole collation runs in ``rl_span_collate`` on chunk indices; the
    host only maps ids to indices and indices back to records."""
    if not chunk_ids:
        return []
    config = config or RAGLiteConfig()
    index = get_index(config)
    local = getattr(index, "local", index) if index is not None else None
    if local is not None and local.chunks is not None and local.chunk_ids is not None:
        ids = [c if isinstance(c, ChunkId) else c.id for c in chunk_ids]
        pos = local._positions()
        idx = [pos[c] for c in ids if c in pos and local._chunk_alive[pos[c]]]
        if len(idx) == len(ids):
            ranked = torch.tensor([idx], dtype=torch.int64, device=local.device)
            out = collate_spans_device(local, ranked, neighbors=neighbors)
            n_span = int(out["n_span"][0])
            member = out["member"][0].tolist()
            start, length = out["span_start"][0, :n_span].tolist(), out["span_len"][0, :n_span].tolist()
            return [ChunkSpan([local.chunks[member[s + j]] for j in range(n)]) for s, n in zip(start, length, strict=True)]
    return _retrieve_chunk_spans_host(chunk_ids, neighbors=neighbors, config=config)


def _retrieve_chunk_spans_host(
    chunk_ids: list[ChunkId] | list[Chunk], *, neighbors: tuple[int, ...] | None = (-1, 1),
    config: RAGLiteConfig | None = None,
) -> list[ChunkSpan]:
    """Group chunks (plus their ``neighbors`` in the same document) into contiguous spans, ordered by
    the summed reciprocal rank ``1 / (i + 1)`` of the chunks they contain (``_search.py:302-361``)."""
    if not chunk_ids:
        return []
    config = config or RAGLiteConfig()
    chunks: list[Chunk] = (
        retrieve_chunks(chunk_ids, config=config)  # type: ignore[arg-type]
        if all(isinstance(c, ChunkId) for c in chunk_ids) else list(chunk_ids)  # type: ignore[arg-type]
    )
    score = {chunk.id: 1 / (i + 1) for i, chunk in enumerate(chunks)}
    pool: dict[tuple[str, int], Chunk] = {(c.document_id, c.index): c for c in chunks}
    if neighbors:
        index = get_index(config)
        local = getattr(index, "local", index) if index is not None else None
        table = {(c.document_id, c.index): c for c in local.live_chunks} if local is not None else {}
        for c in chunks:
            for off in neighbors:
                nb = table.get((c.document_id, c.index + off))
                if nb is not None:
                    pool.setdefault((nb.document_id, nb.index), nb)
    spans: list[ChunkSpan] = []
    run: list[Chunk] = []
    for key in sorted(pool):
        c = pool[key]
        if run and (c.document_id != run[-1].document_id or c.index != run[-1].index + 1):
            spans.append(ChunkSpan(run))
            run = []
        run.append(c)
    if run:
        spans.append(ChunkSpan(run))
    spans.sort(key=lambda s: sum(score.get(c.id, 0.0) for c in s.chunks), reverse=True)
    return spans


def search_and_rerank_chunks(  # noqa: PLR0913
    query: str, *, num_results: int = 8, oversample: int = 4, search: Any = None,
    config: RAGLiteConfig | None = None, metadata_filter: MetadataFilter | None = None,
) -> list[Chunk]:
    """Search ``oversample * num_results`` chunks, rerank, keep ``num_results`` (``_search.py:400-413``).
    The default ``search`` is ``vector_search``; the reference defaults to hybrid search, which
    ``search=raglite_b200.hybrid_search`` gives."""
    search = search or vector_search
    chunk_ids, _ = search(query, num_results=oversample * num_results, metadata_filter=metadata_filter, config=config)
    return rerank_chunks(query, chunk_ids, config=config)[:num_results]


def search_and_rerank_chunk_spans(  # noqa: PLR0913
    query: str, *, num_results: int = 8, oversample: int = 4, neighbors: tuple[int, ...] | None = (-1, 1),
    search: Any = None, config: RAGLiteConfig | None = None, metadata_filter: MetadataFilter | None = None,
) -> list[ChunkSpan]:
    """``search_and_rerank_chunks`` followed by span collation (``_search.py:416-433``); as there, the default ``search``
    is ``vector_search`` and ``search=raglite_b200.hybrid_search`` gives the reference's default."""
    chunks = search_and_rerank_chunks(query, num_results=num_results, oversample=oversample, search=search,
                                      config=config, metadata_filter=metadata_filter)
    return retrieve_chunk_spans(chunks, neighbors=neighbors, config=config)
