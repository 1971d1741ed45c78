"""``RAGLiteConfig`` -- field-for-field mirror of the reference's frozen dataclass
(``raglite/_config.py:42-83``): same names, defaults and ``compare=False`` choices, so a config
written for RAGLite works unchanged.  The reference's import-time dependencies (rerankers,
SQLAlchemy) are not needed here."""

from __future__ import annotations

import os
from dataclasses import dataclass, field
from pathlib import Path
from typing import Any, Literal

from ._typing import ChunkId, MetadataFilter, SearchMethod

try:  # reference: platformdirs.user_data_dir("raglite", ensure_exists=True) (_config.py:23)
    from platformdirs import user_data_dir

    cache_path = Path(user_data_dir("raglite", ensure_exists=True))
except Exception:  # noqa: BLE001
    cache_path = Path.home() / ".local" / "share" / "raglite"


def llama_supports_gpu_offload() -> bool:
    """``raglite._lazy_llama.llama_supports_gpu_offload`` -- False when llama-cpp-python is absent."""
    try:
        from llama_cpp import llama_supports_gpu_offload as f  # type: ignore[import-not-found]

        return bool(f())
    except Exception:  # noqa: BLE001
        return False


def _vector_search(
    query: str, *, num_results: int = 8, metadata_filter: MetadataFilter | None = None,
    config: "RAGLiteConfig | None" = None,
) -> tuple[list[ChunkId], list[float]]:
    """Default search method (``_config.py:28-39``), resolved lazily to avoid a circular import."""
    from ._search import vector_search

    return vector_search(query, num_results=num_results, metadata_filter=metadata_filter, config=config)


def _default_reranker() -> Any:
    """``_config.py:73-79``: ``{"en": ms-marco-MiniLM-L-12-v2, "other": ms-marco-MultiBERT-L-12}``,
    here as GPU cross-encoder rankers that load their weights lazily from ``cache_path``."""
    from ._rerank import B200CrossEncoderRanker

    return {
        "en": B200CrossEncoderRanker("ms-marco-MiniLM-L-12-v2", cache_dir=cache_path),
        "other": B200CrossEncoderRanker("ms-marco-MultiBERT-L-12", cache_dir=cache_path),
    }


@dataclass(frozen=True)
class RAGLiteConfig:
    """RAGLite config (``_config.py:42-83``)."""

    # Database config.  Here the URL keys the registry of device-resident indexes (_index.py).
    db_url: str = f"duckdb:///{(cache_path / 'raglite.db').as_posix()}"
    # LLM config used for generation (unused by the hot path; kept for signature parity).
    llm: str = field(
        default_factory=lambda: (
            "llama-cpp-python/unsloth/Qwen3-8B-GGUF/*Q4_K_M.gguf@8192"
            if llama_supports_gpu_offload()
            else "llama-cpp-python/unsloth/Qwen3-4B-GGUF/*Q4_K_M.gguf@8192"
        )
    )
    llm_max_tries: int = 4
    # Embedder config used for indexing.
    embedder: str = field(
        default_factory=lambda: (
            "llama-cpp-python/lm-kit/bge-m3-gguf/*F16.gguf@512"
            if llama_supports_gpu_offload() or (os.cpu_count() or 1) >= 4  # noqa: PLR2004
            else "llama-cpp-python/lm-kit/bge-m3-gguf/*Q4_K_M.gguf@512"
        )
    )
    embedder_normalize: bool = True
    # Chunk config used to partition documents into chunks.
    chunk_max_size: int = 2048
    # Vector search config.
    # "l1" is not in the reference's annotation, but its PostgreSQL layer renders it (pgvector `<+>`,
    # _typing.py:110-120; halfvec_l1_ops, _database.py:573-578), so PostgreSQL configs may carry it.
    vector_search_distance_metric: Literal["cosine", "dot", "l2", "l1"] = "cosine"
    vector_search_multivector: bool = True
    vector_search_query_adapter: bool = True
    # Reranking config: anything with ``.rank(query=, docs=)`` -> ``.results[i].doc_id``.
    reranker: Any = field(default_factory=_default_reranker, compare=False)
    # Search config.
    search_method: SearchMethod = field(default=_vector_search, compare=False)
    self_query: bool = False
