"""raglite_b200 -- H100-native (sm_90a) implementation of RAGLite's retrieval hot path.

Drop-in surface (reference ``raglite/__init__.py`` names for this path): ``RAGLiteConfig``,
``vector_search``, ``keyword_search``, ``hybrid_search``, ``rerank_chunks``, ``embed_strings``; plus the device-resident ``CorpusIndex`` /
``ShardedIndex`` that replace the database for this path and the batched ``vector_search_batch`` /
``keyword_search_batch``; and
``TokenEmbedderEngine``, the embedding model's encoder on the GPU behind ``embed_strings`` / ``embed_queries`` (from a
Hugging Face directory or the config's GGUF file, ``register_gguf_embedder``); and
``split_sentences`` with ``SaTEngine``, the sentence splitter's SaT model and partition on the GPU; and
``split_chunklets`` / ``split_chunks`` / ``split_documents``, the chunklet and chunk partitions on the GPU; and
``Document`` with ``insert_documents`` / ``delete_documents`` / ``delete_documents_by_metadata``, ingest into the
registered index on the GPU.
"""

from ._chunks import (
    embed_strings_batch,
    markdown_chunklet_boundaries,
    split_chunklets,
    split_chunklets_batch,
    split_chunks,
    split_chunks_batch,
    split_documents,
)
from ._config import RAGLiteConfig
from ._embed import embed_queries, embed_strings, register_gguf_embedder, register_token_embedder
from ._index import Chunk, CorpusIndex, get_index, merge_hits, register_index, unregister_index
from ._insert import Document, delete_documents, delete_documents_by_metadata, insert_documents
from ._query_adapter import update_query_adapter
from ._search import (
    ChunkSpan,
    collate_spans_device,
    hybrid_search,
    keyword_search,
    keyword_search_batch,
    reciprocal_rank_fusion,
    register_keyword_search,
    rerank_chunks,
    retrieve_chunk_spans,
    retrieve_chunks,
    rrf_fuse_device,
    search_and_rerank_chunk_spans,
    search_and_rerank_chunks,
    vector_search,
    vector_search_batch,
    vector_search_batch_async,
)
from ._sentences import (
    SaTEngine,
    markdown_sentence_boundaries,
    register_sentence_splitter,
    sentence_boundary_probas,
    split_sentences,
    split_sentences_batch,
)
from ._xenc import TokenEmbedderEngine

__all__ = [
    "Chunk",
    "ChunkSpan",
    "CorpusIndex",
    "Document",
    "RAGLiteConfig",
    "SaTEngine",
    "TokenEmbedderEngine",
    "collate_spans_device",
    "delete_documents",
    "delete_documents_by_metadata",
    "hybrid_search",
    "keyword_search",
    "keyword_search_batch",
    "markdown_sentence_boundaries",
    "register_keyword_search",
    "register_sentence_splitter",
    "rrf_fuse_device",
    "embed_queries",
    "embed_strings",
    "embed_strings_batch",
    "markdown_chunklet_boundaries",
    "split_chunklets",
    "split_chunklets_batch",
    "split_chunks",
    "split_chunks_batch",
    "split_documents",
    "get_index",
    "insert_documents",
    "merge_hits",
    "register_index",
    "reciprocal_rank_fusion",
    "register_gguf_embedder",
    "register_token_embedder",
    "rerank_chunks",
    "retrieve_chunk_spans",
    "retrieve_chunks",
    "search_and_rerank_chunk_spans",
    "search_and_rerank_chunks",
    "sentence_boundary_probas",
    "split_sentences",
    "split_sentences_batch",
    "unregister_index",
    "update_query_adapter",
    "vector_search",
    "vector_search_batch",
    "vector_search_batch_async",
]
