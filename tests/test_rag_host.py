"""The RAG prompt's ``<source>`` on chunks as ``insert_documents`` builds them (every metadata value a list), with and
without the index's ``Document`` records, and ``get_context_size`` without a registered LLM."""

from __future__ import annotations

import json

import pytest

import raglite_b200 as rl
from raglite_b200 import _insert as I  # noqa: N812


def _span(doc: rl.Document) -> rl.ChunkSpan:
    return rl.ChunkSpan(chunks=I.chunk_records(doc, ["The fox is brown. ", "It runs."]))


@pytest.mark.parametrize("url,filename,want", [(None, "fox.md", "fox.md"), ("https://x/fox", "fox.md", "https://x/fox")])
def test_source_of_inserted_chunks_is_the_documents_url_else_filename(url, filename, want):
    doc = rl.Document.from_text("# Fox\n\nThe fox is brown. It runs.", url=url, filename=filename)
    span = _span(doc)
    assert isinstance(span.chunks[0].metadata_["url"], list)   # the shape insert_documents stores
    assert f"<source>{want}</source>" in span.to_xml(index=1)
    assert json.loads(span.to_json(index=1))["source"] == want
    # with the Document record (as retrieve_chunk_spans and add_context attach it from the index)
    from raglite_b200._search import with_documents

    class _Index:
        documents = {doc.id: doc}

    (with_doc,) = with_documents([span], _Index())
    assert with_doc.document is doc and f"<source>{want}</source>" in with_doc.to_xml()


def test_source_of_a_chunk_without_url_or_filename_is_empty():
    span = rl.ChunkSpan(chunks=[rl.Chunk(id="c", document_id="d", metadata_={"url": [None], "filename": [None]})])
    assert "<source></source>" in span.to_xml()


def test_context_size_without_a_registered_llm():
    from raglite_b200._rag import get_context_size

    assert get_context_size(rl.RAGLiteConfig(llm="llama-cpp-python/org/repo/m.gguf@4096", reranker=None)) == 4096
    with pytest.warns(UserWarning, match="using 2048"):
        assert get_context_size(rl.RAGLiteConfig(llm="llama-cpp-python/org/repo/m.gguf", reranker=None)) == 2048
    with pytest.raises(ValueError, match="context size"):
        get_context_size(rl.RAGLiteConfig(llm="gpt-4o", reranker=None), fallback=0)
    msg = rl.add_context("Why?", [_span(rl.Document.from_text("The fox.", filename="fox.md"))],
                         rl.RAGLiteConfig(llm="llama-cpp-python/org/repo/m.gguf@4096", db_url="none://x", reranker=None))
    assert "<source>fox.md</source>" in msg["content"]
