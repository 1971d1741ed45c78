"""Retrieval-augmented generation on the GPU: RAGLite's programmable RAG path (``retrieve_context`` + ``add_context`` +
``rag``) with the config's Qwen3 GGUF generating (``_llm.LlmEngine``).

Restated in behaviour from the reference (``_rag.py``): the token estimate ``len // 3``, the left clip of the
messages and the proportional trim of the context to the context window, and the RAG instruction template.  ``rag``
renders ChatML as llama-cpp-python's chat handler does without tools and samples with the settings RAGLite ends up with
for a ``qwen3`` model.  When the last message carries no context, the model may search the knowledge base on its own:
RAGLite's ``search_knowledge_base`` tool through the function-calling protocol of ``_tools.chat_completion``.
"""

from __future__ import annotations

import asyncio
import contextlib
import json
import logging
import warnings
from collections.abc import AsyncIterator, Callable, Iterator, Mapping, Sequence
from typing import Any

import numpy as np

from ._config import RAGLiteConfig
from ._gguf import parse_embedder
from ._index import Chunk, get_index
from ._llm import find_llm, get_llm
from ._search import ChunkSpan, retrieve_chunk_spans, with_documents
from ._tools import chat_completion, render_chatml_tools

logger = logging.getLogger(__name__)

RAG_INSTRUCTION_TEMPLATE = """
---
The following context is intended to support answering the question below.
Use this information as the primary source when forming your response.
Provide a direct answer to the question without referencing how the information was supplied.
---

<context>
{context}
</context>

{user_prompt}
""".strip()

# RAGLite's qwen3 settings (its LiteLLM adapter over the chat handler's defaults): temperature 0.6, top_p 0.95, top_k 20,
# min_p 0; llama-cpp-python's repeat_penalty 1.1.
QWEN3_SAMPLING = {"temperature": 0.6, "top_p": 0.95, "top_k": 20, "min_p": 0.0, "repeat_penalty": 1.1}


def get_context_size(config: RAGLiteConfig, *, fallback: int = 2048) -> int:
    """The LLM's context window: the registered engine's ``n_ctx``; without one, the ``@n_ctx`` of a
    ``llama-cpp-python/...`` llm string, else ``fallback`` with a warning (as the reference falls back when it cannot
    tell), so that ``add_context`` works without a registered LLM."""
    engine = find_llm(config)
    if engine is not None:
        return engine.n_ctx
    if str(config.llm).startswith("llama-cpp-python/"):
        with contextlib.suppress(ValueError):
            n_ctx = parse_embedder(str(config.llm))[2]
            if n_ctx > 0:
                return n_ctx
    if fallback > 0:
        warnings.warn(f"Could not determine the context size of {config.llm}: no LLM is registered for it, using "
                      f"{fallback}.", stacklevel=2)
        return fallback
    raise ValueError(f"Could not determine the context size of {config.llm}.")


def retrieve_context(query: str, *, num_chunks: int = 10, metadata_filter: Any = None,
                     config: RAGLiteConfig | None = None) -> list[ChunkSpan]:
    """Search with ``config.search_method`` and return the hits as chunk spans."""
    config = config or RAGLiteConfig()
    results = config.search_method(query, num_results=num_chunks, metadata_filter=metadata_filter, config=config)
    if isinstance(results, tuple):
        return retrieve_chunk_spans(results[0], config=config)
    if all(isinstance(r, Chunk) for r in results):
        return retrieve_chunk_spans(results, config=config)
    if all(isinstance(r, ChunkSpan) for r in results):
        return with_documents(list(results), get_index(config))
    return []


def _count_tokens(item: str) -> int:
    return len(item) // 3


def _last_idx(messages: Sequence[Mapping[str, str]], role: str) -> int | None:
    return next((i for i in range(len(messages) - 1, -1, -1) if messages[i].get("role") == role), None)


def _token_counts(items: Sequence[Any]) -> list[int]:
    return [_count_tokens(x.to_xml()) if isinstance(x, ChunkSpan) else _count_tokens(json.dumps(x, ensure_ascii=False))
            if isinstance(x, dict) else _count_tokens(x) if isinstance(x, str) else 0 for x in items]


def _cutoff_idx(counts: list[int], max_tokens: int, *, reverse: bool = False) -> int:
    cum = np.cumsum(counts[::-1] if reverse else counts)
    i = int(np.searchsorted(cum, max_tokens, side="right"))
    return len(counts) - i if reverse else i


def _limit_chunkspans(tool_chunk_spans: dict[str, list[ChunkSpan]], config: RAGLiteConfig, *,
                      messages: list[dict[str, str]] | None = None, user_prompt: str | None = None,
                      template: str = RAG_INSTRUCTION_TEMPLATE) -> dict[str, list[ChunkSpan]]:
    """Trim each list of spans (most relevant first) so that all fit in the context window beside the messages'
    last system / user / assistant message or the instruction, each list cut in proportion to its tokens."""
    if messages:
        buffer = sum(_count_tokens(json.dumps(messages[i])) for r in ("user", "system", "assistant")
                     if (i := _last_idx(messages, r)) is not None)
    elif user_prompt:
        buffer = _count_tokens(template.format(context="", user_prompt=user_prompt))
    else:
        buffer = 0
    max_tokens = get_context_size(config) - buffer
    counts = {k: _token_counts(v) for k, v in tool_chunk_spans.items()}
    total = sum(sum(c) for c in counts.values())
    if total <= max_tokens:
        return tool_chunk_spans
    ratio = max_tokens / total
    out = {k: v[:_cutoff_idx(counts[k], int(ratio * sum(counts[k])))] if v else [] for k, v in tool_chunk_spans.items()}
    kept, before = sum(map(len, out.values())), sum(map(len, tool_chunk_spans.values()))
    if kept < before:
        logger.warning("RAG context was limited to %d out of %d chunks due to context window size.", kept, before)
    return out


def add_context(user_prompt: str, context: list[ChunkSpan], config: RAGLiteConfig, *,
                rag_instruction_template: str = RAG_INSTRUCTION_TEMPLATE) -> dict[str, str]:
    """A user message carrying ``context`` (trimmed to the context window) and the prompt.  Each span's source is its
    document's url or filename, from the records of the index registered for ``config.db_url`` when it holds them."""
    if config is not None:
        context = with_documents(list(context), get_index(config))
    limited = _limit_chunkspans({"temp": context}, config, user_prompt=user_prompt)["temp"]
    body = "\n".join(s.to_xml(index=i + 1) for i, s in enumerate(limited))
    return {"role": "user", "content": rag_instruction_template.format(context=body, user_prompt=user_prompt.strip())}


def _clip(messages: list[dict[str, str]], max_tokens: int) -> list[dict[str, str]]:
    """Drop messages from the left until the rest fit in ``max_tokens``; when even the last user message would go,
    keep the last system and user messages if they fit together, else the user message alone if it fits, else none."""
    counts = _token_counts(messages)
    cut = _cutoff_idx(counts, max_tokens, reverse=True)
    iu = _last_idx(messages, "user")
    if cut == len(messages) or (iu is not None and iu < cut):
        logger.warning("Context window of %d tokens exceeded.", max_tokens)
        isys = _last_idx(messages, "system")
        if iu is not None and isys is not None and isys < iu and counts[iu] + counts[isys] <= max_tokens:
            return [messages[isys], messages[iu]]
        if iu is not None and counts[iu] <= max_tokens:
            return [messages[iu]]
        return []
    return messages[cut:]


def render_chatml(messages: Sequence[Mapping[str, Any]]) -> str:
    """ChatML of the system, user and assistant messages with content, then the assistant's turn.  This equals the
    chat handler's rendering (``render_chatml_tools``, which ``rag()`` uses) for messages of those roles only; the
    handler also renders every message's header, an assistant's tool calls and a ``tool`` message's header."""
    parts = [f"<|im_start|>{m['role']}\n{m['content']}<|im_end|>\n" for m in messages
             if m.get("role") in ("system", "user") or (m.get("role") == "assistant" and m.get("content"))]
    return "".join(parts) + "<|im_start|>assistant\n"


def _has_context(message: Mapping[str, Any]) -> bool:
    content = str(message.get("content") or "")
    return any(tag in content for tag in ("<context>", "<document", "from_chunk_id"))


# RAGLite's tool for searching the knowledge base (``_rag.py``'s ``_get_tools``).
SEARCH_KNOWLEDGE_BASE_TOOL = {
    "type": "function",
    "function": {
        "name": "search_knowledge_base",
        "description": (
            "Search the knowledge base.\n"
            "IMPORTANT: You MAY NOT use this function if the question can be answered with common knowledge or "
            "straightforward reasoning.\n"
            "For multi-faceted questions, call this function once for each facet."),
        "parameters": {
            "type": "object",
            "properties": {
                "query": {
                    "type": "string",
                    "description": (
                        "The `query` string MUST be a precise single-faceted question in the user's language.\n"
                        "The `query` string MUST resolve all pronouns to explicit nouns."),
                },
            },
            "required": ["query"],
            "additionalProperties": False,
        },
    },
}


def _run_tools(tool_calls: list[dict[str, Any]], on_retrieval: Callable[[list[ChunkSpan]], None] | None,
               config: RAGLiteConfig, *, messages: list[dict[str, Any]]) -> list[dict[str, Any]]:
    """Run each ``search_knowledge_base`` call in order, limit all their spans together to the context window, and
    return one ``tool`` message per call (``on_retrieval`` gets each non-empty list)."""
    spans: dict[str, list[ChunkSpan]] = {}
    for call in tool_calls:
        try:
            if call["function"]["name"] != "search_knowledge_base":
                raise ValueError(f"Unknown function {call['function']['name']}.")
            kwargs = json.loads(call["function"]["arguments"])
            spans[call["id"]] = retrieve_context(**kwargs, config=config)
        except Exception as e:
            raise ValueError(f"Error executing tool: {e}") from e
    spans = _limit_chunkspans(spans, config, messages=messages)
    out = []
    for call in tool_calls:
        found = spans.get(call["id"], [])
        out.append({"role": "tool", "content": '{"documents": [' + ", ".join(s.to_json(index=i + 1) for i, s in
                                                                            enumerate(found)) + "]}",
                    "tool_call_id": call["id"]})
        if found and callable(on_retrieval):
            on_retrieval(found)
    return out


def _stream_answer(stream: Iterator[str], messages: list[dict[str, Any]]) -> Iterator[str]:
    pieces = []
    for piece in stream:
        pieces.append(piece)
        yield piece
    messages.append({"role": "assistant", "content": "".join(pieces)})


def _rag_with_tools(messages: list[dict[str, Any]], *, tools: list[dict[str, Any]], tool_choice: Any,
                    on_retrieval: Callable[[list[ChunkSpan]], None] | None, config: RAGLiteConfig,
                    max_tokens: int | None, seed: int | None) -> Iterator[str]:
    """``rag()``'s function-calling path with the given tools (each one run as ``search_knowledge_base``)."""
    engine = get_llm(config)
    calls, stream = chat_completion(engine, _clip(messages, engine.n_ctx), tools=tools, tool_choice=tool_choice,
                                    max_tokens=max_tokens, seed=seed, sampling=QWEN3_SAMPLING)
    if calls:
        messages.append({"role": "assistant", "content": None, "tool_calls": calls})
        messages.extend(_run_tools(calls, on_retrieval, config, messages=messages))
        _, stream = chat_completion(engine, _clip(messages, engine.n_ctx), max_tokens=max_tokens, seed=seed,
                                    sampling=QWEN3_SAMPLING)
    yield from _stream_answer(stream if stream is not None else iter(()), messages)


def rag(messages: list[dict[str, str]], *, on_retrieval: Callable[[list[ChunkSpan]], None] | None = None,
        config: RAGLiteConfig, max_tokens: int | None = None, seed: int | None = None) -> Iterator[str]:
    """Stream the registered LLM's answer to ``messages``, then append it to ``messages`` as the assistant's message.

    When the last message carries its context (from ``retrieve_context`` + ``add_context``), the LLM answers it.
    Otherwise the LLM may first call ``search_knowledge_base`` on the index registered for ``config.db_url``: the
    tool-call message and one ``tool`` message per call are appended before the answer, and ``on_retrieval`` gets each
    call's spans.  ``max_tokens`` bounds the answer."""
    engine = get_llm(config)
    clipped = _clip(messages, engine.n_ctx)
    if clipped and _has_context(clipped[-1]):
        prompt = engine.tokenizer.encode(render_chatml_tools(clipped))   # the handler's text, tool rounds included
        yield from _stream_answer(engine.generate(prompt, max_tokens=max_tokens, seed=seed, **QWEN3_SAMPLING), messages)
        return
    if not clipped or _has_context(messages[-1]) or get_index(config) is None:
        raise NotImplementedError(
            "rag() without context in the last message lets the LLM search the knowledge base, which needs an index "
            f"registered for db_url={config.db_url!r} (register_index, or insert_documents); else retrieve the context "
            "with retrieve_context and add it with add_context first")
    yield from _rag_with_tools(messages, tools=[SEARCH_KNOWLEDGE_BASE_TOOL], tool_choice="auto",
                               on_retrieval=on_retrieval, config=config, max_tokens=max_tokens, seed=seed)


async def async_rag(messages: list[dict[str, str]], *, on_retrieval: Callable[[list[ChunkSpan]], None] | None = None,
                    config: RAGLiteConfig, max_tokens: int | None = None, seed: int | None = None) -> AsyncIterator[str]:
    """``rag`` as an async generator: each step of the synchronous path runs in a worker thread, off the event loop,
    and the same messages are appended."""
    it = rag(messages, on_retrieval=on_retrieval, config=config, max_tokens=max_tokens, seed=seed)
    done = object()
    try:
        while (piece := await asyncio.to_thread(next, it, done)) is not done:
            yield piece
    finally:   # a consumer that stops early closes the synchronous path here, not in the garbage collector
        await asyncio.to_thread(it.close)
