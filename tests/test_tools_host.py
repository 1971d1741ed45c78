"""RAGLite's function-calling protocol on the host: the template renderer against the reference template rendered
with jinja2 (``tests/golden/chatml_tools.json``), and ``chat_completion`` over a scripted engine that emits each raw
output token by token through the NumPy mask of its grammar, against the reference handler run on the same outputs
(every completion's prompt, grammar, temperature and token limit, and the calls).  Then ``rag()``'s tool path and
``async_rag`` with a stub search."""

from __future__ import annotations

import asyncio
import json
from pathlib import Path

import pytest

import grammar_oracle as go
import raglite_b200 as rl
from raglite_b200 import _rag
from raglite_b200._grammar import json_schema_to_gbnf
from raglite_b200._tools import chat_completion, render_chatml_tools, tojson

GOLDEN = json.loads((Path(__file__).parent / "golden" / "chatml_tools.json").read_text())
SAMPLING = dict(_rag.QWEN3_SAMPLING)


def test_tojson_is_jinjas():
    assert tojson({"b": "<a href='x'>&</a>", "a": [1, "é"]}) == (
        '{"a": [1, "\\u00e9"], "b": "\\u003ca href=\\u0027x\\u0027\\u003e\\u0026\\u003c/a\\u003e"}')


@pytest.mark.parametrize("case", GOLDEN["renders"], ids=lambda c: f"{c['messages']}-{c['tools']}")
def test_renderer_equals_the_reference_template(case):
    tools = GOLDEN["toolsets"][case["tools"]] if case["tools"] else []
    assert render_chatml_tools(GOLDEN["lists"][case["messages"]], tools, tool_calls=case["tool_calls"]) == case["text"]


def _grammar_text(g):
    if g is None:
        return None
    kind, text = g
    return text if kind == "gbnf" else json_schema_to_gbnf(text)


@pytest.mark.parametrize("run", GOLDEN["protocol"], ids=lambda r: f"{r['scenario']}-{r['messages']}")
def test_protocol_replays_the_reference_handler(run):
    eng = go.ScriptedEngine(run["raw"])
    tools = GOLDEN["toolsets"][run["tools"]]
    calls, stream = chat_completion(eng, GOLDEN["lists"][run["messages"]], tools=tools, tool_choice=run["tool_choice"],
                                    sampling=SAMPLING)
    text = None if stream is None else "".join(stream)
    assert len(eng.calls) == len(run["calls"]) and not eng.raw
    for got, want in zip(eng.calls, run["calls"], strict=True):
        assert got["prompt"] == want["prompt"]
        assert got["grammar"] == _grammar_text(want["grammar"])
        assert got["temperature"] == want["temperature"] and got["max_tokens"] == want["max_tokens"]
    if "text" in run["result"]:
        assert calls is None and text == run["result"]["text"]
    else:
        assert [[c["function"]["name"], c["function"]["arguments"]] for c in calls] == run["result"]["tool_calls"]
        assert all(c["type"] == "function" and c["id"].startswith(f"call__{i}_") for i, c in enumerate(calls))


def test_the_cap_is_seventeen_calls():
    run = next(r for r in GOLDEN["protocol"] if r["scenario"] == "cap")
    assert len(run["result"]["tool_calls"]) == 17 and len(run["calls"]) == 35


def test_max_tokens_bounds_the_message_only():
    eng = go.ScriptedEngine(["<message>", "The fox is brown.<|im_end|>"])
    _, stream = chat_completion(eng, [{"role": "user", "content": "q"}], tools=GOLDEN["toolsets"]["kb"],
                                tool_choice="auto", max_tokens=3, sampling=SAMPLING)
    assert "".join(stream) == "The"
    assert [c["max_tokens"] for c in eng.calls] == [None, 3]


class _Span:
    def __init__(self, i: int) -> None:
        self.i = i

    def to_json(self, index: int) -> str:
        return json.dumps({"index": index, "id": f"doc{self.i}"})


@pytest.fixture
def tool_config(monkeypatch):
    """A config whose llm is a scripted engine, with an index registered and retrieve_context stubbed."""
    cfg = rl.RAGLiteConfig(db_url="tools-host://index", llm="llama-cpp-python/test/scripted/x.gguf@4096", reranker=None)
    queries: list[str] = []

    def retrieve(query: str, *, config):  # noqa: ANN001, ANN202
        queries.append(query)
        return [_Span(len(queries) * 10 + k) for k in range(2)]

    monkeypatch.setattr(_rag, "retrieve_context", retrieve)
    monkeypatch.setattr(_rag, "get_index", lambda config: object() if config.db_url == cfg.db_url else None)
    return cfg, queries


def _register(cfg, raw):
    eng = go.ScriptedEngine(raw)
    rl.register_llm(cfg, eng)
    return eng


def test_rag_calls_the_tool_and_answers(tool_config):
    from raglite_b200 import _llm

    cfg, queries = tool_config
    raw = ["<function_calls>\nfunctions.search_knowledge_base:", '{"query": "fox colour"}<|im_end|>',
           "functions.search_knowledge_base:", '{"query": "dog"}<|im_end|>', "</function_calls>",
           "Brown.<|im_end|>"]
    eng = _register(cfg, raw)
    got_spans = []
    messages = [{"role": "user", "content": "What colour is the fox?"}]
    try:
        out = "".join(rl.rag(messages, on_retrieval=got_spans.append, config=cfg))
    finally:
        _llm._LLMS.pop(cfg.llm, None)
    assert out == "Brown." and queries == ["fox colour", "dog"]
    assert [m["role"] for m in messages] == ["user", "assistant", "tool", "tool", "assistant"]
    a = messages[1]
    assert a["content"] is None and [c["function"]["arguments"] for c in a["tool_calls"]] == [
        '{"query": "fox colour"}', '{"query": "dog"}']
    assert [m["tool_call_id"] for m in messages[2:4]] == [c["id"] for c in a["tool_calls"]]
    assert messages[2]["content"] == '{"documents": [{"index": 1, "id": "doc10"}, {"index": 2, "id": "doc11"}]}'
    assert [[s.i for s in x] for x in got_spans] == [[10, 11], [20, 21]]
    assert messages[-1] == {"role": "assistant", "content": "Brown."}
    # the answer's prompt: the final messages rendered without tools (a tool message is its header only)
    assert eng.calls[-1]["prompt"] == render_chatml_tools(messages[:-1])
    assert "<|im_start|>tool\n<|im_start|>tool\n<|im_start|>assistant\n" in eng.calls[-1]["prompt"]


def test_on_retrieval_gets_the_limited_spans(tool_config, monkeypatch):
    from raglite_b200 import _llm

    cfg, _ = tool_config
    monkeypatch.setattr(_rag, "_limit_chunkspans", lambda spans, config, messages: {k: v[:1] for k, v in spans.items()})
    _register(cfg, ["<function_calls>\nfunctions.search_knowledge_base:", '{"query": "q"}<|im_end|>', "<|im_end|>",
                    "A.<|im_end|>"])
    got = []
    messages = [{"role": "user", "content": "Q"}]
    try:
        list(rl.rag(messages, on_retrieval=got.append, config=cfg))
    finally:
        _llm._LLMS.pop(cfg.llm, None)
    assert [[s.i for s in x] for x in got] == [[10]]
    assert messages[2]["content"] == '{"documents": [{"index": 1, "id": "doc10"}]}'


def test_rag_message_branch_and_async_rag_yield_the_same(tool_config):
    from raglite_b200 import _llm

    cfg, queries = tool_config
    raw = ["<think>\nno need</think>\n\n<message>", "Hello there.<|im_end|>"]
    try:
        _register(cfg, raw)
        m1 = [{"role": "user", "content": "hi"}]
        sync = list(rl.rag(m1, config=cfg, seed=1))
        _register(cfg, raw)
        m2 = [{"role": "user", "content": "hi"}]

        async def collect():  # noqa: ANN202
            return [p async for p in rl.async_rag(m2, config=cfg, seed=1)]

        assert asyncio.run(collect()) == sync and "".join(sync) == "Hello there."
        assert m1 == m2 and [m["role"] for m in m1] == ["user", "assistant"] and not queries
    finally:
        _llm._LLMS.pop(cfg.llm, None)


def test_bad_arguments_raise_error_executing_tool(tool_config):
    from raglite_b200 import _llm

    cfg, _ = tool_config
    calls = [{"id": "c0", "type": "function", "function": {"name": "search_knowledge_base", "arguments": "{bad"}}]
    with pytest.raises(ValueError, match="Error executing tool"):
        _rag._run_tools(calls, None, cfg, messages=[])
    calls[0]["function"] = {"name": "other", "arguments": "{}"}
    with pytest.raises(ValueError, match="Error executing tool: Unknown function other"):
        _rag._run_tools(calls, None, cfg, messages=[])
    _llm._LLMS.pop(cfg.llm, None)


def test_without_an_index_rag_and_async_rag_raise(tool_config):
    from raglite_b200 import _llm

    cfg, _ = tool_config
    other = rl.RAGLiteConfig(db_url="tools-host://none", llm=cfg.llm, reranker=None)
    _register(other, [])
    try:
        with pytest.raises(NotImplementedError, match="retrieve_context") as e:
            list(rl.rag([{"role": "user", "content": "hi"}], config=other))
        assert "register_index" in str(e.value) and "insert_documents" in str(e.value)

        async def first():  # noqa: ANN202
            return [p async for p in rl.async_rag([{"role": "user", "content": "hi"}], config=other)]

        with pytest.raises(NotImplementedError, match="register_index"):
            asyncio.run(first())
    finally:
        _llm._LLMS.pop(cfg.llm, None)


def test_a_follow_up_turn_with_context_renders_the_tool_round(tool_config):
    from raglite_b200 import _llm

    cfg, queries = tool_config
    eng = _register(cfg, ["Brown.<|im_end|>"])
    call = {"id": "c0", "type": "function", "function": {"name": "search_knowledge_base", "arguments": '{"query": "q"}'}}
    messages = [{"role": "user", "content": "Q"}, {"role": "assistant", "content": None, "tool_calls": [call]},
                {"role": "tool", "content": '{"documents": []}', "tool_call_id": "c0"},
                {"role": "assistant", "content": "A."}, {"role": "user", "content": "<context>\nx\n</context>\nQ2"}]
    try:
        out = "".join(rl.rag(messages, config=cfg))
    finally:
        _llm._LLMS.pop(cfg.llm, None)
    assert out == "Brown." and not queries
    assert eng.calls[0]["prompt"] == render_chatml_tools(messages[:-1])
    assert "<function_calls>\nfunctions.search_knowledge_base:\n" in eng.calls[0]["prompt"]


def test_async_rag_closes_the_synchronous_path_when_left_early(tool_config):
    from raglite_b200 import _llm

    cfg, _ = tool_config
    _register(cfg, ["<message>", "one two three<|im_end|>"])
    messages = [{"role": "user", "content": "hi"}]
    closed = []
    real = _rag.rag

    def spy(*a, **k):  # noqa: ANN002, ANN003, ANN202
        it = real(*a, **k)
        try:
            yield from it
        finally:
            closed.append(True)

    async def first_piece():  # noqa: ANN202
        gen = rl.async_rag(messages, config=cfg)
        piece = await gen.__anext__()
        await gen.aclose()
        return piece

    try:
        import unittest.mock as um

        with um.patch.object(_rag, "rag", spy):
            assert asyncio.run(first_piece())
    finally:
        _llm._LLMS.pop(cfg.llm, None)
    assert closed == [True] and messages == [{"role": "user", "content": "hi"}]
