"""RAGLite's function-calling protocol on the GPU decoder: the chat handler that lets ``rag()`` decide to search the
knowledge base on its own (the reference's ``_chatml_function_calling.py`` over llama-cpp-python).

``render_chatml_tools`` reproduces the handler's ChatML template text exactly, including its quirks: a ``tool`` message
renders as its header only (the template has no branch for that role), a tool-call message closes with
``<function_calls>`` (no slash), and parameters are jinja's ``tojson`` (sorted keys, HTML characters escaped).
``chat_completion`` makes the handler's completions, each one re-tokenizing its whole prompt:

1. a temperature-0 decision under ``DECISION_GRAMMAR`` (message or function calls, an optional ``<think>`` block kept);
2. for a message, an unconstrained completion of the prompt rendered without tools;
3. for function calls, at most 17 rounds of: the arguments under the grammar of the tool's JSON schema, then a
   temperature-0 follow-up under ``FOLLOW_UP_GRAMMAR`` that names the next tool or ends the calls.
"""

from __future__ import annotations

import json
import uuid
from collections.abc import Iterator, Mapping, Sequence
from typing import Any

from ._grammar import json_schema_to_gbnf

DEFAULT_STOP = ("<|im_end|>", "<|endoftext|>")
MAX_TOOL_CALLS = 17   # the handler's loop runs while it holds at most 16 completions

DECISION_GRAMMAR = ('root ::= think? ("<function_calls>" "\\n" functions | "<message>")\n'
                    "functions ::= {names}\n"
                    'think ::= "<think>" [^<]* "</think>" "\\n\\n"\n')
FIXED_DECISION_GRAMMAR = ('root ::= think? "<function_calls>" "\\n" functions\n'
                          "functions ::= {names}\n"
                          'think ::= "<think>" [^<]* "</think>" "\\n\\n"\n')
FOLLOW_UP_GRAMMAR = 'root ::= functions | "</function_calls>" | "<|im_end|>" | "<|endoftext|>"\nfunctions ::= {names}\n'

_TOOLS_PREAMBLE = "\n\nYou have access to the following functions:\n"
_TOOLS_FORMAT = (
    "\nYou must decide whether to respond to the user directly, or to first make one or more function calls before "
    "responding.\nUse the following format to respond directly:\n\n<message>\n...\n</message>\n\nUse the following "
    'format to first make one or more function calls:\n\n<function_calls>\nfunctions.function_name_1:\n{ "arg1": '
    '"value1", "arg2": "value2", ... }\nfunctions.function_name_2:\n{ "arg1": "value1", "arg2": "value2", ... }\n'
    "</function_calls>")


def tojson(value: Any) -> str:
    """jinja2's ``tojson`` filter: ``json.dumps`` with sorted keys, then ``<``, ``>``, ``&`` and ``'`` escaped."""
    return (json.dumps(value, sort_keys=True).replace("<", "\\u003c").replace(">", "\\u003e").replace("&", "\\u0026")
            .replace("'", "\\u0027"))


def render_chatml_tools(messages: Sequence[Mapping[str, Any]], tools: Sequence[Mapping[str, Any]] = (), *,
                        tool_calls: bool = False) -> str:
    """The handler's template text for ``messages`` (with the generation prompt); ``tool_calls`` lists ``tools`` in
    the system message and wraps assistant content in ``<message>``."""
    out = []   # values printed with str(), as jinja prints them (None as "None")
    for m in messages:
        role = m["role"]
        out.append(f"<|im_start|>{role}\n")
        if role == "system":
            out.append(str(m["content"]))
            if tool_calls:
                out.append(_TOOLS_PREAMBLE)
                for t in tools:
                    f = t["function"]
                    out.append("\n")
                    if f.get("description"):
                        out.append(f"/* {str(f['description']).strip()} */")
                    out.append(f"\nfunctions.{f['name']}:\n{tojson(f['parameters'])}\n")
                out.append(_TOOLS_FORMAT)
            out.append("<|im_end|>\n")
        elif role == "user":
            out.append(f"{m['content']}<|im_end|>\n")
        elif role == "assistant":
            if "content" in m and m["content"]:
                body = str(m["content"])
                out.append(f"<message>\n{body}\n</message>" if tool_calls else body)
                out.append("<|im_end|>\n")
            if "tool_calls" in m:
                out.append("<function_calls>\n")
                for c in m["tool_calls"]:
                    out.append(f"functions.{c['function']['name']}:\n{c['function']['arguments']}")
                out.append("\n<function_calls><|im_end|>\n")
    return "".join(out) + "<|im_start|>assistant\n"


def _names(tools: Sequence[Mapping[str, Any]]) -> str:
    return " | ".join(f'"functions.{t["function"]["name"]}:"' for t in tools)


def chat_completion(engine: Any, messages: Sequence[Mapping[str, Any]], *, tools: Sequence[Mapping[str, Any]] | None = None,
                    tool_choice: str | Mapping[str, Any] | None = None, stop: Sequence[str] = (),
                    max_tokens: int | None = None, seed: int | None = None, sampling: Mapping[str, float]
                    ) -> tuple[list[dict[str, Any]] | None, Iterator[str] | None]:
    """One chat completion as the handler makes it: ``(tool_calls, None)`` when the model calls tools, else
    ``(None, stream of the message's text)``.  ``max_tokens`` bounds the message only; the decision, argument and
    follow-up completions run until the grammar ends them.  ``seed`` seeds every completion."""
    stops = [*stop, *DEFAULT_STOP]

    def complete(prompt: str, *, grammar: str | None = None, temperature: float | None = None,
                 extra_stop: Sequence[str] = (), limit: int | None = None) -> Iterator[str]:
        kw = {**sampling, **({} if temperature is None else {"temperature": temperature})}
        return engine.generate(engine.tokenizer.encode(prompt), stop=[*stops, *extra_stop], max_tokens=limit, seed=seed,
                               grammar=grammar, **kw)

    if not tools or tool_choice is None or tool_choice == "none":
        return None, complete(render_chatml_tools(messages), limit=max_tokens)
    if not any(m["role"] == "system" for m in messages):   # the tool block goes into a system message, appended last
        messages = [*messages, {"role": "system", "content": ""}]
    if isinstance(tool_choice, Mapping):
        tools = [t for t in tools if t["function"]["name"] == tool_choice["function"]["name"]]
        if not tools:
            raise ValueError(f"tool_choice names no given tool: {tool_choice!r}")
    elif tool_choice != "auto":
        raise ValueError(f"tool_choice={tool_choice!r} unsupported ('auto', 'none' or a function)")
    names = _names(tools)
    prompt = render_chatml_tools(messages, tools, tool_calls=True)
    decision = (DECISION_GRAMMAR if tool_choice == "auto" else FIXED_DECISION_GRAMMAR).format(names=names)
    think, text = "", "".join(complete(prompt, grammar=decision, temperature=0))
    if "</think>\n\n" in text:
        think, text = text.split("</think>\n\n", maxsplit=1)
        think += "</think>\n\n"
        prompt += think
    text = text.strip()
    if text.startswith("<message>"):
        return None, complete(render_chatml_tools(messages) + think, limit=max_tokens)
    name = text.split("\n")[-1][len("functions."):].rstrip(":")
    follow_up = FOLLOW_UP_GRAMMAR.format(names=names)
    by_name = {t["function"]["name"]: t for t in tools}
    prompt += "<function_calls>\n"
    calls: list[tuple[str, str]] = []
    while name in by_name and len(calls) < MAX_TOOL_CALLS:
        prompt += f"functions.{name}:\n"
        grammar = json_schema_to_gbnf(json.dumps(by_name[name]["function"]["parameters"]))
        args = "".join(complete(prompt, grammar=grammar))
        calls.append((name, args))
        prompt += args + "\n"
        nxt = "".join(complete(prompt, grammar=follow_up, temperature=0, extra_stop=(":", "</function_calls>")))
        name = nxt[len("functions."):]
    cid = f"cmpl-{uuid.uuid4()}"
    return [{"id": f"call__{i}_{n}_{cid}", "type": "function", "function": {"name": n, "arguments": a}}
            for i, (n, a) in enumerate(calls)], None
