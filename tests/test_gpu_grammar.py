"""Grammar-constrained generation on the GPU: ``rl_grammar_token_index`` bit for bit against the NumPy walk,
``rl_llm_sample_masked`` against ``llm_oracle.sample`` on pre-masked logits, constrained generation with the Qwen3
fixture model against the host DFA, and ``rag()``'s function-calling path end to end."""

from __future__ import annotations

import copy
import ctypes as C

import numpy as np
import pytest
import torch

import grammar_oracle as go
import llm_oracle
import raglite_b200 as rl
from qwen3_fixtures import make_model, write_qwen3_gguf
from raglite_b200 import _lib, _rag
from raglite_b200._grammar import MAX_STATES, compile_gbnf, json_schema_to_gbnf
from raglite_b200._tools import DECISION_GRAMMAR, DEFAULT_STOP, FIXED_DECISION_GRAMMAR, FOLLOW_UP_GRAMMAR, render_chatml_tools
from test_gpu_rag import DOCS, config  # noqa: F401  (the fixture)

pytestmark = pytest.mark.gpu

NAMES = '"functions.search_knowledge_base:"'
PROTOCOL = [DECISION_GRAMMAR.format(names=NAMES), FIXED_DECISION_GRAMMAR.format(names=NAMES),
            FOLLOW_UP_GRAMMAR.format(names=NAMES),
            json_schema_to_gbnf(_rag.SEARCH_KNOWLEDGE_BASE_TOOL["function"]["parameters"])]
BOUNDED = {"type": "object", "properties": {"query": {"type": "string", "minLength": 3, "maxLength": 12}},
           "required": ["query"], "additionalProperties": False}


def synthetic_vocab(V: int = 151936, seed: int = 0) -> list[bytes]:
    """Seeded byte pieces: empty ones, ones over 64 bytes, partial UTF-8 characters, protocol fragments."""
    rng = np.random.default_rng(seed)
    frag = [b"<", b"function", b"_calls", b">", b"\n", b"functions", b".", b"search", b"_knowledge_base", b":",
            b'{"', b"query", b'":', b' "', b'"}', b" ", b"\xc3", b"\xa9", b"\xe4\xb8", b"\xad", b"<think>", b"</think>",
            b"message", b"<|im_end|>", b"\\u00", b"</function_calls>"]
    out = []
    for v in range(V):
        r = rng.random()
        if r < 0.01:
            out.append(b"")
        elif r < 0.02:
            out.append(bytes(rng.integers(0, 256, size=int(rng.integers(65, 130)), dtype=np.uint8)))
        elif r < 0.35:
            out.append(b"".join(frag[int(i)] for i in rng.integers(0, len(frag), size=int(rng.integers(1, 4)))))
        elif r < 0.6:
            out.append(bytes(rng.integers(32, 127, size=int(rng.integers(1, 9)), dtype=np.uint8)))
        else:
            out.append(bytes(rng.integers(0, 256, size=int(rng.integers(1, 7)), dtype=np.uint8)))
    out[:256] = [bytes([b]) for b in range(256)]
    return out


def device_index(trans: np.ndarray, pieces: list[bytes]) -> np.ndarray:
    lib = _lib.load()
    offs = np.zeros(len(pieces) + 1, dtype=np.int64)
    offs[1:] = np.cumsum([len(p) for p in pieces])
    flat = torch.from_numpy(np.frombuffer(b"".join(pieces) + b"\0", dtype=np.uint8).copy()).cuda()
    t = torch.from_numpy(np.ascontiguousarray(trans, dtype=np.int16)).cuda()
    o = torch.from_numpy(offs).cuda()
    idx = torch.empty((len(trans), len(pieces)), dtype=torch.int16, device="cuda")
    _lib.check(lib.rl_grammar_token_index(t.data_ptr(), len(trans), flat.data_ptr(), o.data_ptr(), len(pieces),
                                          idx.data_ptr(), torch.cuda.current_stream().cuda_stream), "index")
    return idx.cpu().numpy()


@pytest.fixture(scope="module")
def big_vocab():
    return synthetic_vocab()


@pytest.fixture(scope="module")
def fixture_vocab(engine):
    """The Qwen3 fixture's 640 pieces (control tokens as their text), padded with empty ones."""
    pieces = list(engine.tokenizer.token_bytes)
    return pieces + [b""] * (engine.plan.vocab - len(pieces))


_HOST_INDEX: dict = {}


def _host_index(text: str, V: int, pieces: list[bytes]):  # noqa: ANN202
    if (text, V) not in _HOST_INDEX:
        dfa = compile_gbnf(text)
        _HOST_INDEX[text, V] = dfa, go.token_index(dfa.trans, pieces)
    return _HOST_INDEX[text, V]


@pytest.mark.parametrize("g", range(len(PROTOCOL)))
def test_token_index_equals_the_numpy_walk(g, big_vocab, fixture_vocab):
    for pieces in (fixture_vocab, big_vocab):
        dfa, want = _host_index(PROTOCOL[g], len(pieces), pieces)
        assert np.array_equal(device_index(dfa.trans, pieces), want)


def test_token_index_near_the_state_cap(fixture_vocab):
    dfa = compile_gbnf('root ::= [a-z\\u00e0-\\u00ff]{0,%d} "."' % (MAX_STATES // 2 - 8))
    assert MAX_STATES - 20 <= dfa.n_states <= MAX_STATES
    pieces = fixture_vocab + synthetic_vocab(4000, seed=3)
    assert np.array_equal(device_index(dfa.trans, pieces), go.token_index(dfa.trans, pieces))


def _sample_masked(logits, hist, index, accept, eog, state, **kw):
    lib = _lib.load()
    V = logits.shape[0]
    d = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in
         (("l", logits.astype(np.float32)), ("h", np.asarray(hist or [0], dtype=np.int32)), ("i", index),
          ("a", accept.astype(np.uint8)), ("s", np.array([state], dtype=np.int32)))}
    out = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    ws = torch.empty(int(lib.rl_llm_sample_workspace_bytes(V)), dtype=torch.uint8, device="cuda")
    e = (C.c_int32 * max(1, len(eog)))(*eog)
    _lib.check(lib.rl_llm_sample_masked(d["l"].data_ptr(), V, d["h"].data_ptr(), len(hist), kw["temperature"], kw["top_k"],
                                        kw["top_p"], kw["min_p"], kw["penalty"], kw["u"], d["i"].data_ptr(), len(accept),
                                        d["a"].data_ptr(), e, len(eog), d["s"].data_ptr(), out.data_ptr(), ws.data_ptr(),
                                        ws.numel(), torch.cuda.current_stream().cuda_stream), "masked")
    return int(out.item()), int(d["s"].item())


# greedy, the qwen3 settings, and no top-p (where only the cut to the allowed count keeps masked ids out of the draw)
SETTINGS = [dict(temperature=0.0, top_k=20, top_p=0.95, min_p=0.0, penalty=1.1),
            dict(temperature=0.6, top_k=20, top_p=0.95, min_p=0.0, penalty=1.1),
            dict(temperature=1.0, top_k=40, top_p=1.0, min_p=0.0, penalty=1.0)]


@pytest.mark.parametrize("V", [640, 151936])
@pytest.mark.parametrize("si", range(len(SETTINGS)))
def test_masked_sampler_equals_the_masked_chain(V, si, big_vocab, fixture_vocab):
    pieces = fixture_vocab if V == 640 else big_vocab
    rng = np.random.default_rng(V + si)
    eog = [V - 1, V - 3]
    for text in PROTOCOL:
        dfa, idx = _host_index(text, V, pieces)
        for st in range(0, dfa.n_states, max(1, dfa.n_states // 12)):
            logits = (rng.standard_normal(V) * 3).astype(np.float32)
            hist = rng.integers(0, V, size=40).tolist()
            for u in (float(np.float32(rng.random())), float(np.nextafter(np.float32(1), np.float32(0)))):
                kw = dict(SETTINGS[si], u=u)
                want = go.sample_masked(logits, hist, idx, dfa.accept, eog, st, **kw)
                got = _sample_masked(logits, hist, idx, dfa.accept, eog, st, **kw)
                ok = go.allowed(idx, dfa.accept, eog, st)
                masked = np.where(ok, logits, np.float32(-np.inf))
                close = SETTINGS[si]["temperature"] > 0 and llm_oracle.sample_margin(
                    masked, hist, u, **{**SETTINGS[si], "top_k": min(SETTINGS[si]["top_k"], int(ok.sum()))}) < 1e-5
                assert got == want or close, (st, u)   # a draw within float32 ulps of a CDF step may differ in exp
                if got[0] >= 0:
                    assert ok[got[0]]
                    assert got[1] == (st if got[0] in eog else dfa.walk(pieces[got[0]], st))


def test_few_allowed_ids_and_eog_only_in_accepting_states():
    V = 640
    rng = np.random.default_rng(5)
    trans = np.full((2, 256), -1, dtype=np.int16)
    trans[0, ord("a")] = 1
    trans[0, ord("b")] = 1
    accept = np.array([False, True])
    pieces = [bytes([b]) for b in range(256)] + [b"zz"] * (V - 256)
    idx = go.token_index(trans, pieces)
    eog = [V - 1]
    logits = rng.standard_normal(V).astype(np.float32)
    logits[V - 1] = 50.0   # the end-of-generation id dominates wherever it is allowed
    for u in (0.0, 0.5, float(np.nextafter(np.float32(1), np.float32(0)))):
        kw = dict(SETTINGS[1], u=u)
        tok, st = _sample_masked(logits, [], idx, accept, eog, 0, **kw)
        assert tok in (ord("a"), ord("b")) and st == 1 and (tok, st) == go.sample_masked(logits, [], idx, accept, eog, 0, **kw)
        tok, st = _sample_masked(logits, [], idx, accept, eog, 1, **kw)
        assert (tok, st) == (V - 1, 1)
    assert _sample_masked(logits, [], idx, np.array([False, False]), eog, 1, **SETTINGS[1], u=0.3) == (-1, 1)


@pytest.fixture(scope="module")
def engine(tmp_path_factory):
    from raglite_b200._llm import LlmEngine

    path = tmp_path_factory.mktemp("grammar") / "q.gguf"
    write_qwen3_gguf(path, make_model(layers=1, tied=True, seed=5), mode="Q8_0", seed=2)
    return LlmEngine.from_gguf(path, n_ctx=1024, prefill_chunk=128)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_constrained_generation_follows_the_dfa(engine, seed):
    import json

    import jsonschema

    text = json_schema_to_gbnf(BOUNDED)
    dfa = compile_gbnf(text)
    prompt = engine.tokenizer.encode("<|im_start|>user\nfind foxes<|im_end|>\n<|im_start|>assistant\n")
    state, ids = 0, []
    it = engine.generate_ids(prompt, grammar=text, seed=seed, **_rag.QWEN3_SAMPLING)
    for t in it:
        ids.append(t)
        state = dfa.walk(engine.tokenizer.token_bytes[t], state)
        assert state >= 0 and state == int(engine.grammar_state.item())
    assert dfa.accept[state] and int(engine.grammar_state.item()) == state   # ended by an end-of-generation id
    out = engine.tokenizer.decode_bytes(ids).decode()
    jsonschema.validate(json.loads(out), BOUNDED)
    again = engine.tokenizer.decode_bytes(list(engine.generate_ids(prompt, grammar=text, seed=seed,
                                                                   **_rag.QWEN3_SAMPLING))).decode()
    assert again == out


def _insert(config):  # noqa: F811
    docs = [rl.Document.from_text(text, filename=name, url=url) for text, name, url in DOCS]
    rl.insert_documents(docs, config=config)


def test_rag_with_a_fixed_tool_end_to_end(config, monkeypatch):  # noqa: F811
    _insert(config)
    tool = copy.deepcopy(_rag.SEARCH_KNOWLEDGE_BASE_TOOL)
    tool["function"]["parameters"] = BOUNDED
    queries, got = [], []
    real = _rag.retrieve_context

    def spy(query, **kw):  # noqa: ANN001, ANN003, ANN202
        queries.append(query)
        return real(query, **kw)

    monkeypatch.setattr(_rag, "retrieve_context", spy)
    messages = [{"role": "user", "content": "What colour is the fox?"}]
    out = "".join(_rag._rag_with_tools(messages, tools=[tool], tool_choice={"type": "function", "function": {
        "name": "search_knowledge_base"}}, on_retrieval=got.append, config=config, max_tokens=12, seed=4))
    roles = [m["role"] for m in messages]
    n = len(messages[1]["tool_calls"])
    assert roles == ["user", "assistant"] + ["tool"] * n + ["assistant"] and 1 <= n <= 17
    import json

    assert queries == [json.loads(c["function"]["arguments"])["query"] for c in messages[1]["tool_calls"]]
    assert got and all(isinstance(s, rl.ChunkSpan) for x in got for s in x)
    engine = _rag.get_llm(config)
    prompt = engine.tokenizer.encode(render_chatml_tools(_rag._clip(messages[:-1], engine.n_ctx)))
    want = "".join(engine.generate(prompt, stop=DEFAULT_STOP, max_tokens=12, seed=4, **_rag.QWEN3_SAMPLING))
    assert out == want and messages[-1] == {"role": "assistant", "content": want}


def test_rag_auto_replays_on_the_host_protocol(config):  # noqa: F811
    from raglite_b200 import _llm

    _insert(config)
    engine = _rag.get_llm(config)
    seen = []
    real = engine.generate_ids

    def spy(prompt_ids, **kw):  # noqa: ANN001, ANN003, ANN202
        rec = {"prompt": engine.tokenizer.decode_bytes(prompt_ids).decode(), "ids": [], "error": None}
        seen.append(rec)
        try:
            for t in real(prompt_ids, **kw):
                rec["ids"].append(t)
                yield t
        except ValueError as e:   # a prompt past n_ctx: the replay raises it at the same completion
            rec["error"] = e
            raise

    engine.generate_ids = spy

    def run(messages):  # noqa: ANN001, ANN202
        try:
            return "".join(rl.rag(messages, config=config, max_tokens=10, seed=3)), None
        except ValueError as e:   # arguments the fixture model left unparseable (cut at n_ctx)
            return None, str(e)

    try:
        m1 = [{"role": "user", "content": "What colour is the fox?"}]
        out, err = run(m1)
    finally:
        del engine.generate_ids
    raw = [r["error"] or engine.tokenizer.decode_bytes(r["ids"]).decode(errors="replace") + "<|im_end|>" for r in seen]
    scripted = go.ScriptedEngine(raw)
    rl.register_llm(config, scripted)
    try:
        m2 = [{"role": "user", "content": "What colour is the fox?"}]
        out2, err2 = run(m2)
    finally:
        _llm.register_llm(config, engine)
    assert [c["prompt"] for c in scripted.calls] == [r["prompt"] for r in seen]
    assert [m["role"] for m in m2] == [m["role"] for m in m1] and (err is None) == (err2 is None)
    if out is not None:   # the replay's byte tokens are shorter, so its 10-token answer is a prefix
        assert out.startswith(out2)
