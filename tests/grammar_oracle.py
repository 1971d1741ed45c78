"""Independent statements of grammar-constrained generation for the tests: a set-based backtracking matcher over the
parsed GBNF AST that decodes UTF-8 itself (full acceptance and prefix liveness, with no DFA), the token index as a
NumPy walk, the masked sampler as ``llm_oracle.sample`` on pre-masked logits, and a scripted engine that emits given
texts token by token through the NumPy mask."""

from __future__ import annotations

from collections.abc import Iterator, Sequence
from typing import Any

import numpy as np

import llm_oracle
from raglite_b200._grammar import SURROGATES, parse_gbnf
from raglite_b200._llm import LlmEngine

EOF = -1   # "the input ran out while this node could still go on"

_LEAD = [(0x00, 0x7F, 1, 0x00), (0xC2, 0xDF, 2, 0x80), (0xE0, 0xEF, 3, 0x800), (0xF0, 0xF4, 4, 0x10000)]


def _cp_range(data: bytes, i: int) -> tuple[int, int, int] | None:
    """The code points whose strict UTF-8 encoding starts with ``data[i:]`` (cut at one character): (lo, hi, length
    consumed) with length 0 when the input ends inside the character; None when no valid encoding starts so."""
    b0 = data[i]
    lead = next((x for x in _LEAD if x[0] <= b0 <= x[1]), None)
    if lead is None:
        return None
    n = lead[2]
    if n == 1:
        return b0, b0, 1
    cp = b0 & (0x7F >> n)
    have = min(n, len(data) - i)
    for k in range(1, have):
        c = data[i + k]
        if c & 0xC0 != 0x80:
            return None
        cp = (cp << 6) | (c & 0x3F)
    missing = n - have
    lo, hi = cp << (6 * missing), (cp << (6 * missing)) | ((1 << (6 * missing)) - 1)
    lo, hi = max(lo, lead[3]), min(hi, 0x10FFFF)   # no overlong forms, nothing past U+10FFFF
    if lo > hi:
        return None
    return lo, hi, (n if missing == 0 else 0)


def _in_class(ranges: Sequence[tuple[int, int]], lo: int, hi: int) -> bool:
    """Some code point of [lo, hi], surrogates excluded, is in the class."""
    for a, b in ranges:
        x, y = max(a, lo), min(b, hi)
        while x <= y:
            if SURROGATES[0] <= x <= SURROGATES[1]:
                x = SURROGATES[1] + 1
                continue
            return True
    return False


class Matcher:
    """Runs the AST over a byte string: ``ends(node, i)`` is the set of positions where a match of ``node`` starting at
    ``i`` can end, plus EOF when the input ends inside a match that could go on."""

    def __init__(self, text: str) -> None:
        self.rules = parse_gbnf(text)

    def ends(self, node: Any, data: bytes, i: int) -> set[int]:
        kind = node[0]
        n = len(data)
        if kind == "lit":
            lit = node[1]
            if data[i:i + len(lit)] == lit:
                return {i + len(lit)}
            return {EOF} if n - i < len(lit) and lit.startswith(data[i:]) else set()
        if kind == "cls":
            if i == n:
                return {EOF}
            r = _cp_range(data, i)
            if r is None or not _in_class(node[1], r[0], r[1]):
                return set()
            return {EOF} if r[2] == 0 else {i + r[2]}
        if kind == "ref":
            return self.ends(self.rules[node[1]], data, i)
        if kind == "alt":
            return set().union(*(self.ends(a, data, i) for a in node[1]))
        if kind == "seq":
            cur, out_eof = {i}, False
            for item in node[1]:
                nxt: set[int] = set()
                for p in cur:
                    nxt |= self.ends(item, data, p)
                out_eof |= EOF in nxt
                cur = nxt - {EOF}
            return cur | ({EOF} if out_eof else set())
        if kind == "rep":
            _, body, lo, hi = node
            out, cur, seen, count = set(), {i}, set(), 0
            while cur:
                if count >= lo:
                    out |= cur
                if hi is not None and count == hi:
                    break
                nxt: set[int] = set()
                for p in cur:
                    nxt |= self.ends(body, data, p)
                if EOF in nxt:
                    out.add(EOF)
                cur = nxt - {EOF}
                count += 1
                if count > lo:   # past the minimum only new positions matter
                    cur -= seen
                    seen |= cur
            return out
        raise AssertionError(kind)

    def accepts(self, data: bytes) -> bool:
        return len(data) in self.ends(("ref", "root"), data, 0)

    def live(self, data: bytes) -> bool:
        """Some string of the language starts with ``data``."""
        e = self.ends(("ref", "root"), data, 0)
        return EOF in e or len(data) in e

    def generate(self, rng: np.random.Generator, *, max_rep: int = 4) -> bytes:
        """A seeded string of the language (each repetition at most its minimum + ``max_rep``)."""
        return self._gen(("ref", "root"), rng, max_rep)

    def _gen(self, node: Any, rng: np.random.Generator, max_rep: int) -> bytes:
        kind = node[0]
        if kind == "lit":
            return node[1]
        if kind == "cls":
            while True:
                a, b = node[1][int(rng.integers(len(node[1])))]
                cp = int(rng.integers(a, min(b, a + 0x3000) + 1)) if rng.random() < 0.5 else int(rng.integers(a, b + 1))
                if not SURROGATES[0] <= cp <= SURROGATES[1]:
                    return chr(cp).encode()
        if kind == "ref":
            return self._gen(self.rules[node[1]], rng, max_rep)
        if kind == "alt":
            return self._gen(node[1][int(rng.integers(len(node[1])))], rng, max_rep)
        if kind == "seq":
            return b"".join(self._gen(x, rng, max_rep) for x in node[1])
        _, body, lo, hi = node
        top = lo + max_rep if hi is None else min(hi, lo + max_rep)
        return b"".join(self._gen(body, rng, max_rep) for _ in range(int(rng.integers(lo, top + 1))))


# ---- the token index and the masked draw ---------------------------------------------------------------------------
def token_index(trans: np.ndarray, pieces: Sequence[bytes]) -> np.ndarray:
    """index[s, v]: the state after piece v's bytes from s, -1 on a missing transition or an empty piece (every state
    and token walked together, one byte position at a time)."""
    S, V = len(trans), len(pieces)
    lens = np.array([len(p) for p in pieces])
    L = int(lens.max(initial=0))
    buf = np.zeros((V, max(L, 1)), dtype=np.int64)
    for v, p in enumerate(pieces):
        buf[v, :len(p)] = np.frombuffer(p, dtype=np.uint8)
    st = np.where(lens[None, :] > 0, np.arange(S)[:, None], -1)
    for j in range(L):
        cols = np.flatnonzero(lens > j)   # the tokens still walking at byte j
        cur = st[:, cols]
        st[:, cols] = np.where(cur >= 0, trans[np.clip(cur, 0, None), buf[cols, j][None, :]], -1)
    return st.astype(np.int16)


def allowed(index: np.ndarray, accept: np.ndarray, eog: Sequence[int], state: int) -> np.ndarray:
    ok = index[state] >= 0
    for e in eog:
        ok[e] = bool(accept[state])
    return ok


def sample_masked(logits: np.ndarray, hist: list[int], index: np.ndarray, accept: np.ndarray, eog: Sequence[int],
                  state: int, **kw: float) -> tuple[int, int]:
    """(id, next state): ``llm_oracle.sample`` on the logits with disallowed ids (and ids whose own logit is -inf or
    NaN) at -inf and top-k cut to the allowed count; (-1, state) when nothing is allowed."""
    ok = allowed(index, accept, eog, state) & (np.asarray(logits, dtype=np.float32) > -np.inf)
    if not ok.any():
        return -1, state
    w = np.where(ok, np.asarray(logits, dtype=np.float32), np.float32(-np.inf)).astype(np.float32)
    kw = dict(kw)
    kw["top_k"] = min(int(kw["top_k"]), int(ok.sum()))
    t = llm_oracle.sample(w, hist, **kw)
    return t, state if t in eog else int(index[state, t])


# ---- a scripted engine ----------------------------------------------------------------------------------------------
class ByteTokenizer:
    """256 byte tokens, then extra multi-byte pieces, then the end-of-generation tokens (their text as bytes)."""

    def __init__(self, extra: Sequence[str] = ("functions", ".search", "_knowledge", "<function_calls>", "query",
                                               '": "', "é", "\U0001f98a")) -> None:
        self.token_bytes = [bytes([b]) for b in range(256)] + [e.encode() for e in extra] + [b"<|im_end|>",
                                                                                            b"<|endoftext|>"]
        self.ids = {"<|im_end|>": len(self.token_bytes) - 2, "<|endoftext|>": len(self.token_bytes) - 1}

    def encode(self, text: str) -> list[int]:
        return list(text.encode())


class ScriptedEngine(LlmEngine):
    """An engine whose completions are given raw outputs (text, then an end-of-generation token, or an exception to
    raise): each one emitted
    token by token, longest allowed piece first, each token checked against the NumPy mask of its grammar.  It records
    every completion's prompt text and settings; ``LlmEngine.generate`` applies the stop strings."""

    def __init__(self, raw: Sequence[str], n_ctx: int = 1 << 20) -> None:   # no device state
        from raglite_b200._grammar import compile_gbnf

        self.tokenizer = ByteTokenizer()
        self.n_ctx = n_ctx
        self.raw = list(raw)
        self.calls: list[dict[str, Any]] = []
        self._compile = compile_gbnf
        self._index: dict[str, tuple[Any, np.ndarray]] = {}

    def generate_ids(self, prompt_ids: Sequence[int], *, max_tokens: int | None = None, temperature: float = 0.6,
                     top_k: int = 20, top_p: float = 0.95, min_p: float = 0.0, repeat_penalty: float = 1.1,
                     seed: int | None = None, grammar: str | None = None) -> Iterator[int]:
        self.calls.append({"prompt": bytes(prompt_ids).decode(), "grammar": grammar, "temperature": temperature,
                           "max_tokens": max_tokens})
        raw = self.raw.pop(0)
        if isinstance(raw, Exception):   # a completion that failed where it was recorded
            raise raw
        text = raw.encode()
        eog = sorted(self.stop_ids())
        if grammar is not None and grammar not in self._index:
            g = self._compile(grammar)
            self._index[grammar] = (g, token_index(g.trans, self.tokenizer.token_bytes))
        g, idx = self._index[grammar] if grammar is not None else (None, None)
        pos, state, n = 0, 0, 0
        while pos < len(text) and (max_tokens is None or n < max_tokens):
            # the end-of-generation text is that token where the grammar allows it, else plain text
            if any(text.startswith(self.tokenizer.token_bytes[e], pos) for e in eog) and (g is None or g.accept[state]):
                return
            cands = [v for v, p in enumerate(self.tokenizer.token_bytes) if v not in eog and p and text.startswith(p, pos)]
            if g is not None:
                cands = [v for v in cands if idx[state, v] >= 0]
            if not cands:
                raise AssertionError(f"the grammar masks every token at byte {pos} of {text!r}")
            v = max(cands, key=lambda c: len(self.tokenizer.token_bytes[c]))
            if g is not None:
                state = int(idx[state, v])
            pos += len(self.tokenizer.token_bytes[v])
            n += 1
            yield v
        if max_tokens is not None and n >= max_tokens:
            return
        if g is not None:
            assert allowed(idx, g.accept, eog, state)[eog[0]], "end of generation outside an accepting state"
