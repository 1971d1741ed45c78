"""Grammar-constrained generation, host side: a GBNF subset compiled to a byte-level DFA over UTF-8, and JSON schema to
GBNF as llama-cpp-python's ``json_schema_to_gbnf`` writes it, for the subset RAGLite's function calling uses.

The GBNF subset: rules ``name ::= ...``, string literals with escapes, character classes with ranges and negation,
``.``, grouping, ``|``, ``?``, ``*``, ``+``, ``{m}``, ``{m,}``, ``{m,n}``.  Recursive rules are refused: the languages are
regular, so the grammar becomes one DFA whose transitions are bytes.  A character class is a set of code points; it
becomes the strict UTF-8 encodings of those code points (no overlong forms, no surrogates, nothing above U+10FFFF), so a
token that ends inside a multi-byte character leaves the DFA mid-character and invalid UTF-8 has no transition.

``Grammar.trans`` is ``int16 [S, 256]`` (next state or -1), ``Grammar.accept`` ``bool [S]``, state 0 the start.  The DFA
is minimal and every state can still reach acceptance, so every prefix it holds can be completed.  ``MAX_STATES`` caps
it: the device's token index is ``S x V`` int16 (311 MB at 1024 states and Qwen3's 151,936 tokens).
"""

from __future__ import annotations

import json
from collections.abc import Iterator
from dataclasses import dataclass
from typing import Any

import numpy as np

MAX_STATES = 1024
_MAX_BUILD_STATES = 8 * MAX_STATES   # the unminimized DFA, before minimization merges states
MAX_CODE_POINT = 0x10FFFF
SURROGATES = (0xD800, 0xDFFF)

# ---- AST: ("lit", bytes) | ("cls", ((lo, hi), ...)) | ("seq", [n...]) | ("alt", [n...]) | ("rep", n, min, max|None)
# ---- | ("ref", name)


class GrammarError(ValueError):
    """A grammar text that does not parse."""


def _normalize(ranges: list[tuple[int, int]]) -> tuple[tuple[int, int], ...]:
    out: list[list[int]] = []
    for lo, hi in sorted(r for r in ranges if r[0] <= r[1]):
        if out and lo <= out[-1][1] + 1:
            out[-1][1] = max(out[-1][1], hi)
        else:
            out.append([lo, hi])
    return tuple((a, b) for a, b in out)


def _negate(ranges: tuple[tuple[int, int], ...]) -> tuple[tuple[int, int], ...]:
    out, lo = [], 0
    for a, b in ranges:
        if a > lo:
            out.append((lo, a - 1))
        lo = b + 1
    if lo <= MAX_CODE_POINT:
        out.append((lo, MAX_CODE_POINT))
    return tuple(out)


class _Parser:
    def __init__(self, text: str) -> None:
        self.s, self.i = text, 0

    def error(self, msg: str) -> GrammarError:
        line = self.s.count("\n", 0, self.i) + 1
        return GrammarError(f"grammar line {line}: {msg} at {self.s[self.i:self.i + 20]!r}")

    def skip(self, newlines: bool) -> None:
        while self.i < len(self.s):
            c = self.s[self.i]
            if c == "#":
                while self.i < len(self.s) and self.s[self.i] != "\n":
                    self.i += 1
            elif c in " \t\r" or (newlines and c == "\n"):
                self.i += 1
            else:
                return

    def name(self) -> str:
        j = self.i
        while j < len(self.s) and (self.s[j].isalnum() or self.s[j] in "-_"):
            j += 1
        if j == self.i:
            raise self.error("expected a rule name")
        out, self.i = self.s[self.i:j], j
        return out

    def at_rule_start(self) -> bool:
        j = self.i
        while j < len(self.s) and (self.s[j].isalnum() or self.s[j] in "-_"):
            j += 1
        k = j
        while k < len(self.s) and self.s[k] in " \t":
            k += 1
        return j > self.i and self.s.startswith("::=", k)

    def escape(self) -> int:
        c = self.s[self.i]
        self.i += 1
        simple = {"n": 10, "t": 9, "r": 13, "\\": 92, '"': 34, "[": 91, "]": 93, "-": 45, "^": 94, "/": 47}
        if c in simple:
            return simple[c]
        width = {"x": 2, "u": 4, "U": 8}.get(c)
        if width is None:
            raise self.error(f"unknown escape \\{c}")
        digits = self.s[self.i:self.i + width]
        if len(digits) != width or any(d not in "0123456789abcdefABCDEF" for d in digits):
            raise self.error(f"bad \\{c} escape")
        self.i += width
        return int(digits, 16)

    def char(self) -> int:
        if self.i >= len(self.s):
            raise self.error("unexpected end")
        c = self.s[self.i]
        self.i += 1
        return self.escape() if c == "\\" else ord(c)

    def grammar(self) -> dict[str, Any]:
        rules: dict[str, Any] = {}
        self.skip(True)
        while self.i < len(self.s):
            name = self.name()
            self.skip(False)
            if not self.s.startswith("::=", self.i):
                raise self.error("expected '::='")
            self.i += 3
            if name in rules:
                raise self.error(f"rule {name!r} defined twice")
            rules[name] = self.alternatives()
            self.skip(True)
        if "root" not in rules:
            raise GrammarError("grammar has no 'root' rule")
        return rules

    def alternatives(self) -> Any:
        alts = [self.sequence()]
        while True:
            self.skip(True)
            if self.i < len(self.s) and self.s[self.i] == "|":
                self.i += 1
                alts.append(self.sequence())
            else:
                break
        return alts[0] if len(alts) == 1 else ("alt", alts)

    def sequence(self) -> Any:
        items: list[Any] = []
        while True:
            self.skip(True)
            if self.i >= len(self.s) or self.s[self.i] in "|)" or self.at_rule_start():
                break
            items.append(self.postfix(self.atom()))
        return items[0] if len(items) == 1 else ("seq", items)

    def atom(self) -> Any:
        c = self.s[self.i]
        if c == '"':
            self.i += 1
            out = []
            while self.i < len(self.s) and self.s[self.i] != '"':
                out.append(chr(self.char()))
            if self.i >= len(self.s):
                raise self.error("unterminated literal")
            self.i += 1
            return ("lit", "".join(out).encode("utf-8", errors="surrogatepass"))
        if c == "[":
            self.i += 1
            neg = self.s.startswith("^", self.i)
            self.i += neg
            ranges = []
            while self.i < len(self.s) and self.s[self.i] != "]":
                lo = self.char()
                hi = lo
                if self.s.startswith("-", self.i) and not self.s.startswith("-]", self.i):
                    self.i += 1
                    hi = self.char()
                if hi < lo:
                    raise self.error("inverted range")
                ranges.append((lo, hi))
            if self.i >= len(self.s):
                raise self.error("unterminated character class")
            self.i += 1
            norm = _normalize(ranges)
            return ("cls", _negate(norm) if neg else norm)
        if c == ".":
            self.i += 1
            return ("cls", ((0, MAX_CODE_POINT),))
        if c == "(":
            self.i += 1
            node = self.alternatives()
            self.skip(True)
            if not self.s.startswith(")", self.i):
                raise self.error("expected ')'")
            self.i += 1
            return node
        if c.isalnum() or c in "-_":
            return ("ref", self.name())
        raise self.error("unexpected character")

    def postfix(self, node: Any) -> Any:
        while self.i < len(self.s):
            c = self.s[self.i]
            if c in "?*+":
                self.i += 1
                node = ("rep", node, 1 if c == "+" else 0, 1 if c == "?" else None)
            elif c == "{":
                j = self.s.find("}", self.i)
                if j < 0:
                    raise self.error("unterminated repetition")
                body = self.s[self.i + 1:j].replace(" ", "")
                try:
                    if "," in body:
                        a, b = body.split(",", 1)
                        lo, hi = int(a), (int(b) if b else None)
                    else:
                        lo = hi = int(body)
                except ValueError as e:
                    raise self.error("bad repetition") from e
                if hi is not None and hi < lo:
                    raise self.error("bad repetition bounds")
                self.i = j + 1
                node = ("rep", node, lo, hi)
            else:
                break
        return node


def parse_gbnf(text: str) -> dict[str, Any]:
    """The rules of a GBNF text as AST nodes (see the module's comment), by name."""
    return _Parser(text).grammar()


# ---- UTF-8 ---------------------------------------------------------------------------------------------------------
def _utf8_len(cp: int) -> int:
    return 1 if cp < 0x80 else 2 if cp < 0x800 else 3 if cp < 0x10000 else 4


def _split_utf8(lo: int, hi: int) -> Iterator[list[tuple[int, int]]]:
    """Byte-range sequences whose product is exactly the UTF-8 encodings of [lo, hi] (no surrogates inside)."""
    if lo > hi:
        return
    for b in (0x7F, 0x7FF, 0xFFFF):
        if lo <= b < hi:
            yield from _split_utf8(lo, b)
            yield from _split_utf8(b + 1, hi)
            return
    if hi < 0x80:
        yield [(lo, hi)]
        return
    n = _utf8_len(lo)
    for i in range(1, n):
        m = (1 << (6 * i)) - 1
        if lo & ~m != hi & ~m:
            if lo & m:
                yield from _split_utf8(lo, lo | m)
                yield from _split_utf8((lo | m) + 1, hi)
                return
            if hi & m != m:
                yield from _split_utf8(lo, (hi & ~m) - 1)
                yield from _split_utf8(hi & ~m, hi)
                return
    a, b = chr(lo).encode(), chr(hi).encode()
    yield list(zip(a, b, strict=True))


def class_sequences(ranges: tuple[tuple[int, int], ...]) -> list[list[tuple[int, int]]]:
    """The UTF-8 byte-range sequences of a code-point class (surrogates removed)."""
    out = []
    for lo, hi in ranges:
        parts = [(lo, min(hi, SURROGATES[0] - 1)), (max(lo, SURROGATES[1] + 1), hi)]
        for a, b in parts:
            out.extend(_split_utf8(a, min(b, MAX_CODE_POINT)))
    return out


# ---- NFA (Thompson) -> DFA -----------------------------------------------------------------------------------------
class _Nfa:
    def __init__(self) -> None:
        self.eps: list[list[int]] = []
        self.edges: list[list[tuple[int, int, int]]] = []

    def state(self) -> int:
        self.eps.append([])
        self.edges.append([])
        return len(self.eps) - 1


def _build(nfa: _Nfa, rules: dict[str, Any], node: Any, s: int, stack: tuple[str, ...]) -> int:
    """Add ``node`` from state ``s``; returns its end state."""
    kind = node[0]
    if kind == "lit":
        for b in node[1]:
            t = nfa.state()
            nfa.edges[s].append((b, b, t))
            s = t
        return s
    if kind == "cls":
        e = nfa.state()
        for seq in class_sequences(node[1]):
            cur = s
            for k, (lo, hi) in enumerate(seq):
                t = e if k == len(seq) - 1 else nfa.state()
                nfa.edges[cur].append((lo, hi, t))
                cur = t
        return e
    if kind == "seq":
        for item in node[1]:
            s = _build(nfa, rules, item, s, stack)
        return s
    if kind == "alt":
        e = nfa.state()
        for item in node[1]:
            a = nfa.state()
            nfa.eps[s].append(a)
            nfa.eps[_build(nfa, rules, item, a, stack)].append(e)
        return e
    if kind == "ref":
        name = node[1]
        if name not in rules:
            raise GrammarError(f"undefined rule {name!r}")
        if name in stack:
            raise NotImplementedError(f"recursive grammar rule {name!r} ({' -> '.join((*stack, name))}): only regular "
                                      "grammars (no rule reaching itself) are supported")
        return _build(nfa, rules, rules[name], s, (*stack, name))
    if kind == "rep":
        _, body, lo, hi = node
        for _ in range(lo):
            s = _build(nfa, rules, body, s, stack)
        if hi is None:   # s -> body -> s, and out
            a = nfa.state()
            nfa.eps[s].append(a)
            nfa.eps[_build(nfa, rules, body, a, stack)].append(s)
            e = nfa.state()
            nfa.eps[s].append(e)
            return e
        e = nfa.state()
        for _ in range(hi - lo):
            nfa.eps[s].append(e)
            s = _build(nfa, rules, body, s, stack)
        nfa.eps[s].append(e)
        return e
    raise AssertionError(kind)


def _closure(nfa: _Nfa, states: set[int]) -> frozenset[int]:
    out, todo = set(states), list(states)
    while todo:
        for t in nfa.eps[todo.pop()]:
            if t not in out:
                out.add(t)
                todo.append(t)
    return frozenset(out)


def _subset(nfa: _Nfa, start: int, final: int) -> tuple[np.ndarray, np.ndarray]:
    s0 = _closure(nfa, {start})
    ids = {s0: 0}
    order = [s0]
    rows: list[np.ndarray] = []
    for cur in order:   # grows while iterating
        row = np.full(256, -1, dtype=np.int64)
        edges = [e for q in cur for e in nfa.edges[q]]
        cuts = sorted({lo for lo, _, _ in edges} | {hi + 1 for _, hi, _ in edges})
        for a, b in zip(cuts, cuts[1:], strict=False):
            tgt = {t for lo, hi, t in edges if lo <= a and b - 1 <= hi}
            if not tgt:
                continue
            nxt = _closure(nfa, tgt)
            if nxt not in ids:
                if len(order) >= _MAX_BUILD_STATES:
                    raise NotImplementedError(f"grammar DFA exceeds {_MAX_BUILD_STATES} states before minimization")
                ids[nxt] = len(order)
                order.append(nxt)
            row[a:b] = ids[nxt]
        rows.append(row)
    return np.stack(rows), np.array([final in s for s in order])


def _minimize(trans: np.ndarray, accept: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """Drop states that cannot reach acceptance (their transitions become -1), merge equivalent states (Moore's
    refinement) and renumber breadth-first from the start."""
    S = len(trans)
    live = accept.copy()
    while True:
        nxt = live | np.any((trans >= 0) & live[np.clip(trans, 0, None)], axis=1)
        if np.array_equal(nxt, live):
            break
        live = nxt
    if not live[0]:
        raise GrammarError("the grammar accepts no string")
    t = np.where((trans >= 0) & live[np.clip(trans, 0, None)], trans, -1)
    cls = np.where(live, accept.astype(np.int64), -1)
    while True:
        sig = np.concatenate([cls[:, None], np.where(t >= 0, cls[np.clip(t, 0, None)], -1)], axis=1)
        _, new = np.unique(sig, axis=0, return_inverse=True)
        new = np.where(live, new.reshape(-1), -1)
        if len(np.unique(new[live])) == len(np.unique(cls[live])):
            cls = new
            break
        cls = new
    order, seen = [], {int(cls[0])}
    todo = [int(cls[0])]
    rep = {}
    for s in range(S):
        if live[s]:
            rep.setdefault(int(cls[s]), s)
    while todo:
        c = todo.pop(0)
        order.append(c)
        for b in range(256):
            d = t[rep[c], b]
            if d >= 0 and int(cls[d]) not in seen:
                seen.add(int(cls[d]))
                todo.append(int(cls[d]))
    num = {c: i for i, c in enumerate(order)}
    out = np.full((len(order), 256), -1, dtype=np.int64)
    acc = np.zeros(len(order), dtype=bool)
    for c, i in num.items():
        r = t[rep[c]]
        out[i] = [num[int(cls[d])] if d >= 0 else -1 for d in r]
        acc[i] = accept[rep[c]]
    return out, acc


@dataclass(frozen=True)
class Grammar:
    """A compiled grammar: ``text`` (its GBNF), ``trans`` int16 [S, 256] (-1: no transition), ``accept`` bool [S]."""

    text: str
    trans: np.ndarray
    accept: np.ndarray

    @property
    def n_states(self) -> int:
        return len(self.trans)

    def walk(self, data: bytes, state: int = 0) -> int:
        """The state after ``data`` from ``state``, -1 once a byte has no transition."""
        for b in data:
            if state < 0:
                return -1
            state = int(self.trans[state, b])
        return state

    def matches(self, data: bytes) -> bool:
        s = self.walk(data)
        return s >= 0 and bool(self.accept[s])


def compile_gbnf(text: str, *, max_states: int = MAX_STATES) -> Grammar:
    """Compile a GBNF text (the subset in the module's comment) to its minimal byte-level DFA."""
    rules = parse_gbnf(text)
    nfa = _Nfa()
    start = nfa.state()
    final = _build(nfa, rules, ("ref", "root"), start, ())
    trans, accept = _minimize(*_subset(nfa, start, final))
    if len(trans) > max_states:
        raise NotImplementedError(f"grammar DFA has {len(trans)} states, more than {max_states}")
    return Grammar(text, trans.astype(np.int16), accept)


# ---- JSON schema -> GBNF (llama-cpp-python's json_schema_to_gbnf, restated for a subset) ---------------------------
SPACE_RULE = '| " " | "\\n" [ \\t]{0,20}'
CHAR_RULE = r'[^"\\\x7F\x00-\x1F] | [\\] (["\\bfnrt] | "u" [0-9a-fA-F]{4})'
PRIMITIVE_RULES = {
    "boolean": '("true" | "false") space',
    "decimal-part": "[0-9]{1,16}",
    "integral-part": "[0] | [1-9] [0-9]{0,15}",
    "number": '("-"? integral-part) ("." decimal-part)? ([eE] [-+]? integral-part)? space',
    "integer": '("-"? integral-part) space',
    "null": '"null" space',
    "char": CHAR_RULE,
}
_PRIMITIVE_DEPS = {"number": ("integral-part", "decimal-part"), "integer": ("integral-part",)}
_SCHEMA_KEYS_IGNORED = {"description", "title", "$schema", "default", "examples"}


def _gbnf_literal(s: str) -> str:
    esc = {"\r": "\\r", "\n": "\\n", '"': '\\"', "\\": "\\\\"}
    return '"' + "".join(esc.get(c, c) for c in s) + '"'


def _repetition(item: str, lo: int, hi: int | None, sep: str | None = None) -> str:
    if sep is None:
        if lo == 0 and hi == 1:
            return f"{item}?"
        if hi is None:
            return f"{item}*" if lo == 0 else f"{item}+" if lo == 1 else f"{item}{{{lo},}}"
        return f"{item}{{{lo}}}" if lo == hi else f"{item}{{{lo},{hi}}}"
    if hi == 0:
        return ""
    rest = _repetition(f"({sep} {item})", max(lo - 1, 0), None if hi is None else hi - 1)
    body = f"{item} {rest}"
    return f"({body})?" if lo == 0 else f"({body})"


class _SchemaConverter:
    def __init__(self) -> None:
        self.rules: dict[str, str] = {"space": SPACE_RULE}

    def add(self, name: str, body: str) -> str:
        key, i = name or "root", 0
        while key in self.rules and self.rules[key] != body:
            i += 1
            key = f"{name or 'root'}{i}"
        self.rules[key] = body
        return key

    def primitive(self, name: str) -> str:
        for dep in _PRIMITIVE_DEPS.get(name, ()):
            self.rules[dep] = PRIMITIVE_RULES[dep]
        self.rules[name] = PRIMITIVE_RULES[name]
        return name

    def visit(self, schema: Any, name: str) -> str:
        if not isinstance(schema, dict):
            raise NotImplementedError(f"schema {schema!r}: only object schemas are supported")
        unknown = set(schema) - _SCHEMA_KEYS_IGNORED - {"type", "properties", "required", "additionalProperties",
                                                        "minLength", "maxLength", "enum", "const", "items", "minItems",
                                                        "maxItems", "anyOf", "oneOf"}
        if unknown:
            raise NotImplementedError(f"JSON schema keywords {sorted(unknown)} are not supported")
        rule = name or "root"
        if "anyOf" in schema or "oneOf" in schema:
            alts = schema.get("anyOf", schema.get("oneOf"))
            return self.add(rule, " | ".join(self.visit(a, f"{rule}-{i}") for i, a in enumerate(alts)))
        if "const" in schema:
            return self.add(rule, _gbnf_literal(json.dumps(schema["const"])) + " space")
        if "enum" in schema:
            return self.add(rule, "(" + " | ".join(_gbnf_literal(json.dumps(v)) for v in schema["enum"]) + ") space")
        ty = schema.get("type")
        if isinstance(ty, list):
            return self.add(rule, " | ".join(self.visit({**schema, "type": t}, f"{rule}-{t}") for t in ty))
        if ty == "object":
            return self.add(rule, self.object_rule(schema, rule))
        if ty == "array":
            if not isinstance(schema.get("items"), dict):
                raise NotImplementedError("array schemas need a single 'items' schema")
            item = self.visit(schema["items"], f"{rule}-item")
            rep = _repetition(item, int(schema.get("minItems", 0)), schema.get("maxItems"), '"," space')
            return self.add(rule, f'"[" space {rep} "]" space')
        if ty == "string":
            self.primitive("char")
            lo, hi = int(schema.get("minLength", 0)), schema.get("maxLength")
            return self.add(rule, f'"\\"" {_repetition("char", lo, None if hi is None else int(hi))} "\\"" space')
        if ty in ("integer", "number", "boolean", "null"):
            if set(schema) - _SCHEMA_KEYS_IGNORED - {"type"}:
                raise NotImplementedError(f"keywords on a {ty} schema are not supported")
            return self.primitive(ty)
        raise NotImplementedError(f"JSON schema type {ty!r} is not supported")

    def object_rule(self, schema: dict[str, Any], name: str) -> str:
        if schema.get("additionalProperties") is not False:   # else any extra key, whose value grammar recurses
            raise NotImplementedError("object schemas need additionalProperties: false")
        props = schema.get("properties", {})
        required = [k for k in props if k in set(schema.get("required", []))]
        optional = [k for k in props if k not in set(required)]
        kv = {k: self.add(f"{name}-{k}-kv", f"{_gbnf_literal(json.dumps(k))} space \":\" space "
                                             f"{self.visit(props[k], f'{name}-{k}')}") for k in props}

        def rest(ks: list[str], first_optional: bool) -> str:
            k, *more = ks
            out = f'( "," space {kv[k]} )?' if first_optional else kv[k]
            if more:
                out += " " + self.add(f"{name}-{k}-rest", rest(more, True))
            return out

        body = '"{" space ' + ' "," space '.join(kv[k] for k in required)
        if optional:
            body += " ("
            if required:
                body += ' "," space ( '
            body += " | ".join(rest(optional[i:], False) for i in range(len(optional)))
            if required:
                body += " )"
            body += " )?"
        return body + ' "}" space'


def json_schema_to_gbnf(schema: dict[str, Any] | str) -> str:
    """The GBNF of a JSON schema (``object`` with ``additionalProperties: false``, ``string`` with ``minLength`` /
    ``maxLength``, ``integer``, ``number``, ``boolean``, ``null``, ``enum``, ``const``, ``array`` of ``items`` with
    ``minItems`` / ``maxItems``, ``anyOf`` / ``oneOf``).  Anything else raises ``NotImplementedError``."""
    conv = _SchemaConverter()
    conv.visit(json.loads(schema) if isinstance(schema, str) else schema, "")
    return "".join(f"{k} ::= {v}\n" for k, v in sorted(conv.rules.items()))
