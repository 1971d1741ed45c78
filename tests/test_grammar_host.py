"""The grammar compiler on the host: the byte-level DFA against the backtracking matcher of ``grammar_oracle`` (full
acceptance and prefix liveness on seeded strings of each language, their byte mutations and every truncation), the
JSON-schema grammars against ``json.loads`` + ``jsonschema``, and the refusals."""

from __future__ import annotations

import json
import zlib

import jsonschema
import numpy as np
import pytest

import grammar_oracle as go
from raglite_b200._grammar import MAX_STATES, GrammarError, compile_gbnf, json_schema_to_gbnf
from raglite_b200._tools import DECISION_GRAMMAR, FIXED_DECISION_GRAMMAR, FOLLOW_UP_GRAMMAR

NAMES = '"functions.search_knowledge_base:"'
NAMES2 = '"functions.search_knowledge_base:" | "functions.lookup:"'
PROTOCOL = {"decision": DECISION_GRAMMAR.format(names=NAMES), "fixed": FIXED_DECISION_GRAMMAR.format(names=NAMES),
            "follow_up": FOLLOW_UP_GRAMMAR.format(names=NAMES2)}
SCHEMAS = {
    "query": {"type": "object", "properties": {"query": {"type": "string"}}, "required": ["query"],
              "additionalProperties": False},
    "query_bounded": {"type": "object", "properties": {"query": {"type": "string", "minLength": 1, "maxLength": 6}},
                      "required": ["query"], "additionalProperties": False},
    "scalars": {"type": "object", "properties": {
        "n": {"type": "integer"}, "b": {"type": "boolean"}, "z": {"type": "null"}, "e": {"enum": ["a", 1, None]},
        "c": {"const": "k<&>"}}, "required": ["n", "b"], "additionalProperties": False},
    "array_number": {"type": "object", "properties": {
        "x": {"type": "number"},
        "tags": {"type": "array", "items": {"type": "string", "maxLength": 2}, "minItems": 1, "maxItems": 3},
        "opt": {"anyOf": [{"type": "string", "maxLength": 3}, {"type": "null"}]}},
        "required": ["tags"], "additionalProperties": False},
    "optional_only": {"type": "object", "properties": {"a": {"type": "integer"}, "b": {"type": "boolean"}},
                      "additionalProperties": False},
}
HAND = {
    "negated": 'root ::= [^a-c"\\\\] [^\\x00-\\x7F]',
    "utf8_class": "root ::= [é-ü\\u4e00-\\u4e10\\U0001F600-\\U0001F64F]+",
    "counted": 'root ::= "x"{2} [0-9]{1,3} "y"{2,} ("-" [a-b]{0,2}){1,2}',
    "nested_optional": 'root ::= ("a" ("b" ("c")?)?)? "d"? (e f?)*\ne ::= "e"\nf ::= [fg]',
    "dot": 'root ::= "<" . . ">"',
    "space": 'root ::= "{" space "}"\nspace ::= | " " | "\\n" [ \\t]{0,20}',
}
ALL = {**PROTOCOL, **{f"schema_{k}": json_schema_to_gbnf(v) for k, v in SCHEMAS.items()}, **HAND}


def _mutations(s: bytes, rng: np.random.Generator) -> list[bytes]:
    out = []
    for _ in range(4):
        m = bytearray(s)
        i = int(rng.integers(len(m) + 1))
        op = int(rng.integers(3))
        if op == 0 and m:
            m[min(i, len(m) - 1)] = int(rng.choice([0x80, 0xBF, 0xC0, 0xE0, 0xED, 0xF4, 0xF5, 0x22, 0x5C, rng.integers(256)]))
        elif op == 1:
            m.insert(i, int(rng.integers(256)))
        elif m:
            del m[min(i, len(m) - 1)]
        out.append(bytes(m))
    return out


@pytest.mark.parametrize("name", sorted(ALL))
def test_dfa_agrees_with_the_backtracking_matcher(name):
    text = ALL[name]
    g, m = compile_gbnf(text), go.Matcher(text)
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    for _ in range(25):
        s = m.generate(rng)
        assert m.accepts(s) and g.matches(s), s
        for cand in [s, *_mutations(s, rng)]:
            assert g.matches(cand) == m.accepts(cand), cand
            for cut in range(len(cand) + 1):
                assert (g.walk(cand[:cut]) >= 0) == m.live(cand[:cut]), cand[:cut]


@pytest.mark.parametrize("name", sorted(ALL))
def test_every_state_reaches_acceptance_and_fits_int16(name):
    g = compile_gbnf(ALL[name])
    assert g.trans.dtype == np.int16 and g.n_states <= MAX_STATES
    live = g.accept.copy()
    for _ in range(g.n_states):
        live |= np.any((g.trans >= 0) & live[np.clip(g.trans, 0, None)], axis=1)
    assert live.all()


def test_a_token_ending_inside_a_character_leaves_the_dfa_mid_character():
    g = compile_gbnf(HAND["utf8_class"])
    e_acute = "é".encode()
    s = g.walk(e_acute[:1])
    assert s >= 0 and not g.accept[s]
    assert g.walk(e_acute[1:], s) >= 0 and g.accept[g.walk(e_acute[1:], s)]
    assert g.walk(b"\xc3\xc3") == -1          # a lead byte where a continuation must come
    assert g.walk(b"\xe0\x80") == -1          # overlong
    assert g.walk(b"\xed\xa0\x80") == -1      # a surrogate
    assert g.walk(e_acute[1:]) == -1          # a continuation byte taken as a character


@pytest.mark.parametrize("name", sorted(SCHEMAS))
def test_strings_of_a_schema_grammar_parse_and_validate(name):
    text = json_schema_to_gbnf(SCHEMAS[name])
    m = go.Matcher(text)
    rng = np.random.default_rng(7)
    for _ in range(40):
        s = m.generate(rng)
        jsonschema.validate(json.loads(s.decode()), SCHEMAS[name])


def test_recalled_json_rules_are_written_as_recalled():
    text = json_schema_to_gbnf(SCHEMAS["array_number"]) + json_schema_to_gbnf(SCHEMAS["scalars"])
    assert 'space ::= | " " | "\\n" [ \\t]{0,20}' in text
    assert 'char ::= [^"\\\\\\x7F\\x00-\\x1F] | [\\\\] (["\\\\bfnrt] | "u" [0-9a-fA-F]{4})' in text
    assert "integral-part ::= [0] | [1-9] [0-9]{0,15}" in text


@pytest.mark.parametrize("schema", [
    {"type": "object", "properties": {"a": {"$ref": "#"}}, "additionalProperties": False},
    {"type": "object", "properties": {"a": {"type": "string", "pattern": "x+"}}, "additionalProperties": False},
    {"type": "object", "properties": {}},
    {"type": "string", "format": "date"},
    {"type": "array"},
])
def test_unsupported_schemas_raise(schema):
    with pytest.raises(NotImplementedError):
        json_schema_to_gbnf(schema)


def test_recursive_and_oversized_grammars_raise():
    with pytest.raises(NotImplementedError, match="recursive"):
        compile_gbnf('root ::= "[" item? "]"\nitem ::= root | "x"')
    with pytest.raises(NotImplementedError, match="states"):
        compile_gbnf("root ::= [a-z]{0,9000}")   # past the unminimized cap: refused before minimization
    with pytest.raises(GrammarError):
        compile_gbnf('root ::= "unterminated')
    with pytest.raises(GrammarError):
        compile_gbnf("root ::= undefined-rule")
