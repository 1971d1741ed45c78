"""ts_rank keyword search, host side: the tsvector text parser, the query analysis of ``raglite_b200._pgfts``, the
oracle's arithmetic (``tsrank_oracle``) on pinned values, and the C-ABI's refusals (no GPU needed)."""

from __future__ import annotations

import ctypes
import string

import numpy as np
import pytest

import tsrank_oracle as to
from raglite_b200 import _pgfts


# ---- tsvector text ----------------------------------------------------------------------------------------------------
def test_tsvector_parser_quotes_backslashes_and_positions():
    text = r"'a':1 'it''s':2,5,9 'back\\slash':3 'q''''':4 'naïve':7,8 'sp ace':10 'strip'"
    lex, npos = _pgfts.parse_tsvector(text, "c0")
    assert lex == ["a", "it's", "back\\slash", "q''", "naïve", "sp ace", "strip"]
    assert npos == [1, 3, 1, 1, 2, 1, 1]          # a lexeme without positions counts as one (POSNULL)
    assert _pgfts.parse_tsvector("", "c1") == ([], [])
    many = "'x':" + ",".join(str(p) for p in range(1, 257))
    assert _pgfts.parse_tsvector(many, "c2") == (["x"], [256])
    assert _pgfts.parse_tsvector("'x':16383", "c3") == (["x"], [1])
    # the oracle's own writer round-trips
    held = {"b": [1, 4], "a'b": [2], "c\\d": [], "é": [3, 5, 7]}
    assert _pgfts.parse_tsvector(to.tsvector_text(held)) == (sorted(held, key=str.encode), [1, 2, 1, 3])


@pytest.mark.parametrize("text,why", [
    ("'a':1A", "weight"), ("'a':1,2B", "weight"), ("'a':3C", "weight"),
    ("'x':" + ",".join(str(p) for p in range(1, 258)), "257 positions"),
    ("'a':1D", "malformed"), ("'a':0", "range"), ("'a':16384", "range"), ("'a':99999", "range"), ("'a':01", "range"),
    ("'a':-1", "range"), ("'a':", "malformed"), ("'a':1,", "malformed"), ("a:1", "malformed"),
    ("'a'  'b'", "malformed"), ("'a' ", "malformed"), ("'a''", "malformed"), ("'a'\t'b'", "malformed"), ("''", "empty"),
    ("'a':1 'a':2", "twice"), ("'a\\b'", "malformed"), ("'a':1 'b':x", "malformed"),
])
def test_tsvector_parser_refusals(text, why):
    with pytest.raises(ValueError, match="chunk 'cid-7'"):
        _pgfts.parse_tsvector(text, "cid-7")


def test_tsvector_parser_refuses_non_text():
    with pytest.raises(ValueError, match="chunk 3"):
        _pgfts.parse_tsvector(None, 3)


# ---- query analysis ---------------------------------------------------------------------------------------------------
def test_every_ascii_punctuation_character_separates_operands():
    for c in string.punctuation:
        assert _pgfts.tsquery_operands(f"ab{c}cd") == ["ab", "cd"], c
        assert _pgfts.query_lexemes(f"ab{c}cd") == ["ab", "cd"], c
    assert _pgfts.query_lexemes(string.punctuation) == []


def test_whitespace_ascii_and_unicode():
    assert _pgfts.tsquery_operands("a\tb\nc\r\nd\x0be\x0cf") == list("abcdef")
    assert _pgfts.tsquery_operands("a b c　d e\x85f") == list("abcdef")
    assert _pgfts.query_lexemes("  \t\n ") == []


def test_duplicates_case_and_byte_order():
    assert _pgfts.query_lexemes("Cat cat CAT dog") == ["cat", "dog"]
    # byte order: digits < upper < lower ASCII < multi-byte; a prefix before its extensions
    assert _pgfts.query_lexemes("zeta 9lives éclair alpha alphabet b2b") == ["9lives", "alpha", "alphabet", "b2b", "zeta",
                                                                             "éclair"]
    assert _pgfts.query_lexemes("ж z ä 中") == ["z", "ä", "ж", "中"]


def test_letters_and_digits_make_one_token():
    assert _pgfts.query_lexemes("covid19 2024 x86") == ["2024", "covid19", "x86"]
    assert _pgfts.query_lexemes("COVID-19") == ["19", "covid"]          # '-' is punctuation: two operands


def test_non_ascii_lower_casing():
    assert _pgfts.query_lexemes("ΣΊΣΥΦΟΣ") == ["σίσυφοσ"]              # no final-sigma rule: towlower per character
    assert _pgfts.query_lexemes("İstanbul") == ["istanbul"]             # U+0130 -> i
    assert _pgfts.query_lexemes("ÅNGSTRÖM Ünïcödé") == ["ångström", "ünïcödé"]


def test_phrase_operands_are_refused():
    for q in ("what’s up", "naïve café l’été", "áb", "x·y"):
        with pytest.raises(NotImplementedError, match="phrase"):
            _pgfts.query_lexemes(q)


def test_dropped_operands():
    assert _pgfts.query_lexemes("€ ™ ½ keep") == ["keep"]                # no token: the operand is dropped
    assert _pgfts.query_lexemes("a" * 2046 + " b") == ["a" * 2046, "b"]
    assert _pgfts.query_lexemes("a" * 2047 + " b") == ["b"]             # MAXSTRLEN bytes and more: not indexed
    assert _pgfts.query_lexemes("é" * 1023 + " é" + "a" * 2045) == ["é" * 1023]   # 2046 bytes kept, 2047 dropped
    assert _pgfts.query_lexemes("") == [] and _pgfts.query_lexemes("!!!") == []


# ---- oracle pins --------------------------------------------------------------------------------------------------------
def test_one_and_two_occurrences():
    assert str(to.rank([1], 1)) == "0.06079271" and str(to.rank([2], 1)) == "0.075990885"
    assert to.rank([1], 1).dtype == np.float32


def test_contribution_of_every_npos():
    """Each n in 1..256 against an independent restatement in Python floats rounded through float32 at each step; and the
    two roundings the issue names matter: skipping (0.1 + resj) - 0.1 or dividing in float changes some values."""
    f32 = lambda x: float(np.float32(x))  # noqa: E731
    resj, skipped, in_float = 0.0, 0, 0
    for n in range(1, 257):
        resj = f32(resj + f32(f32(0.1) / f32(n * n)))
        t = f32(f32(f32(0.1) + resj) - f32(0.1))
        assert to.CONTRIB[n - 1] == t / 1.64493406685, n
        skipped += f32(resj / 1.64493406685) != f32(t / 1.64493406685)
        in_float += f32(np.float32(t) / np.float32(1.64493406685)) != f32(t / 1.64493406685)
    assert skipped > 0 and in_float > 0
    assert (np.diff(to.CONTRIB) >= 0).all() and to.CONTRIB[0] > 0
    assert to.CONTRIB[-1] < 0.1 * 2 / 1.64493406685


def test_unknown_entries_count_in_the_divisor():
    table = {0: {"cat": 1}, 1: {"cat": 2, "dog": 1}, 2: {"emu": 3}}
    one = to.ts_rank_table(table, ["cat"])
    two = to.ts_rank_table(table, ["cat", "unknownword"])
    assert set(one) == {0, 1} and set(two) == {0, 1}
    assert two[0] == np.float32(one[0] / np.float32(2))
    both = to.ts_rank_table(table, ["dog", "cat"])
    assert both[1] == to.rank([2, 1], 2) and both[0] == to.rank([1], 2)
    assert to.ts_rank_table(table, []) == {} and to.ts_rank_table(table, ["zzz"]) == {}


def test_csr_restatement_matches_the_table_restatement():
    vocab = [f"w{i}" for i in range(300)] + ["Zulu", "alpha", "é"]
    texts, table = to.make_tsvectors(800, 3, vocab=vocab)
    ids: dict[str, int] = {}
    for c in range(len(texts)):
        for x in _pgfts.parse_tsvector(texts[c], c)[0]:
            ids.setdefault(x, len(ids))
    csr = to.csr_from_table(table, ids)
    rng = np.random.default_rng(4)
    queries = [list(rng.choice(vocab, size=int(rng.integers(1, 12)))) + (["nope"] if i % 3 == 0 else []) for i in range(40)]
    plans = [sorted(set(q), key=str.encode) for q in queries]
    q_off = np.concatenate([[0], np.cumsum([len(p) for p in plans])]).astype(np.int32)
    q_terms = np.asarray([ids.get(x, -1) for p in plans for x in p], np.int32)
    scores, matched = to.tsrank_csr_scores(*csr, q_off, q_terms, len(texts))
    for b, q in enumerate(queries):
        want = to.ts_rank_table(table, q)
        assert set(np.flatnonzero(matched[b])) == set(want)
        assert all(scores[b, c] == s for c, s in want.items())
    ids_, sc, cnt = to.tsrank_topk(scores, matched, None, 64)
    for b in range(len(queries)):
        s = sc[b, : cnt[b]]
        assert (np.diff(s) <= 0).all()
        tie = np.diff(s) == 0
        assert (np.diff(ids_[b, : cnt[b]])[tie] > 0).all()


# ---- C-ABI refusals -----------------------------------------------------------------------------------------------------
def test_tsrank_abi_refusals_before_any_cuda_call():
    from raglite_b200 import _lib

    lib = _lib.load()
    d = ctypes.c_void_p(16)
    call = lib.rl_tsrank_topk_global
    # (term_off, doc, npos, n_terms, n_chunks, mask, q_off, q_terms, B, k, chunk_base, out, ws, ws_bytes, stream)
    assert call(d, d, d, 1, 10, None, d, d, 0, 1, 0, d, d, 80, None) == 0                  # B = 0: nothing to do
    assert call(d, d, d, 1, 10, None, d, d, -1, 1, 0, d, d, 80, None) == -1                # B < 0
    assert call(d, d, d, -1, 10, None, d, d, 1, 1, 0, d, d, 80, None) == -1                # n_terms < 0
    assert call(d, d, d, 1, 1 << 31, None, d, d, 1, 1, 0, d, d, 80, None) == -1            # n_chunks > INT32_MAX
    assert call(d, d, d, 1, 10, None, d, d, 1, 1, -5, d, d, 80, None) == -1                # chunk_base < 0
    assert call(d, d, d, 1, 10, None, d, d, 1, 0, 0, d, d, 80, None) == -1                 # k = 0
    assert "k=0 outside [1, 4096]" in lib.rl_last_error().decode()
    assert call(d, d, d, 1, 10, None, d, d, 1, 4097, 0, d, d, 80, None) == -1              # k > 4096
    assert call(None, d, d, 1, 10, None, d, d, 1, 1, 0, d, d, 80, None) == -1              # term_off
    assert call(d, d, None, 1, 10, None, d, d, 1, 1, 0, d, d, 80, None) == -1              # npos
    assert call(d, d, d, 1, 10, None, d, d, 1, 1, 0, d, None, 80, None) == -1              # workspace
    assert call(d, d, d, 1, 10, None, d, d, 1, 1, 0, ctypes.c_void_p(24), d, 80, None) == -1   # out not 16-aligned
    assert "rl_tsrank_topk_global" in lib.rl_last_error().decode()
    assert call(d, d, d, 1, 10, None, d, d, 1, 1, 0, d, d, 79, None) == -3                 # workspace below one query
    assert "holds no query (needs 80)" in lib.rl_last_error().decode()


def test_postgresql_keyword_search_refusals_without_a_device():
    import raglite_b200 as rl

    cfg = rl.RAGLiteConfig(db_url="postgresql://u@h/none")
    with pytest.raises(NotImplementedError, match=r"ts_rank.*add_tsvector_rows.*to_tsvector\('simple', body\)::text"):
        rl.keyword_search("x", config=cfg)
    with pytest.raises(NotImplementedError, match="add_tsvector_rows"):
        rl.keyword_search_batch(["x"], config=cfg)
    with pytest.raises(NotImplementedError, match="self_query"):
        rl.keyword_search("x", config=rl.RAGLiteConfig(db_url="postgresql://u@h/none", self_query=True))
