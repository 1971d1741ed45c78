"""The device analysis of the BM25 index (csrc/fts.cu, ``_fts.analyze_on_device``), host side: the class and stop tables
it is given, the tokenizer automaton it runs restated in Python, against ``_fts.tokenize`` itself, and the refusals of
its C-ABI before any CUDA call."""

from __future__ import annotations

import ctypes

import numpy as np
import pytest

from raglite_b200 import _fts

SEP, WORD, ODD = 0, 1, 2


def _letter(c: int) -> str:
    return chr(ord("a") + c - 1)


def test_class_table_agrees_with_the_tokenizer_for_every_code_point():
    """``a·ch·b`` and ``\\·ch·b`` through ``tokenize``, predicted from the class of ``ch`` alone: a letter joins the word
    (and is swallowed by the backslash), a dropped code point vanishes (so the backslash swallows the ``b``), a
    separator splits (and is swallowed itself, with the backslash)."""
    table = _fts.class_table()
    assert table.shape == (0x110000,) and table.dtype == np.uint8
    assert ((table >= 1) & (table <= 26)).sum() == 542 and (table == _fts.CLASS_DROP).sum() == 1985
    bad = []
    for cp in range(0x110000):
        ch, c = chr(cp), int(table[cp])
        if ch == "\\":   # a separator that swallows the b; two backslashes pair up
            want = (["a"], ["b"])
        elif c == _fts.CLASS_DROP:
            want = (["ab"], [])
        elif 1 <= c <= 26:
            want = ([f"a{_letter(c)}b"], ["b"])
        else:
            want = (["a", "b"], ["b"])
        got = (_fts.tokenize("a" + ch + "b"), _fts.tokenize("\\" + ch + "b"))
        if got != want:
            bad.append((hex(cp), got, want))
    assert not bad, bad[:10]
    assert (table[ord("É")], table[0x0130], table[0x212A], table[0x0301]) == (5, 9, 11, _fts.CLASS_DROP)


def _automaton_words(text: str, table: np.ndarray) -> list[str]:
    """The words of ``rl_fts_mark``'s automaton, one code point at a time: a letter starts a word in SEP, continues it
    in WORD and is swallowed in ODD; a backslash moves to ODD, or back to SEP from ODD; a dropped code point changes
    nothing; any other separator moves to SEP."""
    words, cur, s = [], [], SEP
    for ch in text:
        c = int(table[ord(ch)])
        if ch == "\\":
            s = SEP if s == ODD else ODD
        elif c == _fts.CLASS_DROP:
            continue
        elif 1 <= c <= 26:
            if s == ODD:
                s = SEP
            else:
                cur.append(_letter(c))
                s = WORD
                continue
        else:
            s = SEP
        if cur:
            words.append("".join(cur))
            cur = []
    if cur:
        words.append("".join(cur))
    return words


def test_backslash_parity_rule_matches_the_tokenizer():
    table = _fts.class_table()
    alphabet = ["a", "b", "Z", "\\", "\n", " ", "\u0301", "é", "İ", "1", "ß", "\u212a"]
    rng = np.random.default_rng(7)
    for _ in range(40_000):
        text = "".join(alphabet[i] for i in rng.integers(0, len(alphabet), size=int(rng.integers(0, 24))))
        assert _automaton_words(text, table) == _fts.tokenize(text), repr(text)
    for n in range(1, 12):   # long runs, and runs broken by marks and newlines
        for tail in ("b", "\nb", "\u0301b", "\\\u0301b"):
            text = "a" + "\\" * n + tail
            assert _automaton_words(text, table) == _fts.tokenize(text), repr(text)


def test_stop_table_is_the_letter_only_stop_words():
    table = _fts.stop_table()
    assert table.dtype == np.uint64 and table.shape[1] == 2
    words = [(int(hi).to_bytes(8, "big") + int(lo).to_bytes(8, "big")).rstrip(b"\0").decode() for hi, lo in table]
    assert words == sorted(words)   # the padded strings in byte order: what the device's binary search needs
    assert set(words) == {w for w in _fts.STOPWORDS if w.isascii() and w.isalpha() and w.islower()}
    assert len(words) == len(set(words)) and max(map(len, words)) == 13


def test_groups_respect_the_byte_budget():
    assert _fts._groups([], 10) == []
    assert _fts._groups([5, 5, 5, 100, 1, 1], 12) == [(0, 2), (2, 3), (3, 4), (4, 6)]
    assert _fts._groups([0, 0, 0], 1) == [(0, 1), (1, 2), (2, 3)]
    sizes = np.random.default_rng(1).integers(0, 50, size=500).tolist()
    groups = _fts._groups(sizes, 200)
    assert groups[0][0] == 0 and groups[-1][1] == 500 and all(a[1] == b[0] for a, b in zip(groups, groups[1:]))
    assert all(b - a == 1 or sum(sizes[a:b]) + (b - a) <= 200 for a, b in groups)


def test_add_stems_appends_in_the_order_given():
    an = _fts.Analyzer()
    an.analyze(["cats and dogs"])
    assert an.add_stems(["dog", "zebra", "cat", "zebra", "ant"]).tolist() == [1, 2, 0, 2, 3]
    assert an.term_ids == {"cat": 0, "dog": 1, "zebra": 2, "ant": 3}


def test_a_body_over_the_limit_is_refused_before_any_launch(monkeypatch):
    monkeypatch.setattr(_fts, "MAX_BODY_BYTES", 8)
    with pytest.raises(ValueError, match="at most 8"):
        _fts.analyze_on_device(_fts.Analyzer(), ["short", "é" * 5], "cuda:0")


def test_fts_abi_refusals_before_any_cuda_call():
    from raglite_b200 import _lib

    lib = _lib.load()
    d = ctypes.c_void_p(16)
    assert lib.rl_fts_workspace_bytes(-1) == 0 and lib.rl_fts_workspace_bytes(1) > 0
    assert lib.rl_fts_workspace_bytes(1 << 20) >= 2 * (1 << 20) // 4096
    # rl_fts_mark(text, n_bytes, class_table, mark, workspace, workspace_bytes, stream)
    assert lib.rl_fts_mark(None, 0, None, None, None, 0, None) == 0
    assert lib.rl_fts_mark(d, -1, d, d, d, 1 << 20, None) == -1
    assert lib.rl_fts_mark(None, 10, d, d, d, 1 << 20, None) == -1
    assert lib.rl_fts_mark(d, 10, None, d, d, 1 << 20, None) == -1
    assert lib.rl_fts_mark(d, 10, d, None, d, 1 << 20, None) == -1
    assert lib.rl_fts_mark(d, 10, d, d, None, 1 << 20, None) == -1
    need = lib.rl_fts_workspace_bytes(1 << 20)
    assert lib.rl_fts_mark(d, 1 << 20, d, d, d, need - 1, None) == -3
    assert "rl_fts_mark" in lib.rl_last_error().decode()
    # rl_fts_stem(letters, word_off, n_words, stop, n_stop, hash_bits, keep, tail, hash, stream)
    assert lib.rl_fts_stem(None, None, 0, None, 0, 64, None, None, None, None) == 0
    assert lib.rl_fts_stem(d, d, -1, d, 1, 64, d, d, d, None) == -1
    assert lib.rl_fts_stem(d, d, 5, d, -1, 64, d, d, d, None) == -1
    for bits in (0, 65):
        assert lib.rl_fts_stem(d, d, 5, d, 1, bits, d, d, d, None) == -1
    for k in range(9):
        args = [d, d, 5, d, 1, 64, d, d, d, None]
        if k in (2, 4, 5):
            continue
        args[k] = None
        assert lib.rl_fts_stem(*args) == -1, k
    assert "rl_fts_stem" in lib.rl_last_error().decode()
    # rl_fts_verify(letters, word_off, keep, tail, word_a, word_b, n, differ, stream)
    # rl_fts_stem_bytes(letters, word_off, keep, tail, words, n, out_off, out, stream)
    for name, n_at in (("rl_fts_verify", 6), ("rl_fts_stem_bytes", 5)):
        fn = getattr(lib, name)
        args = [None] * 9
        args[n_at] = 0
        assert fn(*args) == 0
        args = [d] * 8 + [None]
        args[n_at] = -1
        assert fn(*args) == -1
        for k in range(8):
            args = [d] * 8 + [None]
            args[n_at] = 3
            if k != n_at:
                args[k] = None
                assert fn(*args) == -1, (name, k)
        assert name in lib.rl_last_error().decode()
    # rl_fts_term_keys(tok_stem, owner, n, stem_term, chunk_base, key, stream)
    assert lib.rl_fts_term_keys(None, None, 0, None, 0, None, None) == 0
    assert lib.rl_fts_term_keys(d, d, -1, d, 0, d, None) == -1
    assert lib.rl_fts_term_keys(d, d, 3, d, -1, d, None) == -1
    for k in (0, 1, 3, 5):
        args = [d, d, 3, d, 0, d, None]
        args[k] = None
        assert lib.rl_fts_term_keys(*args) == -1, k
    assert "rl_fts_term_keys" in lib.rl_last_error().decode()
