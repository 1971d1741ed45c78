"""The NumPy restatements of ``fts_oracle`` that the fts kernel tests compare against, held to ``_fts`` on the CPU: the
mark restatement to ``_fts.tokenize`` and to the automaton of ``test_fts_device_host``, the vectorized stem hash to
Python integers, and the stop table's ``(hi, lo)`` order to the order of the words."""

from __future__ import annotations

import numpy as np
import pytest

import fts_oracle as fo
from raglite_b200 import _fts
from test_fts_device_host import _automaton_words


@pytest.fixture(scope="module")
def table():
    return _fts.class_table()


def _marks_agree(text: str, table) -> None:
    raw = text.encode("utf-8", "surrogatepass")
    mark = fo.mark_oracle(raw, table)
    assert np.isin(np.flatnonzero(mark), fo.decode_leads(np.frombuffer(raw, np.uint8))[0]).all()
    words = fo.words_from_marks(mark)
    assert words == _fts.tokenize(text) == _automaton_words(text, table), repr(text)


def test_mark_oracle_matches_the_tokenizer_on_seeded_strings(table):
    alphabet = ["a", "b", "Z", "\\", "\n", " ", "\u0301", "é", "\u0130", "1", "ß", "\u212a"]
    rng = np.random.default_rng(7)
    for _ in range(40_000):
        _marks_agree("".join(alphabet[i] for i in rng.integers(0, len(alphabet), size=int(rng.integers(0, 24)))), table)
    for n in range(1, 12):
        for tail in ("b", "\nb", "\u0301b", "\\\u0301b"):
            _marks_agree("a" + "\\" * n + tail, table)


def test_mark_oracle_matches_the_tokenizer_on_hazards_and_lone_surrogates(table):
    for text in fo.HAZARDS:
        _marks_agree(text, table)
    for text in ("\ud800", "a\udbffb", "x\udc00\\\udfffy z", "\\\ud800q", "é\udfffé", "\U0001f600 pair"):
        _marks_agree(text, table)
    _marks_agree(" ".join(fo.HAZARDS), table)


def test_mark_oracle_writes_each_letter_at_its_lead_byte(table):
    raw = "\u00c9a \\\\b \\c K\u0301x \u1e31".encode()
    mark = fo.mark_oracle(raw, table)
    want = np.zeros(len(raw), np.uint8)
    for i, c in ((0, "E"), (2, "a"), (6, "B"), (11, "K"), (14, "x"), (16, "K")):   # '\c' swallows c; U+0301 drops
        want[i] = ord(c)
    assert mark.tolist() == want.tolist()


def test_mark_oracle_decodes_invalid_utf8_by_the_documented_rule(table):
    """Truncated sequences read missing bytes as 0, a stray continuation byte is no symbol, a lead above 0xF7 reads its
    low 3 bits, and an overlong encoding is decoded like any other (0xC1 0x9C is a backslash)."""
    pos, cp = fo.decode_leads(np.frombuffer(b"a\xc3\x80\xe2\x84\xaa\xf0\x9f\x98\x80\xc3", np.uint8))
    assert pos.tolist() == [0, 1, 3, 6, 10] and cp.tolist() == [0x61, 0xC0, 0x212A, 0x1F600, 0xC0]
    assert fo.decode_leads(np.frombuffer(b"\xe1\x80", np.uint8))[1].tolist() == [0x1000]
    assert fo.decode_leads(np.frombuffer(b"\xff\xbf\xbf\xbf", np.uint8))[1].tolist() == [0x1FFFFF]   # > 0x10FFFF
    assert fo.decode_leads(np.frombuffer(b"\x80\xbfa", np.uint8))[0].tolist() == [2]
    assert fo.mark_oracle(b"\xc1\x9cab", table).tolist() == [0, 0, 0, ord("B")]          # overlong backslash
    assert fo.mark_oracle(b"ab\xc3", table).tolist() == [ord("A"), ord("b"), ord("a")]    # 0xC3 + 0 = U+00C0 = 'a'
    assert fo.mark_oracle(b"a\xff\xbf\xbf\xbfb", table).tolist() == [ord("A"), 0, 0, 0, 0, ord("B")]
    assert fo.mark_oracle(b"a\xe2\x84", table).tolist() == [ord("A"), 0, 0]              # U+2100: a separator
    assert fo.mark_oracle(b"", table).tolist() == []


@pytest.mark.parametrize("bits", [1, 7, 31, 32, 63, 64])
def test_stem_hash_matches_python_integers(bits):
    rng = np.random.default_rng(bits)
    stems = [bytes(rng.integers(ord("a"), ord("z") + 1, size=int(n)).astype(np.uint8))
             for n in rng.integers(0, 40, size=300)]
    stems += [b"", b"a", b"hope", b"z" * 64, b"y" * 65, b"ab" * 300, b"q" * 5000]
    got = fo.stem_hash(stems, bits)
    want = [fo.stem_hash_int(s, bits) for s in stems]
    assert got.tolist() == want
    assert fo.stem_hash([], bits).shape == (0,)
    if bits >= 31:   # a hash that collapsed to a few values would still give right answers: keep it spread
        assert len(set(want)) == len(set(stems))


def test_stop_table_order_is_the_order_of_the_padded_words():
    """The device's binary search compares ``(hi, lo)`` pairs; that order must be the byte order of the words for every
    stop word and every word one letter longer or shorter, and the search must find exactly the stop words."""
    table = _fts.stop_table()
    stops = [(int(h).to_bytes(8, "big") + int(lo).to_bytes(8, "big")).rstrip(b"\0") for h, lo in table]
    cands = set(stops)
    for w in stops:
        cands.add(w[:-1])
        cands.update(w + bytes([c]) for c in range(ord("a"), ord("z") + 1))
        cands.update(w[:i] + bytes([c]) + w[i + 1:] for i in range(len(w)) for c in (ord("a"), ord("z")))
    cands.discard(b"")
    cands = sorted(cands)
    keys = [fo.stop_key(w) for w in cands]
    assert keys == sorted(keys) and len(set(keys)) == len(keys)
    stop_set = set(stops)
    assert [fo.is_stop(w, table) for w in cands] == [w in stop_set for w in cands]
    assert not fo.is_stop(b"a" * 17, table) and fo.is_stop(b"unfortunately", table)


def test_words_to_csr_offsets():
    letters, off = fo.words_to_csr(["ab", "", "cde"], base=5)
    assert bytes(letters) == b"qqqqqabcde" and off.tolist() == [5, 7, 7, 10]
    letters, off = fo.words_to_csr([])
    assert letters.size == 0 and off.tolist() == [0]


def test_y_window_words_reach_the_deepest_deciding_mark():
    """The y-mark window of ``rl_fts_stem`` keeps the marks of the last 32 letters.  A mark decides a stem only in the
    shape ``Y v c e`` with the ``Y`` first (step 5a's short-syllable test), at most 16 letters from the end.  The words
    the GPU test stems reach that depth: with the window cut to 16 letters their stems change, with 17 or more they
    do not, and at 32 the windowed port is ``_fts.stem``."""
    words = fo.y_window_words()
    assert [fo.stem_y_window(w, 32) for w in words] == [_fts.stem(w) for w in words]
    cut = [w for w in words if fo.stem_y_window(w, 16) != _fts.stem(w)]
    assert "yoteativenessings" in cut and {len(w) for w in cut} == {17}
    assert fo.stem_y_window("yoteativenessings", 16) == "yot" and _fts.stem("yoteativenessings") == "yote"
    for window in (17, 24):
        assert all(fo.stem_y_window(w, window) == _fts.stem(w) for w in words), window
