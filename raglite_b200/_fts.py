"""Text analysis of DuckDB's full-text search, as the reference's ``keyword_search`` runs it (``_search.py:203-225``).

The reference indexes ``chunk.body`` with ``PRAGMA create_fts_index('chunk', 'id', 'body')`` (``_database.py:618``) and
ranks with ``fts_main_chunk.match_bm25(id, query)``, both at their defaults.  What those defaults do is restated here
from memory of DuckDB's ``fts`` extension, which is not part of the reference's source tree; it is recalled, not
verified (DESIGN.md section 5):

* tokenizer: ``lower(strip_accents(text))``, then ``regexp_replace(..., '(\\\\.|[^a-z])+', ' ', 'g')`` -- a backslash
  together with the character after it, and every character outside ``a-z``, is a separator -- then a split on
  whitespace, empty strings dropped;
* document side: tokens in the ``english`` stop list (``fts_stopwords_english.txt``) are dropped, the rest stemmed with
  Snowball's ``porter`` stemmer;
* query side: ``DISTINCT stem(unnest(tokenize(query)), 'porter')`` -- the same tokenizer and stemmer, no stop list.

``Analyzer`` is the batch form the index build uses: it maps chunk bodies to a ``(term id, chunk)`` token stream and
keeps the ``stem -> term id`` dictionary (ids in order of first appearance).
"""

from __future__ import annotations

import functools
import re
import unicodedata
from collections.abc import Iterable, Sequence
from itertools import chain
from pathlib import Path

import numpy as np

_STOP_FILE = Path(__file__).resolve().parent / "fts_stopwords_english.txt"
STOPWORD_ENTRIES: tuple[str, ...] = tuple(
    w for w in (line.strip() for line in _STOP_FILE.read_text(encoding="utf-8").splitlines()) if w and not w.startswith("#"))
STOPWORDS: frozenset[str] = frozenset(STOPWORD_ENTRIES)

_IGNORE = re.compile(r"(\\.|[^a-z])+")


def strip_accents(text: str) -> str:
    """NFD, then every combining mark (Unicode category Mn) dropped."""
    if text.isascii():
        return text
    return "".join(ch for ch in unicodedata.normalize("NFD", text) if unicodedata.category(ch) != "Mn")


def tokenize(text: str) -> list[str]:
    """The ``fts`` tokenizer at ``create_fts_index``'s defaults (``strip_accents=1, lower=1``)."""
    return _IGNORE.sub(" ", strip_accents(text).lower()).split()


# ---- Snowball 'porter' (the Porter algorithm as published in Snowball's porter.sbl) ----------------------------
_V = frozenset("aeiouy")
_NON_V_WXY = frozenset("aeiouywxY")
_STEP2 = {"tional": "tion", "enci": "ence", "anci": "ance", "abli": "able", "entli": "ent", "eli": "e", "izer": "ize",
          "ization": "ize", "ational": "ate", "ation": "ate", "ator": "ate", "alli": "al", "alism": "al", "aliti": "al",
          "fulness": "ful", "ousli": "ous", "ousness": "ous", "iveness": "ive", "iviti": "ive", "biliti": "ble"}
_STEP3 = {"alize": "al", "icate": "ic", "iciti": "ic", "ical": "ic", "ative": "", "ful": "", "ness": ""}
_STEP4 = ("al", "ance", "ence", "er", "ic", "able", "ible", "ant", "ement", "ment", "ent", "ou", "ism", "ate", "iti", "ous",
          "ive", "ize", "ion")


def _longest(s: str, suffixes: Iterable[str]) -> str | None:
    best = None
    for suf in suffixes:
        if s.endswith(suf) and (best is None or len(suf) > len(best)):
            best = suf
    return best


def _shortv(s: str) -> bool:
    """``non-v_WXY v non-v`` at the end of ``s``."""
    return len(s) >= 3 and s[-1] not in _NON_V_WXY and s[-2] in _V and s[-3] not in _V


@functools.lru_cache(maxsize=1 << 20)
def stem(word: str) -> str:
    """``stem(word, 'porter')``: Snowball's ``porter`` stemmer (lower-case input)."""
    chars = list(word)
    y_found = False
    for i, ch in enumerate(chars):   # 'y' at the start or after a vowel is a consonant: mark it 'Y'
        if ch == "y" and (i == 0 or chars[i - 1] in _V):
            chars[i], y_found = "Y", True
    n = len(chars)

    def region_after(start: int) -> int:   # gopast v  gopast non-v
        i = start
        while i < n and chars[i] not in _V:
            i += 1
        while i < n and chars[i] in _V:
            i += 1
        return i + 1 if i < n else n

    p1 = region_after(0)
    p2 = region_after(p1) if p1 < n else n
    s = "".join(chars)
    # Step 1a
    if s.endswith("sses") or s.endswith("ies"):
        s = s[:-2]
    elif s.endswith("s") and not s.endswith("ss"):
        s = s[:-1]
    # Step 1b
    if s.endswith("eed"):
        if len(s) - 3 >= p1:
            s = s[:-1]
    else:
        suf = "ed" if s.endswith("ed") else "ing" if s.endswith("ing") else None
        if suf is not None and any(c in _V for c in s[: -len(suf)]):
            s = s[: -len(suf)]
            if s.endswith(("at", "bl", "iz")):
                s += "e"
            elif len(s) >= 2 and s[-1] == s[-2] and s[-1] in "bdfgmnprt":
                s = s[:-1]
            elif len(s) == p1 and _shortv(s):
                s += "e"
    # Step 1c
    if s.endswith(("y", "Y")) and any(c in _V for c in s[:-1]):
        s = s[:-1] + "i"
    # Steps 2 and 3: the longest listed suffix, replaced when it lies in R1
    for table in (_STEP2, _STEP3):
        suf = _longest(s, table)
        if suf is not None and len(s) - len(suf) >= p1:
            s = s[: len(s) - len(suf)] + table[suf]
    # Step 4: the longest listed suffix, deleted when it lies in R2 ('ion' only after 's' or 't')
    suf = _longest(s, _STEP4)
    if suf is not None and len(s) - len(suf) >= p2:
        base = s[: len(s) - len(suf)]
        if suf != "ion" or base.endswith(("s", "t")):
            s = base
    # Step 5a / 5b
    if s.endswith("e") and (len(s) - 1 >= p2 or (len(s) - 1 >= p1 and not _shortv(s[:-1]))):
        s = s[:-1]
    if s.endswith("ll") and len(s) - 1 >= p2:
        s = s[:-1]
    return s.replace("Y", "y") if y_found else s


def document_terms(body: str) -> list[str]:
    """The stemmed terms of one document, in order, stop words dropped (what ``create_fts_index`` stores)."""
    return [stem(w) for w in tokenize(body) if w not in STOPWORDS]


def query_terms(query: str) -> list[str]:
    """``DISTINCT stem(unnest(tokenize(query)), 'porter')`` (no stop list), in order of first appearance."""
    return list(dict.fromkeys(stem(w) for w in tokenize(query)))


# ---- batch analysis for the index build ---------------------------------------------------------------------
_ASCII_MAP = bytes((c | 0x20) if chr(c).isalpha() and c < 128 else 0x20 for c in range(256))


class Analyzer:
    """Chunk bodies -> ``(term id, chunk)`` token stream, with the ``stem -> term id`` dictionary it grows.

    Most bodies are ASCII without backslashes; for those the tokenizer is one ``bytes.translate`` (upper case folded,
    everything outside ``a-z`` mapped to a space) and a split, and each distinct word is stop-listed and stemmed once.
    Anything else goes through ``tokenize``."""

    def __init__(self) -> None:
        self.term_ids: dict[str, int] = {}
        self._word: dict[bytes, int] = {}   # document word -> term id, -1 for a stop word

    def _word_id(self, w: bytes) -> int:
        s = w.decode("ascii")
        if s in STOPWORDS:
            tid = -1
        else:
            t = stem(s)
            tid = self.term_ids.get(t)
            if tid is None:
                tid = self.term_ids[t] = len(self.term_ids)
        self._word[w] = tid
        return tid

    @staticmethod
    def _words(body: str) -> list[bytes]:
        if body.isascii() and "\\" not in body:
            return body.encode("ascii").translate(_ASCII_MAP).split()
        return [w.encode("ascii") for w in tokenize(body)]

    def analyze(self, bodies: Sequence[str], *, batch: int = 8192) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
        """``(term int32 [T], chunk int32 [T], doc_len int32 [len(bodies)])``: the kept tokens of every body in order
        (``chunk`` counts from 0 within ``bodies``) and the number of kept tokens per body."""
        terms, owners, lens = [], [], np.zeros(len(bodies), dtype=np.int32)
        word, word_id = self._word, self._word_id
        for c0 in range(0, len(bodies), batch):
            lists = [self._words(b) for b in bodies[c0:c0 + batch]]
            counts = np.fromiter(map(len, lists), dtype=np.int64, count=len(lists))
            flat = list(chain.from_iterable(lists))
            for w in dict.fromkeys(flat):   # new words in order of first appearance: term ids do not depend on hashing
                if w not in word:
                    word_id(w)
            ids = np.fromiter(map(word.__getitem__, flat), dtype=np.int32, count=len(flat))
            own = np.repeat(np.arange(c0, c0 + len(lists), dtype=np.int32), counts)
            keep = ids >= 0
            terms.append(ids[keep])
            owners.append(own[keep])
            lens[c0:c0 + len(lists)] = np.bincount(own[keep] - c0, minlength=len(lists))
        if not terms:
            return np.zeros(0, np.int32), np.zeros(0, np.int32), lens
        return np.concatenate(terms), np.concatenate(owners), lens

    def query_ids(self, query: str) -> np.ndarray:
        """Distinct term ids of a query's stems that are in the dictionary, ascending (unknown stems are ignored)."""
        ids = {self.term_ids[t] for t in query_terms(query) if t in self.term_ids}
        return np.fromiter(sorted(ids), dtype=np.int32, count=len(ids))

    def query_plan(self, queries: Sequence[str]) -> tuple[np.ndarray, list[str], np.ndarray]:
        """The entries of a sharded search: each query's distinct stems sorted by code point (stems are ASCII, so that
        order is the same on every shard whatever its dictionary).  Returns ``(q_off int32 [B + 1], stems [J], ids int32
        [J])``: query ``b`` is entries ``q_off[b] .. q_off[b + 1]``, ``ids`` the local term ids, ``-1`` for a stem this
        dictionary does not hold.  Unlike ``query_ids``, unknown stems stay: another shard may hold them."""
        per = [sorted(set(query_terms(q))) for q in queries]
        q_off = np.zeros(len(per) + 1, dtype=np.int32)
        np.cumsum([len(s) for s in per], out=q_off[1:])
        stems = list(chain.from_iterable(per))
        get = self.term_ids.get
        ids = np.fromiter((get(t, -1) for t in stems), dtype=np.int32, count=len(stems))
        return q_off, stems, ids
