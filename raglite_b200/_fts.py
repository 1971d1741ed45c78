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

``Analyzer`` is the batch form of the host: it maps chunk bodies to a ``(term id, chunk)`` token stream and keeps the
``stem -> term id`` dictionary (ids in order of first appearance).  ``analyze_on_device`` is what the index build runs:
the same analysis in CUDA (csrc/fts.cu), bit for bit, with the dictionary kept by the same ``Analyzer``.
"""

from __future__ import annotations

import functools
import re
import threading
import time
import unicodedata
import warnings
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

    def add_stems(self, stems: Sequence[str]) -> np.ndarray:
        """Term ids of ``stems`` (int32), a stem not in the dictionary getting the next id: in the order given, which is
        the order of first appearance when ``stems`` lists a group's distinct stems that way."""
        ids = self.term_ids
        return np.fromiter((ids.setdefault(t, len(ids)) for t in stems), dtype=np.int32, count=len(stems))

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


# ---- analysis on the device (csrc/fts.cu) --------------------------------------------------------------------------
GROUP_BYTES = 128 << 20  # UTF-8 bytes of text analysed at a time (a longer body is a group of its own)
HASH_BITS = 64           # stem hash width; hash collisions are resolved exactly whatever it is
MAX_BODY_BYTES = (1 << 31) - 1
N_CODE_POINTS = 0x110000
CLASS_DROP = 0xFF


@functools.lru_cache(maxsize=1)
def class_table() -> np.ndarray:
    """uint8 [0x110000]: what ``lower(strip_accents(ch))`` makes of each code point -- 1..26 the letter a..z,
    ``CLASS_DROP`` when it vanishes (combining marks, and what decomposes into marks only), 0 for a separator."""
    # Each code point's strip_accents(ch).lower(), all at once: NFD over the code points joined by NUL (a starter, so no
    # mark is reordered across it), the combining marks deleted, lower(), then split at the NULs again.
    mn = dict.fromkeys(cp for cp in range(N_CODE_POINTS) if unicodedata.category(chr(cp)) == "Mn")
    parts = unicodedata.normalize("NFD", "\0".join(map(chr, range(1, N_CODE_POINTS)))).translate(mn).lower().split("\0")
    assert len(parts) == N_CODE_POINTS - 1
    lens = np.fromiter(map(len, parts), dtype=np.int64, count=len(parts))
    chars = np.frombuffer("".join(parts).encode("utf-32-le", "surrogatepass"), dtype=np.uint32)
    first = chars[np.minimum(np.cumsum(lens) - lens, len(chars) - 1)]
    letter = (lens == 1) & (first >= ord("a")) & (first <= ord("z"))
    table = np.zeros(N_CODE_POINTS, dtype=np.uint8)   # code point 0 (NUL) is a separator
    table[1:][lens == 0] = CLASS_DROP
    table[1:][letter] = (first[letter] - ord("a") + 1).astype(np.uint8)
    return table


def stop_table() -> np.ndarray:
    """uint64 [n, 2]: the stop words made of a-z only (no other entry can equal a token), each zero-padded to 16 bytes
    and read as two big-endian words, sorted ascending -- the byte order of the padded strings."""
    keys = sorted({w.encode("ascii").ljust(16, b"\0") for w in STOPWORDS if re.fullmatch("[a-z]{1,16}", w)})
    return np.array([(int.from_bytes(k[:8], "big"), int.from_bytes(k[8:], "big")) for k in keys], dtype=np.uint64)


_tables_lock = threading.Lock()
_tables: dict = {}


def _device_tables(device):
    """The class and stop tables on ``device``, uploaded once per process and device."""
    import torch

    with _tables_lock:
        t = _tables.get(device)
        if t is None:
            with torch.cuda.device(device):
                t = _tables[device] = (torch.from_numpy(class_table()).to(device),
                                       torch.from_numpy(stop_table().view(np.int64)).to(device))
                torch.cuda.current_stream().synchronize()
        return t


def _groups(sizes: Sequence[int], budget: int) -> list[tuple[int, int]]:
    """Consecutive bodies whose bytes (and one separator each) fit in ``budget``; a larger body is a group alone."""
    out, a, used = [], 0, 0
    for i, n in enumerate(sizes):
        if i > a and used + n + 1 > budget:
            out.append((a, i))
            a, used = i, 0
        used += n + 1
    if a < len(sizes):
        out.append((a, len(sizes)))
    return out


def analyze_on_device(analyzer: Analyzer, bodies: Sequence[str], device, *, chunk_base: int = 0,
                      hash_bits: int = HASH_BITS, seconds: dict | None = None):
    """``analyzer.analyze(bodies)`` on ``device``, as postings keys: returns ``(key int64 [T], doc_len int32
    [len(bodies)])`` on the device, ``key = term << 32 | (chunk_base + chunk)`` for every kept token in order, with
    ``analyzer.term_ids`` grown exactly as ``analyze`` grows it.  Per group of at most ``GROUP_BYTES`` bytes: one upload of
    the UTF-8 text, the words (``rl_fts_mark``), their stems (``rl_fts_stem``), the distinct stems in order of first
    appearance (hashes grouped with ``torch.unique``, every token checked byte for byte against its group's first token
    by ``rl_fts_verify``: the tokens of a colliding stem are grouped again among themselves), one download of those
    stems, their ids from the dictionary, one upload of the ids and the keys (``rl_fts_term_keys``).  ``seconds``, when
    given, accumulates ``encode`` (host UTF-8 encoding), ``device`` and ``dictionary`` (download, lookup, upload).
    Raises ``ValueError`` for a body over 2^31 - 1 bytes, before any launch."""
    import torch

    from . import _lib

    t0 = time.perf_counter()
    # surrogatepass: a lone surrogate is a separator on the device, as on the host
    sizes = [len(b) if b.isascii() else len(b.encode("utf-8", "surrogatepass")) for b in bodies]
    if sizes and max(sizes) > MAX_BODY_BYTES:
        raise ValueError(f"a body of {max(sizes)} UTF-8 bytes: at most {MAX_BODY_BYTES} can be analysed")
    t_enc, t_dict = time.perf_counter() - t0, 0.0
    lib = _lib.load()
    cls_d, stop_d = _device_tables(device)
    n_stop = int(stop_d.numel()) // 2
    ptr = lambda t: int(t.data_ptr())   # noqa: E731
    keys, lens = [], []
    with torch.cuda.device(device):
        stream = int(torch.cuda.current_stream().cuda_stream)
        i64 = dict(dtype=torch.int64, device=device)
        for a, b in _groups(sizes, GROUP_BYTES):
            t1 = time.perf_counter()
            text = " ".join(bodies[a:b]).encode("utf-8", "surrogatepass")   # a space between bodies: no word spans two
            starts = np.zeros(b - a, dtype=np.int64)
            np.cumsum(np.asarray(sizes[a:b - 1], dtype=np.int64) + 1, out=starts[1:])
            t_enc += time.perf_counter() - t1
            N = len(text)
            with warnings.catch_warnings():   # a read-only buffer: torch only reads it, for the copy
                warnings.simplefilter("ignore", UserWarning)
                text_d = torch.frombuffer(text, dtype=torch.uint8) if N else torch.zeros(0, dtype=torch.uint8)
            text_d = text_d.to(device)
            mark = torch.empty(N, dtype=torch.uint8, device=device)
            ws = torch.empty(max(int(lib.rl_fts_workspace_bytes(N)), 1), dtype=torch.uint8, device=device)
            _lib.check(lib.rl_fts_mark(ptr(text_d), N, ptr(cls_d), ptr(mark), ptr(ws), ws.numel(), stream), "rl_fts_mark")
            del text_d, ws
            is_letter = mark != 0
            letters = mark[is_letter] | 0x20
            wpos = torch.nonzero(is_letter & (mark < ord("a"))).squeeze(1)
            W = int(wpos.numel())
            word_off = torch.empty(W + 1, **i64)
            word_off[:W] = torch.cumsum(is_letter, 0, dtype=torch.int32)[wpos] - 1
            word_off[W] = letters.numel()
            del mark, is_letter
            owner = torch.searchsorted(torch.from_numpy(starts).to(device), wpos, right=True) - 1
            keep = torch.empty(W, dtype=torch.int32, device=device)
            tail, hsh = torch.empty(W, **i64), torch.empty(W, **i64)
            _lib.check(lib.rl_fts_stem(ptr(letters), ptr(word_off), W, ptr(stop_d), n_stop, int(hash_bits), ptr(keep),
                                       ptr(tail), ptr(hsh), stream), "rl_fts_stem")
            kept = torch.nonzero(keep >= 0).squeeze(1)   # the word of each kept token
            tok_owner = owner[kept]
            lens.append(torch.bincount(tok_owner, minlength=b - a).to(torch.int32))
            rep = _first_of_each_stem(lib, hsh[kept], kept, (letters, word_off, keep, tail), stream)
            first, tok_stem = torch.unique(rep, return_inverse=True)   # ascending token index: first appearance
            stem_word = kept[first]
            n_tail = (tail[stem_word].view(torch.uint8).view(-1, 8) != 0).sum(1)
            stem_off = torch.zeros(len(first) + 1, **i64)
            torch.cumsum(keep[stem_word].to(torch.int64) + n_tail, 0, out=stem_off[1:])
            raw = torch.empty(max(int(stem_off[-1]), 1), dtype=torch.uint8, device=device)
            _lib.check(lib.rl_fts_stem_bytes(ptr(letters), ptr(word_off), ptr(keep), ptr(tail), ptr(stem_word),
                                             len(first), ptr(stem_off), ptr(raw), stream), "rl_fts_stem_bytes")
            t2 = time.perf_counter()
            raw_h, off_h = raw.cpu().numpy().tobytes(), stem_off.cpu().tolist()
            stems = [raw_h[x:y].decode("ascii") for x, y in zip(off_h[:-1], off_h[1:])]
            stem_term = torch.from_numpy(analyzer.add_stems(stems)).to(device)
            t_dict += time.perf_counter() - t2
            key = torch.empty(len(kept), **i64)
            _lib.check(lib.rl_fts_term_keys(ptr(tok_stem), ptr(tok_owner), len(kept), ptr(stem_term), chunk_base + a,
                                            ptr(key), stream), "rl_fts_term_keys")
            keys.append(key)
        key = torch.cat(keys) if keys else torch.zeros(0, **i64)
        doc_len = torch.cat(lens) if lens else torch.zeros(0, dtype=torch.int32, device=device)
        torch.cuda.current_stream().synchronize()
    if seconds is not None:
        total = time.perf_counter() - t0
        seconds["encode"] = seconds.get("encode", 0.0) + t_enc
        seconds["dictionary"] = seconds.get("dictionary", 0.0) + t_dict
        seconds["device"] = seconds.get("device", 0.0) + total - t_enc - t_dict
    return key, doc_len


def _first_of_each_stem(lib, hsh, kept, stems, stream: int):
    """For each kept token, the index of the first kept token with the same stem (int64 [T]).  Tokens are grouped by
    hash and each is compared byte for byte with its group's first token; the tokens that differ (a hash collision)
    are grouped again among themselves, until none is left.  Every round settles at least the first stem of each group,
    and all tokens of one stem move together, so the representative is always the stem's first token."""
    import torch

    from . import _lib

    letters, word_off, keep, tail = stems
    T = int(hsh.numel())
    rep = torch.empty(T, dtype=torch.int64, device=hsh.device)
    idx = torch.arange(T, dtype=torch.int64, device=hsh.device)
    while idx.numel():
        uniq, inv = torch.unique(hsh[idx], return_inverse=True)
        first = torch.full((len(uniq),), len(idx), dtype=torch.int64, device=hsh.device)
        first.scatter_reduce_(0, inv, torch.arange(len(idx), dtype=torch.int64, device=hsh.device), "amin")
        cand = idx[first[inv]]
        wa, wb = kept[idx], kept[cand]
        differ = torch.empty(len(idx), dtype=torch.uint8, device=hsh.device)
        _lib.check(lib.rl_fts_verify(int(letters.data_ptr()), int(word_off.data_ptr()), int(keep.data_ptr()),
                                     int(tail.data_ptr()), int(wa.data_ptr()), int(wb.data_ptr()), len(idx),
                                     int(differ.data_ptr()), stream), "rl_fts_verify")
        same = differ == 0
        rep[idx[same]] = cand[same]
        idx = idx[~same]
    return rep
