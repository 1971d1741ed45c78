"""NumPy restatements of the BM25 text-analysis kernels' outputs (csrc/fts.cu), as include/raglite_b200.h defines them,
built from the definitions and not from the kernels' structure.

* ``mark_oracle``: ``rl_fts_mark``.  Lead bytes are decoded by the kernel's documented rule, each code point is looked
  up in the class table, the dropped ones are removed, and a letter is kept when the backslash run right before it has
  even length (run lengths from a ``cumsum``, no automaton, no loop over the text).
* ``stem_hash``: ``rl_fts_stem``'s hash, FNV-1a 64 over the stem, ``^ len``, splitmix64's finaliser, cut to ``bits``.
* ``words_to_csr``: the ``(letters, word_off)`` pair the stem kernels take.
* ``stem_y_window``: porter as ``rl_fts_stem`` runs it with its window of y marks as a parameter, and
  ``y_window_words``, the words that probe that window."""

from __future__ import annotations

import numpy as np

CLASS_DROP = 0xFF
MAX_CODE_POINT = 0x10FFFF

FNV_OFFSET = 0xCBF29CE484222325
FNV_PRIME = 0x100000001B3
MIX1, MIX2 = 0xBF58476D1CE4E5B9, 0x94D049BB133111EB

# Bodies that reach every rule of the tokenizer: separators only, backslash runs, accented and non-Latin letters,
# marks inside words, stop words in any case, lone surrogates, NUL bytes, the Kelvin sign and dotted capital I.
HAZARDS = [
    "", " ", " \t\n.,;!?-", "123 456", "\\\\\\", "\n\n",
    "Café résumé naïve façade Ærøskøbing Straße İstanbul ﬁne K ÉTÉ",           # accented Latin, ligature, Kelvin sign
    "Ελληνικά κείμενα με τόνους", "漢字かな交じり文 한국어", "emoji 😀🎉 mixed😀in words",  # Greek, CJK, emoji
    "ét́e combining̈marks à́̂b ́start end́",         # marks inside words
    "THE The thé Thé AND aNd alls ALL c'mon don't it's",                          # stop words, any case, accented
    "lone \ud800 surrogate \udfff here x\ud800y", "nul\x00byte\x00 and \x00",
    "Kelvin İi ẞ",
]
for _n in range(1, 6):   # backslash runs before letters, newlines, marks and the end of a body
    HAZARDS += ["a" + "\\" * _n + "bc d", "x" + "\\" * _n + "\nyz", "p" + "\\" * _n + "́q r", "\\" * _n,
                "k" + "\\" * _n + "́\\́m n", "\\" * _n + "word"]


def decode_leads(b: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """``(lead byte positions, code points)`` of UTF-8 bytes ``b`` by the kernel's rule: a byte ``10xxxxxx`` is not a
    lead; a lead below 0x80 is one byte, below 0xE0 two, below 0xF0 three, else four (its low 3 bits); each following
    byte adds its low 6 bits whatever it is, and a byte past the end reads as 0."""
    b = np.asarray(b, dtype=np.uint8)
    pos = np.flatnonzero((b & 0xC0) != 0x80)
    lead = b[pos].astype(np.uint32)
    extra = np.where(lead < 0x80, 0, np.where(lead < 0xE0, 1, np.where(lead < 0xF0, 2, 3)))
    cp = np.where(extra == 0, lead, np.where(extra == 1, lead & 0x1F, np.where(extra == 2, lead & 0x0F, lead & 0x07)))
    padded = np.concatenate([b, np.zeros(3, np.uint8)]).astype(np.uint32)
    for k in (1, 2, 3):
        cp = np.where(extra >= k, (cp << 6) | (padded[pos + k] & 0x3F), cp)
    return pos, cp


def mark_oracle(text: bytes | np.ndarray, table: np.ndarray) -> np.ndarray:
    """``rl_fts_mark``'s output for ``text`` (uint8 [n]): the letter at the lead byte of each kept letter, upper case
    when the symbol before it (dropped code points removed) is not a kept letter; 0 at every other byte."""
    b = np.frombuffer(text, dtype=np.uint8) if isinstance(text, (bytes, bytearray)) else np.asarray(text, np.uint8)
    out = np.zeros(len(b), dtype=np.uint8)
    pos, cp = decode_leads(b)
    is_bs = cp == ord("\\")
    cls = np.where(cp <= MAX_CODE_POINT, table[np.minimum(cp, MAX_CODE_POINT)], 0)
    live = is_bs | (cls != CLASS_DROP)
    pos, cls, is_bs = pos[live], cls[live], is_bs[live]
    is_letter = ~is_bs & (cls >= 1) & (cls <= 26)
    # backslashes ending at each symbol: the distance to the last non-backslash at or before it
    idx = np.arange(len(pos))
    last_other = np.maximum.accumulate(np.where(is_bs, -1, idx)) if len(pos) else idx
    run_here = idx - last_other
    run_before = np.concatenate([[0], run_here[:-1]]) if len(pos) else run_here
    kept = is_letter & (run_before % 2 == 0)
    starts = kept & ~np.concatenate([[False], kept[:-1]]) if len(pos) else kept
    letter = (cls[kept] + ord("a") - 1).astype(np.uint8)
    out[pos[kept]] = np.where(starts[kept], letter - 32, letter)
    return out


def words_from_marks(mark: np.ndarray) -> list[str]:
    """The words of a mark array: its letters in order, a new word at every upper-case letter."""
    letters = bytes(mark[mark != 0])
    if not letters:
        return []
    starts = [i for i, c in enumerate(letters) if c < ord("a")] + [len(letters)]
    return [letters[a:z].decode().lower() for a, z in zip(starts[:-1], starts[1:])]


def _mix64(x: np.ndarray) -> np.ndarray:
    x = x ^ (x >> np.uint64(30))
    x = x * np.uint64(MIX1)
    x = x ^ (x >> np.uint64(27))
    x = x * np.uint64(MIX2)
    return x ^ (x >> np.uint64(31))


def _mask(bits: int) -> int:
    return (1 << 64) - 1 if bits == 64 else (1 << bits) - 1


def stem_hash(stems: list[bytes], bits: int) -> np.ndarray:
    """``rl_fts_stem``'s hash of each stem (int64): FNV-1a 64 over its bytes, ``^ len``, splitmix64's finaliser, the low
    ``bits`` bits.  One column of bytes at a time over all stems still that long; the few very long ones finish in
    Python integers."""
    n = len(stems)
    lens = np.fromiter(map(len, stems), dtype=np.int64, count=n)
    order = np.argsort(-lens, kind="stable")
    flat = np.frombuffer(b"".join(stems[i] for i in order), dtype=np.uint8)
    off = np.concatenate([[0], np.cumsum(lens[order])])[:-1]
    h = np.full(n, FNV_OFFSET, dtype=np.uint64)
    prime = np.uint64(FNV_PRIME)
    sorted_lens = lens[order]
    with np.errstate(over="ignore"):
        for col in range(min(int(sorted_lens[0]), 64) if n else 0):
            active = int(np.searchsorted(-sorted_lens, -col, side="left"))   # the rows longer than col
            c = flat[off[:active] + col].astype(np.uint64)
            h[:active] = (h[:active] ^ c) * prime
        for r in range(int(np.searchsorted(-sorted_lens, -64, side="left"))):   # the rows longer than 64
            x = int(h[r])
            for c in flat[off[r] + 64: off[r] + sorted_lens[r]].tobytes():
                x = ((x ^ c) * FNV_PRIME) & ((1 << 64) - 1)
            h[r] = x
        out = _mix64(h ^ sorted_lens.astype(np.uint64)) & np.uint64(_mask(bits))
    res = np.empty(n, dtype=np.int64)
    res[order] = out.view(np.int64)
    return res


def stem_hash_int(stem: bytes, bits: int) -> int:
    """The same hash of one stem in Python integers, as a signed int64."""
    m64 = (1 << 64) - 1
    h = FNV_OFFSET
    for c in stem:
        h = ((h ^ c) * FNV_PRIME) & m64
    x = h ^ len(stem)
    x ^= x >> 30
    x = (x * MIX1) & m64
    x ^= x >> 27
    x = (x * MIX2) & m64
    x ^= x >> 31
    x &= _mask(bits)
    return x - (1 << 64) if x >> 63 else x


def words_to_csr(words: list[str] | list[bytes], *, base: int = 0) -> tuple[np.ndarray, np.ndarray]:
    """``(letters uint8, word_off int64 [W + 1])`` of ``words``, with ``base`` filler letters ('q') before the first
    word, so ``word_off[0] == base``."""
    bs = [w.encode("ascii") if isinstance(w, str) else w for w in words]
    letters = np.frombuffer(b"q" * base + b"".join(bs), dtype=np.uint8).copy()
    off = np.empty(len(bs) + 1, dtype=np.int64)
    off[0] = base
    np.cumsum(np.fromiter(map(len, bs), dtype=np.int64, count=len(bs)), out=off[1:])
    off[1:] += base
    return letters, off


def stop_key(word: bytes) -> tuple[int, int]:
    """A word zero-padded to 16 bytes, read as two big-endian uint64 ``(hi, lo)``: the stop table's entry format."""
    k = word.ljust(16, b"\0")
    return int.from_bytes(k[:8], "big"), int.from_bytes(k[8:16], "big")


def is_stop(word: bytes, table: np.ndarray) -> bool:
    """The device's stop-list lookup: words over 16 letters are refused, the rest found by a lower-bound binary search
    over ``(hi, lo)``."""
    if len(word) > 16:
        return False
    key = stop_key(word)
    a, b = 0, len(table)
    while a < b:
        m = (a + b) >> 1
        if (int(table[m, 0]), int(table[m, 1])) < key:
            a = m + 1
        else:
            b = m
    return a < len(table) and (int(table[a, 0]), int(table[a, 1])) == key


# ---- the y-mark window of rl_fts_stem -------------------------------------------------------------------------------
_V = frozenset("aeiouy")


def _shortv(s: str) -> bool:
    return len(s) >= 3 and s[-1] not in "aeiouywxY" and s[-2] in _V and s[-3] not in _V


def stem_y_window(word: str, window: int) -> str:
    """Snowball porter as ``rl_fts_stem`` runs it when only the y marks of the last ``window`` letters are kept: R1, R2
    and the first vowel come from the fully marked word, and a letter farther from the end reads as ``y`` where it was
    marked.  At ``window = 32`` this is ``_fts.stem`` (for the words the tests use); a smaller window shows which words
    depend on a mark that far back."""
    from raglite_b200 import _fts

    n = len(word)
    chars = list(word)
    for i, ch in enumerate(chars):
        if ch == "y" and (i == 0 or chars[i - 1] in _V):
            chars[i] = "Y"

    def region_after(start: int) -> int:
        i = start
        while i < n and chars[i] not in _V:
            i += 1
        while i < n and chars[i] in _V:
            i += 1
        return i + 1 if i < n else n

    p1 = region_after(0)
    p2 = region_after(p1) if p1 < n else n
    fv = next((i for i, c in enumerate(chars) if c in _V), n)
    s = "".join(c if c != "Y" or n - 1 - i < window else "y" for i, c in enumerate(chars))
    if s.endswith("sses") or s.endswith("ies"):
        s = s[:-2]
    elif s.endswith("s") and not s.endswith("ss"):
        s = s[:-1]
    if s.endswith("eed"):
        if len(s) - 3 >= p1:
            s = s[:-1]
    else:
        suf = "ed" if s.endswith("ed") else "ing" if s.endswith("ing") else None
        if suf is not None and fv < len(s) - len(suf):
            s = s[: -len(suf)]
            if s.endswith(("at", "bl", "iz")):
                s += "e"
            elif len(s) >= 2 and s[-1] == s[-2] and s[-1] in "bdfgmnprt":
                s = s[:-1]
            elif len(s) == p1 and _shortv(s):
                s += "e"
    if s.endswith(("y", "Y")) and fv < len(s) - 1:
        s = s[:-1] + "i"
    for table in (_fts._STEP2, _fts._STEP3):
        suf = _fts._longest(s, table)
        if suf is not None and len(s) - len(suf) >= p1:
            s = s[: len(s) - len(suf)] + table[suf]
    suf = _fts._longest(s, _fts._STEP4)
    if suf is not None and len(s) - len(suf) >= p2:
        base = s[: len(s) - len(suf)]
        if suf != "ion" or base.endswith(("s", "t")):
            s = base
    if s.endswith("e") and (len(s) - 1 >= p2 or (len(s) - 1 >= p1 and not _shortv(s[:-1]))):
        s = s[:-1]
    if s.endswith("ll") and len(s) - 1 >= p2:
        s = s[:-1]
    return s.replace("Y", "y")


def y_deciding_words() -> list[str]:
    """Words whose stem is ``Y v c e`` with the marked ``Y`` as their first letter: the only shape in which a y mark
    decides a step (step 5a's short-syllable test keeps the ``e`` only because ``Y`` is not a vowel).  The ``e`` is
    exposed by step 3 (``ative``, ``ful``, ``ness`` deleted, after step 2's ``iveness`` / ``fulness``), after step 1a
    and 1b deletions, so the ``Y`` sits up to 16 letters from the end (``yoteativenessings``)."""
    tails = ["", "ative", "ful", "ness", "ativeness", "fulness", "iveness"]
    ends = ["", "s", "es", "ed", "ing", "eds", "ings", "sses"]
    return sorted({"y" + v + c + "e" + t + e for v in "aeiou" for c in "bcdflmnprstv" for t in tails for e in ends})


def y_window_words() -> list[str]:
    """``P + "y" + S``: ``S`` ends in a chain of porter suffixes (steps 4, 3, 2, then 1b / 1a) after filler, and the
    ``y`` sits 16 to 36 letters from the end, around the 32-letter window of y marks; contexts before the ``y`` make it
    marked or not.  Then every word of ``y_deciding_words``, whose stems depend on a mark up to 16 letters back."""
    from raglite_b200 import _fts

    rng = np.random.default_rng(31)
    ends = ["", "s", "ing", "ed", "ings", "es", "eds"]
    chains = sorted({a + b + c + e for a in ("", *_fts._STEP4) for b in ("", *_fts._STEP3) for c in ("", *_fts._STEP2)
                     for e in ends})
    chains = [chains[i] for i in rng.choice(len(chains), size=250, replace=False)]
    chains += ["ationalizations", "alizationally", "icationalism", "ementalities", "ousnesses", "ativenesses",
               "fulnesses", "ivenesses", "abilities", "izationing", "ate", "ize", "ive", "e", "ye", "yes"]
    out = set(y_deciding_words())
    for pre in ("", "a", "e", "o", "ba", "ab", "tr", "eu", "ay", "by"):
        for d in range(16, 37):
            for ch in chains:
                if len(ch) <= d:
                    for fill in ("tanor" * 8, "rst" * 12):
                        out.add(pre + "y" + fill[: d - len(ch)] + ch)
    return sorted(out)
