"""The BM25 text-analysis kernels (csrc/fts.cu) at the C-ABI, against the restatements of ``fts_oracle`` and against
``_fts`` itself, at the places the end-to-end test cannot aim at:

* ``rl_fts_mark`` byte for byte against ``fts_oracle.mark_oracle``: lengths on both sides of every scan boundary
  (16-byte threads, 512-byte warps, 4096-byte tiles, 1 MiB chunks of ``fts_tile_carry``), text and mark pointers at
  every offset mod 16 with canaries around the mark and a workspace of exactly the documented size filled with 0xFF,
  crafted cases straddling each boundary at every split point, 3 MiB backslash runs, invalid UTF-8 at the end of the
  buffer, and ``n_bytes = 2^31 - 1`` built and checked on the device.
* ``rl_fts_stem``: the ``(keep, tail)`` representation and the hash at 1 to 64 bits against ``_fts.stem`` and
  ``fts_oracle.stem_hash``; stop words and their neighbours; the y-mark window; words of 10^6 letters; offsets; and one
  launch of 9 000 000 words, past the 8 388 608 one pass of the grid covers.
* ``rl_fts_verify``, ``rl_fts_stem_bytes`` and ``rl_fts_term_keys`` on crafted splits and on launches above the
  16 777 216 items one pass of their grids covers.
* ``analyze_on_device`` at the default ``GROUP_BYTES`` over about 300 MiB of bodies, against the result computed from
  each vocabulary token analysed alone."""

from __future__ import annotations

import numpy as np
import pytest
import torch

import fts_oracle as fo
from raglite_b200 import _fts

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
CANARY = 0xA5
GUARD = 64                    # canary bytes on each side of a mark buffer
MIB = 1 << 20
STEM_WRAP = 65536 * 128       # words one pass of fts_stem's grid covers
ITEM_WRAP = 65536 * 256       # items one pass of fts_verify's, fts_stem_bytes' and fts_term_keys' grids covers
STOP_AZ = sorted(w for w in _fts.STOPWORDS if w.isascii() and w.isalpha() and w.islower())


def _lib():
    from raglite_b200 import _lib as L

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return L, L.load()


_STREAM: list = []


def _stream() -> torch.cuda.Stream:
    if not _STREAM:
        _STREAM.append(torch.cuda.Stream(DEV))
    return _STREAM[0]


def _check(rc: int, name: str) -> None:
    L, _ = _lib()
    L.check(rc, name)


def _need(gib: float) -> None:
    free, _ = torch.cuda.mem_get_info(DEV)
    if free < gib * (1 << 30):
        pytest.skip(f"needs {gib} GiB of free device memory, {free / (1 << 30):.1f} GiB free")


# ---- rl_fts_mark ----------------------------------------------------------------------------------------------------
_SYMBOLS = ["a", "b", "e", "o", "t", "s", "y", "Q", "Z", "é", "\u0130", "\u212a", "\u1e01", "\U0001f600", "\u0301",
            "\\", " ", "\n", "0", "7", "\ud800", "\udfff", "\U000101fd"]
_WEIGHTS = [8, 6, 6, 5, 5, 5, 3, 2, 2, 2, 1, 1, 1, 1, 2, 6, 6, 2, 1, 1, 1, 1, 1]


def random_text(n: int, seed: int, weights=_WEIGHTS) -> np.ndarray:
    """``n`` bytes of seeded UTF-8 (``surrogatepass``) over a mixed alphabet: ASCII letters, é, dotted capital I, the
    Kelvin sign, a 3-byte letter, an emoji, U+0301, backslashes, spaces, newlines, digits, lone surrogates and a 4-byte
    dropped code point.  The cut at ``n`` may split the last code point."""
    enc = [s.encode("utf-8", "surrogatepass") for s in _SYMBOLS]
    tab = np.zeros((len(enc), 4), np.uint8)
    for i, e in enumerate(enc):
        tab[i, :len(e)] = np.frombuffer(e, np.uint8)
    lens = np.array([len(e) for e in enc])
    p = np.asarray(weights, np.float64) / np.sum(weights)
    rng = np.random.default_rng(seed)
    idx = rng.choice(len(enc), size=int(n / (p @ lens)) + 64, p=p)
    out = tab[idx][np.arange(4)[None, :] < lens[idx][:, None]]
    while len(out) < n:
        out = np.concatenate([out, out])
    return out[:n].copy()


def _run_mark(text_d: torch.Tensor, n: int, *, mark_off: int = 0) -> torch.Tensor:
    """``rl_fts_mark`` on the first ``n`` bytes at ``text_d``, the mark written at ``mark_off`` mod 16 inside a buffer
    guarded by canaries, the workspace exactly ``rl_fts_workspace_bytes(n)`` bytes of 0xFF.  Returns the mark."""
    _, lib = _lib()
    cls_d, _ = _fts._device_tables(DEV)
    st = _stream()
    with torch.cuda.stream(st):
        need = int(lib.rl_fts_workspace_bytes(n))
        ws = torch.full((need,), 0xFF, dtype=torch.uint8, device=DEV)
        buf = torch.full((GUARD + mark_off + n + GUARD,), CANARY, dtype=torch.uint8, device=DEV)
        mark = buf[GUARD + mark_off: GUARD + mark_off + n]
        assert mark.data_ptr() % 16 == mark_off % 16
        _check(lib.rl_fts_mark(text_d.data_ptr(), n, cls_d.data_ptr(), mark.data_ptr(), ws.data_ptr(), need,
                               st.cuda_stream), "rl_fts_mark")
        st.synchronize()
        assert bool((buf[:GUARD + mark_off] == CANARY).all()) and bool((buf[GUARD + mark_off + n:] == CANARY).all())
    return mark


def _mark(raw: np.ndarray, *, text_off: int = 0, mark_off: int = 0) -> np.ndarray:
    n = len(raw)
    tbuf = torch.empty(text_off + n, dtype=torch.uint8, device=DEV)
    text = tbuf[text_off:]
    text.copy_(torch.from_numpy(np.ascontiguousarray(raw)))
    assert text.data_ptr() % 16 == text_off % 16
    torch.cuda.current_stream().synchronize()
    return _run_mark(text, n, mark_off=mark_off).cpu().numpy()


def _assert_marks(raw: np.ndarray, **kw) -> np.ndarray:
    got = _mark(raw, **kw)
    want = fo.mark_oracle(raw, _fts.class_table())
    bad = np.flatnonzero(got != want)
    assert not len(bad), (len(bad), bad[:8].tolist(), got[bad[:8]].tolist(), want[bad[:8]].tolist())
    return got


@pytest.mark.parametrize("n", [1, 15, 16, 17, 511, 512, 513, 4095, 4096, 4097, MIB - 1, MIB, MIB + 1, 2 * MIB + 17,
                               64 * MIB])
def test_mark_lengths(n):
    mark = _assert_marks(random_text(n, seed=n))
    if n >= 4096:
        assert (mark >= ord("a")).any() and ((mark > 0) & (mark < ord("a"))).any()


@pytest.mark.parametrize("off", range(16))
def test_mark_unaligned_buffers(off):
    raw = random_text(3 * 4096 + 77 + 31 * off, seed=100 + off)
    _assert_marks(raw, text_off=off, mark_off=(7 * off + 3) % 16)
    _assert_marks(raw[: 16 * (off + 1) + off], text_off=off, mark_off=off)


BOUNDARY_CASES = [s.encode("utf-8") for s in (
    "x\\b", "x\\\\b", "x\\\\\\b", "x\\\\\\\\b", "\\" * 17 + "q", "\\" * 32 + "q",   # odd and even backslash runs
    "word",                                                                       # a word
    "aéb", "a\u212ab", "a\u1e01b", "a\U0001f600b", "a\U000101fdb",   # 2-, 3- and 4-byte code points
    "\\\u0301b", "a\\\u0301\\\u0301b",                                            # a dropped mark after a backslash
    "a\\\\\nb", "\\\\\\\\\nb")]                                                   # even runs before a newline


def test_mark_cases_straddling_every_scan_boundary():
    """Each case at each split point across a carry-chunk boundary (k MiB), a tile boundary, a warp boundary and a
    thread boundary, in random text; the 4-byte code points are a dropped one and an emoji (no 4-byte code point is a
    letter)."""
    splits = lambda c: range(1, len(c)) if len(c) <= 8 else (1, 2, 3, len(c) // 2, len(c) - 3, len(c) - 2, len(c) - 1)
    placed = [(c, k) for c in BOUNDARY_CASES for k in splits(c)]
    raw = random_text((len(placed) + 1) * MIB + 4096, seed=9)
    inner = (0, 5 * 4096, 7 * 4096 + 3 * 512, 9 * 4096 + 5 * 512 + 7 * 16)   # carry, tile, warp, thread
    for m, (c, k) in enumerate(placed, start=1):
        for d in inner:
            p = m * MIB + d
            inst = b"  " + c + b"  "
            raw[p - k - 2: p - k - 2 + len(inst)] = np.frombuffer(inst, np.uint8)
    mark = _assert_marks(raw)
    assert (mark[MIB - 64: MIB + 64] != 0).any()


@pytest.mark.parametrize("odd", [False, True])
def test_mark_long_backslash_runs(odd):
    """3 MiB of backslashes (768 tiles, three carry chunks) between a letter and a word: the carry is ODD or SEP all
    the way, and decides whether the first letter after the run is swallowed."""
    run = 3 * MIB - int(odd)
    raw = np.frombuffer(b"a" + b"\\" * run + b"xy z", np.uint8).copy()
    mark = _assert_marks(raw)
    tail = bytes(mark[1 + run:]).replace(b"\0", b"")
    assert mark[0] == ord("A") and not mark[1:1 + run].any() and tail == (b"YZ" if odd else b"XyZ")


@pytest.mark.parametrize("seed", range(4))
def test_mark_random_text(seed):
    weights = list(_WEIGHTS)
    weights[_SYMBOLS.index("\\")] = 4 + 20 * seed     # from sparse backslashes to runs of them
    _assert_marks(random_text(300_000 + 4099 * seed, seed=1000 + seed, weights=weights))


@pytest.mark.parametrize("raw", [b"ab\xc3", b"ab\xe2\x84", b"ab\xf0\x9f\x98", b"a\xf0", b"\x80\xbf\xbfa",
                                 b"a\xff\xbf\xbf\xbfb\xfe", b"\xc1\x9cab\\\xc1\x9cc", b"x\xed\xa0\x80y\xc3\xa9",
                                 b"q" * 15 + b"\xe1\x80", b"q" * 4094 + b"\xf0\x9f", b"word \\\xcc"])
def test_mark_invalid_utf8_at_the_end(raw):
    for off in (0, 1):
        _assert_marks(np.frombuffer(raw, np.uint8).copy(), text_off=off, mark_off=off)


def test_mark_at_the_size_limit():
    """``n_bytes = 2^31 - 1`` (524 288 tiles, 2048 trips of the carry loop): a period of P bytes, P odd and so coprime
    to 4096, repeated on the device; each period starts in SEP (it ends in a space), so the marks are the oracle's marks
    of one period repeated, then of the last partial period.  Compared on the device."""
    _need(6.0)
    n = (1 << 31) - 1
    period = "ab\\\\\\cd é\\\u0301f \u212ax\\\\\ny \U0001f600z\u0301w \\\\\\\\word\\ ".encode()
    if len(period) % 2 == 0:
        period += b" "
    P = len(period)
    q, r = divmod(n, P)
    per = torch.from_numpy(np.frombuffer(period, np.uint8).copy()).to(DEV)
    text = torch.empty(n, dtype=torch.uint8, device=DEV)
    text[:q * P].view(q, P).copy_(per.expand(q, P))
    text[q * P:] = per[:r]
    torch.cuda.current_stream().synchronize()
    mark = _run_mark(text, n)
    del text
    table = _fts.class_table()
    want = torch.from_numpy(fo.mark_oracle(period, table)).to(DEV)
    assert bool((want != 0).any())
    rows = (256 * MIB) // P
    for a in range(0, q, rows):
        b = min(q, a + rows)
        assert torch.equal(mark[a * P:b * P].view(b - a, P), want.expand(b - a, P)), (a, b)
    last = torch.from_numpy(fo.mark_oracle(period[:r], table)).to(DEV)
    assert torch.equal(mark[q * P:], last)


def test_mark_is_deterministic():
    raw = random_text(8 * MIB + 3, seed=77)
    text = torch.from_numpy(raw).to(DEV)
    torch.cuda.current_stream().synchronize()
    assert torch.equal(_run_mark(text, len(raw), mark_off=0), _run_mark(text, len(raw), mark_off=0))


# ---- rl_fts_stem ----------------------------------------------------------------------------------------------------
def _stem(words, *, bits: int = 64, stop: bool = True, base: int = 0, odd: bool = False):
    """``rl_fts_stem`` on ``words`` (``word_off[0] = base``; the letters at an odd address when ``odd``), outputs
    pre-filled with values the kernel never writes.  Returns numpy ``(keep int32, tail uint64, hash int64)``."""
    _, lib = _lib()
    _, stop_d = _fts._device_tables(DEV)
    letters, off = fo.words_to_csr(words, base=base)
    W = len(words)
    st = _stream()
    with torch.cuda.stream(st):
        lbuf = torch.zeros(len(letters) + 2, dtype=torch.uint8, device=DEV)
        lt = lbuf[int(odd):int(odd) + len(letters)]
        lt.copy_(torch.from_numpy(letters))
        off_d = torch.from_numpy(off).to(DEV)
        keep = torch.full((W,), -2, dtype=torch.int32, device=DEV)
        tail = torch.full((W,), 0x5A5A5A5A5A5A5A5A, dtype=torch.int64, device=DEV)
        hsh = torch.full((W,), 0x5A5A5A5A5A5A5A5A, dtype=torch.int64, device=DEV)
        assert lt.data_ptr() % 2 == int(odd)
        _check(lib.rl_fts_stem(lt.data_ptr(), off_d.data_ptr(), W, stop_d.data_ptr() if stop else None,
                               stop_d.numel() // 2 if stop else 0, bits, keep.data_ptr(), tail.data_ptr(),
                               hsh.data_ptr(), st.cuda_stream), "rl_fts_stem")
        st.synchronize()
        return keep.cpu().numpy(), tail.cpu().numpy().view(np.uint64), hsh.cpu().numpy()


def _tail_bytes(t: int) -> bytes:
    """The appended letters of a tail: its non-zero bytes low first, which must be followed by zeros only."""
    raw = int(t).to_bytes(8, "little")
    k = len(raw.rstrip(b"\0"))
    assert b"\0" not in raw[:k], hex(int(t))
    return raw[:k]


def _check_stems(words, keep, tail, hsh, bits: int, *, stop: bool = True) -> list[bytes]:
    """Every word's ``(keep, tail, hash)`` against ``_fts.stem`` and ``fts_oracle.stem_hash``; returns the stems."""
    stems, live = [], []
    for i, w in enumerate(words):
        if stop and w in _fts.STOPWORDS:
            assert (keep[i], tail[i], hsh[i]) == (-1, 0, 0), w
            stems.append(None)
            continue
        assert 0 <= keep[i] <= len(w), (w, keep[i])
        s = w[:keep[i]].encode() + _tail_bytes(tail[i])
        assert s.decode() == _fts.stem(w), (w, s, _fts.stem(w))
        stems.append(s)
        live.append(i)
    want = fo.stem_hash([stems[i] for i in live], bits)
    got = hsh[live]
    bad = np.flatnonzero(got != want)
    assert not len(bad), [(words[live[j]], int(got[j]), int(want[j])) for j in bad[:5]]
    return stems


def _stop_neighbours() -> list[str]:
    words = set(STOP_AZ)
    for w in STOP_AZ:
        words.add(w[:-1])
        words.update(w + c for c in "abcdefghijklmnopqrstuvwxyz")
        for L in (13, 16, 17):   # the 16-byte key's edges, on a stop word's prefix
            if len(w) < L:
                words.add((w + "sesame" * 3)[:L])
    words.discard("")
    words.update(("unfortunately" + "s" * 4)[:L] for L in range(10, 18))
    return sorted(words)


@pytest.mark.parametrize("bits", [1, 2, 31, 32, 33, 63, 64])
def test_stem_stop_words_and_their_neighbours(bits):
    words = _stop_neighbours()
    keep, tail, hsh = _stem(words, bits=bits)
    stems = _check_stems(words, keep, tail, hsh, bits)
    assert sum(s is None for s in stems) == len(STOP_AZ)
    if bits >= 31:
        live = {s: int(h) for s, h in zip(stems, hsh) if s is not None}
        assert len(set(live.values())) == len(live)


def test_stem_without_a_stop_list():
    words = STOP_AZ + ["hoping", "the" * 6]
    keep, tail, hsh = _stem(words, stop=False)
    _check_stems(words, keep, tail, hsh, 64, stop=False)
    assert (keep >= 0).all()


def test_stem_y_mark_window():
    """Words with a ``y`` 16 to 36 letters from the end behind suffix chains, and every word of the one shape whose stem
    a y mark decides, up to 16 letters back (``fts_oracle.y_window_words``)."""
    words = fo.y_window_words()
    keep, tail, hsh = _stem(words)
    _check_stems(words, keep, tail, hsh, 64)


def test_stem_long_words():
    rng = np.random.default_rng(6)
    vow = np.frombuffer(b"aeiouybcst", np.uint8)
    words = ["ay" * 50_000, "y" * 100_000 + "ing", "x" * 99_993 + "ational",
             bytes(rng.choice(vow, size=1_000_000)).decode() + "ization", "ab" * 500_000, "e" * 999_999 + "s"]
    keep, tail, hsh = _stem(words)
    _check_stems(words, keep, tail, hsh, 64)
    keep, tail, hsh = _stem(words, bits=33, odd=True, base=3)
    _check_stems(words, keep, tail, hsh, 33)


def _vocab(n: int, seed: int) -> list[str]:
    import keyword_oracle as ko

    bases = ["connect", "gener", "relat", "hope", "hop", "run", "fil", "sing", "poni", "agre", "happi", "sky", "formal",
             "adopt", "ration", "bake", "control", "roll", "motor", "condit", "digit", "analog", "sensibl", "rate", "y"]
    sufs = ["", "s", "es", "ies", "ed", "ing", "eed", "y", "ly", "e", *_fts._STEP2, *_fts._STEP3, *_fts._STEP4]
    words = set(ko.make_vocab(n, seed)) | {b + s for b in bases for s in sufs} | set(STOP_AZ[:40])
    return sorted(w for w in words if len(w) <= 20)


def test_stem_offsets():
    words = _vocab(1500, 3)
    for base, odd in ((1, False), (1_000_001, True), (7, True)):
        keep, tail, hsh = _stem(words, base=base, odd=odd, bits=63)
        _check_stems(words, keep, tail, hsh, 63)


def _stem_device(letters_d, off_d, W, *, bits=64):
    _, lib = _lib()
    _, stop_d = _fts._device_tables(DEV)
    st = _stream()
    with torch.cuda.stream(st):
        keep = torch.full((W,), -2, dtype=torch.int32, device=DEV)
        tail = torch.full((W,), 0x5A5A5A5A5A5A5A5A, dtype=torch.int64, device=DEV)
        hsh = torch.full((W,), 0x5A5A5A5A5A5A5A5A, dtype=torch.int64, device=DEV)
        _check(lib.rl_fts_stem(letters_d.data_ptr(), off_d.data_ptr(), W, stop_d.data_ptr(), stop_d.numel() // 2, bits,
                               keep.data_ptr(), tail.data_ptr(), hsh.data_ptr(), st.cuda_stream), "rl_fts_stem")
        st.synchronize()
    return keep, tail, hsh


def _gather_words(words: list[str], idx: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """The letters CSR of ``words[idx[0]], words[idx[1]], ...``, built from a padded table."""
    M = max(map(len, words))
    tab = np.zeros((len(words), M), np.uint8)
    for i, w in enumerate(words):
        tab[i, :len(w)] = np.frombuffer(w.encode(), np.uint8)
    lens = np.array([len(w) for w in words], np.int64)
    letters = tab[idx][np.arange(M)[None, :] < lens[idx][:, None]]
    off = np.zeros(len(idx) + 1, np.int64)
    np.cumsum(lens[idx], out=off[1:])
    return letters, off


def test_stem_grid_stride_wrap():
    """9 000 000 words in one launch (one pass of the grid covers 8 388 608): every occurrence of a vocabulary word
    gets the (keep, tail, hash) its word gets in a small launch, which is checked against ``_fts.stem``."""
    _need(1.5)
    vocab = _vocab(3000, 11)
    small = _stem(vocab)
    _check_stems(vocab, *small, 64)
    n = 9_000_000
    assert n > STEM_WRAP
    idx = np.random.default_rng(12).integers(0, len(vocab), size=n)
    letters, off = _gather_words(vocab, idx)
    keep, tail, hsh = _stem_device(torch.from_numpy(letters).to(DEV), torch.from_numpy(off).to(DEV), n)
    idx_d = torch.from_numpy(idx).to(DEV)
    for got, want in zip((keep, tail, hsh), small):
        want_d = torch.from_numpy(want.view(np.int64) if want.dtype == np.uint64 else want).to(DEV)
        assert torch.equal(got, want_d[idx_d])


# ---- rl_fts_verify and rl_fts_stem_bytes ----------------------------------------------------------------------------
def _split_representations():
    """Stems given directly as (word, keep, tail): equal stems with different splits (an 8-letter tail against none),
    stems that differ only in the tail, only in the kept prefix, or by one letter."""
    reps = []

    def add(word, keep, tail):
        reps.append((word, keep, tail))

    w = "abcdefghij"
    for k in range(2, 11):
        add(w, k, w[k:])                           # every split of one stem, tails of 8 down to 0 letters
    add(w, 2, "cdefghik")                          # differs only in the last tail letter
    add("xbcdefghij", 2, "cdefghij")               # differs only in the kept prefix
    add(w, 9, "")                                  # one letter shorter
    add(w, 2, "cdefghi")                           # one letter shorter, in the tail
    add("abcdefghijz", 10, "z")                    # one letter longer, in the tail
    add("abcdefghijzzz", 11, "")                   # one letter longer, in the prefix
    add("", 0, "abcdefgh")                         # only a tail
    add("abcdefgh", 0, "abcdefgh")
    add("abcdefgh", 8, "")
    add("q", 0, "")                                # the empty stem
    add("", 0, "")
    return reps


def _upload_reps(reps):
    words = [r[0] for r in reps]
    letters, off = fo.words_to_csr(words, base=5)
    keep = np.array([r[1] for r in reps], np.int32)
    tail = np.array([int.from_bytes(r[2].encode().ljust(8, b"\0"), "little") for r in reps], np.uint64)
    stems = [(r[0][:r[1]] + r[2]).encode() for r in reps]
    dev = [torch.from_numpy(np.concatenate([letters, np.zeros(1, np.uint8)])).to(DEV), torch.from_numpy(off).to(DEV),
           torch.from_numpy(keep).to(DEV), torch.from_numpy(tail.view(np.int64)).to(DEV)]
    return dev, stems


def _verify(dev, a: np.ndarray, b: np.ndarray) -> np.ndarray:
    _, lib = _lib()
    st = _stream()
    with torch.cuda.stream(st):
        a_d, b_d = torch.from_numpy(np.asarray(a, np.int64)).to(DEV), torch.from_numpy(np.asarray(b, np.int64)).to(DEV)
        differ = torch.full((len(a),), 0xAA, dtype=torch.uint8, device=DEV)
        _check(lib.rl_fts_verify(*(t.data_ptr() for t in dev), a_d.data_ptr(), b_d.data_ptr(), len(a),
                                 differ.data_ptr(), st.cuda_stream), "rl_fts_verify")
        st.synchronize()
        return differ.cpu().numpy()


def _stem_bytes(dev, words: np.ndarray, lens: np.ndarray) -> np.ndarray:
    _, lib = _lib()
    st = _stream()
    with torch.cuda.stream(st):
        out_off = np.zeros(len(words) + 1, np.int64)
        np.cumsum(lens, out=out_off[1:])
        w_d, o_d = torch.from_numpy(np.asarray(words, np.int64)).to(DEV), torch.from_numpy(out_off).to(DEV)
        out = torch.zeros(max(int(out_off[-1]), 1) + 16, dtype=torch.uint8, device=DEV)
        _check(lib.rl_fts_stem_bytes(*(t.data_ptr() for t in dev), w_d.data_ptr(), len(words), o_d.data_ptr(),
                                     out.data_ptr(), st.cuda_stream), "rl_fts_stem_bytes")
        st.synchronize()
        res = out.cpu().numpy()
    assert not res[int(out_off[-1]):].any()
    return res[:int(out_off[-1])]


def test_verify_and_stem_bytes_on_crafted_splits():
    reps = _split_representations()
    dev, stems = _upload_reps(reps)
    R = len(reps)
    a, b = np.divmod(np.arange(R * R), R)
    got = _verify(dev, a, b)
    want = np.array([stems[i] != stems[j] for i, j in zip(a, b)], np.uint8)
    assert np.array_equal(got, want)
    assert (want == 0).sum() > R   # equal stems under different splits
    order = np.random.default_rng(2).permutation(np.tile(np.arange(R), 3))
    lens = np.array([len(stems[i]) for i in order])
    assert bytes(_stem_bytes(dev, order, lens)) == b"".join(stems[i] for i in order)


def _stemmed_vocab(n: int, seed: int):
    """A vocabulary stemmed on the device (checked against ``_fts.stem``), its stop words dropped: the device
    arrays, the stems, and stem ids (equal ids for equal stems)."""
    vocab = [w for w in _vocab(n, seed) if w not in _fts.STOPWORDS]
    keep, tail, hsh = _stem(vocab)
    stems = _check_stems(vocab, keep, tail, hsh, 64)
    letters, off = fo.words_to_csr(vocab)
    dev = [torch.from_numpy(np.concatenate([letters, np.zeros(1, np.uint8)])).to(DEV), torch.from_numpy(off).to(DEV),
           torch.from_numpy(keep).to(DEV), torch.from_numpy(tail.view(np.int64)).to(DEV)]
    ids = {}
    sid = np.array([ids.setdefault(s, len(ids)) for s in stems], np.int64)
    return vocab, dev, stems, sid, keep, tail


def test_verify_equal_stems_with_different_splits():
    """Pairs of words whose stems are equal but split differently between kept prefix and tail (``hoping``/``hope``),
    found by search over the vocabulary; pairs with a == b; and all pairs within each stem's neighbourhood."""
    vocab, dev, stems, sid, keep, tail = _stemmed_vocab(2000, 4)
    n_tail = np.array([len(_tail_bytes(t)) for t in tail])
    by_stem: dict = {}
    for i, s in enumerate(stems):
        by_stem.setdefault(s, []).append(i)
    split_pairs = [(i, j) for g in by_stem.values() for i in g for j in g
                   if (keep[i], n_tail[i]) != (keep[j], n_tail[j])]
    assert len(split_pairs) >= 20, len(split_pairs)
    assert any({vocab[i], vocab[j]} == {"hoping", "hope"} for i, j in split_pairs) or "hoping" not in vocab
    a = np.array([p[0] for p in split_pairs] + list(range(len(vocab))))
    b = np.array([p[1] for p in split_pairs] + list(range(len(vocab))))
    assert not _verify(dev, a, b).any()
    # near neighbours in sorted stem order: shared prefixes, one letter more or less
    order = sorted(range(len(stems)), key=lambda i: stems[i])
    a = np.array([order[k] for k in range(len(order) - 1)] * 2)
    b = np.array([order[k + 1] for k in range(len(order) - 1)] + [order[min(k + 2, len(order) - 1)]
                                                                  for k in range(len(order) - 1)])
    assert np.array_equal(_verify(dev, a, b), (sid[a] != sid[b]).astype(np.uint8))


def test_verify_grid_stride_wrap():
    """17 000 000 pairs in one launch (one pass covers 16 777 216), half of them of equal stems, against stem ids."""
    _need(1.0)
    vocab, dev, stems, sid, _, _ = _stemmed_vocab(4000, 5)
    n = 17_000_000
    assert n > ITEM_WRAP
    rng = np.random.default_rng(13)
    a = rng.integers(0, len(vocab), size=n)
    order = np.argsort(sid, kind="stable")
    start = np.searchsorted(sid[order], np.arange(sid.max() + 1))
    size = np.bincount(sid)
    same = order[start[sid[a]] + (rng.random(n) * size[sid[a]]).astype(np.int64)]
    b = np.where(rng.random(n) < 0.5, same, rng.integers(0, len(vocab), size=n))
    got = _verify(dev, a, b)
    want = (sid[a] != sid[b]).astype(np.uint8)
    assert np.array_equal(got, want) and 0.3 < want.mean() < 0.7


def test_stem_bytes_shuffled_repeated_and_past_one_grid_pass():
    vocab, dev, stems, sid, _, _ = _stemmed_vocab(3000, 6)
    lens = np.array([len(s) for s in stems])
    order = np.random.default_rng(3).permutation(np.tile(np.arange(len(vocab)), 2))
    assert bytes(_stem_bytes(dev, order, lens[order])) == b"".join(stems[i] for i in order)
    _need(1.5)
    n = 17_000_000
    assert n > ITEM_WRAP
    idx = np.random.default_rng(14).integers(0, len(vocab), size=n)
    got = _stem_bytes(dev, idx, lens[idx])
    want, _ = _gather_words([s.decode() for s in stems], idx)
    assert np.array_equal(got, want)


# ---- rl_fts_term_keys -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chunk_base", [0, (1 << 30) + 12345])
def test_term_keys(chunk_base):
    """key == term << 32 | (chunk_base + owner) for 17 000 000 tokens (one pass covers 16 777 216), term ids up to
    2^31 - 1 and chunk_base + owner up to 2^31 - 1."""
    _need(1.0)
    _, lib = _lib()
    n, S = 17_000_000, 5000
    rng = np.random.default_rng(chunk_base % 1000)
    stem_term = rng.integers(0, 1 << 31, size=S).astype(np.int32)
    stem_term[:3] = [0, (1 << 31) - 1, 1]
    tok_stem = rng.integers(0, S, size=n)
    tok_stem[:3] = [0, 1, 2]
    tok_stem[-3:] = [1, 0, 2]
    top = (1 << 31) - 1 - chunk_base
    owner = np.sort(rng.integers(0, top + 1, size=n))
    owner[-1] = top
    st = _stream()
    with torch.cuda.stream(st):
        ts, ow, term = (torch.from_numpy(x).to(DEV) for x in (tok_stem, owner, stem_term))
        key = torch.full((n,), -7, dtype=torch.int64, device=DEV)
        _check(lib.rl_fts_term_keys(ts.data_ptr(), ow.data_ptr(), n, term.data_ptr(), chunk_base, key.data_ptr(),
                                    st.cuda_stream), "rl_fts_term_keys")
        st.synchronize()
        got = key.cpu().numpy()
    want = (stem_term[tok_stem].astype(np.int64) << 32) | (chunk_base + owner)
    assert np.array_equal(got, want)
    assert got[-1] & 0xFFFFFFFF == (1 << 31) - 1 and (got >> 32).max() == (1 << 31) - 1


# ---- analyze_on_device at the default group budget ------------------------------------------------------------------
def _e2e_vocab(seed: int) -> list[str]:
    rng = np.random.default_rng(seed)
    letters = np.array(list("abcdefghilmnoprstuy"))
    plain = sorted({"".join(rng.choice(letters, size=int(rng.integers(2, 7)))) for _ in range(3000)})
    accent = str.maketrans("aeiou", "áéíóú")
    vocab = plain[:1500]
    vocab += [w.upper() for w in plain[1500:1800]] + [w.capitalize() for w in plain[1800:2000]]
    vocab += [w.translate(accent) for w in plain[2000:2300]] + [w[:1] + "\u0301" + w[1:] for w in plain[2300:2400]]
    vocab += [w[:2] + "\\" + w[2:] for w in plain[2400:2500]] + [w + "\\\\" + w for w in plain[2500:2550]]
    vocab += ["\\\\" + w for w in plain[2550:2600]] + ["don't", "e.g.", "x2y", "\u212aelvin", "\u0130nn", "naïve"]
    vocab += ["hoping", "hope", "running", "ponies", "connection", "generalizations"]
    return vocab


def test_analyze_at_the_default_group_size():
    """About 300 MiB of bodies at the default ``GROUP_BYTES``: two multi-body groups, one body over 128 MiB alone,
    then one more multi-body group.  Tokens of a vocabulary that mixes case, accents, marks and backslashes, separated
    by single spaces, so each analyses as it does alone.  The body over 128 MiB holds more than 16 777 216 kept
    tokens, so every per-token kernel runs past one pass of its grid.  Term ids, keys and doc_len are computed in NumPy
    from each vocabulary token's own analysis."""
    _need(5.0)
    assert _fts.GROUP_BYTES == 128 * MIB
    vocab = _e2e_vocab(21)
    stops = ["the", "and", "of", "The", "AND", "it's"]
    V = len(vocab)
    tokens = vocab + stops
    toks_b = [t.encode() for t in tokens]
    # each token alone: its kept stems
    per = [_fts.document_terms(t) for t in tokens]
    stem_names = sorted({s for p in per for s in p})
    stem_index = {s: i for i, s in enumerate(stem_names)}
    cnt = np.array([len(p) for p in per], np.int64)
    s_off = np.zeros(len(tokens) + 1, np.int64)
    np.cumsum(cnt, out=s_off[1:])
    s_flat = np.array([stem_index[s] for p in per for s in p], np.int64)
    # the token stream: stop words rare; bytes = each token then a space
    tok_len = np.array([len(b) + 1 for b in toks_b], np.int64)
    M = int(tok_len.max())
    tab = np.full((len(tokens), M), 0x20, np.uint8)
    for i, b in enumerate(toks_b):
        tab[i, :len(b)] = np.frombuffer(b, np.uint8)
    p = np.full(len(tokens), 1.0)
    p[V:] = 0.2
    p /= p.sum()
    rng = np.random.default_rng(22)
    body_bytes = [150 * MIB, 136 * MIB, 16 * MIB]
    bodies, idx_parts, n_tok_per_body = [], [], []
    for part, nbytes in enumerate(body_bytes):
        m = int(nbytes / (p @ tok_len))
        idx = rng.choice(len(tokens), size=m, p=p).astype(np.int32)
        lens = tok_len[idx]
        raw = tab[idx][np.arange(M)[None, :] < lens[:, None]]
        ends = np.cumsum(lens)
        if part == 1:
            cuts = np.array([0, m])
        else:
            sizes = rng.integers(1, 40_000, size=m // 1000)
            cuts = np.unique(np.concatenate([[0], np.minimum(np.cumsum(sizes), m), [m]]))
        starts_b = np.concatenate([[0], ends])[cuts]
        for a, z in zip(starts_b[:-1], starts_b[1:]):
            bodies.append(raw[a:z - 1].tobytes().decode("utf-8") if z > a else "")
        n_tok_per_body.append(np.diff(cuts))
        idx_parts.append(idx)
        del raw
    idx = np.concatenate(idx_parts)
    del idx_parts
    n_tok = np.concatenate(n_tok_per_body)
    assert len(bodies[len(n_tok_per_body[0])].encode()) > 128 * MIB
    groups = _fts._groups([len(b.encode()) for b in bodies], _fts.GROUP_BYTES)
    assert len(groups) == 4 and sum(b - a > 1 for a, b in groups) == 3
    # expected: each token's stems in order, term ids in order of first appearance, owners and doc_len
    c = cnt[idx]
    body_of_tok = np.repeat(np.arange(len(bodies), dtype=np.int64), n_tok)
    owner = np.repeat(body_of_tok, c)
    del body_of_tok
    tok_rep = np.repeat(idx, c)
    within = np.arange(len(tok_rep), dtype=np.int64) - np.repeat(np.cumsum(c) - c, c)
    stem_ids = s_flat[s_off[tok_rep] + within]
    del tok_rep, within
    uniq, first = np.unique(stem_ids, return_index=True)
    term_of = np.empty(len(stem_names), np.int64)
    term_of[uniq[np.argsort(first)]] = np.arange(len(uniq))
    want_key = (term_of[stem_ids] << 32) | owner
    want_len = np.bincount(owner, minlength=len(bodies)).astype(np.int32)
    big = len(n_tok_per_body[0])
    assert want_len[big] > ITEM_WRAP and n_tok[big] > STEM_WRAP
    del stem_ids, owner
    an = _fts.Analyzer()
    key, doc_len = _fts.analyze_on_device(an, bodies, DEV)
    assert list(an.term_ids) == [stem_names[s] for s in uniq[np.argsort(first)]]
    assert list(an.term_ids.values()) == list(range(len(uniq)))
    assert np.array_equal(doc_len.cpu().numpy(), want_len)
    got = key.cpu().numpy()
    assert len(got) == len(want_key) and np.array_equal(got, want_key)
