"""The BM25 index's text analysis on the device (csrc/fts.cu behind ``_fts.analyze_on_device`` and
``KeywordIndex.extend``) against the host analyzer it replaces, ``_fts.Analyzer.analyze``: the same kept tokens in the
same order, the same owners and ``doc_len``, and the same ``stem -> term id`` dictionary, ids included."""

from __future__ import annotations

import itertools
import threading

import numpy as np
import pytest
import torch

import keyword_oracle as ko
from raglite_b200 import _fts

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _device(bodies, *, analyzer=None, chunk_base=0, hash_bits=_fts.HASH_BITS):
    an = analyzer if analyzer is not None else _fts.Analyzer()
    key, doc_len = _fts.analyze_on_device(an, bodies, DEV, chunk_base=chunk_base, hash_bits=hash_bits)
    key = key.cpu().numpy()
    return (key >> 32).astype(np.int32), (key & 0xFFFFFFFF) - chunk_base, doc_len.cpu().numpy(), an


def _check(bodies, **kw):
    terms, owners, lens = (host := _fts.Analyzer()).analyze(bodies)
    d_terms, d_owners, d_lens, dev = _device(bodies, **kw)
    assert list(dev.term_ids.items()) == list(host.term_ids.items())
    assert np.array_equal(d_terms, terms) and np.array_equal(d_owners, owners) and np.array_equal(d_lens, lens)
    return dev


HAZARDS = [
    "", " ", " \t\n.,;!?-", "123 456", "\\\\\\", "\n\n",
    "Café résumé naïve façade Ærøskøbing Straße İstanbul ﬁne K ÉTÉ",           # accented Latin, ligature, Kelvin sign
    "Ελληνικά κείμενα με τόνους", "漢字かな交じり文 한국어", "emoji 😀🎉 mixed😀in words",  # Greek, CJK, emoji
    "ét́e combining̈marks à́̂b ́start end́",         # marks inside words
    "THE The thé Thé AND aNd alls ALL c'mon don't it's",                          # stop words, any case, accented
    "lone \ud800 surrogate \udfff here x\ud800y", "nul\x00byte\x00 and \x00",
    "Kelvin İi ẞ",
]
for n in range(1, 6):   # backslash runs before letters, newlines, marks and the end of a body
    HAZARDS += ["a" + "\\" * n + "bc d", "x" + "\\" * n + "\nyz", "p" + "\\" * n + "́q r", "\\" * n,
                "k" + "\\" * n + "́\\́m n", "\\" * n + "word"]


def test_generated_corpora_and_hazards():
    for seed in (0, 1):
        _check(ko.make_bodies(3000, seed, vocab=800) + HAZARDS)
    _check(HAZARDS)
    _check([""] * 5)
    _check([])


@pytest.mark.parametrize("pattern", ["a{}b", "\\{}b"])
def test_every_code_point(pattern):
    chars = [chr(cp) for cp in range(0x110000)]
    bodies = [" ".join(pattern.format(ch) for ch in chars[i:i + 4096]) for i in range(0, len(chars), 4096)]
    bodies += ["".join(pattern.format(ch) for ch in chars[i:i + 4096]) for i in range(0, len(chars), 4096)]
    _check(bodies)


def test_stemmer_coverage():
    letters = "abcdefghijklmnopqrstuvwxyz"
    short = ["".join(p) for n in range(1, 5) for p in itertools.product(letters, repeat=n)]
    assert len(short) == 475_254
    _check(short)
    bases = ["connect", "gener", "relat", "hope", "run", "fil", "sing", "poni", "cat", "agre", "happi", "sky", "formal",
             "electr", "adopt", "ration", "bake", "control", "roll", "motor", "condit", "valenc", "digit", "conform",
             "radic", "differ", "analog", "sensibl", "feud", "rate", "y", "ay", "oy", "by"]
    sufs = ["s", "es", "ies", "sses", "ed", "ing", "eed", "y", "ly", *_fts._STEP2, *_fts._STEP3, *_fts._STEP4]
    words = [b + s for b in bases for s in sufs] + [b + s + t for b in bases for s in sufs for t in ("s", "ing", "ed")]
    rng = np.random.default_rng(5)
    words += ["".join(rng.choice(list("abeiouyyyyst"), size=int(rng.integers(1, 16)))) for _ in range(40_000)]
    words += ["a" * 64, "ab" * 32, "y" * 64, ("ay" * 500), "ization" * 143, ("ay" * 2500) + "ing",
              "x" * 1000 + "ational", "biliti" * 800 + "ness", "sses" * 1250, "y" * 5000]
    dev = _check(words)
    assert all(_fts.stem(w) in dev.term_ids for w in words[-10:])


def test_dictionary_across_calls_and_groups(monkeypatch):
    """``KeywordIndex.extend`` in pieces, with the group budget cut so that a call spans many groups and some bodies
    exceed it: ids and postings equal one host pass over everything."""
    from raglite_b200._keyword import KeywordIndex

    bodies = ko.make_bodies(1500, 4, vocab=600) + HAZARDS + ["word " * 400 + "épée " * 50]
    monkeypatch.setattr(_fts, "GROUP_BYTES", 700)
    kw = KeywordIndex(DEV)
    for a, b in ((0, 1), (1, 400), (400, 401), (401, 1200), (1200, len(bodies))):
        kw.extend(bodies[a:b])
    host = _fts.Analyzer()
    terms, owners, lens = host.analyze(bodies)
    assert list(kw.analyzer.term_ids.items()) == list(host.term_ids.items())
    keys, tf = np.unique((terms.astype(np.int64) << 32) | owners, return_counts=True)
    term_off = np.searchsorted(keys >> 32, np.arange(len(host.term_ids) + 1))
    assert np.array_equal(kw.term_off.cpu().numpy(), term_off)
    assert np.array_equal(kw.doc.cpu().numpy(), (keys & 0xFFFFFFFF).astype(np.int32))
    assert np.array_equal(kw.tf.cpu().numpy(), tf) and np.array_equal(kw.doc_len.cpu().numpy(), lens)
    assert set(kw.analysis_seconds) == {"encode", "device", "dictionary"}


@pytest.mark.parametrize("bits", [1, 3, 9])
def test_forced_hash_collisions(bits):
    bodies = ko.make_bodies(400, 6, vocab=300) + HAZARDS
    _check(bodies, hash_bits=bits)


def test_determinism_and_two_streams():
    from raglite_b200._keyword import KeywordIndex

    corpora = [ko.make_bodies(2000, 8, vocab=900) + HAZARDS, ko.make_bodies(2000, 9, vocab=900)[::-1]]

    def build(bodies, out, i, stream=None):
        with torch.cuda.stream(stream) if stream is not None else torch.cuda.device(DEV):
            kw = KeywordIndex(DEV)
            kw.extend(bodies)
            out[i] = (dict(kw.analyzer.term_ids), kw.term_off.cpu().numpy(), kw.doc.cpu().numpy(), kw.tf.cpu().numpy(),
                      kw.doc_len.cpu().numpy())

    seq = [None, None]
    for i in range(2):
        build(corpora[i], seq, i)
    again = [None]
    build(corpora[0], again, 0)
    streams, par = [torch.cuda.Stream(DEV), torch.cuda.Stream(DEV)], [None, None]
    threads = [threading.Thread(target=build, args=(corpora[i], par, i, streams[i])) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for a, b in ((seq[0], again[0]), (seq[0], par[0]), (seq[1], par[1])):
        assert list(a[0].items()) == list(b[0].items())
        assert all(np.array_equal(x, y) for x, y in zip(a[1:], b[1:]))


def test_sharded_search_over_non_ascii_bodies():
    """A one-rank ShardedIndex over a device-built index, on accented bodies: the oracle's results over sorted stems."""
    from synth import make_corpus

    import raglite_b200 as rl
    from raglite_b200._dist import ShardedIndex

    vocab = ko.make_vocab(300, 12)
    rng = np.random.default_rng(12)
    accent = str.maketrans("aeiou", "áéíóú")
    bodies = [" ".join((w.translate(accent).upper() if rng.random() < 0.3 else w) for w in rng.choice(vocab, size=int(n)))
              for n in rng.integers(1, 40, size=600)]
    E, off = make_corpus(len(bodies), 1, 16, seed=0)
    ids = [f"c{c}" for c in range(len(bodies))]
    idx = rl.CorpusIndex(E, off, chunk_ids=ids,
                         chunks=[rl.Chunk(id=ids[c], document_id="d", index=c, body=b) for c, b in enumerate(bodies)])
    queries = [" ".join(rng.choice(vocab, size=3)) for _ in range(12)] + ["ÁBÁCÚS", vocab[0].translate(accent)]
    fts = ko.create_fts_index(bodies)
    g_ids, g_scores, g_counts = rl.keyword_search_batch(queries, num_results=20, index=idx)
    s_ids, s_scores, s_counts = rl.keyword_search_batch(queries, num_results=20, index=ShardedIndex(idx))
    host = _fts.Analyzer()
    host.analyze(bodies)
    by_id = idx.keyword_index().analyzer.term_ids
    assert list(by_id.items()) == list(host.term_ids.items())
    by_stem = {t: i for i, t in enumerate(sorted(fts.dict))}
    for b, q in enumerate(queries):
        for (ids_, sc, cnt), order in (((g_ids, g_scores, g_counts), by_id), ((s_ids, s_scores, s_counts), by_stem)):
            w_ids, w_scores = ko.keyword_search(fts, q, num_results=20, term_order=order)
            assert cnt[b] == len(w_ids) and np.allclose(sc[b, :cnt[b]], w_scores, rtol=1e-12, atol=0)
