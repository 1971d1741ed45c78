"""ts_rank oracle: PostgreSQL's ``calc_rank_or`` (``tsrank.c``; default weights, normalization 0, every position of
weight D) restated in NumPy float32 with its one float64 step, as the reference's PostgreSQL ``keyword_search`` runs it
(``_search.py:176-201``).  Test infrastructure beside the tests.  Recalled, not checked against a server.

For an entry held with ``n`` positions: ``resj = sum_{j<n} fl(0.1f / (float)((j+1)^2))`` (float32, ascending j),
``t = fl(fl(0.1f + resj) - fl(0.1f / 1))``, contribution ``(double)t / 1.64493406685``.  Per chunk, over the query's
entries in ascending UTF-8 byte order: ``res = (float)((double)res + contribution)``; finally ``res = fl(res /
(float)size)`` with ``size`` the number of entries, known to the index or not.
"""

from __future__ import annotations

import numpy as np

F = np.float32
W_D = F(0.1)
PI2_6 = 1.64493406685
MAX_POS = 256


def contributions() -> np.ndarray:
    """float64 [256]: the contribution of an entry held with n = 1..256 positions."""
    out = np.zeros(MAX_POS, np.float64)
    resj = F(0.0)
    for j in range(MAX_POS):
        resj = F(resj + F(W_D / F((j + 1) * (j + 1))))
        t = F(F(W_D + resj) - F(W_D / F(1.0)))
        out[j] = np.float64(t) / PI2_6
    return out


CONTRIB = contributions()


def rank(nposes: list[int], size: int) -> np.float32:
    """``calc_rank_or`` of one chunk: ``nposes`` = the npos of each entry it holds, in entry order; ``size`` entries."""
    res = F(0.0)
    for n in nposes:
        res = F(np.float64(res) + CONTRIB[min(max(int(n), 1), MAX_POS) - 1])
    return F(res / F(size))


def ts_rank_table(table: dict[int, dict[str, int]], lexemes: list[str]) -> dict[int, np.float32]:
    """``ts_rank`` of every matching chunk of ``table`` (chunk -> {lexeme: npos}) for a query with the entries
    ``lexemes`` (distinct, any order: they are summed in UTF-8 byte order)."""
    entries = sorted(set(lexemes), key=lambda s: s.encode())
    out = {}
    for c, held in table.items():
        ns = [held[x] for x in entries if x in held]
        if ns:
            out[c] = rank(ns, len(entries))
    return out


def tsrank_csr_scores(term_off, doc, npos, q_off, q_terms, n_chunks):
    """``rl_tsrank_topk_global``'s scores over the CSR: ``(score float32 [B, C], matched bool [B, C])``, each chunk's
    sum over the entries in the given order."""
    term_off, q_off, q_terms = np.asarray(term_off, np.int64), np.asarray(q_off, np.int64), np.asarray(q_terms, np.int64)
    doc, npos = np.asarray(doc, np.int64), np.asarray(npos, np.int64)
    V, B = len(term_off) - 1, len(q_off) - 1
    res = np.zeros((B, n_chunks), np.float32)
    matched = np.zeros((B, n_chunks), bool)
    for q in range(B):
        for j in range(q_off[q], q_off[q + 1]):
            t = q_terms[j]
            if t < 0 or t >= V:
                continue
            d = doc[term_off[t]:term_off[t + 1]]
            c = CONTRIB[np.clip(npos[term_off[t]:term_off[t + 1]], 1, MAX_POS) - 1]
            res[q, d] = (res[q, d].astype(np.float64) + c).astype(np.float32)
            matched[q, d] = True
        size = q_off[q + 1] - q_off[q]
        if size:
            res[q] = res[q] / F(size)
    return res, matched


def tsrank_topk(scores, matched, mask, k, chunk_base=0):
    """The top k by (score desc, chunk asc) over the matched chunks ``mask`` allows, in the packed layout: ``(chunk
    int64 [B, k] (-1 padded, chunk_base added), score float64 [B, k] (the float32 widened, -inf padded), count [B])``."""
    B = len(scores)
    ids = np.full((B, k), -1, np.int64)
    out = np.full((B, k), -np.inf, np.float64)
    count = np.zeros(B, np.int32)
    for q in range(B):
        keep = matched[q] if mask is None else matched[q] & np.asarray(mask, bool)
        cand = np.flatnonzero(keep)
        top = cand[np.lexsort((cand, -scores[q][cand].astype(np.float64)))[:k]]
        n = len(top)
        ids[q, :n], out[q, :n], count[q] = top + chunk_base, scores[q][top], n
    return ids, out, count


def csr_from_table(table: dict[int, dict[str, int]], lexeme_ids: dict[str, int]):
    """``(term_off int64 [V + 1], doc int32 [P], npos int32 [P])`` of ``table`` under the ids ``lexeme_ids``."""
    V = len(lexeme_ids)
    per: list[list[tuple[int, int]]] = [[] for _ in range(V)]
    for c in sorted(table):
        for x, n in table[c].items():
            per[lexeme_ids[x]].append((c, n))
    term_off = np.concatenate([[0], np.cumsum([len(p) for p in per])]).astype(np.int64)
    doc = np.asarray([c for p in per for c, _ in p], np.int32)
    npos = np.asarray([n for p in per for _, n in p], np.int32)
    return term_off, doc, npos


def tsvector_text(held: dict[str, list[int]]) -> str:
    """PostgreSQL's text output of a tsvector: lexemes in byte order, ``'`` and ``\\`` doubled, positions listed (an
    empty list: a stripped lexeme)."""
    parts = []
    for x in sorted(held, key=lambda s: s.encode()):
        q = "'" + x.replace("\\", "\\\\").replace("'", "''") + "'"
        parts.append(q + (":" + ",".join(str(p) for p in held[x]) if held[x] else ""))
    return " ".join(parts)


def make_tsvectors(n: int, seed: int, *, vocab: list[str], max_words: int = 60, max_npos: int = 300):
    """Seeded chunk tsvectors: ``(texts [n], table chunk -> {lexeme: npos})``.  Zipf lexemes of ``vocab``; a few lexemes
    repeated up to ``max_npos`` times (positions capped at 256, as PostgreSQL does), some chunks empty, some stripped."""
    rng = np.random.default_rng(seed)
    p = 1.0 / np.arange(1, len(vocab) + 1) ** 1.07
    p /= p.sum()
    texts, table = [], {}
    for c in range(n):
        m = int(rng.integers(0, max_words + 1)) if rng.random() > 0.03 else 0
        words = [vocab[i] for i in rng.choice(len(vocab), size=m, p=p)]
        if m and rng.random() < 0.05:
            words += [words[0]] * int(rng.integers(1, max_npos))
        held: dict[str, list[int]] = {}
        for i, w in enumerate(words):
            held.setdefault(w, []).append(min(i + 1, 16383))
        held = {w: sorted(set(ps))[:MAX_POS] for w, ps in held.items()}
        stripped = rng.random() < 0.02
        texts.append(tsvector_text({w: [] for w in held} if stripped else held))
        table[c] = {w: (1 if stripped else len(ps)) for w, ps in held.items()}
    return texts, table
