"""Float64 / plain-loop restatements of ``split_sentences`` (TEST INFRASTRUCTURE).

* ``sat_probas_f64``: wtpsplit's ``predict_proba(doc, stride=128, block_size=256, weighting="hat")`` as recalled in
  ``raglite_b200/_sentences.py`` (blocks, hat weights, token -> character map, sigmoid), with a ``transformers``
  ``XLMRobertaForTokenClassification`` run block by block in float64.  Every rule is written again here as a loop.
* ``split_sentences_post``: the reference's post-processing (``_split_sentences.py:183-219`` and ``:56-143``) step by
  step: the override, the whitespace-run propagation, the two dynamic programs with NumPy float32 scores and float64 dp.
* The device kernels of ``csrc/sentences.cu`` restated in their own float32 order, for bit-exact checks at the C-ABI:
  ``fmaf`` and ``sat_head`` (``rl_sat_token_logits``), ``sat_char_logits`` and ``propagate_runs``
  (``rl_sat_char_probas`` up to and after its sigmoid), ``partition_cuts`` (``rl_sentence_partition``).
"""

from __future__ import annotations

from collections import deque

import numpy as np

BLOCK_SIZE, STRIDE = 256, 128
SKIP_PIECES = ("<s>", "</s>", "<pad>", "▁")
PARTITION_FAILED = "Sentence partition failed: no valid split satisfies the constraints."


# ---- item by item, as loops ---------------------------------------------------------------------------------------------
def plan_loop(T: int, block_size: int = BLOCK_SIZE, stride: int = STRIDE) -> tuple[int, list[int]]:
    if T == 0:
        return 0, []
    B = min(block_size - 2, T)
    starts = []
    k = 0
    while True:
        s = k * stride
        if s + B >= T:
            starts.append(T - B)
            return B, starts
        starts.append(s)
        k += 1


def hat_loop(B: int) -> np.ndarray:
    lo, hi = -(1 - 1 / B), 1 - 1 / B
    w = []
    for k in range(B):
        x = lo + k * ((hi - lo) / (B - 1)) if B > 1 else lo
        if B > 1 and k == B - 1:
            x = hi
        w.append(1 - abs(x))
    return np.array(w, dtype=np.float32)


def char_targets_loop(ends, skip, n: int) -> list[int]:   # noqa: ANN001
    owner: dict[int, int] = {}
    for i, (e, s) in enumerate(zip(ends, skip, strict=True)):
        if not s:
            c = int(e) - 1
            owner[c + n if c < 0 else c] = i
    out = [-1] * len(ends)
    for c, i in owner.items():
        out[i] = c
    return out


def sat_probas_f64(model, tokenizer, doc: str) -> np.ndarray:  # noqa: ANN001
    """float64 character probabilities of one document; ``model`` an ``XLMRobertaForTokenClassification``."""
    import copy

    import torch

    enc = tokenizer.encode(doc, add_special_tokens=False)
    ids, T = list(enc.ids), len(enc.ids)
    if T == 0:
        return np.zeros(len(doc))
    bos, eos = tokenizer.token_to_id("<s>"), tokenizer.token_to_id("</s>")
    B, starts = plan_loop(T)
    w = hat_loop(B).astype(np.float64)
    m = copy.deepcopy(model).double().eval()
    NL = int(m.config.num_labels)
    num, den = np.zeros((T, NL)), np.zeros(T)
    with torch.no_grad():
        for s in starts:
            x = torch.tensor([[bos, *ids[s:s + B], eos]])
            lg = m(input_ids=x, attention_mask=torch.ones_like(x)).logits[0, 1:B + 1].numpy()
            for k in range(B):
                num[s + k] += w[k] * lg[k]
                den[s + k] += w[k]
    stitched = num / den[:, None]
    logit = np.full(len(doc), stitched.min())
    skip_ids = {tokenizer.token_to_id(p) for p in SKIP_PIECES}
    tgt = char_targets_loop([e for _, e in enc.offsets], [i in skip_ids for i in ids], len(doc))
    for t, c in enumerate(tgt):
        if c >= 0:
            logit[c] = stitched[t, 0]
    return 1 / (1 + np.exp(-logit))


# ---- the reference's post-processing --------------------------------------------------------------------------------------
def _partition(probas: np.ndarray, n: int, min_len: int, max_len: int | None) -> list[int] | None:
    """Boundaries (last character of each sentence but the final one) of ``_split_sentences``; None = one sentence.
    Raises the reference's ValueError."""
    lo, hi = min_len - 1, n - min_len - 1
    if hi < lo:
        return None
    score = probas - 0.25                      # float32, as NumPy computes it
    dp = np.full(n, -np.inf)
    back = np.full(n, -1, dtype=np.intp)
    if max_len is None:
        run, run_at = -np.inf, -1
        for i in range(lo, hi + 1):
            j = i - min_len
            if j >= lo and dp[j] > run:
                run, run_at = dp[j], j
            dp[i] = score[i]
            if run > -np.inf and run + score[i] > dp[i]:
                dp[i], back[i] = run + score[i], run_at
    else:
        window: deque[tuple[float, int]] = deque()
        for i in range(lo, hi + 1):
            j = i - min_len
            if j >= lo and np.isfinite(dp[j]):
                while window and window[-1][0] <= dp[j]:
                    window.pop()
                window.append((dp[j], j))
            while window and window[0][1] < i - max_len:
                window.popleft()
            if i + 1 <= max_len:
                dp[i] = score[i]
            if window and window[0][0] + score[i] > dp[i]:
                dp[i], back[i] = window[0][0] + score[i], window[0][1]
    first = lo if max_len is None else max(lo, n - max_len - 1)
    whole_ok = max_len is None or max_len >= n
    best, last = (0.0 if whole_ok else -np.inf), -1
    for i in range(first, hi + 1):
        if dp[i] > best:
            best, last = dp[i], i
    if last == -1:
        if whole_ok:
            return None
        raise ValueError(PARTITION_FAILED)
    out = []
    while last >= 0:
        out.append(last)
        last = back[last]
    return out[::-1]


def _cut(doc: str, bounds: list[int] | None) -> list[str]:
    if bounds is None:
        return [doc]
    edges = [0, *[b + 1 for b in bounds], len(doc)]
    return [doc[a:e] for a, e in zip(edges[:-1], edges[1:], strict=True)]


def propagate(doc: str, probas: np.ndarray) -> np.ndarray:
    """The whitespace-run step on a copy: for each run bounded by non-space characters on both sides."""
    p = probas.copy()
    sp = [c.isspace() for c in doc]
    i = 0
    while i < len(doc) - 1:
        if not sp[i] and sp[i + 1]:
            j = i + 1
            while j < len(doc) and sp[j]:
                j += 1
            if j < len(doc):
                seg = p[i:j]
                mn, mx = np.min(seg), np.max(seg)
                p[i:j - 1] = mn
                p[j - 1] = mx
            i = j
        else:
            i += 1
    return p


def split_sentences_post(doc: str, predicted: np.ndarray, *, min_len: int = 4, max_len: int | None = None,
                         known: np.ndarray | None = None) -> list[str]:
    """``split_sentences(doc, min_len, max_len, boundary_probas=known)`` with ``predicted`` in place of SaT's output
    (``known`` None: the Markdown headings' probabilities of ``markdown_boundaries``)."""
    if len(doc) <= min_len:
        return [doc]
    if known is None:
        known = markdown_boundaries(doc)
    p = np.asarray(predicted, dtype=np.float32).copy()
    fin = np.isfinite(known)
    p[fin] = known[fin]
    p = propagate(doc, p)
    sentences = _cut(doc, _partition(p, len(doc), min_len, None))
    if max_len is None:
        return sentences
    out, pos = [], 0
    for s in sentences:
        out.extend([s] if len(s) <= max_len else _cut(s, _partition(p[pos:pos + len(s)], len(s), min_len, max_len)))
        pos += len(s)
    return out


def partition_cuts(p: np.ndarray, n: int, min_len: int, max_len: int | None) -> list[int]:
    """The cut indices (sentence starts after the first) that ``rl_sentence_partition`` writes for one document of n
    characters with final probabilities ``p``: stage 1 with no maximum, then stage 2 on every stage-1 sentence longer
    than ``max_len`` (None or 0: none), as ``split_sentences_post`` runs them.  Raises the reference's ValueError."""
    cuts = [b + 1 for b in _partition(p, n, min_len, None) or []]
    if not max_len:
        return cuts
    out = []
    for s, (a, e) in enumerate(zip([0, *cuts], [*cuts, n], strict=True)):
        if e - a > max_len:
            out += [a + b + 1 for b in _partition(p[a:e], e - a, min_len, max_len) or []]
        if s < len(cuts):
            out.append(e)
    return out


# ---- the device kernels, in their own float32 order --------------------------------------------------------------------
def fmaf(a, b, c) -> np.ndarray:  # noqa: ANN001
    """IEEE ``fmaf(a, b, c)`` of float32 arrays: a b + c rounded once.  The float64 product of two float32 values is
    exact; TwoSum gives s + e = a b + c exactly; s rounded to float32 is the answer except when s lies exactly halfway
    between two float32 values and e != 0, where the exact sum is on e's side of the midpoint."""
    a, b, c = (np.asarray(x, np.float32).astype(np.float64) for x in (a, b, c))
    p = a * b
    s = p + c
    bp = s - c
    e = (p - bp) + (c - (s - bp))
    r = s.astype(np.float32)
    r64 = r.astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        other = np.nextafter(r, np.where(r64 < s, np.float32(np.inf), np.float32(-np.inf)))
        mid = (r64 != s) & ((r64 + other.astype(np.float64)) / 2 == s)
    toward = mid & (e != 0) & ((e > 0) == (s > r64))
    return np.where(toward, other, r).astype(np.float32)


def sat_head(hidden: np.ndarray, W: np.ndarray, bias: np.ndarray) -> np.ndarray:
    """``sat_head_kernel``: lane l of a row's warp runs ``acc = fmaf(h[k], w[k], acc)`` over k = l, l + 32, ...; the
    butterfly adds lane l ^ o for o = 16 ... 1; lane 0 adds the bias.  float32 [rows, NL]."""
    R, H = hidden.shape
    out = np.empty((R, len(bias)), np.float32)
    lanes = np.arange(32)
    for lab in range(len(bias)):
        acc = np.zeros((R, 32), np.float32)
        for k0 in range(0, H, 32):
            k = (k0 + lanes)[k0 + lanes < H]
            acc[:, :len(k)] = fmaf(hidden[:, k], W[lab, k][None, :], acc[:, :len(k)])
        for o in (16, 8, 4, 2, 1):
            acc = acc + acc[:, lanes ^ o]
        out[:, lab] = acc[:, 0] + bias[lab]
    return out


def sat_char_logits(logits: np.ndarray, doc_tok_off: np.ndarray, doc_char_off: np.ndarray, doc_block: np.ndarray,
                    blk_off: np.ndarray, blk_start: np.ndarray, blk_row: np.ndarray, hat: np.ndarray,
                    tok_char: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """``rl_sat_char_probas`` before its sigmoid: (the logit of every character, the stitched logits [T, NL]).

    A token t of document d takes the blocks b of d with start <= t < start + B in ascending order, and sums
    fl(w_k lg) and w_k in float32 (k = t - start, w_k = hat[B (B - 1) / 2 + k]), then divides once.  A document's
    characters get the minimum stitched logit over its tokens and labels (-inf without tokens); each token with
    ``tok_char >= 0`` then writes its label-0 logit there."""
    NL, D = logits.shape[1], len(doc_block)
    T, N = int(doc_tok_off[-1]), int(doc_char_off[-1])
    tok_doc = np.repeat(np.arange(D), np.diff(doc_tok_off))
    t = np.arange(T, dtype=np.int64) - doc_tok_off[tok_doc]
    B = doc_block[tok_doc].astype(np.int64)
    blk_doc = np.repeat(np.arange(D), np.diff(blk_off))
    starts = blk_start.astype(np.int64)
    key = (blk_doc.astype(np.int64) << 32) + starts + 1024            # ascending: documents in order, starts within
    b = np.searchsorted(key, (tok_doc.astype(np.int64) << 32) + t - B + 1024, side="right")   # first start > t - B
    end = blk_off[tok_doc + 1]
    num, den = np.zeros((T, NL), np.float32), np.zeros(T, np.float32)
    live = np.nonzero(b < end)[0]
    live = live[starts[b[live]] <= t[live]]
    while len(live):
        bb = b[live]
        k = t[live] - starts[bb]
        wk = hat[B[live] * (B[live] - 1) // 2 + k]
        num[live] = num[live] + wk[:, None] * logits[blk_row[bb] + k]
        den[live] = den[live] + wk
        b[live] += 1
        live = live[b[live] < end[live]]
        live = live[starts[b[live]] <= t[live]]
    with np.errstate(divide="ignore", invalid="ignore"):
        stitched = num / den[:, None]
    dmin = np.full(D, -np.inf, np.float32)
    has = np.diff(doc_tok_off) > 0
    if has.any():
        dmin[has] = np.minimum.reduceat(stitched.min(axis=1), doc_tok_off[:-1][has])
    char_doc = np.searchsorted(doc_char_off, np.arange(N), side="right") - 1
    out = dmin[char_doc]
    hit = tok_char >= 0
    out[tok_char[hit]] = stitched[hit, 0]
    return out, stitched


def propagate_runs(p: np.ndarray, is_space: np.ndarray, doc_char_off: np.ndarray) -> np.ndarray:
    """``propagate`` over a batch at once, from the whitespace flags: for each run of spaces after a non-space character
    i and before the first non-space j of the same document, p[i .. j-2] = min(p[i .. j-1]), p[j-1] = max(...)."""
    N = len(p)
    sp = np.asarray(is_space, dtype=bool)
    out = p.copy()
    i = np.nonzero(~sp[:-1] & sp[1:])[0]
    ns = np.nonzero(~sp)[0]
    at = np.searchsorted(ns, i + 1)
    j = np.where(at < len(ns), ns[np.minimum(at, len(ns) - 1)], N)
    doc_end = doc_char_off[np.searchsorted(doc_char_off, i, side="right")]
    keep = j < doc_end
    i, j = i[keep], j[keep]
    if not len(i):
        return out
    ext = np.append(p, p.dtype.type(0))
    idx = np.ravel(np.column_stack([i, j]))
    mn, mx = np.minimum.reduceat(ext, idx)[::2], np.maximum.reduceat(ext, idx)[::2]
    L = j - i - 1                                                       # p[i .. j-2] takes the minimum
    pos = np.repeat(i, L) + (np.arange(L.sum()) - np.repeat(np.cumsum(L) - L, L))
    out[pos] = np.repeat(mn, L)
    out[j - 1] = mx
    return out


def markdown_boundaries(doc: str) -> np.ndarray:
    """NaN / 0 / 1 per character from the heading_open tokens of markdown-it, line spans over ``str.splitlines``."""
    from markdown_it import MarkdownIt

    starts = [0]
    for line in doc.splitlines(keepends=True):
        starts.append(starts[-1] + len(line))
    out = np.full(len(doc), np.nan)
    for tok in MarkdownIt().parse(doc):
        if tok.type != "heading_open":
            continue
        a, e = starts[tok.map[0]], starts[tok.map[1]] + 1
        if a >= 1 and a - 1 < len(doc):
            out[a - 1] = 1.0
        for c in range(a, min(e - 1, len(doc))):
            out[c] = 0.0
        if 0 <= e - 1 < len(doc):
            out[e - 1] = 1.0
    return out
