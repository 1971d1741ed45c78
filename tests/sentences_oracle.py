"""Float64 / plain-loop restatements of ``split_sentences`` (TEST INFRASTRUCTURE).

* ``sat_probas_f64``: wtpsplit's ``predict_proba(doc, stride=128, block_size=256, weighting="hat")`` as recalled in
  ``raglite_b200/_sentences.py`` (blocks, hat weights, token -> character map, sigmoid), with a ``transformers``
  ``XLMRobertaForTokenClassification`` run block by block in float64.  Every rule is written again here as a loop.
* ``split_sentences_post``: the reference's post-processing (``_split_sentences.py:183-219`` and ``:56-143``) step by
  step: the override, the whitespace-run propagation, the two dynamic programs with NumPy float32 scores and float64 dp.
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
