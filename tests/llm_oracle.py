"""NumPy statements of the decoder's steps: the sampler chain token for token (float32, in the device's order), and
float64 references of QK-norm + NEOX RoPE and causal GQA attention."""

from __future__ import annotations

import numpy as np


def sample(logits: np.ndarray, hist: list[int], *, temperature: float, top_k: int, top_p: float, min_p: float,
           penalty: float, u: float) -> int:
    """llama-cpp-python's chain at RAGLite's parameters: repeat penalty over the distinct ids of ``hist``, top-k
    (ties by ascending id), top-p on the softmax at temperature 1 (the crossing token kept), min-p, temperature, the
    inverse CDF at ``u``.  ``temperature == 0``: argmax after the penalty, lowest id on ties."""
    w = np.asarray(logits, dtype=np.float32).copy()
    for t in dict.fromkeys(int(h) for h in hist):
        if 0 <= t < len(w):
            w[t] = w[t] * np.float32(penalty) if w[t] <= 0 else w[t] / np.float32(penalty)
    k = 1 if temperature == 0 else min(top_k, len(w))
    order = np.lexsort((np.arange(len(w)), -w.astype(np.float64)))[:k]
    cl, ci = w[order], order
    if temperature == 0:
        return int(ci[0])
    n = k
    if top_p < 1:
        e = np.exp(cl - cl[0]).astype(np.float32)
        s = np.float32(0)
        for x in e:
            s = np.float32(s + x)
        cum = np.float32(0)
        for i in range(n):
            cum = np.float32(cum + np.float32(e[i] / s))
            if cum >= np.float32(top_p):
                n = i + 1
                break
    if min_p > 0:
        cut = np.float32(cl[0] + np.float32(np.log(np.float32(min_p))))
        m = 1
        while m < n and cl[m] >= cut:
            m += 1
        n = m
    z = (cl[:n] / np.float32(temperature)).astype(np.float32)
    e = np.exp(z - z[0]).astype(np.float32)
    s = np.float32(0)
    for x in e:
        s = np.float32(s + x)
    target = np.float32(np.float32(u) * s)
    cum = np.float32(0)
    for i in range(n):
        cum = np.float32(cum + e[i])
        if target < cum:
            return int(ci[i])
    return int(ci[n - 1])


def sample_margin(logits: np.ndarray, hist: list[int], u: float, **kw: float) -> float:
    """How far ``u`` lies from the nearest CDF boundary of the draw (float64): a draw closer than a few float32 ulps
    may differ between exp implementations."""
    w = np.asarray(logits, dtype=np.float64).copy()
    pen = kw["penalty"]
    for t in dict.fromkeys(int(h) for h in hist):
        w[t] = w[t] * pen if w[t] <= 0 else w[t] / pen
    order = np.lexsort((np.arange(len(w)), -w))[:kw["top_k"]]
    cl = w[order]
    e = np.exp(cl - cl[0])
    p = np.cumsum(e / e.sum())
    n = int(np.searchsorted(p, kw["top_p"] - 1e-9) + 1) if kw["top_p"] < 1 else len(cl)
    z = cl[:n] / kw["temperature"]
    q = np.cumsum(np.exp(z - z[0]))
    q /= q[-1]
    return float(np.min(np.abs(q - u)))


def rope_ref(x: np.ndarray, pos: np.ndarray, base: float) -> np.ndarray:
    """NEOX rotation of x [..., 128] at positions pos (float64): pairs (i, i + 64), angle pos / base^(2 i / 128)."""
    i = np.arange(64, dtype=np.float64)
    ang = pos[..., None].astype(np.float64) / base ** (2 * i / 128)
    c, s = np.cos(ang), np.sin(ang)
    a, b = x[..., :64], x[..., 64:]
    return np.concatenate([a * c - b * s, b * c + a * s], axis=-1)


def rms_norm_ref(x: np.ndarray, w: np.ndarray, eps: float) -> np.ndarray:
    x = x.astype(np.float64)
    return x / np.sqrt((x * x).mean(-1, keepdims=True) + eps) * w.astype(np.float64)


def attention_ref(q: np.ndarray, k: np.ndarray, v: np.ndarray, p0: int) -> np.ndarray:
    """q [T, n_head, 128] at positions p0 + t; k, v [n_keys, n_kv, 128]; head h reads KV head h // group (float64)."""
    T, nh, _ = q.shape
    nkv = k.shape[1]
    G = nh // nkv
    out = np.zeros((T, nh, 128))
    for t in range(T):
        L = p0 + t + 1
        for h in range(nh):
            s = k[:L, h // G].astype(np.float64) @ q[t, h].astype(np.float64) / np.sqrt(128.0)
            p = np.exp(s - s.max())
            out[t, h] = (p / p.sum()) @ v[:L, h // G].astype(np.float64)
    return out
