"""The cross-encoder's attention step (``rl_xenc_attention``: the same setup and launches as ``rl_xenc_score``)
against float64, element by element."""

from __future__ import annotations

import json
import tempfile
import time
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HEAD_DIM = 32
GUARD_ROWS = 512          # NaN rows behind the T real rows of qkv and ctx
LENGTHS = (1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, 129, 200, 255, 256, 257, 300, 383, 384, 385,
           511, 512)
PATTERNS = ("gauss", "peaked", "uniform", "negative")


def _record(name: str, payload: dict) -> None:
    """Append a line (case + measured error) to xenc_bounds.jsonl in the temporary directory."""
    with (Path(tempfile.gettempdir()) / "xenc_bounds.jsonl").open("a") as f:
        f.write(json.dumps({"test": name, **payload}) + "\n")


def _fill(Q, K, V, t0, L, pattern, g):
    """Write one sequence's Q, K, V ([L, heads, 32] slices starting at row t0) for a value pattern."""
    import torch

    nh = Q.shape[1]
    dev = Q.device
    sl = slice(t0, t0 + L)
    V[sl] = torch.randn((L, nh, HEAD_DIM), generator=g, device=dev)
    if pattern == "gauss":
        Q[sl] = torch.randn((L, nh, HEAD_DIM), generator=g, device=dev)
        K[sl] = torch.randn((L, nh, HEAD_DIM), generator=g, device=dev)
    elif pattern == "peaked":
        # Query i of head h aims at key tgt[i, h] with logit 40; every other logit is ~N(0, 7^2).  The target lies
        # past the first 64-key block whenever there is one, often in the 32-key tail block, so the running maximum
        # rises after the first block (the O / l rescale decides the result).
        k = torch.randn((L, nh, HEAD_DIM), generator=g, device=dev)
        lo = 64 if L > 64 else L // 2
        tgt = lo + torch.randint(0, L - lo, (L, nh), generator=g, device=dev)
        kt = k.gather(0, tgt[..., None].expand(L, nh, HEAD_DIM))
        K[sl] = k
        Q[sl] = 40.0 * HEAD_DIM**0.5 * kt / (kt * kt).sum(-1, keepdim=True)
    elif pattern == "uniform":
        Q[sl] = torch.randn((L, nh, HEAD_DIM), generator=g, device=dev)
        K[sl] = torch.randn((1, nh, HEAD_DIM), generator=g, device=dev).expand(L, nh, HEAD_DIM)
    else:
        # Every valid logit near -30 and V with mean 3: a padding key (score 0, V = 0) left unmasked would take
        # almost all the weight and pull the output towards 0.
        u = torch.randint(0, 2, (1, nh, HEAD_DIM), generator=g, device=dev).float() * 2 - 1
        Q[sl] = 2.3 * u + 0.3 * torch.randn((L, nh, HEAD_DIM), generator=g, device=dev)
        K[sl] = -2.3 * u + 0.3 * torch.randn((L, nh, HEAD_DIM), generator=g, device=dev)
        V[sl] += 3.0


def _run_case(lib, name, hidden, lengths, patterns, seed):
    """One packed call of ``rl_xenc_attention``; every element of ctx against the float64 reference.  Returns the
    largest |err| / bound."""
    import torch

    nh = hidden // HEAD_DIM
    dev = torch.device("cuda")
    g = torch.Generator(device="cuda").manual_seed(seed)
    lens = np.asarray(lengths, dtype=np.int64)
    P, T, max_len = len(lens), int(lens.sum()), int(lens.max())
    cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    Q = torch.empty((T, nh, HEAD_DIM), device=dev)
    K, V = torch.empty_like(Q), torch.empty_like(Q)
    for s in range(P):
        _fill(Q, K, V, int(cu[s]), int(lens[s]), patterns[s], g)
    qkv = torch.full((T + GUARD_ROWS, 3 * hidden), float("nan"), dtype=torch.float16, device=dev)
    qkv[:T] = torch.cat([Q.reshape(T, hidden), K.reshape(T, hidden), V.reshape(T, hidden)], dim=1).half()
    ctx = torch.full((T + GUARD_ROWS, hidden), float("nan"), dtype=torch.float16, device=dev)
    d_cu = torch.from_numpy(cu).to(dev)
    ws = torch.empty(4 * P + 16, dtype=torch.uint8, device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    rc = lib.rl_xenc_attention(qkv.data_ptr(), d_cu.data_ptr(), P, T, max_len, hidden, nh, ctx.data_ptr(), ws.data_ptr(),
                               ws.numel(), stream)
    assert rc == 0, lib.rl_last_error()
    torch.cuda.synchronize()
    assert torch.isnan(ctx[T:]).all(), f"{name}: ctx written past row T"
    # float64 reference from the fp16 values the kernel reads, sequences of one length batched together
    q16 = qkv[:T].double().reshape(T, 3, nh, HEAD_DIM)
    got = ctx[:T].double().reshape(T, nh, HEAD_DIM)
    worst = {p: 0.0 for p in PATTERNS}                          # largest |err| / bound per value pattern
    first_fail = {}
    for L in sorted(set(lens.tolist())):
        seqs = np.nonzero(lens == L)[0]
        per = max(1, int(2**28 // (nh * L * L * 8)))          # at most ~256 MB per score tensor
        for c0 in range(0, len(seqs), per):
            part = seqs[c0:c0 + per]
            rows = torch.from_numpy(cu[part][:, None] + np.arange(L)[None, :]).to(dev).long()   # [n, L]
            x = q16[rows].permute(0, 2, 3, 1, 4)                # [n, L, 3, nh, 32] -> [n, 3, nh, L, 32]
            q, k, v = x[:, 0], x[:, 1], x[:, 2]
            p = torch.softmax(q @ k.transpose(-1, -2) / HEAD_DIM**0.5, dim=-1)   # [n, nh, L, L]
            ref = p @ v
            A = p @ v.abs()
            dz = 2.0**-18 * (q.abs() @ k.abs().transpose(-1, -2)).amax(-1, keepdim=True) / HEAD_DIM**0.5 + 2.0**-20
            vmax = v.abs().amax(-2, keepdim=True)
            bound = 2.0**-11 * ref.abs() + (2.0**-11 + L * 2.0**-23 + 2.1 * dz) * A + L * 2.0**-25 * vmax + 1e-6
            o = got[rows].permute(0, 2, 1, 3)                   # [n, nh, L, 32]
            assert torch.isfinite(o).all(), f"{name}: non-finite output at L={L}"
            r = (o - ref).abs() / bound
            r_seq = r.flatten(1).amax(1).tolist()
            for n_i, s in enumerate(part.tolist()):
                pat = patterns[s]
                worst[pat] = max(worst[pat], r_seq[n_i])
                if r_seq[n_i] > 1.0 and pat not in first_fail:
                    h, i, d = np.unravel_index(int(r[n_i].argmax()), tuple(r[n_i].shape))
                    first_fail[pat] = (f"sequence {s} (L={L}), head {h}, row {i}, column {d}: got "
                                       f"{float(o[n_i, h, i, d]):.6g}, want {float(ref[n_i, h, i, d]):.6g}")
    if first_fail:
        pytest.fail(f"{name}: |err| / bound per pattern {({p: float(f'{w:.3g}') for p, w in worst.items()})}; first "
                    "failures: " + "; ".join(f"{p}: {msg}" for p, msg in first_fail.items()))
    return max(worst.values())


def test_attention_matches_float64():
    """``ctx = softmax(Q K^T / sqrt(32)) V`` per sequence and head, every element of rows < T, against float64 from
    the fp16 Q, K, V.  Per element, with A = sum p |v| / sum p, dz = 2^-18 max_j sum_t |q_t k_jt| / sqrt(32) + 2^-20:

        |o - ref| <= 2^-11 |ref| + (2^-11 + L 2^-23 + 2.1 dz) A + L 2^-25 max|v| + 1e-6

    - 2^-11 |ref|: the fp16 output.
    - 2^-11 A and L 2^-25 max|v|: P is rounded to fp16 for the P V product while l sums the unrounded values
      (relative 2^-11, absolute 2^-25 below fp16's normal range, and sum p >= 1 because the row maximum has p = 1).
    - L 2^-23 A: fp32 accumulation of O (tensor-core MMAs) and of l over up to L keys, and the rescales.
    - 2.1 dz A: a relative error dz of a weight moves the output by at most 2 dz A.  dz covers the fp32
      accumulation of the 32-term score (2^-18 = 32 * 2^-23 of sum |q k|, in logit units), and the fmaf, the
      rounded scale and ex2.approx in the exponent (2^-20).  The running maximum's own rounding cancels: every
      weight and every rescale is taken against the same stored maximum.
    - 1e-6: outputs below fp16's normal range.

    Value patterns per sequence: Gaussian; peaked logits (+-40) whose row maximum lies past the first key block;
    all keys equal (uniform weights); every logit near -30 with V of mean 3 (an unmasked padding key would dominate).
    qkv holds 512 NaN rows behind the T real rows and ctx is NaN-filled: K / V reads past a sequence, unwritten
    rows and writes past T show up."""
    import torch

    from raglite_b200 import _lib

    lib = _lib.load()
    torch.cuda.set_device(0)
    rng = np.random.default_rng(0)
    cases = []
    for hidden in (384, 160, 512, 32):
        # every length with every pattern, twice: equal lengths tie in the longest-first counting sort
        lengths = [L for L in LENGTHS for _ in range(2 * len(PATTERNS))]
        patterns = [PATTERNS[i % len(PATTERNS)] for i in range(len(lengths))]
        cases.append((f"h{hidden}_max512", hidden, lengths, patterns))
    short = [L for L in LENGTHS if L <= 256]                        # max_len <= 256: K / V of 256 keys fill the smem
    cases.append(("h384_max256", 384, [L for L in short for _ in range(len(PATTERNS))],
                  [p for _ in short for p in PATTERNS]))
    many = rng.choice([1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65], size=1100)   # P > 1024: seq_order_kernel loops
    many[rng.integers(0, len(many))] = 300                           # and one long sequence (sorted first)
    cases.append(("h384_p1100", 384, many.tolist(), [PATTERNS[i % len(PATTERNS)] for i in range(len(many))]))
    worst_all = 0.0
    for seed, (name, hidden, lengths, patterns) in enumerate(cases):
        order = rng.permutation(len(lengths))                        # shuffled: long and short sequences interleave
        lengths, patterns = [lengths[i] for i in order], [patterns[i] for i in order]
        t = time.perf_counter()
        worst = _run_case(lib, name, hidden, lengths, patterns, seed)
        _record("attention", {"case": name, "sequences": len(lengths), "tokens": int(sum(lengths)),
                              "max_err_over_bound": worst, "seconds": round(time.perf_counter() - t, 2)})
        worst_all = max(worst_all, worst)
    assert worst_all <= 1.0
