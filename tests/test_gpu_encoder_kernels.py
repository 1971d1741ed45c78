"""The encoder's LayerNorms and classifier head (``csrc/xenc.cu``) one kernel at a time against float64, through the test
hooks that call the forward's own launch functions (``rl_xenc_embed_ln``, ``rl_xenc_add_ln``, ``rl_xenc_cls_head``), and
the whole forward as exactly the chain of those hooks, ``rl_xenc_linear`` and the attention hooks, bit for bit.

Each test appends its worst |err| / bound (fp32 outputs) or its two-value count (fp16 outputs, ``tests/rounding.py``)
to ``xenc_bounds.jsonl`` in the temporary directory."""

from __future__ import annotations

import ctypes as C
import json
import tempfile
import time
from pathlib import Path

import numpy as np
import pytest
import rounding as rd

pytestmark = pytest.mark.gpu

U = 2.0**-24                          # unit roundoff of float32
GUARD = 8                             # NaN rows / entries behind every output and behind gamma / beta
HS = (32, 160, 384, 512, 544, 768, 800, 1024)   # NC 16 / 32 x vectorised (H % 128 == 0) / scalar
EPS = (1e-12, 1e-5)                   # BERT's and XLM-RoBERTa's ln_eps
PATTERNS = ("gauss", "cancel", "var1e-6", "var1e-5", "var1e-4", "const", "big")


def _record(name: str, payload: dict) -> None:
    with (Path(tempfile.gettempdir()) / "xenc_bounds.jsonl").open("a") as f:
        f.write(json.dumps({"test": name, **payload}) + "\n")


def _lib():
    from raglite_b200 import _lib

    return _lib.load()


def _stream() -> int:
    import torch

    return torch.cuda.current_stream().cuda_stream


def _ok(lib, rc: int) -> None:
    assert rc == 0, lib.rl_last_error()


# ---- LayerNorm reference ------------------------------------------------------------------------------------------
def _kernel_mean(x32: np.ndarray, vec: bool) -> np.ndarray:
    """The kernel's fp32 row mean of x32 [T, H] (float32), reproduced exactly: each lane sums its columns in order
    (scalar path: columns lane + 32 i; vectorised path: pieces (x0 + x1) + (x2 + x3) of columns 128 i + 4 lane + 0..3),
    ``warp_sum_f``'s butterfly adds lane l ^ o for o = 16 ... 1, then one IEEE division by H.  A chain of fp32 additions
    in a fixed order cannot be contracted or reassociated, so numpy's float32 gives the kernel's bits."""
    T, H = x32.shape
    if vec:
        p = x32.reshape(T, H // 128, 32, 4)
        pieces = (p[..., 0] + p[..., 1]) + (p[..., 2] + p[..., 3])
    else:
        pieces = x32.reshape(T, H // 32, 32)
    s = np.zeros((T, 32), np.float32)
    for i in range(pieces.shape[1]):
        s = s + pieces[:, i]
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        s = s + s[:, lanes ^ o]
    return s[:, 0] / np.float32(H)


def _ln_reference(x32: np.ndarray, vec: bool, g: np.ndarray, b: np.ndarray, eps: float):
    """float64 ``v = (x - mean) r g + beta`` with the kernel's fp32 mean and ``r = 1 / sqrt(sum (x - mean)^2 / H + eps)``
    (eps as the fp32 the kernel receives), and the bound ``bnd`` on the kernel's fp32 value (see the add_ln docstring)."""
    T, H = x32.shape
    mu = _kernel_mean(x32, vec).astype(np.float64)[:, None]
    d = x32.astype(np.float64) - mu
    S = (d * d).sum(1, keepdims=True)
    e32 = float(np.float32(eps))
    var = S / H + e32
    r = 1.0 / np.sqrt(var)
    g64, b64 = g.astype(np.float64)[None], b.astype(np.float64)[None]
    v = d * r * g64 + b64
    A = np.abs(d) * r * np.abs(g64)
    eps_v = (H // 32 + 7) * U * (S / H) / var + 2 * U
    eps_r = 0.5 * eps_v + 2.0**-22
    bnd = (A * (3 * U + eps_r) + U * np.abs(v)) * (1 + 2.0**-20)
    return v, bnd


def _rows(T: int, H: int, first: int, g):
    """x and res fp16 [T, H] on the device, row t of pattern PATTERNS[(first + t) % 7]:
    gauss: both N(0, 1); cancel: x = 200, res N(0, 0.01^2); var1e-*: both N(0, s^2 / 2), the row's variance s^2 below,
    at and above the two eps; const: x = c, res = 0 (variance exactly 0); big: |x| in [50 000, 65 504] with random signs,
    res N(0, 3000^2)."""
    import torch

    dev = torch.device("cuda")
    x = torch.empty((T, H), device=dev)
    r = torch.empty((T, H), device=dev)
    pats = [PATTERNS[(first + t) % len(PATTERNS)] for t in range(T)]
    for p in PATTERNS:
        idx = torch.tensor([t for t in range(T) if pats[t] == p], dtype=torch.long, device=dev)
        n = len(idx)
        if n == 0:
            continue
        if p == "gauss":
            xs, rs = torch.randn((n, H), generator=g, device=dev), torch.randn((n, H), generator=g, device=dev)
        elif p == "cancel":
            xs, rs = torch.full((n, H), 200.0, device=dev), 0.01 * torch.randn((n, H), generator=g, device=dev)
        elif p.startswith("var"):
            s = float(p[3:]) ** 0.5 / 2**0.5
            xs, rs = s * torch.randn((n, H), generator=g, device=dev), s * torch.randn((n, H), generator=g, device=dev)
        elif p == "const":
            c = torch.randint(-12, 13, (n, 1), generator=g, device=dev).float() * 0.375
            xs, rs = c.expand(n, H).clone(), torch.zeros((n, H), device=dev)
        else:
            sign = torch.randint(0, 2, (n, H), generator=g, device=dev).float() * 2 - 1
            xs = sign * (50000.0 + 15504.0 * torch.rand((n, H), generator=g, device=dev))
            rs = 3000.0 * torch.randn((n, H), generator=g, device=dev)
        x[idx], r[idx] = xs, rs
    return x.half(), r.half(), pats


def _gamma_beta(H: int, g):
    """fp32 gamma = 1 + N(0, 0.1^2), beta = N(0, 0.1^2) with GUARD NaN entries behind each (a read past column H shows)."""
    import torch

    gam = torch.full((H + 4 * GUARD,), float("nan"), device="cuda")
    bet = torch.full((H + 4 * GUARD,), float("nan"), device="cuda")
    gam[:H] = 1.0 + 0.1 * torch.randn(H, generator=g, device="cuda")
    bet[:H] = 0.1 * torch.randn(H, generator=g, device="cuda")
    return gam, bet


def test_add_ln_matches_float64():
    """``out = LayerNorm(x + res) gamma + beta`` of ``rl_xenc_add_ln`` against float64, every element of every row.

    The kernel (one warp per token): x_i = fp32(x + res) (reproduced in float32); the mean m = fp32 sum / H in the
    lane-sequential-then-butterfly order (reproduced bit for bit, ``_kernel_mean``: its worst-case bound alone would be
    (H/32 + 5) u mean|x|, about 1.4e-4 on the cancellation rows -- 14 fp16 steps of their outputs); d_i = x_i - m; the
    variance sum S of d_i^2 in the same order; r = rsqrtf(S / H + eps); y = (d r) g + beta.  Against
    v = (x - m) r g + beta in float64 with exact d and S (u = 2^-24, A = |d| r |g|):

    - S: d_i rounded (2u relative on d^2), the square rounded unless fused (u), H/32 - 1 lane additions and 5 butterfly
      levels, each within u of a partial sum <= S: (H/32 + 7) u S in all.  / H and + eps: one rounding each (2u).
    - r: half of S's relative error, weighted by S/H / (S/H + eps), plus rsqrtf's 2 ulp (2^-22 relative).
    - y: d (u), d r (u), (d r) g (u unless fused) and r's error, all on A; + beta rounds once (u |y|).

        |y - v| <= A (3u + eps_r) + u |v|   (x (1 + 2^-20) for second-order terms)

    fp32 outputs are held to that bound; fp16 outputs are the fp16 rounding of y, so ``rd.check`` holds them to
    f16(v -+ b) with the two-value count capped at 1 % (a loose bound fails).  Rows: Gaussian; x = 200 with res of
    sigma 0.01 (cancellation); variances 1e-6 / 1e-5 / 1e-4 against eps 1e-12 and 1e-5; constant rows, where the
    output must be exactly beta; |x| near the fp16 maximum.  H covers 16 and 32 columns per lane, vectorised and
    scalar; T = 1, 7, 9 and 1100 (blocks of 8 tokens: partial blocks).  In place (out == res, as the forward runs it)
    must give the out-of-place bits, fp16 out must be f16 of fp32 out bit for bit (the two instantiations share every
    operation before the store), and NaN guard rows behind T and NaN entries behind gamma / beta stay unread /
    unwritten."""
    import torch

    lib = _lib()
    torch.cuda.set_device(0)
    s = _stream()
    g = torch.Generator(device="cuda").manual_seed(0)
    worst32, two_max, cases = 0.0, (0, 1), 0
    t0 = time.perf_counter()
    for hi, H in enumerate(HS):
        vec = H % 128 == 0
        for ei, eps in enumerate(EPS):
            for T in (1, 7, 9, 1100):
                x, r, pats = _rows(T, H, first=3 * hi + ei + T, g=g)
                gam, bet = _gamma_beta(H, g)
                x32 = x.float().cpu().numpy() + r.float().cpu().numpy()   # fp32(x + res): one rounding, as the kernel
                v, bnd = _ln_reference(x32, vec, gam[:H].cpu().numpy(), bet[:H].cpu().numpy(), eps)
                what = f"add_ln H={H} eps={eps:g} T={T}"
                # fp32 out
                o32 = torch.full((T + GUARD, H), float("nan"), device="cuda")
                _ok(lib, lib.rl_xenc_add_ln(x.data_ptr(), r.data_ptr(), gam.data_ptr(), bet.data_ptr(), eps, T, H, 1,
                                            o32.data_ptr(), s))
                # fp16 out, out of place
                o16 = torch.full((T + GUARD, H), float("nan"), dtype=torch.float16, device="cuda")
                _ok(lib, lib.rl_xenc_add_ln(x.data_ptr(), r.data_ptr(), gam.data_ptr(), bet.data_ptr(), eps, T, H, 0,
                                            o16.data_ptr(), s))
                # fp16 out in place over res (NaN guard rows behind it too)
                rin = torch.full((T + GUARD, H), float("nan"), dtype=torch.float16, device="cuda")
                rin[:T] = r
                _ok(lib, lib.rl_xenc_add_ln(x.data_ptr(), rin.data_ptr(), gam.data_ptr(), bet.data_ptr(), eps, T, H, 0,
                                            rin.data_ptr(), s))
                torch.cuda.synchronize()
                for name, o in (("fp32", o32), ("fp16", o16), ("in place", rin)):
                    assert torch.isnan(o[T:]).all(), f"{what} {name}: written past row T"
                y32 = o32[:T].cpu().numpy().astype(np.float64)
                err = np.abs(y32 - v) / bnd
                ratio = float(np.nan_to_num(err, nan=np.inf).max())
                if not ratio <= 1.0:
                    t, c = np.unravel_index(int(np.nan_to_num(err, nan=np.inf).argmax()), err.shape)
                    pytest.fail(f"{what} fp32: |err| / bound {ratio:.3g} at row {t} ({pats[t]}), column {c}: got "
                                f"{y32[t, c]!r}, want {v[t, c]!r} +- {bnd[t, c]:.3g}")
                worst32 = max(worst32, ratio)
                y16 = o16[:T].cpu().numpy()
                n_two = rd.check(y16, v, bnd, rd.f16, what=what)
                if n_two / y16.size > two_max[0] / two_max[1]:
                    two_max = (n_two, y16.size)
                np.testing.assert_array_equal(rin[:T].cpu().numpy().view(np.uint16), y16.view(np.uint16),
                                              err_msg=f"{what}: in place differs from out of place")
                np.testing.assert_array_equal(o32[:T].half().cpu().numpy().view(np.uint16), y16.view(np.uint16),
                                              err_msg=f"{what}: fp16 out is not f16(fp32 out)")
                const = np.array([p == "const" for p in pats])
                if const.any():                              # variance exactly 0: the output is beta
                    want = np.broadcast_to(bet[:H].cpu().numpy(), (int(const.sum()), H))
                    np.testing.assert_array_equal(o32[:T].cpu().numpy()[const], want, err_msg=f"{what}: constant row")
                cases += 1
    _record("add_ln", {"cases": cases, "max_err_over_bound_fp32": worst32, "max_two_value": list(two_max),
                       "seconds": round(time.perf_counter() - t0, 2)})


# ---- embeddings + LayerNorm ---------------------------------------------------------------------------------------
def test_embed_ln_matches_float64():
    """``rl_xenc_embed_ln``: ``LayerNorm(word[id] + pos[pos_id] + type[type_id]) gamma + beta`` in fp16 against float64.
    The kernel forms x = fp32(fp32(word + pos) + type) (reproduced in float32), then runs add_ln's scalar arithmetic
    (columns lane + 32 i) with eps = the weights' ln_eps: the same mean, bound and fp16 bracket as
    ``test_add_ln_matches_float64``.  Tables: BERT-like (2 token types, positions 0 ... 511 of 512) and XLM-RoBERTa-like
    (1 token type, positions 2 + i up to 513 of 514), ids 0 and vocab - 1 among random ids, entries N(0, 0.5^2) with a
    per-row offset (the rows' means differ); both eps at every H.  NaN guard rows behind T stay unwritten."""
    import torch

    from raglite_b200 import _lib as L

    lib = _lib()
    torch.cuda.set_device(0)
    s = _stream()
    g = torch.Generator(device="cuda").manual_seed(1)
    rng = np.random.default_rng(1)
    vocab, T = 1000, 1100
    two_max, cases = (0, 1), 0
    t0 = time.perf_counter()
    for H in HS:
        for eps in EPS:
            for family, max_pos, type_vocab, pos0 in (("bert", 512, 2, 0), ("xlmr", 514, 1, 2)):
                def table(n):
                    return (0.5 * torch.randn((n, H), generator=g, device="cuda")
                            + torch.randn((n, 1), generator=g, device="cuda")).half()

                word, pos, typ = table(vocab), table(max_pos), table(type_vocab)
                gam, bet = _gamma_beta(H, g)
                ids = rng.integers(0, vocab, size=T).astype(np.int32)
                ids[:4] = [0, vocab - 1, 0, vocab - 1]
                pos_ids = (pos0 + np.arange(T) % (max_pos - pos0)).astype(np.int32)    # up to max_pos - 1
                type_ids = rng.integers(0, type_vocab, size=T).astype(np.int32)
                w = L.XencWeights()
                w.hidden, w.vocab, w.max_pos, w.type_vocab, w.ln_eps = H, vocab, max_pos, type_vocab, eps
                w.word_emb, w.pos_emb, w.type_emb = word.data_ptr(), pos.data_ptr(), typ.data_ptr()
                w.emb_ln_g, w.emb_ln_b = gam.data_ptr(), bet.data_ptr()
                d_in = torch.from_numpy(np.concatenate([ids, type_ids, pos_ids])).cuda()
                out = torch.full((T + GUARD, H), float("nan"), dtype=torch.float16, device="cuda")
                _ok(lib, lib.rl_xenc_embed_ln(C.byref(w), d_in.data_ptr(), d_in[T:].data_ptr(), d_in[2 * T:].data_ptr(), T,
                                              out.data_ptr(), s))
                torch.cuda.synchronize()
                what = f"embed_ln H={H} eps={eps:g} {family}"
                assert torch.isnan(out[T:]).all(), f"{what}: written past row T"
                wv, pv, tv = (t.float().cpu().numpy() for t in (word, pos, typ))
                x32 = (wv[ids] + pv[pos_ids]) + tv[type_ids]
                v, bnd = _ln_reference(x32, False, gam[:H].cpu().numpy(), bet[:H].cpu().numpy(), float(w.ln_eps))
                y = out[:T].cpu().numpy()
                n_two = rd.check(y, v, bnd, rd.f16, what=what)
                if n_two / y.size > two_max[0] / two_max[1]:
                    two_max = (n_two, y.size)
                cases += 1
    _record("embed_ln", {"cases": cases, "max_two_value": list(two_max), "seconds": round(time.perf_counter() - t0, 2)})


# ---- pooler + classifier + score ----------------------------------------------------------------------------------
def test_cls_head_matches_float64():
    """``rl_xenc_cls_head``: logit_j = Wc_j . tanh(Wp h + bp) + bc_j on each sequence's [CLS] row h, score sigmoid(l) at
    one label and softmax(l)[1] at two, against float64.  Only the [CLS] rows are finite (every other row is NaN), so a
    read of any other row poisons the logit.  Bounds (u = 2^-24; nw = min(H/32, 16) warps; Z_o = sum_c |Wp_oc h_c| +
    |bp_o|):

    - pre-activation z_o: H/32 lane-sequential FMAs and 5 butterfly levels, each within u of a partial <= Z_o, and + bp:
      E_z = (H/32 + 6) u Z_o.
    - t_o = tanhf(z_o): |tanh'| <= 1, plus tanhf's 2 ulp: E_t = E_z + 2^-22 |t| + 2^-126.
    - logit: each warp's H/nw outputs accumulate t wc in order (a rounding per step, another unless fused), then bc
      plus the nw partials in warp order: E_l = (H/nw + nw + 1) u (|bc| + sum_o |t_o wc_o|) + sum_o |wc_o| E_t.
    - score: x = -l (one label) or fp32(l0 - l1) (two, one more rounding), e = __expf(x) within (2 + 1.2 |x|) ulp,
      flushed below 2^-126 and +inf above 88.7, 1 + e and the division one rounding each:
      |s - s_ref| <= s (1 - s) (E_x + (2 + 1.2 |x|) 2^-23) + 2u s + 1e-37.

    Logits are scaled to reach +-100, so scores saturate to exactly 0 / 1 and must not turn NaN.  H 32 ... 1024 (1 to
    16 warps; 48 / 64 pooler outputs per warp at 768 / 1024), 1 and 2 labels, P = 1, 2, 3, 1101 (odd P leaves a CTA's
    second slot empty).  NaN guard rows behind the T token rows, and NaN guard entries behind the P logits / scores,
    which stay unwritten."""
    import torch
    from scipy.special import expit

    from raglite_b200 import _lib as L

    lib = _lib()
    torch.cuda.set_device(0)
    s = _stream()
    g = torch.Generator(device="cuda").manual_seed(2)
    rng = np.random.default_rng(2)
    worst = {"logit": 0.0, "score": 0.0}
    saturated, cases = 0, 0
    t0 = time.perf_counter()
    for H in (32, 160, 384, 512, 768, 1024):
        nw = min(H // 32, 16)
        for NL in (1, 2):
            for P in (1, 2, 3, 1101):
                lens = rng.integers(1, 6, size=P)
                lens[rng.random(P) < 0.8] += 1                        # mostly >= 2 tokens: row cu + 1 is not a [CLS]
                cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
                T = int(cu[-1])
                hid = torch.full((T + GUARD, H), float("nan"), dtype=torch.float16, device="cuda")
                hid[torch.from_numpy(cu[:-1]).long().cuda()] = torch.randn((P, H), generator=g, device="cuda").half()
                Wp = torch.randn((H, H), generator=g, device="cuda") / H**0.5
                bp = 0.5 * torch.randn(H, generator=g, device="cuda")
                Wc = 60.0 / H**0.5 * torch.randn((NL, H), generator=g, device="cuda")
                bc = torch.tensor([3.0, -2.0][:NL], device="cuda")
                w = L.XencWeights()
                w.hidden, w.n_labels = H, NL
                w.pooler_w, w.pooler_b, w.cls_w, w.cls_b = Wp.data_ptr(), bp.data_ptr(), Wc.data_ptr(), bc.data_ptr()
                d_cu = torch.from_numpy(cu).cuda()
                logit = torch.full((P * NL + GUARD,), float("nan"), device="cuda")
                score = torch.full((P + GUARD,), float("nan"), device="cuda")
                _ok(lib, lib.rl_xenc_cls_head(C.byref(w), hid.data_ptr(), d_cu.data_ptr(), P, logit.data_ptr(),
                                              score.data_ptr(), s))
                torch.cuda.synchronize()
                what = f"cls_head H={H} NL={NL} P={P}"
                assert torch.isnan(logit[P * NL:]).all() and torch.isnan(score[P:]).all(), f"{what}: written past P"
                h = hid[torch.from_numpy(cu[:-1]).long().cuda()].double().cpu().numpy()        # [P, H]
                Wp64, bp64 = Wp.double().cpu().numpy(), bp.double().cpu().numpy()
                Wc64, bc64 = Wc.double().cpu().numpy(), bc.double().cpu().numpy()
                z = h @ Wp64.T + bp64
                t = np.tanh(z)
                lg = t @ Wc64.T + bc64                                                          # [P, NL]
                Ez = (H / 32 + 6) * U * (np.abs(h) @ np.abs(Wp64).T + np.abs(bp64))
                Et = Ez + 2.0**-22 * np.abs(t) + 2.0**-126
                El = ((H / nw + nw + 1) * U * (np.abs(bc64) + np.abs(t) @ np.abs(Wc64).T) + Et @ np.abs(Wc64).T) * (1 + 1e-6)
                got_l = logit[:P * NL].double().cpu().numpy().reshape(P, NL)
                r = np.nan_to_num(np.abs(got_l - lg) / El, nan=np.inf)
                assert r.max() <= 1.0, (what, "logit", float(r.max()), got_l.flat[int(r.argmax())], lg.flat[int(r.argmax())])
                worst["logit"] = max(worst["logit"], float(r.max()))
                if NL == 1:
                    x, Ex = -lg[:, 0], El[:, 0]
                else:
                    x = lg[:, 0] - lg[:, 1]
                    Ex = El[:, 0] + El[:, 1] + U * np.abs(x)
                sc = expit(-x)                                                                  # 1 / (1 + exp(x))
                bs = (sc * (1 - sc) * (Ex + (2 + 1.2 * np.abs(x)) * 2.0**-23) + 2 * U * sc + 1e-37) * 1.01
                got_s = score[:P].double().cpu().numpy()
                rs = np.nan_to_num(np.abs(got_s - sc) / bs, nan=np.inf)
                assert rs.max() <= 1.0, (what, "score", float(rs.max()), got_s[int(rs.argmax())], sc[int(rs.argmax())])
                worst["score"] = max(worst["score"], float(rs.max()))
                saturated += int(((got_s == 0) | (got_s == 1)).sum())
                if P == 1101:
                    assert np.abs(lg).max() > 100, (what, "logits do not reach +-100")
                cases += 1
    assert saturated > 0
    _record("cls_head", {"cases": cases, "max_err_over_bound": worst, "saturated_scores": saturated,
                         "seconds": round(time.perf_counter() - t0, 2)})


# ---- the forward is the chain of the tested kernels -------------------------------------------------------------------
CHAIN_LENS = (1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 511, 512, 3, 100, 7)   # P = 19 (odd)


def _hook_chain(eng, d_ids, d_types, d_pos, d_cu, P: int, T: int, max_len: int, *, out_f32=None, logit=None, score=None):
    """The forward of ``eng`` through the hooks, with the engine's own packed images and pointers: embed_ln, then per layer
    linear(qkv) -> attention -> linear(o) -> add_ln(ln1, in place) -> linear(up, GELU) -> linear(down) -> add_ln(ln2,
    in place, or fp32 into ``out_f32`` on the last layer), then the head when ``logit`` is given."""
    import torch

    lib, w, s = eng.lib, eng.weights, _stream()
    H, F, nh = w.hidden, w.ffn, w.n_heads
    dev = eng.device
    hidden = torch.empty((T, H), dtype=torch.float16, device=dev)
    qkv = torch.empty((T, 3 * H), dtype=torch.float16, device=dev)
    ctx = torch.empty((T, H), dtype=torch.float16, device=dev)
    tmp = torch.empty((T, H), dtype=torch.float16, device=dev)
    ffn = torch.empty((T, F), dtype=torch.float16, device=dev)
    ws = torch.empty(4 * P + 16, dtype=torch.uint8, device=dev)
    attention = lib.rl_xenc_attention if H // nh == 32 and H <= 512 else lib.rl_xenc_encode_attention

    def linear(X, img, bias, Y, N, K, act):
        _ok(lib, lib.rl_xenc_linear(X.data_ptr(), img, bias, Y.data_ptr(), T, N, K, act, s))

    def add_ln(g, b, out, f32):
        _ok(lib, lib.rl_xenc_add_ln(tmp.data_ptr(), hidden.data_ptr(), g, b, w.ln_eps, T, H, f32, out.data_ptr(), s))

    _ok(lib, lib.rl_xenc_embed_ln(C.byref(w), d_ids.data_ptr(), d_types.data_ptr(), d_pos.data_ptr(), T, hidden.data_ptr(), s))
    for l in range(w.n_layers):
        Lr = eng._layers[l]
        linear(hidden, Lr.qkv_img, Lr.qkv_bias, qkv, 3 * H, H, 0)
        _ok(lib, attention(qkv.data_ptr(), d_cu.data_ptr(), P, T, max_len, H, nh, ctx.data_ptr(), ws.data_ptr(), ws.numel(), s))
        linear(ctx, Lr.o_img, Lr.o_bias, tmp, H, H, 0)
        add_ln(Lr.ln1_g, Lr.ln1_b, hidden, 0)
        linear(hidden, Lr.up_img, Lr.up_bias, ffn, F, H, 1)
        linear(ffn, Lr.down_img, Lr.down_bias, tmp, H, F, 0)
        if out_f32 is not None and l == w.n_layers - 1:
            add_ln(Lr.ln2_g, Lr.ln2_b, out_f32, 1)
        else:
            add_ln(Lr.ln2_g, Lr.ln2_b, hidden, 0)
    if logit is not None:
        _ok(lib, lib.rl_xenc_cls_head(C.byref(w), hidden.data_ptr(), d_cu.data_ptr(), P, logit.data_ptr(), score.data_ptr(), s))


@pytest.mark.parametrize("model", ["minilm", "multibert", "xlmr-large", "bge-m3"])
def test_forward_is_the_chain_of_tested_kernels(model):
    """``rl_xenc_score``'s logits and scores (and ``rl_xenc_encode``'s fp32 rows for the bge-m3-shaped embedder) equal the
    hook chain's bit for bit.  Every kernel involved is deterministic (one CTA or warp per output, no atomics), so this
    pins the wiring no per-kernel test sees: which buffer feeds which launch, ln1 against ln2, the eps the forward
    passes, the fp32 switch of the last layer.  Seeded, perturbed 2-layer models: MiniLM (head_dim 32), multilingual
    BERT with 2 labels, XLM-R large with 1 label, bge-m3 (XLM-RoBERTa, 16 x 64); lengths 1 ... 512 across the 32 / 64 /
    128 boundaries in one packed call."""
    import torch
    import xenc_classifiers as xc

    from oracle import embed as oe
    from raglite_b200._xenc import CrossEncoderEngine, TokenEmbedderEngine

    torch.cuda.set_device(0)
    rng = np.random.default_rng(3)
    lens = np.asarray(CHAIN_LENS, dtype=np.int64)
    P, T, max_len = len(lens), int(lens.sum()), int(lens.max())
    t0 = time.perf_counter()
    if model == "bge-m3":
        hf = oe.seeded_model(oe.bge_m3_config(num_hidden_layers=2, vocab_size=5000, max_position_embeddings=514), seed=4)
        eng = TokenEmbedderEngine.from_hf(hf)
        ids = [x.astype(np.int32) for x in (rng.integers(3, 5000, size=int(n)) for n in lens)]
        types = None
    else:
        over = dict(num_hidden_layers=2, vocab_size=5000)
        if model == "xlmr-large":
            over["max_position_embeddings"] = 514
        hf = xc.seeded_classifier(model, seed=5, **over)
        eng = CrossEncoderEngine.from_hf(hf)
        ids, types = xc.random_pairs(0, 5000, rng, xc.SHAPES[model][0], lengths=CHAIN_LENS)
    with torch.cuda.device(eng.device):
        d_ids, d_types, d_pos, d_cu = eng._upload_packed(ids, types, lens, slot=0)
        s = _stream()
        w, H = eng.weights, eng.hidden
        if model == "bge-m3":
            want = torch.full((T, H), float("nan"), device=eng.device)
            _ok(eng.lib, eng.lib.rl_xenc_encode(C.byref(w), d_ids.data_ptr(), d_types.data_ptr(), d_pos.data_ptr(),
                                                d_cu.data_ptr(), P, T, max_len, want.data_ptr(), eng._ws.data_ptr(),
                                                eng._ws.numel(), s))
            got = torch.full((T, H), float("nan"), device=eng.device)
            _hook_chain(eng, d_ids, d_types, d_pos, d_cu, P, T, max_len, out_f32=got)
            torch.cuda.synchronize()
            assert torch.isfinite(want).all()
            assert torch.equal(got.view(torch.int32), want.view(torch.int32)), \
                f"{model}: {int((got != want).sum())} of {got.numel()} hidden values differ"
        else:
            NL = eng.n_labels
            want = torch.full(((NL + 1) * P,), float("nan"), device=eng.device)
            _ok(eng.lib, eng.lib.rl_xenc_score(C.byref(w), d_ids.data_ptr(), d_types.data_ptr(), d_pos.data_ptr(),
                                               d_cu.data_ptr(), P, T, max_len, want.data_ptr(), want[NL * P:].data_ptr(),
                                               eng._ws.data_ptr(), eng._ws.numel(), s))
            got = torch.full(((NL + 1) * P,), float("nan"), device=eng.device)
            _hook_chain(eng, d_ids, d_types, d_pos, d_cu, P, T, max_len, logit=got, score=got[NL * P:])
            torch.cuda.synchronize()
            assert torch.isfinite(want).all()
            assert torch.equal(got.view(torch.int32), want.view(torch.int32)), (model, got.tolist(), want.tolist())
    _record("forward_chain", {"model": model, "tokens": T, "sequences": P, "seconds": round(time.perf_counter() - t0, 2)})
