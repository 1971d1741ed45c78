"""The sentence-splitting kernels (``csrc/sentences.cu``) at their C entry points, against ``sentences_oracle``.

* ``rl_sat_token_logits`` bit for bit against ``sat_head`` (the warp's lanes, ``fmaf`` and butterfly in float32).
* ``rl_sat_char_probas`` bit for bit up to its sigmoid (``sat_char_logits``: stitching, document minimum, fill,
  scatter); the sigmoid within a derived bound of float64; the override exactly; the whitespace step bit for bit as
  ``propagate`` of the device's own values.  Logits, plans, hat tables and character targets are built here, not by
  ``SaTEngine``.
* ``rl_sentence_partition`` per document against ``partition_cuts``, with every document's ``min_len`` / ``max_len``
  its own and infeasible documents among feasible ones.

Every output buffer carries NaN or sentinel guards behind it, and every input a NaN guard, so a read or write past the
end shows.  The sigmoid's worst error over its bound and the share of correctly rounded outputs go to
``sentence_kernels.jsonl`` in the temporary directory.

Sigmoid bound.  The kernel computes P = fl(1 / fl(1 + expf(-x))) with CUDA's ``expf`` within 2 ulp, so
expf(-x) = E (1 + d1), |d1| <= 2^-22, and each of the two other operations adds one relative rounding |d| <= 2^-24.
With p = 1 / (1 + E): P = p (1 + d3) / ((1 + (1 - p) d1)(1 + d2)), so |P - p| <= p ((1 + u) / ((1 - r)(1 - u)) - 1)
with r = (1 - p) 2^-22, u = 2^-24, plus 2^-150 where P is subnormal.  Where E overflows float32 the device returns
exactly 0; in a band of 2^-20 around the overflow threshold it may return 0 or the bounded value."""

from __future__ import annotations

import json
import tempfile
from pathlib import Path

import numpy as np
import pytest
import sentences_oracle as so

from raglite_b200 import _sentences as S

pytestmark = pytest.mark.gpu

GUARD = 8
NAN_BITS = np.uint32(0x7FC0DEAD)          # the guard pattern: any write to a guard changes it
T_VALUES = (0, 1, 2, 253, 254, 255, 382, 383, 384, 5000)
MAX_B = S.SAT_BLOCK_SIZE - 2
F32_MAX = float(np.finfo(np.float32).max)
SENTINEL = -7


def _record(payload: dict) -> None:
    with (Path(tempfile.gettempdir()) / "sentence_kernels.jsonl").open("a") as f:
        f.write(json.dumps(payload) + "\n")


def _lib():
    from raglite_b200 import _lib

    return _lib.load()


def _stream() -> int:
    import torch

    return torch.cuda.current_stream().cuda_stream


def _ok(lib, rc: int) -> None:
    assert rc == 0, lib.rl_last_error()


def _dev(a: np.ndarray):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _guarded(a: np.ndarray, guard: int = GUARD):
    """``a`` (float32) on the device with ``guard`` rows of the NaN guard pattern behind it."""
    g = np.full((guard, *a.shape[1:]), NAN_BITS, np.uint32).view(np.float32)
    return _dev(np.concatenate([a.astype(np.float32), g]))


def _bits(x) -> np.ndarray:  # noqa: ANN001
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


# ---- rl_sat_token_logits ---------------------------------------------------------------------------------------------
def _head(lib, hidden: np.ndarray, W: np.ndarray, b: np.ndarray) -> np.ndarray:
    import torch

    R, H = hidden.shape
    NL = len(b)
    d_h, d_w, d_b = _guarded(hidden), _guarded(W), _guarded(b)
    out = torch.from_numpy(np.full((R + GUARD, NL), NAN_BITS, np.uint32).view(np.float32)).cuda()
    _ok(lib, lib.rl_sat_token_logits(d_h.data_ptr(), R, H, d_w.data_ptr(), d_b.data_ptr(), NL, out.data_ptr(),
                                     _stream()))
    got = out.cpu().numpy()
    assert np.all(got[R:].view(np.uint32) == NAN_BITS), "rl_sat_token_logits wrote past its rows"
    return got[:R]


def _head_inputs(rng, R: int, H: int, NL: int):
    scale = (10.0 ** rng.uniform(-2, 1, size=(R, 1))).astype(np.float32)
    hidden = (rng.standard_normal((R, H)).astype(np.float32) * scale).astype(np.float32)
    W = rng.standard_normal((NL, H)).astype(np.float32)
    b = rng.standard_normal(NL).astype(np.float32)
    return hidden, W, b


@pytest.mark.parametrize("NL", (1, 2, 3, 16))
@pytest.mark.parametrize("H", (1, 31, 32, 33, 384, 768, 1000, 1024))
def test_token_logits_bit_exact(H, NL):
    lib = _lib()
    rng = np.random.default_rng(H * 100 + NL)
    for R in (1, 7, 8, 9):
        hidden, W, b = _head_inputs(rng, R, H, NL)
        got = _head(lib, hidden, W, b)
        np.testing.assert_array_equal(_bits(got), _bits(so.sat_head(hidden, W, b)), err_msg=f"H={H} NL={NL} rows={R}")


def test_token_logits_grid_stride():
    """More rows than one launch has warps (65 536 CTAs x 8): the grid-stride loop runs a second trip."""
    lib = _lib()
    rng = np.random.default_rng(1)
    R, H, NL = 65536 * 8 + 9, 33, 2
    hidden, W, b = _head_inputs(rng, R, H, NL)
    got = _head(lib, hidden, W, b)
    np.testing.assert_array_equal(_bits(got), _bits(so.sat_head(hidden, W, b)))


# ---- rl_sat_char_probas ----------------------------------------------------------------------------------------------
def _plan(T: np.ndarray, dense: bool):
    """(B [D] int32, blk_off [D + 1], blk_start) of the production plan, or a dense plan: a block at every start, of
    min(254, T) tokens in even documents and of min(3 + 53 d mod 250, T) in odd ones (the production plan has one
    block when B < 254, so only here do several blocks of a smaller B overlap and its hat weights matter)."""
    if not dense:
        return S.plan_blocks(T)
    d = np.arange(len(T))
    B = np.minimum(np.where(d % 2 == 0, MAX_B, 3 + (53 * d) % 250), T).astype(np.int32)
    n_blk = np.where(T > 0, T - B + 1, 0)
    off = np.r_[0, np.cumsum(n_blk)].astype(np.int64)
    start = np.concatenate([np.arange(n, dtype=np.int32) for n in n_blk]) if off[-1] else np.zeros(0, np.int32)
    return B, off, start


def _dyadic_hat(rng) -> np.ndarray:
    """Random weights k / 256 for every B; B = 1's weight stays 1, so a one-token document's logit passes exactly."""
    w = (rng.integers(1, 256, size=MAX_B * (MAX_B + 1) // 2) / 256.0).astype(np.float32)
    w[0] = 1
    return w


def _targets(rng, T: int, n: int) -> np.ndarray:
    """Document-relative character targets of T tokens over n characters: distinct, about a fifth of the tokens -1,
    the document's last character always written (when there are tokens and characters)."""
    tgt = np.full(T, -1, np.int64)
    if T == 0 or n == 0:
        return tgt
    k = min(T, n)
    chars = np.sort(rng.choice(n, size=k, replace=False))
    chars[-1] = n - 1
    toks = np.sort(rng.choice(T, size=k, replace=False))
    tgt[toks] = chars
    drop = rng.random(T) < 0.2
    drop[toks[-1]] = False
    tgt[drop] = -1
    return tgt


class Case:
    """One ``rl_sat_char_probas`` call: documents of T[d] tokens and n[d] characters, block rows with NaN gaps."""

    def __init__(self, rng, T, n, NL: int, *, dense: bool = False, dyadic: bool = False, targets=None,
                 logits_fn=None) -> None:
        self.T, self.n = np.asarray(T, np.int64), np.asarray(n, np.int64)
        self.NL, self.D = NL, len(self.T)
        self.tok_off, self.char_off = np.r_[0, np.cumsum(self.T)], np.r_[0, np.cumsum(self.n)]
        self.N, self.NT = int(self.char_off[-1]), int(self.tok_off[-1])
        self.B, self.blk_off, self.blk_start = _plan(self.T, dense)
        blk_B = np.repeat(self.B, np.diff(self.blk_off)).astype(np.int64)
        self.blk_row = (np.cumsum(blk_B + 2) - blk_B - 1).astype(np.int64)              # a NaN row either side
        rows = int(blk_B.sum() + 2 * len(blk_B))
        self.logits = np.full((max(rows, 1), NL), np.nan, np.float32)
        if len(blk_B):
            r = np.repeat(self.blk_row, blk_B) + np.arange(int(blk_B.sum())) - np.repeat(np.cumsum(blk_B) - blk_B, blk_B)
            scale = (10.0 ** rng.uniform(-3, 0.7, size=(len(r), 1))).astype(np.float32)
            self.logits[r] = rng.standard_normal((len(r), NL)).astype(np.float32) * scale
        self.hat = _dyadic_hat(rng) if dyadic else S.hat_table()
        tg = targets if targets is not None else [_targets(rng, int(T), int(c)) for T, c in zip(self.T, self.n)]
        self.tok_char = np.concatenate([np.where(t >= 0, t + self.char_off[d], -1) for d, t in enumerate(tg)] +
                                       [np.zeros(0, np.int64)])
        if logits_fn is not None:
            logits_fn(self)

    def token_rows(self, d: int, t: int) -> np.ndarray:
        """Every logits row of token t of document d (one per block that covers it)."""
        a, e = self.blk_off[d], self.blk_off[d + 1]
        st = self.blk_start[a:e].astype(np.int64)
        cov = (st <= t) & (t < st + self.B[d])
        return self.blk_row[a:e][cov] + t - st[cov]

    def reference(self) -> np.ndarray:
        return so.sat_char_logits(self.logits, self.tok_off, self.char_off, self.B, self.blk_off, self.blk_start,
                                  self.blk_row, self.hat, self.tok_char)[0]

    def run(self, lib, known: np.ndarray | None, is_space: np.ndarray | None, *, no_token_args: bool = False):
        import torch

        d = {k: _dev(v) for k, v in (("tok_off", self.tok_off), ("char_off", self.char_off), ("B", self.B),
                                      ("blk_off", self.blk_off))}
        ptr = {k: v.data_ptr() for k, v in d.items()}
        keep = []
        if no_token_args:
            ptr.update(logits=None, blk_start=None, blk_row=None, hat=None, tok_char=None)
        else:
            for k, v in (("blk_start", np.r_[self.blk_start, 0].astype(np.int32)),
                         ("blk_row", np.r_[self.blk_row, 0]), ("tok_char", np.r_[self.tok_char, -1])):
                keep.append(_dev(v))
                ptr[k] = keep[-1].data_ptr()
            keep += [_guarded(self.logits), _guarded(self.hat, 256)]
            ptr["logits"], ptr["hat"] = keep[-2].data_ptr(), keep[-1].data_ptr()
        d_known = _guarded(known) if known is not None else None
        d_space = _dev(np.r_[is_space.astype(np.uint8), np.ones(GUARD, np.uint8)]) if is_space is not None else None
        need = int(lib.rl_sat_workspace_bytes(self.NT, self.D, self.NL))
        ws = torch.zeros(need + 4096, dtype=torch.uint8, device="cuda")
        out = torch.from_numpy(np.full(self.N + GUARD, NAN_BITS, np.uint32).view(np.float32)).cuda()
        _ok(lib, lib.rl_sat_char_probas(ptr["logits"], self.NL, ptr["tok_off"], ptr["char_off"], ptr["B"], self.D,
                                        self.NT, self.N, ptr["blk_off"], ptr["blk_start"], ptr["blk_row"], ptr["hat"],
                                        ptr["tok_char"], d_known.data_ptr() if d_known is not None else None,
                                        d_space.data_ptr() if d_space is not None else None, out.data_ptr(),
                                        ws.data_ptr(), need, _stream()))
        got = out.cpu().numpy()
        assert np.all(got[self.N:].view(np.uint32) == NAN_BITS), "rl_sat_char_probas wrote past its characters"
        return got[:self.N]


def _check_sigmoid(name: str, got: np.ndarray, x: np.ndarray, known: np.ndarray | None) -> dict:
    """``got`` is ``known`` where that is not NaN, else the kernel's sigmoid of the restated logit ``x`` within the
    bound in the module docstring.  Returns the worst |err| / bound and the share of distinct logits whose output is the
    correctly rounded float32 sigmoid."""
    over = np.zeros(len(got), bool) if known is None else ~np.isnan(known)
    if over.any():
        np.testing.assert_array_equal(_bits(got[over]), _bits(known[over]), err_msg=f"{name}: override")
    g, xv = got[~over].astype(np.float64), x[~over].astype(np.float64)
    with np.errstate(over="ignore"):
        E = np.exp(-xv)
    p = 1.0 / (1.0 + E)
    u, r = 2.0**-24, (1.0 - p) * 2.0**-22
    bnd = p * ((1 + u) / ((1 - r) * (1 - u)) - 1) + 4 * 2.0**-53 * p + 2.0**-150
    overflow = E > F32_MAX * (1 + 2.0**-20)
    band = ~overflow & (E > F32_MAX * (1 - 2.0**-20))
    err = np.abs(g - p)
    assert np.all(g[overflow] == 0), f"{name}: expf(-x) overflows, the probability must be exactly 0"
    ok_band = (g[band] >= 0) & (g[band] <= p[band] + bnd[band])
    assert ok_band.all(), f"{name}: near the overflow threshold"
    mid = ~overflow & ~band
    worst = float((err[mid] / bnd[mid]).max()) if mid.any() else 0.0
    bad = np.nonzero(err[mid] > bnd[mid])[0][:5]
    assert worst <= 1.0, (name, [(float(xv[mid][i]), float(g[mid][i]), float(p[mid][i])) for i in bad])
    _, first = np.unique(xv[mid], return_index=True)             # each distinct logit once (fills repeat one value)
    rn = float((g[mid][first] == p[mid][first].astype(np.float32)).mean()) if mid.any() else 1.0
    stats = {"case": name, "chars": int(len(got)), "sigmoid_checked": int(mid.sum()), "overflow_zero": int(overflow.sum()),
             "worst_err_over_bound": worst, "correctly_rounded": rn}
    _record(stats)
    return stats


def _space_docs(flags: np.ndarray, off: np.ndarray) -> list[str]:
    s = np.where(flags, ord(" "), ord("a")).astype(np.uint32).tobytes().decode("utf-32-le")
    return [s[off[d]:off[d + 1]] for d in range(len(off) - 1)]


def _spaces(rng, n: np.ndarray) -> np.ndarray:
    """Whitespace flags: random runs, plus runs at a document's start and end, a document of spaces only, runs of
    length 1, a run of more than 10^5, and a boundary where a document ending in a non-space meets one starting with
    spaces."""
    N = int(n.sum())
    off = np.r_[0, np.cumsum(n)]
    sp = np.zeros(N, bool)
    for d in range(len(n)):
        a, e = off[d], off[d + 1]
        L = e - a
        if L == 0:
            continue
        kind = d % 5
        seg = rng.random(L) < (0.3 if kind else 0.05)
        if kind == 1:
            seg[:3] = True                           # leading run
        if kind == 2:
            seg[-4:] = True                          # trailing run
        if kind == 3 and L < 400:
            seg[:] = True                            # spaces only
        if kind == 4:
            seg[0] = True                            # the previous document's last character is a non-space
            if L > 2:
                seg[1], seg[-1] = False, False
        if L > 120_000:
            seg[1000:1000 + 110_000] = True          # one run longer than 10^5
            seg[999] = seg[1000 + 110_000] = False
        sp[a:e] = seg
        if kind == 4 and d > 0 and off[d] > off[d - 1]:
            sp[off[d] - 1] = False
    return sp


def _known(rng, N: int, share: float) -> np.ndarray:
    k = np.full(N, np.nan, np.float32)
    pick = rng.random(N) < share
    k[pick] = rng.random(int(pick.sum())).astype(np.float32)
    k[pick & (rng.random(N) < 0.05)] = np.inf        # a finite float64 above the float32 range, as _known_f32 passes it
    return k


def _plant_min(case: Case) -> None:
    """Each document's minimum in its last token, label NL - 1, different per document."""
    for d in range(case.D):
        if case.T[d]:
            case.logits[case.token_rows(d, int(case.T[d]) - 1), case.NL - 1] = -30.0 - 0.5 * d


SIGMOID_X = (-100.0, -89.0, -88.8, -88.73, -88.72, -88.7, -88.0, -87.5, -87.3, -40.0, -17.0, -1e-3, 0.0, 1e-30, 2.0**-20,
             5.0, 16.5, 17.0, 88.0, 100.0)


def _docs(rng, dense: bool):
    """Documents of every T in T_VALUES (5000 only in the production plan with 150 000 characters, else 600), an empty
    document between others (duplicate offsets), a document with characters but no tokens, and one-token documents
    whose logit is each of ``SIGMOID_X``."""
    T, n = [], []
    for t in T_VALUES:
        T.append(t)
        n.append(150_000 if t == 5000 and not dense else t + int(rng.integers(0, 40)) + (t == 0) * 17)
    T[3:3] = [0, 3]
    n[3:3] = [0, 3]
    T += [0, 1] + [1] * len(SIGMOID_X)
    n += [25, 1] + [2] * len(SIGMOID_X)
    return np.array(T), np.array(n)


@pytest.mark.parametrize(("name", "NL", "dense", "dyadic"), [
    ("nl1_prod_plan_prod_hat", 1, False, False), ("nl3_prod_plan_dyadic_hat", 3, False, True),
    ("nl16_dense_plan_dyadic_hat", 16, True, True), ("nl16_prod_plan_prod_hat", 16, False, False)])
def test_char_probas_bit_exact_before_sigmoid(name, NL, dense, dyadic):
    lib = _lib()
    rng = np.random.default_rng(NL * 10 + dense * 2 + dyadic)
    T, n = _docs(rng, dense)
    first_sig = len(T) - len(SIGMOID_X)

    def plant(case: Case) -> None:
        _plant_min(case)
        for i, x in enumerate(SIGMOID_X):
            case.logits[case.token_rows(first_sig + i, 0), 0] = x

    targets = [_targets(rng, int(t), int(c)) for t, c in zip(T, n, strict=True)]
    for i in range(len(SIGMOID_X)):
        targets[first_sig + i] = np.array([1])                 # the one token writes the document's last character
    case = Case(rng, T, n, NL, dense=dense, dyadic=dyadic, targets=targets, logits_fn=plant)
    x = case.reference()
    known = _known(rng, case.N, 0.05)
    for i in range(len(SIGMOID_X)):
        known[case.char_off[first_sig + i]:case.char_off[first_sig + i + 1]] = np.nan
    got = case.run(lib, known, None)
    stats = _check_sigmoid(name, got, x, known)
    assert stats["overflow_zero"] >= 3 and stats["sigmoid_checked"] > 5_000
    assert stats["correctly_rounded"] > 0.3
    for i, v in enumerate(SIGMOID_X):                           # the planted logits reach the sigmoid unchanged
        assert x[case.char_off[first_sig + i] + 1] == np.float32(v)
    for d in np.nonzero((case.T == 0) & (case.n > 0))[0]:       # documents without tokens: 0 unless overridden
        sl = slice(case.char_off[d], case.char_off[d + 1])
        assert np.all(np.where(np.isnan(known[sl]), got[sl], 0) == 0)

    # the whitespace step: propagate, document by document, of the device's own values before it
    sp = _spaces(rng, case.n)
    got_sp = case.run(lib, known, sp)
    docs = _space_docs(sp, case.char_off)
    want = np.concatenate([so.propagate(doc, got[case.char_off[d]:case.char_off[d + 1]]) for d, doc in enumerate(docs)])
    np.testing.assert_array_equal(_bits(got_sp), _bits(want))
    assert not np.array_equal(got_sp, got)


def test_char_probas_known_everywhere():
    """Every character overridden: the propagation's input is the known array itself."""
    lib = _lib()
    rng = np.random.default_rng(21)
    T, n = _docs(rng, False)
    case = Case(rng, T, n, 2)
    known = rng.random(case.N).astype(np.float32)
    known[rng.random(case.N) < 0.01] = np.inf
    np.testing.assert_array_equal(_bits(case.run(lib, known, None)), _bits(known))
    sp = _spaces(rng, case.n)
    want = so.propagate_runs(known, sp, case.char_off)
    np.testing.assert_array_equal(_bits(case.run(lib, known, sp)), _bits(want))
    docs = _space_docs(sp, case.char_off)
    np.testing.assert_array_equal(_bits(want), _bits(np.concatenate(
        [so.propagate(doc, known[case.char_off[d]:case.char_off[d + 1]]) for d, doc in enumerate(docs)])))


def test_char_probas_without_tokens():
    """``n_tokens = 0`` with ``logits``, ``blk_start``, ``blk_row``, ``hat`` and ``tok_char`` null: every probability
    is 0 (sigmoid of -inf) unless overridden, and the whitespace step still runs."""
    lib = _lib()
    rng = np.random.default_rng(22)
    case = Case(rng, [0, 0, 0, 0], [5, 0, 40, 1], 3)
    assert case.NT == 0
    got = case.run(lib, None, None, no_token_args=True)
    assert np.all(_bits(got) == 0)
    known = _known(rng, case.N, 0.3)
    got = case.run(lib, known, None, no_token_args=True)
    np.testing.assert_array_equal(_bits(got), _bits(np.where(np.isnan(known), np.float32(0), known)))
    sp = rng.random(case.N) < 0.4
    got_sp = case.run(lib, known, sp, no_token_args=True)
    np.testing.assert_array_equal(_bits(got_sp), _bits(so.propagate_runs(got, sp, case.char_off)))


def test_char_probas_grid_stride_scale():
    """2^25 + 17 characters and 2^25 + 17 tokens in one call: the stitch, fill, scatter, sigmoid and whitespace
    kernels (at most 2^24 threads a launch) each run a second and a third trip.  Document boundaries sit next to the
    trip boundaries."""
    lib = _lib()
    rng = np.random.default_rng(23)
    T = np.array([2**24 + 3, 7, 0, 2**24 + 7])
    n = np.array([2**24 + 3, 9, 5, 2**24])
    targets = []
    for t, c in zip(T, n, strict=True):
        tg = np.where(np.arange(t) < c, np.arange(t), -1)
        tg[rng.random(t) < 0.1] = -1
        if t and c:
            tg[min(t, c) - 1] = c - 1
        targets.append(tg)
    case = Case(rng, T, n, 1, targets=targets)
    assert case.N == case.NT == 2**25 + 17
    x = case.reference()
    known = _known(rng, case.N, 0.01)
    got = case.run(lib, known, None)
    stats = _check_sigmoid("scale", got, x, known)
    assert stats["sigmoid_checked"] > 2**25 * 0.9
    sp = rng.random(case.N) < 0.1
    sp[2**24 - 2:2**24 + 3] = [False, True, True, True, False]         # a run across the first trip boundary
    got_sp = case.run(lib, known, sp)
    np.testing.assert_array_equal(_bits(got_sp), _bits(so.propagate_runs(got, sp, case.char_off)))


# ---- rl_sentence_partition -------------------------------------------------------------------------------------------
def _partition_docs(rng) -> list[tuple[np.ndarray, int, int]]:
    """(float32 probabilities, min_len, max_len with 0 = none) of every document of one launch."""
    f = np.float32
    docs = [(np.zeros(0, f), 4, 0), (np.zeros(0, f), 1, 3),                                  # n = 0
            (rng.random(3).astype(f), 4, 0), (rng.random(4).astype(f), 4, 2),                  # n <= min_len
            (rng.random(9).astype(f), 5, 0), (rng.random(9).astype(f), 5, 6),                  # min_len < n < 2 min_len
            (rng.random(50).astype(f), 3, 50), (rng.random(50).astype(f), 3, 80),               # max_len >= n
            (rng.random(60).astype(f), 6, 6), (rng.random(61).astype(f), 1, 1),                 # max_len = min_len
            (np.full(13, 0.9, f), 7, 11),           # one stage-1 sentence of 13 > 11 with no split of both >= 7: kept
            (np.zeros(13, f), 5, 6),                                                           # infeasible
            (np.linspace(0.2, 0.0, 900).astype(f), 1, 300),   # strictly decreasing dp: the deque holds the whole window
            (np.linspace(0.2, 0.0, 700).astype(f), 4, 200)]
    for _ in range(150):
        L = int(rng.integers(0, 700))
        lo = int(rng.integers(1, 12))
        hi = int(rng.choice([0, lo, lo + int(rng.integers(0, 30)), int(rng.integers(lo, 3 * lo + 2))]))
        p = rng.choice([0.0, 0.25, 0.5, 0.75, 1.0], size=L, p=[0.3, 0.2, 0.2, 0.2, 0.1]) if rng.random() < 0.5 else \
            rng.random(L) ** 3
        docs.append((p.astype(f), lo, hi))
    for _ in range(10_000):
        L = int(rng.integers(0, 24))
        lo = int(rng.integers(1, 6))
        docs.append((rng.choice([0.0, 0.25, 0.5, 0.75, 1.0], size=L).astype(f), lo, int(rng.choice([0, lo, lo + 3]))))
    order = rng.permutation(len(docs))
    return [docs[i] for i in order]


def test_partition_per_document():
    """One launch of about 10 000 documents, each with its own min_len and max_len: per document, the cuts of
    ``partition_cuts`` and status 0, or status 1 and count 0 where the reference raises; nothing written outside a
    document's slice, and nothing past its count for a successful one."""
    import torch

    lib = _lib()
    rng = np.random.default_rng(31)
    docs = _partition_docs(rng)
    D = len(docs)
    gaps = rng.integers(0, 4, size=D + 1)
    lens = np.array([len(p) for p, _, _ in docs], np.int64)
    off = gaps[0] + np.r_[0, np.cumsum(lens + gaps[1:])[:-1]]
    N = int(off[-1] + lens[-1] + gaps[-1])
    probas = rng.random(N).astype(np.float32)
    for (p, _, _), o in zip(docs, off, strict=True):
        probas[o:o + len(p)] = p
    want, fail = [], []
    for p, lo, hi in docs:
        try:
            want.append(so.partition_cuts(p, len(p), lo, hi))
            fail.append(False)
        except ValueError:
            want.append([])
            fail.append(True)
    assert 0 < sum(fail) < D // 2
    d_p, d_off = _dev(probas), _dev(off.astype(np.int64))
    d_len = _dev(lens.astype(np.int32))
    d_min = _dev(np.array([lo for _, lo, _ in docs], np.int32))
    d_max = _dev(np.array([hi for _, _, hi in docs], np.int32))
    cuts = torch.full((N + GUARD,), SENTINEL, dtype=torch.int32, device="cuda")
    cs = torch.full((2 * D + GUARD,), -5, dtype=torch.int32, device="cuda")
    need = int(lib.rl_sentence_partition_workspace_bytes(N))
    ws = torch.zeros(need + 4096, dtype=torch.uint8, device="cuda")
    t0 = torch.cuda.Event(enable_timing=True)
    t1 = torch.cuda.Event(enable_timing=True)
    t0.record()
    _ok(lib, lib.rl_sentence_partition(d_p.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), d_min.data_ptr(),
                                       d_max.data_ptr(), D, N, cuts.data_ptr(), cs.data_ptr(), cs[D:].data_ptr(),
                                       ws.data_ptr(), need, _stream()))
    t1.record()
    torch.cuda.synchronize()
    h_cuts, h_cs = cuts.cpu().numpy(), cs.cpu().numpy()
    counts, status = h_cs[:D], h_cs[D:2 * D]
    assert np.all(h_cs[2 * D:] == -5)
    owned = np.zeros(N + GUARD, bool)
    for d, ((p, lo, hi), o) in enumerate(zip(docs, off, strict=True)):
        if fail[d]:
            assert status[d] == 1 and counts[d] == 0, (d, len(p), lo, hi, status[d], counts[d])
            owned[o:o + len(p)] = True
            continue
        assert status[d] == 0, (d, len(p), lo, hi)
        assert counts[d] == len(want[d]) and h_cuts[o:o + counts[d]].tolist() == want[d], (d, len(p), lo, hi)
        owned[o:o + counts[d]] = True
    assert np.all(h_cuts[~owned] == SENTINEL), "rl_sentence_partition wrote outside a document's cuts"
    assert sum(len(w) for w in want) > 10_000
    _record({"case": "partition", "docs": D, "chars": N, "failed": int(sum(fail)), "ms": t0.elapsed_time(t1)})
