"""Host side of ``split_sentences``: the post-processing restatement against the reference's own outputs, the Markdown
boundaries, the block plan / hat weights / character targets against plain loops, ``SaTEngine``'s refusals and config
reading, and the public early exit and registration error.  Also the pieces of the kernel restatements that
``test_gpu_sentence_kernels.py`` relies on (``fmaf`` against exact fractions, the head, the stitching and the batched
whitespace propagation against plain loops, ``partition_cuts`` against the post-processing) and the C-ABI refusals of
the three sentence entry points.  No GPU."""

from __future__ import annotations

import ctypes as C
import json
from fractions import Fraction
from pathlib import Path

import numpy as np
import pytest
import sentences_oracle as so

from raglite_b200 import _sentences as S

GOLDEN = Path(__file__).parent / "golden" / "split_sentences.npz"
T_VALUES = (0, 1, 2, 253, 254, 255, 382, 383, 384, 5000)


def _cases():
    z = np.load(GOLDEN)
    return [(c, z[f"pred{i}"], z[f"md{i}"], z[f"known{i}"] if c["known"] else None)
            for i, c in enumerate(json.loads(z["cases"].tobytes()))]


CASES = _cases()


@pytest.mark.parametrize("i", range(len(CASES)), ids=[f"{c['name']}-{c['min_len']}-{c['max_len']}" for c, *_ in CASES])
def test_post_processing_matches_reference(i):
    c, pred, _md, known = CASES[i]
    if c["error"] is not None:
        with pytest.raises(ValueError, match="Sentence partition failed") as e:
            so.split_sentences_post(c["doc"], pred, min_len=c["min_len"], max_len=c["max_len"], known=known)
        assert str(e.value) == c["error"]
        return
    got = so.split_sentences_post(c["doc"], pred, min_len=c["min_len"], max_len=c["max_len"], known=known)
    assert got == c["sentences"]
    assert "".join(got) == c["doc"]


def test_golden_covers_the_issue_cases():
    names = {c["name"] for c, *_ in CASES}
    assert {"headings", "spaces", "multibyte", "len4", "len5", "len8", "infeasible"} <= names
    assert {8, 64, 2048, None} <= {c["max_len"] for c, *_ in CASES}
    assert any(c["error"] for c, *_ in CASES)
    assert any(c["max_len"] == 8 and c["sentences"] and max(map(len, c["sentences"])) <= 8 and len(c["doc"]) > 40
               for c, *_ in CASES)


@pytest.mark.parametrize("doc", sorted({c["doc"] for c, *_ in CASES}))
def test_markdown_boundaries_match_reference(doc):
    want = next(md for c, _p, md, _k in CASES if c["doc"] == doc)
    for got in (S.markdown_sentence_boundaries(doc), so.markdown_boundaries(doc)):
        assert got.dtype == want.dtype and got.shape == want.shape
        np.testing.assert_array_equal(got, want)   # NaN positions equal too


def test_markdown_headings_present():
    doc = next(c["doc"] for c, *_ in CASES if c["name"] == "headings")
    md = S.markdown_sentence_boundaries(doc)
    assert (md == 1).sum() >= 6 and (md == 0).sum() > 20 and np.isnan(md).sum() > 20


@pytest.mark.parametrize("T", T_VALUES)
def test_block_plan_matches_loop(T):
    B, starts = S.block_starts(T)
    wB, wstarts = so.plan_loop(T)
    assert B == wB and starts.tolist() == wstarts
    if T:
        assert starts[-1] + B == T and all(s + B < T for s in starts[:-1])
        covered = np.zeros(T, int)
        for s in starts:
            covered[s:s + B] += 1
        assert covered.min() >= 1 and covered.max() <= -(-B // S.SAT_STRIDE) + 1


def test_batch_plan_equals_per_document():
    T = np.array(T_VALUES + (0, 7, 1000), dtype=np.int64)
    B, off, start = S.plan_blocks(T)
    for d, t in enumerate(T):
        b, s = S.block_starts(int(t))
        assert (t == 0 or B[d] == b) and start[off[d]:off[d + 1]].tolist() == s.tolist()


@pytest.mark.parametrize("B", sorted({1, 2, 3, 127, 128, 253, 254} | {min(254, t) for t in T_VALUES if t}))
def test_hat_weights_match_loop(B):
    w = S.hat_weights(B)
    np.testing.assert_allclose(w, so.hat_loop(B), rtol=0, atol=2e-7)
    assert np.all(w > 0) and np.all(w <= 1) and np.allclose(w, w[::-1])
    table = S.hat_table()
    np.testing.assert_array_equal(table[B * (B - 1) // 2:B * (B + 1) // 2], w)


@pytest.mark.parametrize("T", T_VALUES)
def test_char_targets_match_loop(T):
    rng = np.random.default_rng(T)
    n = max(1, 2 * T)
    ends = np.sort(rng.integers(0, n + 1, size=T))
    skip = rng.random(T) < 0.2
    got = S.token_char_targets(ends, skip, n)
    assert got.tolist() == so.char_targets_loop(ends, skip, n)
    hit = got[got >= 0]
    assert len(np.unique(hit)) == len(hit)


def test_tokenizer_targets_on_multibyte_text():
    """Character offsets from ``tokenizers`` count Python characters: the target of each kept token is a character
    inside the document, and the multi-byte characters keep their own positions."""
    from oracle.embed import unigram_tokenizer

    tok = unigram_tokenizer()
    doc = "héllo  wörld　⊕ the  end.\n\nalpha 😀 x"
    e = tok.encode(doc, add_special_tokens=False)
    ends = np.array([o[1] for o in e.offsets])
    skip = np.isin(e.ids, [tok.token_to_id(p) for p in S.SAT_SKIP_PIECES if tok.token_to_id(p) is not None])
    tgt = S.token_char_targets(ends, skip, len(doc))
    assert tgt.max() < len(doc) and doc[tgt[np.array(e.tokens) == "."][0]] == "."


def test_whitespace_flags_are_str_isspace():
    every = "".join(chr(c) for c in range(0x110000) if not 0xD800 <= c < 0xE000)
    got = S.whitespace_flags(every)
    assert got.tolist() == [c.isspace() for c in every]
    assert S.code_points("a😀é").tolist() == [0x61, 0x1F600, 0xE9]


def _config(**over):
    c = {"model_type": "xlm-token", "architectures": ["SubwordXLMForTokenClassification"], "hidden_size": 768,
         "num_hidden_layers": 1, "num_attention_heads": 12, "intermediate_size": 3072, "max_position_embeddings": 514,
         "hidden_act": "gelu", "layer_norm_eps": 1e-5, "pad_token_id": 1, "vocab_size": 250002, "lookahead": None,
         "num_labels": 111}
    c.update(over)
    return c


def test_config_json_read_as_json(tmp_path):
    (tmp_path / "config.json").write_text(json.dumps(_config()))
    kw = S.read_sat_config(tmp_path)
    assert kw == dict(n_layers=1, hidden=768, n_heads=12, ffn=3072, max_pos=514, ln_eps=1e-5, pos_offset=2)


@pytest.mark.parametrize(("over", "match"), [
    ({"lookahead": 48}, "lookahead"),
    ({"hidden_act": "relu"}, "GELU"),
    ({"num_attention_heads": 6}, "head_dim"),
    ({"hidden_size": 1280, "num_attention_heads": 20}, "at most 1024"),
])
def test_config_refusals(tmp_path, over, match):
    (tmp_path / "config.json").write_text(json.dumps(_config(**over)))
    with pytest.raises(ValueError, match=match):
        S.read_sat_config(tmp_path)
    with pytest.raises(ValueError, match=match):
        S.SaTEngine.from_pretrained(tmp_path)


def test_missing_head_refused(tmp_path):
    import torch
    from safetensors.torch import save_file

    (tmp_path / "config.json").write_text(json.dumps(_config(hidden_size=64, num_attention_heads=1, intermediate_size=128)))
    save_file({"roberta.embeddings.word_embeddings.weight": torch.zeros(10, 64)}, str(tmp_path / "model.safetensors"))
    with pytest.raises(ValueError, match="token-classification head"):
        S.SaTEngine.from_pretrained(tmp_path)
    with pytest.raises(ValueError, match="token-classification head"):
        S.SaTEngine({"roberta.embeddings.word_embeddings.weight": torch.zeros(10, 64)}, n_layers=1, hidden=64,
                    n_heads=1, ffn=128, max_pos=514, tokenizer=None)


def _round_f32(x: Fraction) -> np.float32:
    """The float32 nearest to x, ties to even (x within the float32 range)."""
    r = np.float32(float(x))              # within one float32 step of the answer (float64 first: two roundings)
    cands = [np.nextafter(r, np.float32(-np.inf)), r, np.nextafter(r, np.float32(np.inf))]
    dist = [abs(Fraction(float(c)) - x) for c in cands]
    best = min(dist)
    near = [c for c, e in zip(cands, dist, strict=True) if e == best]
    return min(near, key=lambda c: int(np.array(c, np.float32).view(np.uint32)) & 1)


def _fma_exact(a, b, c) -> np.ndarray:  # noqa: ANN001
    return np.array([_round_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z)))
                     for x, y, z in zip(a, b, c, strict=True)], np.float32)


def _planted_fma() -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Triples whose float64 sum s lies exactly on a float32 midpoint with a nonzero remainder (the products
    +-2^16 (1 - 2^-46) against c near 2^40, where float32 steps are 2^17), and float32 subnormal results."""
    f = np.float32
    a, b, c = [], [], []
    for sa in (1, -1):
        for j in range(4):
            for sc in (1, -1):
                a.append(f(sa * 256 * (1 + 2.0**-23)))
                b.append(f(256 * (1 - 2.0**-23)))
                c.append(f(sc * (2.0**40 + j * 2.0**17)))
    sub = [(2.0**-75 * (1 + 2.0**-23), 2.0**-75 * (1 - 2.0**-23), 2.0**-149), (2.0**-80, 3.0 * 2.0**-70, -(2.0**-149)),
           (2.0**-100, 2.0**-49, 0.0), (-(2.0**-70), 2.0**-70, 2.0**-140), (2.0**-63, 1.5 * 2.0**-63, -(2.0**-126))]
    for x, y, z in sub:
        a.append(f(x))
        b.append(f(y))
        c.append(f(z))
    return np.array(a, f), np.array(b, f), np.array(c, f)


def test_fmaf_emulation_against_fractions():
    """``sentences_oracle.fmaf`` is a correctly rounded a b + c, checked against exact rational arithmetic on random
    triples over a wide exponent range, on planted float32 midpoints and on subnormal results."""
    rng = np.random.default_rng(3)
    n = 4000
    a = (rng.standard_normal(n) * 2.0 ** rng.integers(-60, 60, n)).astype(np.float32)
    b = (rng.standard_normal(n) * 2.0 ** rng.integers(-60, 60, n)).astype(np.float32)
    c = (rng.standard_normal(n) * 2.0 ** rng.integers(-60, 60, n)).astype(np.float32)
    near = rng.random(n) < 0.5                  # c close to -a b: cancellation, the remainder decides the rounding
    c[near] = (-(a[near].astype(np.float64) * b[near]) * (1 + rng.standard_normal(near.sum()) * 2.0**-30)
               ).astype(np.float32)
    got, want = so.fmaf(a, b, c), _fma_exact(a, b, c)
    np.testing.assert_array_equal(got, want)
    pa, pb, pc = _planted_fma()
    got, want = so.fmaf(pa, pb, pc), _fma_exact(pa, pb, pc)
    np.testing.assert_array_equal(got, want)
    naive = (pa.astype(np.float64) * pb + pc).astype(np.float32)
    assert (naive != want).sum() >= 4               # the midpoint correction is exercised
    assert np.any((np.abs(want) < np.finfo(np.float32).tiny) & (want != 0))
    # a product that cancels c exactly gives +0, as IEEE round-to-nearest does
    z = so.fmaf(np.float32([2.0, -0.0]), np.float32([3.0, 1.0]), np.float32([-6.0, -0.0]))
    assert z.view(np.uint32).tolist() == [0, 0x80000000]


def test_sat_head_restatement_within_float64_bound():
    """The lane-by-lane restatement of ``sat_head_kernel`` is a float32 dot product plus bias: within the
    gamma_n bound of float64 (n = H / 32 fmaf steps + 5 butterfly additions + the bias)."""
    rng = np.random.default_rng(4)
    for H in (1, 31, 33, 384, 1000):
        h = rng.standard_normal((7, H)).astype(np.float32)
        W = rng.standard_normal((3, H)).astype(np.float32)
        b = rng.standard_normal(3).astype(np.float32)
        got = so.sat_head(h, W, b).astype(np.float64)
        want = h.astype(np.float64) @ W.T.astype(np.float64) + b
        n = -(-H // 32) + 6
        bnd = n * 2.0**-24 / (1 - n * 2.0**-24) * (np.abs(h).astype(np.float64) @ np.abs(W.T) + np.abs(b))
        assert np.all(np.abs(got - want) <= bnd), H


def test_char_logits_restatement_against_loop():
    """``sat_char_logits`` (vectorised) against a plain loop over every block of every document in float64: stitched
    logits agree to float32 rounding, and fill, scatter and the -inf of a document without tokens exactly by position."""
    rng = np.random.default_rng(6)
    T = np.array([0, 5, 300, 0, 1, 700], np.int64)
    n_chars = np.array([3, 9, 400, 0, 2, 900], np.int64)
    B, blk_off, blk_start = S.plan_blocks(T)
    tok_off, char_off = np.r_[0, np.cumsum(T)], np.r_[0, np.cumsum(n_chars)]
    blk_B = np.repeat(B, np.diff(blk_off)).astype(np.int64)
    blk_row = np.r_[0, np.cumsum(blk_B)[:-1]] + 3 * np.arange(len(blk_B))        # gaps between block rows
    NL = 3
    logits = rng.standard_normal((int(blk_row[-1] + blk_B[-1] + 3), NL)).astype(np.float32)
    hat = S.hat_table()
    tok_char = np.full(int(T.sum()), -1, np.int64)
    for d in range(len(T)):
        for t in range(int(T[d])):
            if rng.random() < 0.8:
                tok_char[tok_off[d] + t] = char_off[d] + min(t, n_chars[d] - 1)
    out, stitched = so.sat_char_logits(logits, tok_off, char_off, B, blk_off, blk_start, blk_row, hat, tok_char)
    for d in range(len(T)):
        lo = char_off[d]
        if T[d] == 0:
            assert np.all(out[lo:char_off[d + 1]] == -np.inf)
            continue
        num, den = np.zeros((int(T[d]), NL)), np.zeros(int(T[d]))
        w = hat[B[d] * (B[d] - 1) // 2:][:B[d]].astype(np.float64)
        for b in range(blk_off[d], blk_off[d + 1]):
            for k in range(B[d]):
                num[blk_start[b] + k] += w[k] * logits[blk_row[b] + k]
                den[blk_start[b] + k] += w[k]
        want = num / den[:, None]
        np.testing.assert_allclose(stitched[tok_off[d]:tok_off[d + 1]], want, rtol=1e-5, atol=1e-5)
        fill = np.full(int(n_chars[d]), stitched[tok_off[d]:tok_off[d + 1]].min(), np.float32)
        for t in range(int(T[d])):
            if tok_char[tok_off[d] + t] >= 0:
                fill[tok_char[tok_off[d] + t] - lo] = stitched[tok_off[d] + t, 0]
        np.testing.assert_array_equal(out[lo:char_off[d + 1]], fill)


def test_propagate_runs_matches_propagate():
    rng = np.random.default_rng(8)
    docs = ["", " ", "   ", "a", "a b", " a  b ", "ab   ", "a" + " " * 40 + "b", "x y z w", "  lead", "trail  "]
    docs += ["".join(rng.choice([" ", "a"], size=int(n), p=[0.4, 0.6])) for n in rng.integers(0, 60, size=200)]
    flat = "".join(docs)
    off = np.r_[0, np.cumsum([len(d) for d in docs])]
    p = rng.random(len(flat)).astype(np.float32)
    p[rng.random(len(flat)) < 0.02] = np.nan
    got = so.propagate_runs(p, np.array([c == " " for c in flat]), off)
    want = np.concatenate([so.propagate(d, p[off[i]:off[i + 1]]) for i, d in enumerate(docs)])
    np.testing.assert_array_equal(got, want)
    assert not np.array_equal(got, p, equal_nan=True)


@pytest.mark.parametrize("i", range(len(CASES)), ids=[f"{c['name']}-{c['min_len']}-{c['max_len']}" for c, *_ in CASES])
def test_partition_cuts_matches_post_processing(i):
    """``partition_cuts`` on the probabilities ``split_sentences_post`` partitions gives its sentences (and the
    reference's own), and raises where it raises."""
    c, pred, md, known = CASES[i]
    doc, min_len, max_len = c["doc"], c["min_len"], c["max_len"]
    known = md if known is None else known
    p = np.asarray(pred, np.float32).copy()
    fin = np.isfinite(known)
    p[fin] = known[fin]
    p = so.propagate(doc, p)
    if c["error"] is not None:
        if len(doc) > min_len:
            with pytest.raises(ValueError, match="Sentence partition failed"):
                so.partition_cuts(p, len(doc), min_len, max_len)
        return
    cuts = so.partition_cuts(p, len(doc), min_len, max_len)
    got = [doc[a:e] for a, e in zip([0, *cuts], [*cuts, len(doc)], strict=True)]
    assert got == c["sentences"] == so.split_sentences_post(doc, pred, min_len=min_len, max_len=max_len, known=known)
    assert cuts == sorted(cuts) and all(0 < x < len(doc) for x in cuts)


# ---- C-ABI refusals, before any CUDA call -------------------------------------------------------------------------------
RL_EINVAL, RL_ENOSPACE = -1, -3


def _abi():
    from raglite_b200 import _lib

    return _lib.load(), C.c_void_p(256)


def test_token_logits_refusals():
    lib, d = _abi()

    def head(rows=4, H=32, NL=2, hidden=d, W=d, bias=d, logits=d):
        return lib.rl_sat_token_logits(hidden, rows, H, W, bias, NL, logits, None)

    assert head(NL=0) == RL_EINVAL and head(NL=17) == RL_EINVAL
    assert "1 <= n_labels <= 16" in lib.rl_last_error().decode()
    assert head(rows=-1) == RL_EINVAL and head(H=0) == RL_EINVAL
    for k in ("hidden", "W", "bias", "logits"):
        assert head(**{k: None}) == RL_EINVAL, k
        assert "null pointer" in lib.rl_last_error().decode()
    assert head(rows=0, hidden=None, W=None, bias=None, logits=None) == 0          # nothing to do


def test_char_probas_refusals():
    lib, d = _abi()
    need = lib.rl_sat_workspace_bytes(100, 3, 2)
    assert need == 1024 + 256 and lib.rl_sat_workspace_bytes(-1, 3, 2) == 0 and lib.rl_sat_workspace_bytes(1, 1, 0) == 0

    def probas(NL=2, D=3, T=100, N=50, ws_bytes=need, **ptr):
        p = {k: d for k in ("logits", "tok_off", "char_off", "block", "blk_off", "blk_start", "blk_row", "hat",
                            "tok_char", "out", "ws")}
        p.update(ptr)
        return lib.rl_sat_char_probas(p["logits"], NL, p["tok_off"], p["char_off"], p["block"], D, T, N, p["blk_off"],
                                      p["blk_start"], p["blk_row"], p["hat"], p["tok_char"], None, None, p["out"],
                                      p["ws"], ws_bytes, None)

    for bad in (dict(NL=0), dict(NL=17), dict(D=-1), dict(T=-1), dict(N=-1)):
        assert probas(**bad) == RL_EINVAL, bad
    for k in ("tok_off", "char_off", "block", "blk_off", "out", "ws"):                # needed whatever T is
        assert probas(**{k: None}) == RL_EINVAL and probas(T=0, **{k: None}) == RL_EINVAL, k
    for k in ("logits", "blk_start", "blk_row", "hat", "tok_char"):                   # needed when T > 0
        assert probas(**{k: None}) == RL_EINVAL, k
        assert "null pointer" in lib.rl_last_error().decode()
    assert probas(ws_bytes=need - 1) == RL_ENOSPACE
    assert "workspace too small" in lib.rl_last_error().decode()
    none = {k: None for k in ("logits", "tok_off", "char_off", "block", "blk_off", "blk_start", "blk_row", "hat",
                              "tok_char", "out", "ws")}
    assert probas(D=0, **none) == 0 and probas(N=0, **none) == 0                       # nothing to do


def test_partition_refusals():
    lib, d = _abi()
    need = lib.rl_sentence_partition_workspace_bytes(100)
    assert need == 1024 + 3 * 512 and lib.rl_sentence_partition_workspace_bytes(-1) == 0

    def part(D=3, N=100, ws_bytes=need, **ptr):
        p = {k: d for k in ("probas", "off", "len", "min", "max", "cuts", "counts", "status", "ws")}
        p.update(ptr)
        return lib.rl_sentence_partition(p["probas"], p["off"], p["len"], p["min"], p["max"], D, N, p["cuts"],
                                         p["counts"], p["status"], p["ws"], ws_bytes, None)

    assert part(D=-1) == RL_EINVAL and part(N=-1) == RL_EINVAL
    for k in ("probas", "off", "len", "min", "max", "cuts", "counts", "status", "ws"):
        assert part(**{k: None}) == RL_EINVAL, k
        assert "null pointer" in lib.rl_last_error().decode()
    assert part(ws_bytes=need - 1) == RL_ENOSPACE
    assert "workspace too small" in lib.rl_last_error().decode()
    assert part(D=0, ws_bytes=0, **{k: None for k in ("probas", "off", "len", "min", "max", "cuts", "counts",
                                                       "status", "ws")}) == 0           # nothing to do


def test_early_exit_and_registration_error():
    saved = list(S._SPLITTER)
    S._SPLITTER.clear()
    try:
        for doc, min_len in (("", 4), ("abcd", 4), ("ab", 2), ("x", 1)):
            assert S.split_sentences(doc, min_len=min_len) == [doc]
        assert S.split_sentences_batch(["abc", "", "abcd"]) == [["abc"], [""], ["abcd"]]
        with pytest.raises(ModuleNotFoundError, match="register_sentence_splitter"):
            S.split_sentences("abcde")
        with pytest.raises(ModuleNotFoundError, match="register_sentence_splitter"):
            S.sentence_boundary_probas(["abc"])
    finally:
        S._SPLITTER[:] = saved
