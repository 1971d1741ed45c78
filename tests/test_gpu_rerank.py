"""GPU parity of the cross-encoder engine against the float32 transformers oracle (seeded weights)."""

from __future__ import annotations

import json
import tempfile
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _random_pairs(n, vocab, rng, lo=6, hi=180, lengths=()):
    """``lengths`` first, then ``n`` pairs of random length in [lo, hi)."""
    ids, types = [], []
    for L in [*lengths, *(int(rng.integers(lo, hi)) for _ in range(n))]:
        q = int(rng.integers(2, max(3, L // 3)))
        a = rng.integers(1000, vocab, size=L).astype(np.int32)
        a[0], a[q], a[-1] = 101, 102, 102                       # [CLS] ... [SEP] ... [SEP]
        t = np.zeros(L, np.int32)
        t[q + 1:] = 1
        ids.append(a); types.append(t)
    return ids, types


def _record(name: str, payload: dict) -> None:
    """Append a line (case + measured error) to xenc_bounds.jsonl in the temporary directory."""
    with (Path(tempfile.gettempdir()) / "xenc_bounds.jsonl").open("a") as f:
        f.write(json.dumps({"test": name, **payload}) + "\n")


def test_linear_layer_matches_torch():
    """``rl_xenc_linear`` against float64 from the fp16-rounded X and W, GELU(erf) exact.  Shapes: the model's, short
    last 128-column passes (N % 128 != 0: stale weight rows may only feed columns that are not stored), K tails
    (K % 64 != 0: the tensor map zero-fills), ragged token tiles, and T = 20000 (more work items than SMs, so every
    CTA loops over items and reuses its stage ring and epilogue staging).  The widths the served models run: BERT-base /
    XLM-R base (qkv 2304 x 768, o 768 x 768, up 3072 x 768 + GELU, down 768 x 3072) and XLM-R large / bge-m3 (qkv
    3072 x 1024, o, up 4096 x 1024 + GELU, down 1024 x 4096: 32 column passes, or 64 K slices, about a dozen trips
    round the stage ring per item), each at T = 1, 129 and 20000."""
    import itertools

    import torch

    from raglite_b200 import _lib

    lib = _lib.load()
    g = torch.Generator(device="cuda").manual_seed(0)
    shapes = [(300, 384, 384, 0), (1000, 1536, 384, 1), (777, 384, 1536, 0), (64, 1152, 384, 0)]
    Ts = (1, 127, 128, 129, 20000)
    shapes += [(T, N, K, act) for N, K, T, act in itertools.product((32, 96, 160, 416, 480), (8, 72, 160, 416), Ts, (0, 1))]
    served = [(2304, 768, 0), (768, 768, 0), (3072, 768, 1), (768, 3072, 0), (3072, 1024, 0), (1024, 1024, 0),
              (4096, 1024, 1), (1024, 4096, 0)]
    shapes += [(T, N, K, act) for (N, K, act), T in itertools.product(served, (1, 129, 20000))]
    s = torch.cuda.current_stream().cuda_stream
    worst, worst_at = 0.0, None
    for (T, N, K, act) in shapes:
        X = (torch.randn((T, K), generator=g, device="cuda") * 0.5).half()
        W = torch.randn((N, K), generator=g, device="cuda") / K**0.5
        b = torch.randn(N, generator=g, device="cuda")
        img = torch.empty(lib.rl_xenc_linear_image_bytes(N, K), dtype=torch.uint8, device="cuda")
        assert lib.rl_xenc_pack_linear(W.data_ptr(), N, K, img.data_ptr(), s) == 0
        Y = torch.full((T, N), float("nan"), dtype=torch.float16, device="cuda")
        assert lib.rl_xenc_linear(X.data_ptr(), img.data_ptr(), b.data_ptr(), Y.data_ptr(), T, N, K, act, s) == 0, lib.rl_last_error()
        Xd, Wd = X.double(), W.half().double()
        ref = Xd @ Wd.T + b.double()
        if act:
            ref = 0.5 * ref * (1.0 + torch.erf(ref / 2.0**0.5))
        # fp16 output rounding + fp32 accumulation over K products (and the bias add) + the erf approximation
        # (<= 8e-7 on the GELU value, xenc.cu)
        bound = 2.0**-11 * ref.abs() + (K + 2) * 2.0**-23 * (Xd.abs() @ Wd.abs().T) + 1e-6
        r = float(((Y.double() - ref).abs() / bound).max())          # (NaN: an output was never written)
        assert r <= 1.0, (T, N, K, act, r)
        if r > worst:
            worst, worst_at = r, (T, N, K, act)
    _record("linear", {"max_err_over_bound": worst, "at_T_N_K_act": worst_at, "shapes": len(shapes)})


def _check_logits(name, model, eng, ids, types):
    from scipy.stats import kendalltau

    from oracle import rerank as orr

    got_logit, got_score = eng.score_tokens(ids, types)
    want = orr.hf_logits(model, ids, types)
    err = np.abs(got_logit - want)
    _record(name, {"pairs": len(ids), "max_len": max(len(x) for x in ids), "max_abs_logit_err": float(err.max()),
                   "logit_spread": float(want.std())})
    assert err.max() < 4e-2, (name, err.max(), len(ids[int(err.argmax())]))
    assert np.abs(got_score - orr.flashrank_scores(want)).max() < 1e-2
    assert kendalltau(got_logit, want)[0] > 0.97


@pytest.mark.parametrize("layers", [2, 12])
def test_cross_encoder_logits_match_transformers_fp32(layers):
    """Every bias, LayerNorm gamma and beta drawn away from its init value (``perturb``), so a forward that dropped
    one of them would not match."""
    from oracle import rerank as orr
    from raglite_b200._xenc import CrossEncoderEngine

    model = orr.seeded_model(seed=layers, perturb=True, num_hidden_layers=layers, vocab_size=5000)
    eng = CrossEncoderEngine.from_hf(model, max_tokens_per_call=4000)       # forces several packed calls
    rng = np.random.default_rng(1)
    ids, types = _random_pairs(48, 5000, rng)
    ids.append(np.array([101, 2000, 102, 2001, 102], np.int32)); types.append(np.array([0, 0, 0, 1, 1], np.int32))
    _check_logits(f"logits_layers{layers}", model, eng, ids, types)


def test_cross_encoder_long_sequences_match_transformers():
    """Pair lengths up to MiniLM's 512 positions: the attention kernel's long key loops, a 32-key tail after several
    64-key blocks, and lengths on either side of every 32 / 64 / 128 / 256 boundary; several packed calls."""
    from oracle import rerank as orr
    from raglite_b200._xenc import CrossEncoderEngine

    model = orr.seeded_model(seed=21, perturb=True, num_hidden_layers=2, vocab_size=5000)
    eng = CrossEncoderEngine.from_hf(model, max_length=512, max_tokens_per_call=3000)
    rng = np.random.default_rng(2)
    lengths = (3, 31, 32, 33, 63, 64, 65, 96, 97, 128, 129, 255, 256, 257, 384, 511, 512)
    ids, types = _random_pairs(24, 5000, rng, lo=3, hi=513, lengths=lengths)
    order = rng.permutation(len(ids))                                # long and short pairs share calls
    ids, types = [ids[i] for i in order], [types[i] for i in order]
    _check_logits("long_sequences", model, eng, ids, types)


@pytest.mark.parametrize(("hidden", "heads", "ffn", "layers"), [(160, 5, 416, 2), (512, 16, 2048, 1)])
def test_cross_encoder_other_widths_match_transformers(hidden, heads, ffn, layers):
    """hidden 160: the scalar LayerNorm (H % 128 != 0), short last linear passes (3H = 480, F = 416 are not multiples
    of 128) and K tails of 32 (K = 160, 416).  hidden 512: the H <= 512 edge of the LayerNorm kernels and 16 warps in
    the pooler / classifier head."""
    from oracle import rerank as orr
    from raglite_b200._xenc import CrossEncoderEngine

    model = orr.seeded_model(seed=hidden, perturb=True, hidden_size=hidden, num_attention_heads=heads,
                             intermediate_size=ffn, num_hidden_layers=layers, vocab_size=5000)
    eng = CrossEncoderEngine.from_hf(model, max_tokens_per_call=4000)
    rng = np.random.default_rng(3)
    ids, types = _random_pairs(40, 5000, rng, lo=3, hi=400)
    _check_logits(f"width{hidden}", model, eng, ids, types)


def test_rerank_chunks_with_b200_cross_encoder(tmp_path):
    """End to end through the reference's call shape: rerank_chunks -> ranker.rank(query=, docs=)."""
    from tokenizers import Tokenizer, models, pre_tokenizers, processors

    import raglite_b200 as rl
    from oracle import rerank as orr
    from raglite_b200._rerank import ScoreFnRanker
    from raglite_b200._xenc import CrossEncoderEngine

    words = ["[PAD]", "[UNK]", "[CLS]", "[SEP]"] + [f"w{i}" for i in range(200)]
    tok = Tokenizer(models.WordPiece({w: i for i, w in enumerate(words)}, unk_token="[UNK]"))
    tok.pre_tokenizer = pre_tokenizers.Whitespace()
    tok.post_processor = processors.TemplateProcessing(single="[CLS] $A [SEP]", pair="[CLS] $A [SEP] $B:1 [SEP]:1",
                                                       special_tokens=[("[CLS]", 2), ("[SEP]", 3)])
    model = orr.seeded_model(seed=5, num_hidden_layers=3, vocab_size=len(words))
    eng = CrossEncoderEngine.from_hf(model, tok, max_length=64)
    rng = np.random.default_rng(0)
    chunks = [rl.Chunk(id=f"c{i}", body=" ".join(f"w{j}" for j in rng.integers(0, 200, size=int(rng.integers(5, 90)))))
              for i in range(20)]
    query = "w1 w2 w3 w4"
    cfg = rl.RAGLiteConfig(reranker=ScoreFnRanker(lambda q, docs: eng.score_pairs([q] * len(docs), list(docs))))
    ranked = rl.rerank_chunks(query, chunks, config=cfg)
    ids, types = eng.encode_pairs([query] * len(chunks), [str(c) for c in chunks])
    assert max(len(x) for x in ids) <= 64                                        # truncation applied
    want = orr.rank_order(orr.flashrank_scores(orr.hf_logits(model, ids, types)))
    got = [int(c.id[1:]) for c in ranked]
    assert sorted(got) == list(range(20))
    # identical order except where float32 scores are within fp16 noise of each other
    ref_scores = orr.flashrank_scores(orr.hf_logits(model, ids, types))
    for a, b in zip(got, want.tolist(), strict=True):
        assert a == b or abs(ref_scores[a] - ref_scores[b]) < 2e-2
