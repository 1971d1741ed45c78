"""The Qwen3 decoder end to end against transformers' Qwen3ForCausalLM in float64 on the CPU, on GGUF files whose
quantized weights the reference model holds exactly (Q8_0 and a Q4_K_M-style mix, tied and separate output weights):
logits after prefill and after each decode step, greedy continuations, chunked prefill, seeded sampling and rag()."""

from __future__ import annotations

import numpy as np
import pytest
import torch

from qwen3_fixtures import hf_model_f64, make_model, write_qwen3_gguf

pytestmark = pytest.mark.gpu

LAYERS = 2
# Tolerance on the logits, relative to their largest magnitude.  Every linear reads fp16 activations and writes fp16
# outputs, and the weights enter the prefill's wgmma as fp16 values of the image: per layer about ten roundings of
# 2^-11 relative (RMSNorm out, Q / K / V, QK-norm + RoPE out, attention out, O, FFN norm out, gate, up, SwiGLU out,
# down), plus the output norm and the head.  Summed linearly: (10 L + 4) 2^-11.
TOL = (10 * LAYERS + 4) * 2.0 ** -11


@pytest.fixture(scope="module", params=[("Q8_0", True), ("Q4_K_M", True), ("Q4_K_M", False), ("Q8_0", False)],
                ids=["Q8_0-tied", "Q4_K_M-tied", "Q4_K_M-untied", "Q8_0-untied"])
def pair(request, tmp_path_factory):
    from raglite_b200._llm import LlmEngine

    mode, tied = request.param
    model = make_model(layers=LAYERS, tied=tied, seed=3)
    path = tmp_path_factory.mktemp("qwen3") / f"{mode}-{tied}.gguf"
    sd = write_qwen3_gguf(path, model, mode=mode, seed=7)
    ref = hf_model_f64(model, sd)
    eng = LlmEngine.from_gguf(path, n_ctx=256, prefill_chunk=64)
    return eng, ref


def _ref_logits(ref, ids: list[int]) -> np.ndarray:
    with torch.no_grad():
        return ref(torch.tensor([ids])).logits[0].numpy()


def _check(got: np.ndarray, want: np.ndarray) -> None:
    err = np.abs(got.astype(np.float64) - want).max()
    assert err <= TOL * np.abs(want).max(), (err, TOL * np.abs(want).max())


def test_logits_after_prefill_and_each_decode_step(pair):
    eng, ref = pair
    rng = np.random.default_rng(0)
    ids2 = rng.integers(0, eng.plan.vocab, size=96).tolist()
    want = _ref_logits(ref, ids2)
    eng.reset()
    _check(eng.prefill(ids2[:90]).cpu().numpy(), want[89])
    eng.reset()
    eng.prefill(ids2[:90])
    for i in range(90, 96):   # one decode step (T = 1, the GEMV path) per token
        _check(eng.prefill([ids2[i]]).cpu().numpy(), want[i])


def test_prefill_in_one_chunk_equals_prefill_in_several(pair):
    eng, _ = pair
    ids = np.random.default_rng(1).integers(0, eng.plan.vocab, size=150).tolist()
    eng.reset()
    a = eng.prefill(ids, chunk=64).cpu().numpy()
    eng.reset()
    b = eng.prefill(ids, chunk=50).cpu().numpy()
    eng.reset()
    c = eng.prefill(ids[:149], chunk=64).cpu().numpy()
    c = eng.prefill(ids[149:]).cpu().numpy()
    want = _ref_logits(pair[1], ids)[-1]
    for x in (a, b, c):
        _check(x, want)


def test_greedy_continuation_equals_the_float64_model_where_its_margin_exceeds_the_bound(pair):
    """Along the engine's own greedy continuation, each token is the float64 model's argmax wherever the model's top-2
    margin exceeds twice the logit bound (closer calls may go either way)."""
    eng, ref = pair
    checked = 0
    for seed in range(6):
        prompt = np.random.default_rng(seed).integers(0, eng.plan.vocab, size=20).tolist()
        got = list(eng.generate_ids(prompt, max_tokens=16, temperature=0.0, repeat_penalty=1.0))
        ids = list(prompt)
        for t in got:
            lg = _ref_logits(ref, ids)[-1]
            top2 = np.sort(lg)[-2:]
            if top2[1] - top2[0] > 2 * TOL * np.abs(lg).max():
                assert t == int(np.argmax(lg))
                checked += 1
            ids.append(t)
    assert checked >= 3   # 55 to 93 of the 96 float64 greedy steps clear the margin on each fixture


def test_fixed_seed_reproduces_its_output(pair):
    eng, _ = pair
    prompt = eng.tokenizer.encode("<|im_start|>user\nThe quick brown fox<|im_end|>\n<|im_start|>assistant\n")
    a = list(eng.generate_ids(prompt, max_tokens=30, seed=11, temperature=1.0))
    b = list(eng.generate_ids(prompt, max_tokens=30, seed=11, temperature=1.0))
    assert a == b and len(a) > 0
    text = "".join(eng.generate(prompt, max_tokens=30, seed=11, temperature=1.0))
    assert text == eng.tokenizer.decode_bytes(a).decode("utf-8", errors="replace")


def test_prompt_longer_than_n_ctx_raises(pair):
    eng, _ = pair
    with pytest.raises(ValueError, match="exceed context window"):
        list(eng.generate_ids([1] * 257, max_tokens=1))


def test_rag_streams_generate_on_the_rendered_prompt(tmp_path):
    import raglite_b200 as rl
    from raglite_b200 import _rag
    from raglite_b200._llm import LlmEngine, register_llm

    model = make_model(layers=1, tied=True, seed=5)
    path = tmp_path / "rag.gguf"
    write_qwen3_gguf(path, model, mode="Q8_0", seed=2)
    eng = LlmEngine.from_gguf(path, n_ctx=512, prefill_chunk=128)
    cfg = rl.RAGLiteConfig(llm="llama-cpp-python/test/qwen3-test/rag.gguf@512", reranker=None)
    register_llm(cfg, eng)
    spans = [rl.ChunkSpan(chunks=[rl.Chunk(id="c0", document_id="d0", index=0, body="The fox is brown.",
                                           metadata_={"filename": "fox.md"})])]
    msg = rl.add_context("What colour is the fox?", spans, cfg)
    assert "<context>" in msg["content"] and "fox.md" in msg["content"]
    messages = [{"role": "system", "content": "Be brief."}, msg]
    prompt = eng.tokenizer.encode(_rag.render_chatml(messages))
    want = "".join(eng.generate(prompt, max_tokens=16, seed=4, **_rag.QWEN3_SAMPLING))
    got = list(rl.rag(messages, config=cfg, max_tokens=16, seed=4))
    assert "".join(got) == want
    assert messages[-1] == {"role": "assistant", "content": want}
    with pytest.raises(NotImplementedError, match="retrieve_context"):
        list(rl.rag([{"role": "user", "content": "hi"}], config=cfg))
    with pytest.raises(NotImplementedError, match="register_gguf_llm"):
        list(rl.rag([msg], config=rl.RAGLiteConfig(llm="llama-cpp-python/x/y/z.gguf", reranker=None)))
