"""``rag()`` end to end on the GPU over a registered index: documents inserted with ``insert_documents`` (a seeded SaT
and a bge-m3-shaped token embedder), ``retrieve_context``, ``add_context`` and ``rag`` with a Qwen3 fixture GGUF.  The
streamed text equals ``generate`` on the rendered prompt, the answer is appended, and each ``<source>`` is its
document's url or filename."""

from __future__ import annotations

import re

import pytest
import torch

import raglite_b200 as rl
from qwen3_fixtures import make_model, write_qwen3_gguf

pytestmark = pytest.mark.gpu

DOCS = [("# Foxes\n\nThe quick brown fox jumps over the lazy dog. The fox is brown and quick.\n", "fox.md", None),
        ("# Dogs\n\nThe lazy dog sleeps all day. It's 2024 and the dog still sleeps.\n", "dog.md", "https://example.org/dog"),
        ("# Clocks\n\nA clock in the frame of the observer ticks. Time of the event.\n", "clock.md", None)]


@pytest.fixture
def config(tmp_path, request):
    """A config whose index, token embedder, sentence splitter and LLM are all registered (undone in teardown)."""
    from transformers import XLMRobertaConfig, XLMRobertaForTokenClassification

    from oracle import embed as oe
    from raglite_b200 import _embed, _llm, _sentences

    tok = oe.unigram_tokenizer()
    torch.manual_seed(0)
    sat_cfg = XLMRobertaConfig(vocab_size=1000, hidden_size=128, num_hidden_layers=1, num_attention_heads=2,
                               intermediate_size=256, max_position_embeddings=514, type_vocab_size=1, pad_token_id=1,
                               layer_norm_eps=1e-5, num_labels=1)
    sat = rl.SaTEngine.from_hf(XLMRobertaForTokenClassification(sat_cfg).eval(), tok)
    model = oe.seeded_model(oe.bge_m3_config(num_hidden_layers=2, vocab_size=1000, max_position_embeddings=514), seed=5)
    embedder = rl.TokenEmbedderEngine.from_hf(model, tokenizer=tok, n_ctx=64)
    path = tmp_path / "rag.gguf"
    write_qwen3_gguf(path, make_model(layers=1, tied=True, seed=5), mode="Q8_0", seed=2)
    llm = rl.LlmEngine.from_gguf(path, n_ctx=2048, prefill_chunk=128)
    cfg = rl.RAGLiteConfig(db_url="rag-test://index", llm="llama-cpp-python/test/qwen3-test/rag.gguf@2048", reranker=None,
                           chunk_max_size=400)
    saved_split, saved_emb = list(_sentences._SPLITTER), _embed._TOKEN_EMBEDDERS.get(cfg.embedder)
    rl.register_sentence_splitter(sat)
    rl.register_token_embedder(cfg.embedder, embedder)
    rl.register_llm(cfg, llm)

    def undo() -> None:
        rl.unregister_index(cfg)
        _llm._LLMS.pop(cfg.llm, None)
        _sentences._SPLITTER[:] = saved_split
        if saved_emb is None:
            _embed._TOKEN_EMBEDDERS.pop(cfg.embedder, None)
        else:
            rl.register_token_embedder(cfg.embedder, saved_emb)

    request.addfinalizer(undo)
    return cfg


def test_rag_over_inserted_documents(config):
    from raglite_b200 import _rag

    docs = [rl.Document.from_text(text, filename=name, url=url) for text, name, url in DOCS]
    rl.insert_documents(docs, config=config)
    want_source = {d.id: d.url or d.filename for d in docs}
    spans = rl.retrieve_context("What colour is the fox?", num_chunks=3, config=config)
    assert spans and all(s.document is not None for s in spans)
    assert [s.source for s in spans] == [want_source[s.document_id] for s in spans]
    msg = rl.add_context("What colour is the fox?", spans, config)
    sources = re.findall(r"<source>(.*)</source>", msg["content"])
    assert sources == [want_source[s.document_id] for s in spans]
    messages = [{"role": "system", "content": "Be brief."}, msg]
    engine = _rag.get_llm(config)
    prompt = engine.tokenizer.encode(_rag.render_chatml(messages))
    want = "".join(engine.generate(prompt, max_tokens=12, seed=4, **_rag.QWEN3_SAMPLING))
    got = list(rl.rag(messages, config=config, max_tokens=12, seed=4))
    assert "".join(got) == want
    assert messages[-1] == {"role": "assistant", "content": want} and len(messages) == 3
