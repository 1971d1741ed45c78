"""``split_chunklets`` / ``split_chunks`` / ``split_documents`` on the GPU through the public path: the reference's own
outputs (``tests/golden/split_chunklets.npz``, ``split_chunks.npz``), batch = single, ``embed_strings_batch`` =
``embed_strings`` bit for bit, and ``split_documents`` = steps 1-4 run one document at a time.

A ``split_chunks`` partition may differ from the reference's only where the device's float32 costs differ from NumPy's
by a rounding: it is accepted when both partitions' costs, evaluated on the float64 cost vector, agree within the sum
of ``chunks_oracle.chunk_cost_bound`` over their cuts.  Every such case is counted in ``chunk_errors.jsonl`` in the
temporary directory."""

from __future__ import annotations

import json
import tempfile
from pathlib import Path

import chunks_oracle as co
import numpy as np
import pytest

import raglite_b200 as rl

pytestmark = pytest.mark.gpu


def _cases(golden_dir, name: str):
    z = np.load(golden_dir / name)
    return json.loads(bytes(z["cases"]).decode()), z


def test_golden_chunklets(golden_dir):
    cases, _ = _cases(golden_dir, "split_chunklets.npz")
    for c in cases:
        if c["error"] is not None:
            with pytest.raises(ValueError, match=c["error"]):
                rl.split_chunklets(c["sentences"], max_size=c["max_size"])
        else:
            assert rl.split_chunklets(c["sentences"], max_size=c["max_size"]) == c["chunklets"], c["name"]
    ok = [c for c in cases if c["error"] is None]
    assert rl.split_chunklets_batch([c["sentences"] for c in ok], max_size=64) == [
        rl.split_chunklets(c["sentences"], max_size=64) for c in ok]


def test_golden_chunks(golden_dir):
    cases, z = _cases(golden_dir, "split_chunks.npz")
    differ = 0
    for i, c in enumerate(cases):
        emb = z[f"emb{i}"]
        if c["error"] is not None:
            with pytest.raises(ValueError, match=c["error"]):
                rl.split_chunks(c["chunklets"], emb, max_size=c["max_size"])
            continue
        chunks, embs = rl.split_chunks(c["chunklets"], emb, max_size=c["max_size"])
        assert "".join(chunks) == "".join(c["chunklets"]) and all(e.dtype == emb.dtype for e in embs)
        cuts = _cuts(c["chunklets"], chunks)
        assert [len(e) for e in embs] == np.diff([0, *cuts, len(emb)]).tolist()
        assert np.array_equal(np.concatenate(embs), emb)
        if chunks == c["chunks"]:
            continue
        sizes = np.array([len(x) for x in c["chunklets"]])
        keep = co.nonoutlying(sizes)
        cost64, info = co.chunk_costs_f64(emb, keep, [co.is_heading(x) for x in c["chunklets"]])
        bound = co.chunk_cost_bound(emb.shape[1], int(keep.sum()), info)
        got, want = cuts, _cuts(c["chunklets"], c["chunks"])
        gap = abs(co.objective(cost64, got) - co.objective(cost64, want))
        assert gap <= sum(bound[x - 1] for x in got) + sum(bound[x - 1] for x in want), (c["name"], gap)
        differ += 1
    with (Path(tempfile.gettempdir()) / "chunk_errors.jsonl").open("a") as f:
        f.write(json.dumps({"golden_chunks": len(cases), "differing_partitions": differ}) + "\n")


def _cuts(items: list[str], pieces: list[str]) -> list[int]:
    ends = np.cumsum([len(s) for s in items]).tolist()
    return [ends.index(e) + 1 for e in np.cumsum([len(p) for p in pieces])[:-1].tolist()]


def test_chunks_batch_equals_single(golden_dir):
    cases, z = _cases(golden_dir, "split_chunks.npz")
    ok = [(c, z[f"emb{i}"]) for i, c in enumerate(cases) if c["error"] is None and max(map(len, c["chunklets"])) <= 600]
    assert len(ok) > 20
    assert len({e.shape[1] for _, e in ok}) > 1 and len({e.dtype for _, e in ok}) > 1   # widths and dtypes mixed
    batch = rl.split_chunks_batch([c["chunklets"] for c, _ in ok], [e for _, e in ok], max_size=600)
    for (c, e), (chunks, embs) in zip(ok, batch, strict=True):
        want_chunks, want_embs = rl.split_chunks(c["chunklets"], e, max_size=600)
        assert chunks == want_chunks and all(np.array_equal(a, b) for a, b in zip(embs, want_embs, strict=True))


@pytest.fixture(scope="module")
def models():
    """A seeded 1-layer SaT and a 2-layer bge-m3-shaped token embedder (n_ctx = 64, so documents take many segments),
    registered for the module."""
    import torch
    from transformers import XLMRobertaConfig, XLMRobertaForTokenClassification

    from oracle import embed as oe
    from raglite_b200 import _embed, _sentences

    tok = oe.unigram_tokenizer()
    torch.manual_seed(0)
    sat_cfg = XLMRobertaConfig(vocab_size=1000, hidden_size=128, num_hidden_layers=1, num_attention_heads=2,
                               intermediate_size=256, max_position_embeddings=514, type_vocab_size=1, pad_token_id=1,
                               layer_norm_eps=1e-5, num_labels=1)
    sat = rl.SaTEngine.from_hf(XLMRobertaForTokenClassification(sat_cfg).eval(), tok)
    cfg = rl.RAGLiteConfig(reranker=None, chunk_max_size=400)
    model = oe.seeded_model(oe.bge_m3_config(num_hidden_layers=2, vocab_size=1000, max_position_embeddings=514), seed=5)
    eng = rl.TokenEmbedderEngine.from_hf(model, tokenizer=tok, n_ctx=64)
    saved_s, saved_e = list(_sentences._SPLITTER), _embed._TOKEN_EMBEDDERS.get(cfg.embedder)
    rl.register_sentence_splitter(sat)
    rl.register_token_embedder(cfg.embedder, eng)
    yield cfg
    _sentences._SPLITTER[:] = saved_s
    if saved_e is None:
        _embed._TOKEN_EMBEDDERS.pop(cfg.embedder, None)
    else:
        rl.register_token_embedder(cfg.embedder, saved_e)


def _documents(n: int, seed: int) -> list[str]:
    rng = np.random.default_rng(seed)
    words = "alpha beta gamma delta light clock rod frame event time of the observer velocity".split()
    docs = []
    for _ in range(n):
        parts = []
        for _ in range(int(rng.integers(1, 8))):
            if rng.random() < 0.4:
                parts.append("# " + " ".join(rng.choice(words, size=3)) + "\n\n")
            sent = [" ".join(rng.choice(words, size=int(rng.integers(3, 20)))).capitalize() + "."
                    for _ in range(int(rng.integers(1, 12)))]
            parts.append(" ".join(sent) + "\n\n")
        docs.append("".join(parts))
    return docs


def test_embed_strings_batch_equals_embed_strings(models):
    cfg = models
    docs = [rl.split_sentences(d, max_len=cfg.chunk_max_size) for d in _documents(12, 3)]
    got = rl.embed_strings_batch(docs, config=cfg)
    nan_rows = 0
    for d, g in zip(docs, got, strict=True):
        want = rl.embed_strings(d, config=cfg)
        assert g.dtype == want.dtype == np.float16 and g.shape == want.shape
        np.testing.assert_array_equal(g.view(np.uint16), want.view(np.uint16))    # bits: NaN rows compare too
        np.testing.assert_array_equal(rl.embed_strings(d, config=cfg).view(np.uint16), want.view(np.uint16))
        nan_rows += int(np.isnan(want).any(axis=1).sum())
    with (Path(tempfile.gettempdir()) / "chunk_errors.jsonl").open("a") as f:
        f.write(json.dumps({"embed_docs": len(docs), "embed_rows": sum(map(len, got)), "nan_rows": nan_rows}) + "\n")


def test_split_documents_equals_one_at_a_time(models):
    cfg = models
    docs = [*_documents(16, 4), "Short."]
    got = rl.split_documents(docs, config=cfg)
    for doc, (chunks, embs) in zip(docs, got, strict=True):
        sentences = rl.split_sentences(doc, max_len=cfg.chunk_max_size)
        chunklets = rl.split_chunklets(sentences, max_size=cfg.chunk_max_size)
        emb = rl.embed_strings(chunklets, config=cfg)
        want_chunks, want_embs = rl.split_chunks(chunklets, emb, max_size=cfg.chunk_max_size)
        assert chunks == want_chunks and "".join(chunks) == doc
        assert len(embs) == len(want_embs) and all(np.array_equal(a, b) for a, b in zip(embs, want_embs, strict=True))
    assert sum(len(c) > 1 for c, _ in got) >= 4
