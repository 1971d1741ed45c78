"""Throughput of ``insert_documents`` on the GPU, late chunking and standard.

On ``bench_split_sentences.py``'s seeded corpus (2000 documents of 20 k characters), with the seeded SaT and the
bge-m3-shaped 2-layer embedder ``bench_split_chunks.py`` builds (n_ctx 512, ``chunk_max_size`` 2048), it reports:

* documents/s and characters/s of ``insert_documents`` end to end into a fresh index, for the default late-chunking
  embedder string and for a standard one;
* for each embedding type, the same work run stage by stage with a synchronise after each: ``split_documents``'s steps
  (``_split_documents_device``), chunk records on the host, the full-chunk forward and pool, the blend, and the append
  into the index (in this run the stages of every document group are summed);
* the card's name and power limit, read in the same run.
"""

from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / "tests"), str(ROOT / "tools")]


def staged(docs, cfg) -> dict:
    """``insert_documents``' stages one after another, each closed by a synchronise (seconds)."""
    import numpy as np

    import raglite_b200 as rl
    from raglite_b200 import _insert as I  # noqa: N812
    from raglite_b200._chunks import _join_pieces, _offsets, _split_documents_device
    from raglite_b200._embed import _mean_pool_device

    t = dict.fromkeys(("split_s", "records_s", "full_chunk_forward_s", "blend_s", "append_s"), 0.0)

    def clock(name, fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        t[name] += time.perf_counter() - t0
        return out

    standard = rl._embed.embedding_type(config=cfg) == "standard"  # noqa: SLF001
    rows, counts, records = [], [], []
    for group in I._document_groups(docs, cfg):  # noqa: SLF001
        chunklets, X, _, cuts = clock("split_s", lambda g=group: _split_documents_device([d.content for d in g], cfg))

        def recs(g=group, chunklets=chunklets, cuts=cuts):
            return [r for d, c, cut in zip(g, chunklets, cuts, strict=True) for r in I.chunk_records(d, _join_pieces(c, cut))]

        rec = clock("records_s", recs)
        n = np.concatenate([np.diff([0, *cut, len(c)]) for c, cut in zip(chunklets, cuts, strict=True)])
        if standard:
            F = clock("full_chunk_forward_s", lambda rec=rec: _mean_pool_device([r.content for r in rec], cfg))
            X = clock("blend_s", lambda X=X, F=F, n=n: I.chunk_embedding_blend(X, F, _offsets(n)))
        rows.append(X)
        counts.append(n)
        records += rec
    X = torch.cat(rows)
    idx = rl.CorpusIndex(X[:0], chunk_ids=[], chunks=[], chunk_metadata=[], storage=I._auto_storage(X))  # noqa: SLF001
    clock("append_s", lambda: idx.append(X, _offsets(np.concatenate(counts)), chunk_ids=[c.id for c in records],
                                         chunks=records, chunk_metadata=[c.metadata_ for c in records]))
    t = {k: round(v, 3) for k, v in t.items()}
    t["rows"], t["chunks"] = int(X.shape[0]), len(records)
    return t


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=2000)
    ap.add_argument("--chars", type=int, default=20000)
    ap.add_argument("--types", default="late_chunking,standard", help="embedding types to measure, comma-separated")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_insert needs a CUDA device")
    from bench_split_sentences import card, corpus, sat_model

    import raglite_b200 as rl
    from oracle import embed as oe

    texts = corpus(a.docs, a.chars)
    n_chars = sum(map(len, texts))
    res: dict = {"metric": "insert_documents_docs_per_s", "docs": a.docs, "chars": n_chars, **card()}
    tok = oe.unigram_tokenizer()
    rl.register_sentence_splitter(rl.SaTEngine.from_hf(sat_model(), tok))
    model = oe.seeded_model(oe.bge_m3_config(num_hidden_layers=2, vocab_size=250002, max_position_embeddings=8194), seed=5)
    eng = rl.TokenEmbedderEngine.from_hf(model, tokenizer=tok, n_ctx=512)
    embedders = {"late_chunking": rl.RAGLiteConfig().embedder, "standard": "bench-standard/bge-m3-shaped"}
    for name in a.types.split(","):
        embedder = embedders[name]
        cfg = rl.RAGLiteConfig(db_url=f"bench-insert://{name}", embedder=embedder, reranker=None)
        rl.register_token_embedder(embedder, eng)
        warm = rl.RAGLiteConfig(db_url=f"bench-insert://{name}-warm", embedder=embedder, reranker=None)
        rl.insert_documents([rl.Document.from_text(x) for x in texts[:4]], config=warm)   # warm-up
        rl.unregister_index(warm)
        docs = [rl.Document.from_text(x) for x in texts]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        rl.insert_documents(docs, config=cfg)
        torch.cuda.synchronize()
        t = time.perf_counter() - t0
        idx = rl.get_index(cfg)
        res[name] = {"insert_s": round(t, 3), "docs_per_s": round(a.docs / t, 2), "chars_per_s": round(n_chars / t),
                     "rows": idx.n_rows, "chunks": idx.n_chunks, "storage": idx.storage}
        print(json.dumps({name: res[name]}), flush=True)   # progress: the stage-by-stage run takes as long again
        res[name]["stages"] = staged(docs, cfg)
        rl.unregister_index(cfg)
        del idx
        torch.cuda.empty_cache()
    res["peak_mem_gb"] = round(torch.cuda.max_memory_allocated() / 2**30, 2)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
