"""Throughput of ``split_chunklets_batch`` / ``split_chunks_batch`` / ``split_documents`` on the GPU.

On ``bench_split_sentences.py``'s seeded corpus (2000 documents of 20 k characters, max_size 2048), cut into sentences
after every '. ' and newline (the SaT model is not needed for steps 2 and 4), it reports:

* characters/s of ``split_chunklets_batch`` and of ``split_chunks_batch`` (seeded fp16 rows, d = 1024), each with its
  host share (Markdown parse, statement counts, quantiles, heading flags, uploads) and device share (kernel events);
* the reference's Python dynamic program and ``linprog`` restated on the host (``tests/chunks_oracle.py``) over a few
  documents, for scale;
* ``split_documents`` end to end with a seeded 1-layer SaT and a 2-layer embedder on a subset;
* the card's name and power limit, read in the same run.
"""

from __future__ import annotations

import argparse
import json
import re
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / "tests"), str(ROOT / "tools")]


def sentences_of(doc: str) -> list[str]:
    return [s for s in re.split(r"(?<=\. )|(?<=\n)", doc) if s]


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t


def kernel_times(chunklets, embs, sents, max_size: int, reps: int = 5) -> dict:
    """Milliseconds per launch of rl_chunk_similarities, rl_chunk_partition and rl_chunklet_partition on the whole batch
    (the median of ``reps`` launches after one warm-up)."""
    from raglite_b200 import _chunks as K
    from raglite_b200 import _lib

    lib, st = _lib.load(), torch.cuda.current_stream().cuda_stream

    def up(x):
        return torch.from_numpy(np.ascontiguousarray(x)).cuda()

    todo = [i for i, c in enumerate(chunklets) if len(c) > 1 and sum(map(len, c)) > max_size]
    D = len(todo)
    off = np.zeros(D + 1, np.int64)
    np.cumsum([len(chunklets[i]) for i in todo], out=off[1:])
    N = int(off[-1])
    X = up(np.concatenate([embs[i] for i in todo]))
    lens = np.concatenate([[len(x) for x in chunklets[i]] for i in todo]).astype(np.int32)
    non = np.concatenate([K._nonoutlying(np.array([len(x) for x in chunklets[i]])) for i in todo]).view(np.uint8)  # noqa: SLF001
    head = np.array([K.is_heading(x) for i in todo for x in chunklets[i]]).view(np.uint8)
    d_off, d_non, d_head, d_len = up(off), up(non), up(head), up(lens)
    d_max = torch.full((max(D, 1),), max_size, dtype=torch.int32, device="cuda")
    costs = torch.empty(max(N, 1), dtype=torch.float32, device="cuda")
    cuts = torch.empty(max(N, 1), dtype=torch.int32, device="cuda")
    cs = torch.empty(2 * max(D, 1), dtype=torch.int32, device="cuda")
    ws_s = torch.empty(int(lib.rl_chunk_similarities_workspace_bytes(N)), dtype=torch.uint8, device="cuda")
    ws_p = torch.empty(int(lib.rl_chunk_partition_workspace_bytes(N, D)), dtype=torch.uint8, device="cuda")
    S = len(sents)
    s_off = np.zeros(S + 1, np.int64)
    np.cumsum([len(x) for x in sents], out=s_off[1:])
    NS = int(s_off[-1])
    p = up(np.concatenate([K.markdown_chunklet_boundaries(x) for x in sents]))
    q = up(np.concatenate([K.num_statements(x) for x in sents]))
    s_len = up(np.array([len(y) for x in sents for y in x], np.int32))
    d_soff = up(s_off)
    s_max = torch.full((S,), max_size, dtype=torch.int32, device="cuda")
    s_cuts = torch.empty(max(NS, 1), dtype=torch.int32, device="cuda")
    s_cs = torch.empty(2 * S, dtype=torch.int32, device="cuda")
    ws_c = torch.empty(int(lib.rl_chunklet_partition_workspace_bytes(NS, S)), dtype=torch.uint8, device="cuda")
    launches = {
        "similarity_kernel_ms": lambda: lib.rl_chunk_similarities(
            X.data_ptr(), 1, X.stride(0), int(X.shape[1]), d_off.data_ptr(), D, N, d_non.data_ptr(), d_head.data_ptr(),
            costs.data_ptr(), cs.data_ptr(), ws_s.data_ptr(), ws_s.numel(), st),
        "chunk_partition_kernel_ms": lambda: lib.rl_chunk_partition(
            costs.data_ptr(), d_len.data_ptr(), d_off.data_ptr(), d_max.data_ptr(), D, N, cuts.data_ptr(),
            cs.data_ptr(), cs[D:].data_ptr(), ws_p.data_ptr(), ws_p.numel(), st),
        "chunklet_partition_kernel_ms": lambda: lib.rl_chunklet_partition(
            p.data_ptr(), q.data_ptr(), s_len.data_ptr(), d_soff.data_ptr(), s_max.data_ptr(), S, NS, s_cuts.data_ptr(),
            s_cs.data_ptr(), s_cs[S:].data_ptr(), ws_c.data_ptr(), ws_c.numel(), st),
    }
    out = {}
    for name, launch in launches.items():
        assert launch() == 0
        times = []
        for _ in range(reps):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record()
            assert launch() == 0
            ev[1].record()
            torch.cuda.synchronize()
            times.append(ev[0].elapsed_time(ev[1]))
        out[name] = round(float(np.median(times)), 2)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=2000)
    ap.add_argument("--chars", type=int, default=20000)
    ap.add_argument("--max-size", type=int, default=2048)
    ap.add_argument("--host-docs", type=int, default=4)
    ap.add_argument("--e2e-docs", type=int, default=100)
    ap.add_argument("--repeat", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_split_chunks needs a CUDA device")
    import chunks_oracle as co
    from bench_split_sentences import card, corpus, sat_model

    import raglite_b200 as rl
    from raglite_b200 import _chunks as K

    docs = corpus(a.docs, a.chars)
    n_chars = sum(map(len, docs))
    sents = [sentences_of(d) for d in docs]
    res: dict = {"metric": "split_chunks_chars_per_s", "docs": a.docs, "chars": n_chars, "max_size": a.max_size,
                 **card()}
    rl.split_chunklets_batch(sents[:8], max_size=a.max_size)                       # warm-up
    for _ in range(a.repeat):
        chunklets, t = timed(lambda: rl.split_chunklets_batch(sents, max_size=a.max_size))
        res.setdefault("chunklets_s", []).append(round(t, 3))
    t_host = time.perf_counter()
    for s in sents:
        K.markdown_chunklet_boundaries(s)
        K.num_statements(s)
    res["chunklets_host_s"] = round(time.perf_counter() - t_host, 3)
    res["chunklets_chars_per_s"] = round(n_chars / min(res["chunklets_s"]))
    rng = np.random.default_rng(0)
    embs = [rng.standard_normal((len(c), 1024)).astype(np.float16) for c in chunklets]
    rl.split_chunks_batch(chunklets[:8], embs[:8], max_size=a.max_size)
    for _ in range(a.repeat):
        _, t = timed(lambda: rl.split_chunks_batch(chunklets, embs, max_size=a.max_size))
        res.setdefault("chunks_s", []).append(round(t, 3))
    res["chunks_chars_per_s"] = round(n_chars / min(res["chunks_s"]))
    res["chunklets_per_doc"] = round(float(np.mean([len(c) for c in chunklets])), 1)
    # device share: each kernel on the whole batch, inputs already on the device, CUDA events around the launches alone
    res.update(kernel_times(chunklets, embs, sents, a.max_size))
    # the reference's algorithms restated on the host, over a few documents
    t = time.perf_counter()
    for s in sents[:a.host_docs]:
        co.chunklet_cuts(K.markdown_chunklet_boundaries(s), K.num_statements(s), [len(x) for x in s], a.max_size, "pow")
    res["host_chunklet_dp_s_per_doc"] = round((time.perf_counter() - t) / a.host_docs, 4)
    t = time.perf_counter()
    for i in range(a.host_docs):
        c = chunklets[i]
        co.linprog_cuts(co.chunk_costs_f32(c, embs[i]), [len(x) for x in c], a.max_size)
    res["host_linprog_s_per_doc"] = round((time.perf_counter() - t) / a.host_docs,4)
    # split_documents end to end with seeded models
    from oracle import embed as oe

    tok = oe.unigram_tokenizer()
    rl.register_sentence_splitter(rl.SaTEngine.from_hf(sat_model(), tok))
    cfg = rl.RAGLiteConfig(reranker=None)
    model = oe.seeded_model(oe.bge_m3_config(num_hidden_layers=2, vocab_size=250002, max_position_embeddings=8194), seed=5)
    rl.register_token_embedder(cfg.embedder, rl.TokenEmbedderEngine.from_hf(model, tokenizer=tok, n_ctx=512))
    sub = docs[:a.e2e_docs]
    rl.split_documents(sub[:2], config=cfg)
    _, t = timed(lambda: rl.split_documents(sub, config=cfg))
    res["split_documents_s"] = round(t, 3)
    res["split_documents_chars_per_s"] = round(sum(map(len, sub)) / t)
    res["e2e_docs"] = len(sub)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
