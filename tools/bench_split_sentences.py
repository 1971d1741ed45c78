"""Benchmark ``split_sentences_batch`` on the GPU: a SaT model of sat-1l's shape on a seeded corpus.

    python tools/bench_split_sentences.py [--docs 2000] [--chars 20000] [--host-docs 4]

Inputs: seeded weights at sat-1l's shape (XLM-RoBERTa, 1 layer, H 768, 12 x 64, FFN 3072, vocabulary 250,002, 514
positions, one label), the seeded Unigram tokenizer of ``oracle/embed.py`` and a seeded corpus.  Prints one JSON line:

* characters/s end to end (``split_sentences_batch`` with ingest's ``max_len=2048``, best of ``--repeat``);
* host tokenization and planning (``SaTEngine._plan`` over the corpus);
* from one ``torch.profiler`` pass: the forward (the encoder's kernels, with TFLOP/s over block tokens), the head and
  stitch kernels, the partition kernel, and the device-to-host copies; the partition kernel alone on the longest
  document (CUDA events);
* the same model in torch float32 on the host threads plus the reference's post-processing restated in Python, over
  ``--host-docs`` documents (not onnxruntime);
* the card's name and power limit, read in the same run.
"""

from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / "tests")]

WORDS = ("alpha", "beta", "gamma", "delta", "light", "clock", "rod", "frame", "event", "time", "of", "the",
         "observer", "velocity", "what", "is", "how", "does", "a", "an", "in", "to")


def corpus(n_docs: int, n_chars: int, seed: int = 0) -> list[str]:
    rng = np.random.default_rng(seed)
    vocab = np.array([*WORDS, *[w.capitalize() + "." for w in WORDS], "é", "\n\n# Heading\n"])
    p = np.r_[np.full(len(WORDS), 0.8 / len(WORDS)), np.full(len(WORDS), 0.19 / len(WORDS)), 0.005, 0.005]
    docs = []
    for _ in range(n_docs):
        words = rng.choice(vocab, size=n_chars // 5, p=p)
        docs.append(" ".join(words.tolist())[:n_chars])
    return docs


def sat_model(seed: int = 0):
    from transformers import XLMRobertaConfig, XLMRobertaForTokenClassification

    cfg = XLMRobertaConfig(vocab_size=250002, hidden_size=768, num_hidden_layers=1, num_attention_heads=12,
                           intermediate_size=3072, max_position_embeddings=514, type_vocab_size=1, layer_norm_eps=1e-5,
                           hidden_act="gelu", pad_token_id=1, bos_token_id=0, eos_token_id=2, num_labels=1,
                           hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    cfg._attn_implementation = "sdpa"   # noqa: SLF001
    torch.manual_seed(seed)
    return XLMRobertaForTokenClassification(cfg).eval()


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=False).stdout.strip().splitlines()
    return {"gpu": q[0] if q else torch.cuda.get_device_name(), "torch_device": torch.cuda.get_device_name()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=2000)
    ap.add_argument("--chars", type=int, default=20000)
    ap.add_argument("--repeat", type=int, default=2)
    ap.add_argument("--host-docs", type=int, default=4)
    ap.add_argument("--max-len", type=int, default=2048)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_split_sentences needs a CUDA device")
    import sentences_oracle as so

    import raglite_b200 as rl
    from oracle.embed import unigram_tokenizer
    from raglite_b200 import _sentences as S

    docs = corpus(a.docs, a.chars)
    n_chars = sum(map(len, docs))
    tok = unigram_tokenizer()
    model = sat_model()
    eng = S.SaTEngine.from_hf(model, tok)
    rl.register_sentence_splitter(eng)
    res: dict = {"metric": "split_sentences_chars_per_s", "docs": a.docs, "chars": n_chars, "max_len": a.max_len, **card()}

    rl.split_sentences_batch(docs[:8], max_len=a.max_len)                # warm every kernel
    best = float("inf")
    for _ in range(a.repeat):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = rl.split_sentences_batch(docs, max_len=a.max_len)
        best = min(best, time.perf_counter() - t0)
    res["e2e_s"] = best
    res["chars_per_s"] = n_chars / best
    res["sentences"] = sum(map(len, out))

    t0 = time.perf_counter()
    block_tokens = 0
    for lo, hi in eng._groups(docs):  # noqa: SLF001
        p = eng._plan(docs[lo:hi])    # noqa: SLF001
        block_tokens += int(p["row_off"][-1])
    res["host_plan_s"] = time.perf_counter() - t0
    res["block_tokens"] = block_tokens

    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        rl.split_sentences_batch(docs, max_len=a.max_len)
        torch.cuda.synchronize()
    cats = {"forward": 0.0, "head_stitch": 0.0, "partition": 0.0, "download": 0.0, "upload": 0.0, "other": 0.0}
    for ev in prof.key_averages():
        us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        n = ev.key
        if "sentence_partition" in n:
            cats["partition"] += us
        elif "sat_" in n:
            cats["head_stitch"] += us
        elif "DtoH" in n:
            cats["download"] += us
        elif "HtoD" in n:
            cats["upload"] += us
        elif "xenc" in n or "wgmma" in n or "ln" in n.lower() or "attn" in n or "linear" in n:
            cats["forward"] += us
        else:
            cats["other"] += us
    res["device_s"] = {k: v / 1e6 for k, v in cats.items()}
    H, F = 768, 3072
    flop_per_tok = 2 * (4 * H * H + 2 * H * F)       # QKV, output, up and down projections; attention over 256 adds ~3 %
    res["forward_tflops"] = block_tokens * flop_per_tok / max(cats["forward"] / 1e6, 1e-9) / 1e12 if cats["forward"] else None

    longest = max(docs, key=len)
    d_p = torch.rand(len(longest), dtype=torch.float32, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    lib = eng.lib
    off = torch.zeros(1, dtype=torch.int64, device="cuda")
    lens = torch.tensor([len(longest), 4, a.max_len], dtype=torch.int32, device="cuda")   # n, min_len, max_len
    cuts = torch.empty(len(longest), dtype=torch.int32, device="cuda")
    cs = torch.empty(2, dtype=torch.int32, device="cuda")
    ws = torch.empty(int(lib.rl_sentence_partition_workspace_bytes(len(longest))), dtype=torch.uint8, device="cuda")
    args = (d_p.data_ptr(), off.data_ptr(), lens.data_ptr(), lens[1:].data_ptr(), lens[2:].data_ptr(), 1, len(longest),
            cuts.data_ptr(), cs.data_ptr(), cs[1:].data_ptr(), ws.data_ptr(), ws.numel(),
            C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert lib.rl_sentence_partition(*args) == 0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        lib.rl_sentence_partition(*args)
    e1.record()
    torch.cuda.synchronize()
    assert int(cs[1]) == 0 and int(cs[0]) > 0
    res["partition_longest_doc"] = {"chars": len(longest), "ms": e0.elapsed_time(e1) / 5}

    # host comparison: the same model in torch float32 on the CPU threads + the restated post-processing
    sub = docs[: a.host_docs]
    cpu_model = model.float().eval()
    t0 = time.perf_counter()
    with torch.no_grad():
        for lo, hi in eng._groups(sub):  # noqa: SLF001
            p = eng._plan(sub[lo:hi])    # noqa: SLF001
            seqs = np.split(p["rows"], p["row_off"][1:-1])
            for i in range(0, len(seqs), 64):
                batch = [s for s in seqs[i:i + 64]]
                L = max(map(len, batch))
                x = torch.ones((len(batch), L), dtype=torch.int64)
                m = torch.zeros((len(batch), L), dtype=torch.int64)
                for r, s in enumerate(batch):
                    x[r, :len(s)] = torch.from_numpy(s.astype(np.int64))
                    m[r, :len(s)] = 1
                cpu_model(input_ids=x, attention_mask=m)
    t_model = time.perf_counter() - t0
    pred = rl.sentence_boundary_probas(sub)
    t0 = time.perf_counter()
    for d, pr in zip(sub, pred, strict=True):
        so.split_sentences_post(d, pr, max_len=a.max_len)
    t_post = time.perf_counter() - t0
    sub_chars = sum(map(len, sub))
    res["host_baseline"] = {"label": "torch fp32 on the host threads + Python post-processing (not onnxruntime)",
                            "docs": len(sub), "chars": sub_chars, "threads": torch.get_num_threads(),
                            "model_s": t_model, "post_s": t_post, "chars_per_s": sub_chars / (t_model + t_post)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
