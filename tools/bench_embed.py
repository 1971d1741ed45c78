"""Token-embedder throughput on one GPU: bge-m3's architecture (XLM-RoBERTa, 24 layers, H = 1024, 16 heads x 64,
FFN 4096, 250,002-token vocabulary) with seeded weights, on two workloads:

- ingest: 2048 segments x 498 tokens (the pool workload's shape plus <s> / </s>);
- queries: 256 single-sentence queries of about 20 tokens.

Reports tokens/s and achieved TFLOP/s from algorithmic FLOPs, layers * (2T(4H^2 + 2HF) + 4H sum L^2), against the data
sheet's 989 TFLOP/s dense FP16; the kernel-time split between linear, attention and LayerNorm from a separate
torch.profiler run; end-to-end ``embed_strings`` on a document (pooling included); a bounded CPU float32 transformers
sample; and the card's name and power limit, read in the same process.  Prints one JSON line."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--segments", type=int, default=2048)
ap.add_argument("--segment-len", type=int, default=498)
ap.add_argument("--queries", type=int, default=256)
ap.add_argument("--query-len", type=int, default=20)
ap.add_argument("--repeats", type=int, default=3)
ap.add_argument("--doc-sentences", type=int, default=2000)
ap.add_argument("--cpu-segments", type=int, default=2, help="segments of the ingest shape run by the CPU float32 arm")
ap.add_argument("--profile-dir", default="", help="write the torch.profiler summary here (default: no trace file)")
args = ap.parse_args()

from fake_llama import make_sentences  # noqa: E402

from oracle import embed as oe  # noqa: E402
from raglite_b200 import RAGLiteConfig, TokenEmbedderEngine, embed_strings, register_token_embedder  # noqa: E402

PEAK_TFLOPS = 989.0


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=False).stdout.strip().splitlines()
    return {"card": q[0] if q else torch.cuda.get_device_name(0)}


cfg = oe.bge_m3_config()
model = oe.seeded_model(cfg, seed=0)
eng = TokenEmbedderEngine.from_hf(model, oe.unigram_tokenizer())
H, F, LYR = cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers
rng = np.random.default_rng(0)


def ids_of(n, L):
    return [np.r_[0, rng.integers(5, cfg.vocab_size, size=L - 2), 2].astype(np.int32) for _ in range(n)]


def flops(lens):
    lens = np.asarray(lens, dtype=np.float64)
    T = lens.sum()
    return LYR * (2.0 * T * (4 * H * H + 2 * H * F) + 4.0 * H * float((lens**2).sum()))


def timed(ids):
    eng.embed_token_ids(ids[: max(1, len(ids) // 8)])                # warm-up (every kernel of the shape)
    torch.cuda.synchronize()
    best = []
    for _ in range(args.repeats):
        t0 = time.perf_counter()
        eng.embed_token_ids(ids)
        torch.cuda.synchronize()
        best.append(time.perf_counter() - t0)
    return best


out = {"metric": "bge-m3-shaped token embedder (24 layers, H 1024, seeded weights), fp16 tensor cores", **card(),
       "tokens_per_call": eng.max_tokens_per_call}
ingest = ids_of(args.segments, args.segment_len)
queries = [np.r_[0, rng.integers(5, cfg.vocab_size, size=int(n)), 2].astype(np.int32)
           for n in rng.integers(args.query_len - 6, args.query_len + 4, size=args.queries)]
for name, ids in (("ingest", ingest), ("queries", queries)):
    ts = timed(ids)
    lens = [len(x) for x in ids]
    t = float(np.median(ts))
    out[name] = {"sequences": len(ids), "tokens": int(sum(lens)), "seconds_median": t, "seconds_all": ts,
                 "tokens_per_s": sum(lens) / t, "tflops": flops(lens) / t / 1e12,
                 "share_of_989": flops(lens) / t / 1e12 / PEAK_TFLOPS}

# kernel-time split (a run of its own: tracing slows the host)
from torch.profiler import ProfilerActivity, profile  # noqa: E402

sample = ingest[:256]
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    eng.embed_token_ids(sample)
    torch.cuda.synchronize()
split = {"linear": 0.0, "attention": 0.0, "layernorm": 0.0, "other": 0.0}
for ev in prof.key_averages():
    us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
    if us <= 0:
        continue
    key = ev.key
    cls = ("linear" if "linear_wgmma" in key else "attention" if "attention" in key or "seq_order" in key
           else "layernorm" if "_ln_kernel" in key else "other")
    split[cls] += us
total = sum(split.values())
out["profile_sample_segments"] = len(sample)
out["kernel_time_share"] = {k: v / total for k, v in split.items()} if total else "not measured"
if args.profile_dir:
    Path(args.profile_dir).mkdir(parents=True, exist_ok=True)
    (Path(args.profile_dir) / "bench_embed_profile.txt").write_text(prof.key_averages().table(sort_by="cuda_time_total", row_limit=30))

# end to end: late-chunking embed_strings of one document at n_ctx = 512, pooling included
conf = RAGLiteConfig(reranker=None)
register_token_embedder(conf.embedder, eng)
doc = make_sentences(args.doc_sentences, seed=1)
embed_strings(doc[:200], config=conf)
torch.cuda.synchronize()
t0 = time.perf_counter()
E = embed_strings(doc, config=conf)
dt = time.perf_counter() - t0
out["embed_strings_document"] = {"sentences": len(doc), "characters": sum(map(len, doc)), "seconds": dt,
                                 "sentences_per_s": len(doc) / dt, "shape": list(E.shape)}

# CPU float32 transformers arm on a bounded sample of the ingest shape
n = args.cpu_segments
torch.set_num_threads(max(1, torch.get_num_threads()))
with torch.no_grad():
    t0 = time.perf_counter()
    for x in ingest[:n]:
        model(input_ids=torch.from_numpy(x.astype(np.int64))[None])
    cpu_dt = time.perf_counter() - t0
out["cpu_fp32_transformers"] = {"segments": n, "tokens": n * args.segment_len, "threads": torch.get_num_threads(),
                                "tokens_per_s": n * args.segment_len / cpu_dt, "seconds": cpu_dt}
out.update(card())
print(json.dumps(out))
