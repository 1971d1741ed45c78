"""Cross-encoder throughput (BASELINE configs[4]: 1024 queries x 100 candidates, MiniLM-L12) on one GPU,
next to the float32 transformers forward on the host cores for a bounded sample.

``--model`` picks the shape, with seeded weights at the full vocabulary: ``minilm`` (ms-marco-MiniLM-L-12-v2's shape,
the default), ``multibert`` (multilingual BERT-base, two labels) or ``xlmr-large`` (XLM-R large, one label).  Besides
throughput the line holds the latency of one ``rerank_chunks``-sized call: 32 pairs of 256-512 tokens."""
import argparse, json, subprocess, sys, time
from pathlib import Path
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
import numpy as np, torch

DENSE_FP16_TFLOPS = 989.0   # H100 SXM data sheet, dense FP16
METRICS = {"minilm": "MiniLM-L12-H384", "multibert": "BERT-base-H768 2 labels", "xlmr-large": "XLM-R-large-H1024"}
CPU_PAIRS = {"minilm": 64, "multibert": 16, "xlmr-large": 8}

ap = argparse.ArgumentParser()
ap.add_argument("--model", choices=sorted(METRICS), default="minilm")
ap.add_argument("--pairs", type=int, default=8192)
ap.add_argument("--mean-len", type=int, default=200)
ap.add_argument("--cpu-pairs", type=int, default=None)
ap.add_argument("--tokens-per-call", type=int, default=None)
ap.add_argument("--latency-reps", type=int, default=50)
args = ap.parse_args()

import xenc_classifiers as xc
from raglite_b200._xenc import CrossEncoderEngine

if args.model == "minilm":
    from oracle import rerank as orr

    model = orr.seeded_model(seed=0)
else:
    model = xc.seeded_classifier(args.model, seed=0, perturb=False)
c = model.config
kw = {} if args.tokens_per_call is None else {"max_tokens_per_call": args.tokens_per_call}
eng = CrossEncoderEngine.from_hf(model, **kw)
rng = np.random.default_rng(0)
lens = np.clip(rng.normal(args.mean_len, 60, size=args.pairs).astype(int), 32, 512)
hi_id = 30000 if args.model == "minilm" else c.vocab_size
ids = [rng.integers(1000, hi_id, size=L).astype(np.int32) for L in lens]
if c.type_vocab_size > 1:
    types = [np.r_[np.zeros(12, np.int32), np.ones(L - 12, np.int32)] for L in lens]
else:
    types = [np.zeros(L, np.int32) for L in lens]
eng.score_tokens(ids[:256], types[:256])
torch.cuda.synchronize()
t0 = time.perf_counter()
logits, scores = eng.score_tokens(ids, types)
torch.cuda.synchronize()
dt = time.perf_counter() - t0
T = int(lens.sum())
H, F, Lyr = c.hidden_size, c.intermediate_size, c.num_hidden_layers


def flops(ls: np.ndarray) -> float:
    return Lyr * (2.0 * float(ls.sum()) * (3 * H * H + H * H + 2 * H * F) + 4.0 * float((ls.astype(np.float64) ** 2).sum()) * H)


# one rerank_chunks-sized call: 32 pairs of 256-512 tokens, host ids in -> host scores out
lat_lens = rng.integers(256, 513, size=32)
lat_ids = [rng.integers(1000, hi_id, size=int(L)).astype(np.int32) for L in lat_lens]
lat_types = [np.zeros(int(L), np.int32) for L in lat_lens]
eng.score_tokens(lat_ids, lat_types)
lat = []
for _ in range(args.latency_reps):
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    eng.score_tokens(lat_ids, lat_types)
    torch.cuda.synchronize()
    lat.append(time.perf_counter() - t1)
n = args.cpu_pairs if args.cpu_pairs is not None else CPU_PAIRS[args.model]
t0 = time.perf_counter()
ref = xc.classifier_logits(model, ids[:n], types[:n])
cpu_dt = time.perf_counter() - t0
got = logits[:n].reshape(n, -1)
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True, timeout=30, check=False).stdout.strip().splitlines()[0]
except Exception:  # noqa: BLE001
    card = torch.cuda.get_device_name()
print(json.dumps({
    "metric": f"cross-encoder pairs/sec ({METRICS[args.model]}, packed varlen, fp16 tensor cores)", "model": args.model,
    "card": card, "pairs": args.pairs,
    "tokens": T, "mean_len": float(lens.mean()), "gpu_pairs_per_s": args.pairs / dt, "gpu_tokens_per_s": T / dt,
    "gpu_tflops": flops(lens) / dt / 1e12, "share_of_dense_fp16": flops(lens) / dt / 1e12 / DENSE_FP16_TFLOPS,
    "seconds": dt, "c5_seconds_extrapolated": 102400 / (args.pairs / dt),
    "latency_32x256_512_ms_median": 1e3 * float(np.median(lat)), "latency_32x256_512_ms_min": 1e3 * float(np.min(lat)),
    "latency_tokens": int(lat_lens.sum()),
    "cpu_pairs_per_s": n / cpu_dt, "cpu_threads": torch.get_num_threads(), "cpu_sample_pairs": n,
    "max_abs_logit_err_vs_fp32": float(np.abs(got - ref).max()),
}))
