"""GGUF token-embedder throughput on one GPU: bge-m3's architecture (XLM-RoBERTa, 24 layers, H = 1024, 16 heads x 64,
FFN 4096, 250,002-token vocabulary) with seeded weights written as F16, Q8_0 and Q4_K_M-style (Q4_K with Q6_K attn_v /
ffn_down in every other layer, Q6_K embeddings) GGUF files, each loaded with ``TokenEmbedderEngine.from_gguf``, beside the
same F16 weights loaded with ``from_hf``.

Per arm: ingest tokens/s (2048 segments x 498 tokens), the latency of one query and of 256 queries (about 20 tokens
each), resident weight bytes and the file's tensor bytes; the card's name and power limit, read in the same process.
The arms alternate over the repeats and the best repeat is reported.  Prints one JSON line."""
import argparse
import json
import subprocess
import sys
import tempfile
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
ap.add_argument("--layers", type=int, default=24)
args = ap.parse_args()

from gguf_fixtures import write_xlmr_gguf  # noqa: E402

from oracle import embed as oe  # noqa: E402
from raglite_b200 import TokenEmbedderEngine  # noqa: E402
from raglite_b200._gguf import GGUFFile  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=False).stdout.strip()
    return {"card": q or torch.cuda.get_device_name(0)}


cfg = oe.bge_m3_config(num_hidden_layers=args.layers, max_position_embeddings=514)
model = oe.seeded_model(cfg, seed=0, perturb=False)
rng = np.random.default_rng(0)
engines, files = {}, {}
for mode in ("F16", "Q8_0", "Q4_K_M"):   # one file of up to 1.1 GB at a time, removed once its engine holds the weights
    with tempfile.TemporaryDirectory(prefix="bench_gguf_") as tmp:
        path = Path(tmp) / f"bge-m3-{mode}.gguf"
        write_xlmr_gguf(path, model, oe.unigram_tokenizer(), mode=mode, rng=np.random.default_rng(1), dequantize=False)
        files[mode] = GGUFFile(path).tensor_bytes()
        engines[mode] = TokenEmbedderEngine.from_gguf(path)
engines["hf_f16"] = TokenEmbedderEngine.from_hf(model, oe.unigram_tokenizer())
del model


def ids_of(n: int, L: int) -> list[np.ndarray]:
    return [np.r_[0, rng.integers(5, cfg.vocab_size, size=L - 2), 2].astype(np.int32) for _ in range(n)]


ingest = ids_of(args.segments, args.segment_len)
queries = ids_of(args.queries, args.query_len)


def timed(eng: TokenEmbedderEngine, ids: list[np.ndarray], reps: int = 1) -> float:
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        eng.embed_token_ids(ids)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


for eng in engines.values():   # warm every shape
    timed(eng, ingest[:64]), timed(eng, queries), timed(eng, queries[:1])
res = {k: {"ingest_s": [], "q1_ms": [], "q256_ms": []} for k in engines}
for _ in range(args.repeats):
    for k, eng in engines.items():
        res[k]["ingest_s"].append(timed(eng, ingest))
        res[k]["q1_ms"].append(1e3 * timed(eng, queries[:1], 50))
        res[k]["q256_ms"].append(1e3 * timed(eng, queries, 10))
T = args.segments * args.segment_len
out = {"workload": f"{args.segments}x{args.segment_len} ingest, 1 / {args.queries} queries of {args.query_len} tokens",
       "layers": args.layers, **card()}
for k, r in res.items():
    out[k] = {"ingest_tokens_per_s": round(T / min(r["ingest_s"])), "query1_ms": round(min(r["q1_ms"]), 3),
              "query256_ms": round(min(r["q256_ms"]), 3), "resident_weight_bytes": engines[k].weight_bytes(),
              "file_tensor_bytes": files.get(k)}
out["q4_k_m_over_f16_ingest"] = round(out["Q4_K_M"]["ingest_tokens_per_s"] / out["F16"]["ingest_tokens_per_s"], 3)
print(json.dumps(out))
