"""Measure the Qwen3 decoder on one GPU with seeded Q4_K_M-style weights at Qwen3-8B's shape (36 layers, hidden 4096,
32 / 8 heads, FFN 12288, vocabulary 151 936, separate Q6_K output) or 4B's (36 layers, hidden 2560, 32 / 8 heads, FFN
9728, tied).  The weights are built in memory, so no GGUF file is needed.

Reports prefill tokens/s at 512 / 2048 / 8192-token prompts, decode ms/token (forward + sampling) at context 1k / 4k /
8k, each decode GEMV's achieved GB/s over its image bytes against the H100 SXM data sheet's 3.35 TB/s, and the card's
name and power limit read in the same process; prints one JSON line.

    python tools/bench_llm.py [--model 8b|4b|both] [--steps 32]
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

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

from raglite_b200._gguf import F32, Q4_K, Q6_K, GGUFTensor, Qwen3Plan  # noqa: E402
from raglite_b200._llm import LlmEngine  # noqa: E402

SHAPES = {"8b": dict(n_layers=36, hidden=4096, n_head=32, n_kv=8, ffn=12288, vocab=151936, tied=False),
          "4b": dict(n_layers=36, hidden=2560, n_head=32, n_kv=8, ffn=9728, vocab=151936, tied=True)}
HBM_BPS = 3.35e12


def _blocks(ty: int, N: int, K: int, rng: np.random.Generator) -> np.ndarray:
    bb = 144 if ty == Q4_K else 210
    b = rng.integers(0, 256, (N * K // 256, bb), dtype=np.uint8)
    scale = rng.uniform(2e-5, 1e-4, (len(b), 2)).astype(np.float16).view(np.uint8)
    if ty == Q4_K:
        b[:, 0:4] = scale
    else:
        b[:, 208:210] = scale[:, :2]
    return b.reshape(-1)


def make_plan(shape: dict, seed: int = 0) -> Qwen3Plan:
    rng = np.random.default_rng(seed)
    H, F, V, nq, nkv = shape["hidden"], shape["ffn"], shape["vocab"], shape["n_head"] * 128, shape["n_kv"] * 128
    ts: dict[str, GGUFTensor] = {}

    def q(name: str, ty: int, N: int, K: int) -> None:
        ts[name] = GGUFTensor(name, ty, (N, K), _blocks(ty, N, K, rng))

    def norm(name: str, n: int) -> None:
        ts[name] = GGUFTensor(name, F32, (n,), (1 + 0.1 * rng.standard_normal(n)).astype("<f4").view(np.uint8))

    q("token_embd.weight", Q4_K, V, H)
    if shape["tied"]:
        ts["output.weight"] = ts["token_embd.weight"]
    else:
        q("output.weight", Q6_K, V, H)
    norm("output_norm.weight", H)
    for i in range(shape["n_layers"]):
        b = f"blk.{i}."
        q6 = Q6_K if i % 2 == 0 else Q4_K   # Q4_K_M: attn_v and ffn_down of half the layers in Q6_K
        for n, ty, N, K in (("attn_q", Q4_K, nq, H), ("attn_k", Q4_K, nkv, H), ("attn_v", q6, nkv, H),
                            ("attn_output", Q4_K, H, nq), ("ffn_gate", Q4_K, F, H), ("ffn_up", Q4_K, F, H),
                            ("ffn_down", q6, H, F)):
            q(b + n + ".weight", ty, N, K)
        for n, d in (("attn_norm", H), ("attn_q_norm", 128), ("attn_k_norm", 128), ("ffn_norm", H)):
            norm(b + n + ".weight", d)
    return Qwen3Plan(shape["n_layers"], H, shape["n_head"], shape["n_kv"], F, V, 40960, 1e6, 1e-6, ts, shape["tied"])


def _time(fn, reps: int) -> float:
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps / 1e3


def bench(name: str, steps: int) -> dict:
    t0 = time.time()
    eng = LlmEngine(make_plan(SHAPES[name]), None, n_ctx=8192 + steps + 1, prefill_chunk=512)
    out: dict = {"model": name, "weight_bytes": eng.weight_bytes(), "kv_cache_bytes": eng.kv_cache_bytes,
                 "load_s": round(time.time() - t0, 1)}
    rng = np.random.default_rng(1)
    V = eng.plan.vocab
    prefill = {}
    for n in (512, 2048, 8192):
        ids = rng.integers(0, V, n).tolist()
        eng.reset()
        eng.prefill(ids[:512])   # warm-up of every prefill shape
        torch.cuda.synchronize()
        eng.reset()
        t = time.perf_counter()
        eng.prefill(ids)
        torch.cuda.synchronize()
        prefill[str(n)] = round(n / (time.perf_counter() - t), 1)
    out["prefill_tok_s"] = prefill
    decode = {}
    for ctx in (1024, 4096, 8192):
        eng.reset()
        eng.prefill(rng.integers(0, V, ctx).tolist())
        hist = rng.integers(0, V, 64).tolist()

        def step() -> None:
            eng._forward_dev(eng._tok.data_ptr(), 1)
            eng.sample(hist, temperature=0.6, top_k=20, top_p=0.95, min_p=0.0, repeat_penalty=1.1, u=0.5)

        eng._tok.fill_(1)
        step()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(steps):
            step()
        e.record()
        torch.cuda.synchronize()
        decode[str(ctx)] = round(s.elapsed_time(e) / steps, 3)
    out["decode_ms_per_token"] = decode
    # each decode GEMV of layer 0 and the LM head alone: bytes of its images over kernel time
    lib, L = eng.lib, eng._layers[0]
    x = torch.randn(max(eng.plan.hidden, eng.plan.ffn, eng.plan.n_head * 128), device="cuda").half()
    gb = {}
    for label, lin in (("attn_q", L.q), ("attn_k", L.k), ("attn_v", L.v), ("attn_output", L.o), ("ffn_gate", L.gate),
                       ("ffn_down", L.down), ("output", eng.weights.output)):
        ws = torch.empty(max(1, int(lib.rl_llm_qgemv_workspace_bytes(lin.N, lin.K))), dtype=torch.uint8, device="cuda")
        y = torch.empty(lin.N, dtype=torch.float32, device="cuda")
        stream = int(torch.cuda.current_stream().cuda_stream)
        parts = {lin.parts[i] for i in range(lin.n_parts)}
        nbytes = sum(t.numel() for t in eng._keep if t.data_ptr() in parts)   # the part images
        sec = _time(lambda lin=lin, ws=ws, y=y: lib.rl_llm_qgemv(C.byref(lin), x.data_ptr(), y.data_ptr(), 1, ws.data_ptr(),
                                                                 ws.numel(), stream), 50)
        gb[label] = {"N": lin.N, "K": lin.K, "us": round(sec * 1e6, 1), "GB_s": round(nbytes / sec / 1e9, 1),
                     "of_3.35TB_s": round(nbytes / sec / HBM_BPS, 3)}
    out["gemv"] = gb
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="both", choices=["8b", "4b", "both"])
    ap.add_argument("--steps", type=int, default=32)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_llm needs a CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=False).stdout.strip().splitlines()
    res = {"device": torch.cuda.get_device_name(0), "nvidia_smi": smi[0] if smi else None,
           "models": [bench(m, a.steps) for m in (["8b", "4b"] if a.model == "both" else [a.model])]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
