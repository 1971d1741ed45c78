"""Where a GGUF embedder's forward spends its time on one GPU: kernel time of each linear of bge-m3's layer (Q | K | V
3072 x 1024, output 1024 x 1024, up 4096 x 1024, down 1024 x 4096) for the fp16 image and the Q8_0 / Q4_K / Q6_K images,
at one query's tokens (T = 20) and at an ingest call's (T = 65536), from CUDA events over repeated launches; then the
kernel-time split of whole forwards (F16 and Q4_K_M-style files, 24 layers) from torch.profiler, by kernel.  Reports
achieved weight-stream bandwidth at the small T and TFLOP/s at the large T, the card's name and power limit.  Prints one
JSON line."""
import json
import subprocess
import sys
import tempfile
from collections import defaultdict
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from gguf_fixtures import Q4_K, Q6_K, Q8_0, random_blocks, write_xlmr_gguf  # noqa: E402

from oracle import embed as oe  # noqa: E402
from raglite_b200 import TokenEmbedderEngine, _lib  # noqa: E402

lib = _lib.load()
s = torch.cuda.current_stream().cuda_stream
rng = np.random.default_rng(0)
SHAPES = {"qkv": (3072, 1024), "out": (1024, 1024), "up": (4096, 1024), "down": (1024, 4096)}


def time_ms(fn, reps: int) -> float:
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


linears = {}
for name, (N, K) in SHAPES.items():
    bias = torch.zeros(N, device="cuda")
    W = torch.randn(N, K, device="cuda") * 0.02
    imgs = {"fp16": torch.empty(int(lib.rl_xenc_linear_image_bytes(N, K)), dtype=torch.uint8, device="cuda")}
    lib.rl_xenc_pack_linear(W.data_ptr(), N, K, imgs["fp16"].data_ptr(), s)
    wbytes = {"fp16": N * K * 2}
    for ty, tn in ((Q8_0, "Q8_0"), (Q4_K, "Q4_K"), (Q6_K, "Q6_K")):
        raw = torch.from_numpy(random_blocks(ty, N, K, rng)).cuda()
        imgs[tn] = torch.empty(int(lib.rl_xenc_qlinear_image_bytes(ty, N, K)), dtype=torch.uint8, device="cuda")
        lib.rl_xenc_pack_qlinear(ty, raw.data_ptr(), N, K, imgs[tn].data_ptr(), s)
        wbytes[tn] = imgs[tn].numel()
    for T, reps in ((20, 200), (65536, 5)):
        X = torch.randn(T, K, device="cuda").half()
        Y = torch.empty(T, N, device="cuda", dtype=torch.float16)
        for tn, img in imgs.items():
            fn = lib.rl_xenc_linear if tn == "fp16" else lib.rl_xenc_linear_q
            ms = time_ms(lambda fn=fn, img=img: fn(X.data_ptr(), img.data_ptr(), bias.data_ptr(), Y.data_ptr(), T, N, K, 0, s),
                         reps)
            r = {"us": round(1e3 * ms, 1)}
            if T == 20:
                r["weight_GB_per_s"] = round(wbytes[tn] / ms / 1e6, 1)
            else:
                r["TFLOP_per_s"] = round(2 * T * N * K / ms / 1e9, 1)
            linears[f"{name} T={T} {tn}"] = r

cfg = oe.bge_m3_config(max_position_embeddings=514)
model = oe.seeded_model(cfg, seed=0, perturb=False)
split = {}
for mode in ("F16", "Q4_K_M"):
    with tempfile.TemporaryDirectory(prefix="profile_gguf_") as tmp:
        path = Path(tmp) / f"m-{mode}.gguf"
        write_xlmr_gguf(path, model, oe.unigram_tokenizer(), mode=mode, rng=np.random.default_rng(1), dequantize=False)
        eng = TokenEmbedderEngine.from_gguf(path)
    for label, ids in (("1 query", [np.arange(4, 24, dtype=np.int32)]),
                       ("ingest 256 x 498", [rng.integers(5, 250000, 498).astype(np.int32) for _ in range(256)])):
        eng.embed_token_ids(ids)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            eng.embed_token_ids(ids)
            torch.cuda.synchronize()
        per = defaultdict(float)
        for e in prof.key_averages():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                key = next((k for k in ("linear_q_wgmma", "linear_wgmma", "attention64", "add_ln", "embed_ln") if k in e.key),
                           "other")
                per[key] += e.self_device_time_total / 1e3
        split[f"{mode} {label}"] = {k: round(v, 3) for k, v in sorted(per.items())} | {"total_ms": round(sum(per.values()), 3)}
    del eng
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                   check=False).stdout.strip()
print(json.dumps({"card": q, "linear_kernels": linears, "forward_kernel_ms": split}))
