"""Benchmark of the l1 metric (pgvector's ``<+>``): ``vector_search_batch`` end to end and the L1 scan alone.

Shapes: c2 (100 k chunks x 8 vectors x 384, float32 and float16 rows, top-20) and one 1024-d float16 shard
(1.25 M chunks x 12 vectors x 1024 = 30.7 GB, top-100, num_hits 400), each at B = 1 (the reference's own call shape:
``vector_search`` takes one query) and B = 256.  Per case one JSON line:

- ``e2e_ms``: wall time per ``vector_search_batch`` call (it ends in a stream synchronisation);
- ``scan_ms``: sample + main scan from the ``RL_FLAG_TIME_KERNELS`` stage events (both passes run the L1 kernel);
- ``fadd_tflops``: ``2 B rows d / scan_ms`` (a FADD counts as one operation), against ``132 * 128 * f_SM`` with the SM
  clock read by ``nvidia-smi`` while the scans run, and against the data sheet's 67 TFLOP/s FP32 / 2;
- ``hbm_frac`` (B = 1): corpus bytes / scan time against 3.35 TB/s;
- ``oracle_ok``: 16 queries, searched B at a time (``oracle_batch``: the timed tile is the one checked), against
  float64 (c2: ``l1_oracle`` on the host over row blocks copied back; the 30.7 GB shard: the same float64 sums on the
  device, block by block, since 16 x 15 M x 1024 terms take too long in NumPy);
- ``numpy_ms_per_query``: the NumPy port ``np.abs(E - q).sum(1)`` on the host cores over a stated row subsample,
  scaled to the full corpus.

Run: ``python tools/bench_l1.py [--shapes c2,shard1024] [--storages fp32,fp16] [--batches 1,256] [--steps 10]
[--warmup 2] [--out FILE]``.
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
import threading
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

PEAK_FP32_TFLOPS = 67.0      # H100 SXM data sheet, dense FP32
HBM_TBS = 3.35
SHAPES = {
    "c2": dict(n_chunks=100_000, vecs=8, d=384, storages=("fp32", "fp16"), k=20),
    "shard1024": dict(n_chunks=1_250_000, vecs=12, d=1024, storages=("fp16",), k=100),
}


def gpu_info() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True, check=False).stdout.strip().splitlines()
    name, power, max_sm = (x.strip() for x in out[0].split(","))
    return {"gpu": name, "power_limit_w": float(power), "max_sm_mhz": float(max_sm)}


def sm_clock_during(fn) -> tuple[float, object]:   # noqa: ANN001
    """Run fn() (device work that ends in a synchronise) while a thread samples the SM clock; median MHz."""
    samples: list[float] = []
    stop = threading.Event()

    def sample() -> None:
        while not stop.is_set():
            r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"],
                               capture_output=True, text=True, check=False).stdout.strip().splitlines()
            if r:
                samples.append(float(r[0]))
            time.sleep(0.05)

    t = threading.Thread(target=sample, daemon=True)
    t.start()
    try:
        res = fn()
    finally:
        stop.set()
        t.join()
    return (float(np.median(samples)) if samples else float("nan")), res


def make_corpus(n_rows: int, d: int, storage: str, seed: int) -> torch.Tensor:
    """Gaussian unit rows on the device, float16-rounded (what RAGLite stores), generated in slices."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    E = torch.empty((n_rows, d), dtype=torch.float16 if storage == "fp16" else torch.float32, device="cuda")
    step = 1 << 20
    for r0 in range(0, n_rows, step):
        x = torch.randn((min(step, n_rows - r0), d), generator=g, device="cuda")
        x /= x.norm(dim=1, keepdim=True)
        E[r0:r0 + len(x)] = x.half().to(E.dtype)
    return E


def oracle_check(E: torch.Tensor, off_vecs: int, Q: np.ndarray, ids: np.ndarray, sims: np.ndarray, counts: np.ndarray,
                 k: int, on_host: bool) -> int:
    """Number of the queries whose (ids, sims) equal the float64 restatement (l1_oracle semantics, ties by index)."""
    from l1_oracle import l1_topn_rows_blocked

    from oracle import vector_search as ovs

    n_keep = ovs.num_hits_rule(k, 4, 2048)
    n_rows = int(E.shape[0])
    block = 1 << 17
    if on_host:
        blocks = ((r0, E[r0:r0 + block].float().cpu().numpy()) for r0 in range(0, n_rows, block))
        top = l1_topn_rows_blocked(blocks, Q, n_keep, f32_ties=True)
    else:
        Qd = torch.from_numpy(Q).cuda().double()
        keep_d = [torch.empty(0, dtype=torch.float32, device="cuda") for _ in Q]
        keep_r = [torch.empty(0, dtype=torch.int64, device="cuda") for _ in Q]
        for r0 in range(0, n_rows, block):
            D = torch.cdist(Qd, E[r0:r0 + block].double(), p=1).float()      # float64 sums, rounded to FLOAT
            for b in range(len(Q)):
                cd = torch.cat([keep_d[b], D[b]])
                cr = torch.cat([keep_r[b], torch.arange(r0, r0 + D.shape[1], device="cuda")])
                o = np.lexsort((cr.cpu().numpy(), cd.cpu().numpy()))[:n_keep]
                o = torch.from_numpy(o).cuda()
                keep_d[b], keep_r[b] = cd[o], cr[o]
        top = [(keep_r[b].cpu().numpy(), keep_d[b].cpu().numpy()) for b in range(len(Q))]
    ok = 0
    for b, (rows, dist) in enumerate(top):
        w_ids, w_sims = ovs.group_hits(dist.astype(np.float32), rows // off_vecs, k)
        n = int(counts[b])
        ok += int(n == len(w_ids) and np.array_equal(ids[b, :n], w_ids) and np.array_equal(sims[b, :n], w_sims))
    return ok


def run_case(rl, name: str, spec: dict, storage: str, E: torch.Tensor, B: int, args, info: dict) -> dict:  # noqa: ANN001
    from raglite_b200._lib import RL_FLAG_TIME_KERNELS

    d, vecs, k = spec["d"], spec["vecs"], spec["k"]
    n_rows = int(E.shape[0])
    idx = rl.CorpusIndex(E, vecs_per_chunk=vecs, storage=storage)
    cfg = rl.RAGLiteConfig(db_url="postgresql://bench/l1", vector_search_distance_metric="l1", reranker=None,
                           vector_search_query_adapter=False)
    g = torch.Generator(device="cuda").manual_seed(B)
    rows = torch.randint(0, n_rows, (B,), generator=g, device="cuda")
    Q = (E[rows].float() + 0.02 * torch.randn((B, d), generator=g, device="cuda")).half().float().contiguous()
    Qh = Q.cpu().numpy()
    num_hits = 4 * max(k, 10)
    for _ in range(args.warmup):
        rl.vector_search_batch(Qh, num_results=k, config=cfg, index=idx)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        ids, sims, counts = rl.vector_search_batch(Qh, num_results=k, config=cfg, index=idx)
    e2e_ms = (time.perf_counter() - t0) * 1e3 / args.steps

    def timed_scans() -> dict:
        for _ in range(args.steps):
            idx.scan(Q, k=k, num_hits=num_hits, metric="l1", flags=RL_FLAG_TIME_KERNELS)
        torch.cuda.synchronize()
        return idx.kernel_times_ms()

    idx.scan(Q, k=k, num_hits=num_hits, metric="l1", flags=RL_FLAG_TIME_KERNELS)
    idx.kernel_times_ms()
    f_mhz, ms = sm_clock_during(timed_scans)
    scan_ms = ms["sample_scan"] + ms["main_scan"]
    fadd = 2.0 * B * n_rows * d
    tflops = fadd / (scan_ms * 1e-3) / 1e12
    issue_peak = 132 * 128 * f_mhz * 1e6 / 1e12
    out = {"shape": name, "storage": storage, "B": B, "k": k, "num_hits": num_hits, "rows": n_rows, "d": d,
           "e2e_ms": round(e2e_ms, 3), "scan_ms": round(scan_ms, 3), "stage_ms": {s: round(v, 3) for s, v in ms.items()},
           "fadd_tflops": round(tflops, 2), "sm_mhz_during_scan": f_mhz,
           "frac_of_issue_at_clock": round(tflops / issue_peak, 3), "frac_of_datasheet_fp32_over_2": round(tflops / (PEAK_FP32_TFLOPS / 2), 3),
           **info}
    if B == 1:
        nbytes = n_rows * d * E.element_size()
        out["hbm_tbs"] = round(nbytes / (scan_ms * 1e-3) / 1e12, 3)
        out["hbm_frac"] = round(out["hbm_tbs"] / HBM_TBS, 3)
    if args.check:
        nq = 16
        if B < 16:   # 16 more queries, searched B at a time: the check runs the tile that was timed
            g2 = torch.Generator(device="cuda").manual_seed(99)
            rows = torch.randint(0, n_rows, (16,), generator=g2, device="cuda")
            Qc = (E[rows].float() + 0.02 * torch.randn((16, d), generator=g2, device="cuda")).half().float().cpu().numpy()
            parts = [rl.vector_search_batch(Qc[i:i + B], num_results=k, config=cfg, index=idx) for i in range(0, 16, B)]
            ids, sims, counts = (np.concatenate([p[j] for p in parts]) for j in range(3))
        else:
            Qc = Qh[:16]
        out["oracle_batch"] = B   # queries per vector_search_batch call in the check
        out["oracle_ok"] = f"{oracle_check(E, vecs, Qc, ids[:nq], sims[:nq], counts[:nq], k, on_host=name == 'c2')}/{nq}"
        out["oracle_where"] = "host float64" if name == "c2" else "device float64"
    idx.close()
    del idx
    return out


def numpy_port(E: torch.Tensor, n_sub: int) -> dict:
    sub = E[:n_sub].float().cpu().numpy()
    q = sub[0] + np.float32(0.01)
    t0 = time.perf_counter()
    np.abs(sub - q).sum(1)
    dt = time.perf_counter() - t0
    return {"numpy_subsample_rows": n_sub, "numpy_ms_per_query": round(dt * 1e3 * E.shape[0] / n_sub, 1)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="c2,shard1024")
    ap.add_argument("--batches", default="1,256")
    ap.add_argument("--storages", default="fp32,fp16", help="row storages to run, where the shape has them")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-check", dest="check", action="store_false")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_l1 needs a CUDA device")
    import raglite_b200 as rl

    info = gpu_info()
    lines = []
    for name in args.shapes.split(","):
        spec = SHAPES[name]
        for storage in (s for s in spec["storages"] if s in args.storages.split(",")):
            E = make_corpus(spec["n_chunks"] * spec["vecs"], spec["d"], storage, seed=7)
            extra = numpy_port(E, 20_000)
            for B in (int(b) for b in args.batches.split(",")):
                line = {**run_case(rl, name, spec, storage, E, B, args, info), **extra}
                print(json.dumps(line), flush=True)
                lines.append(line)
            del E
            torch.cuda.empty_cache()
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text("".join(json.dumps(x) + "\n" for x in lines))


if __name__ == "__main__":
    main()
