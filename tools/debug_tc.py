"""Compare the tensor-core (wgmma) scan's approximate keys with the fp32 scan's, element by element."""
import sys
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parents[1])); sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tests"))
import numpy as np, torch
from synth import make_corpus, make_queries
import raglite_b200 as rl

def run(n_chunks, vecs, dim, B, metric="cosine"):
    E, off = make_corpus(n_chunks, vecs, dim, seed=0)
    Q = make_queries(E, B, seed=1)
    idx = rl.CorpusIndex(E, off)
    Qd = torch.from_numpy(Q).cuda()
    out = {}
    for algo in ("fp32", "tcgen05"):
        idx.scan(Qd, k=5, num_hits=40, metric=metric, algo=algo, sample_stride=1)
        torch.cuda.synchronize()
        out[algo] = idx.debug_dump().cpu().numpy()
    a, b = out["fp32"], out["tcgen05"]
    fin = np.isfinite(a)
    err = np.abs(a[fin] - b[fin])
    print(f"shape n={E.shape[0]} d={dim} B={B} {metric}: dump {a.shape} max|diff|={err.max():.3e} mean={err.mean():.3e} "
          f"inf-mismatch={(np.isfinite(a) != np.isfinite(b)).sum()}")
    if err.max() > 5e-3:
        bad = np.argwhere(np.abs(np.where(fin, a - b, 0)) > 5e-3)
        print("  first bad (query, pos):", bad[:10].tolist())
        print("  fp32   :", a[0, :8]); print("  tcgen05:", b[0, :8])
        cols = np.unique(bad[:, 0]); rows = np.unique(bad[:, 1] % 128)
        print("  bad queries:", cols[:20], " bad rows%128:", rows[:40])

if len(sys.argv) > 1 and sys.argv[1] == "stress":
    for args in [(40000, 8, 1024, 256), (100000, 8, 384, 256), (30000, 12, 1024, 200), (150000, 4, 128, 64)]:
        run(*args)
    sys.exit(0)
for args in [(64, 2, 64, 16), (100, 3, 128, 40), (300, 4, 384, 256), (200, 8, 1024, 128), (500, 2, 100, 7), (400, 4, 64, 300)]:
    run(*args)
run(300, 2, 64, 16, "dot"); run(300, 2, 64, 16, "l2")
