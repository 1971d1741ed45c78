"""The coarse scan's key contract, checked directly: every approximate key lies within the kernel's own ``eps[b]``
of the exact key.

Exact top-k rests on this bound.  The finalize step only re-scores rows inside a band of 2 eps around the cut, so a
row whose coarse key is off by more than eps is dropped without a trace when it sits at the cut -- something
end-to-end tests on random data almost never see.  Here every (query, row) key of a scan with ``sample_stride=1``
(every block is a sample block, so the dump holds all rows, position p = row p) is compared with the key computed
in float64 from the stored values, against the eps the kernels wrote into the workspace (``debug_eps``), for the
tensor-core scan's loader paths and for the float32 scan.  The largest ``|err| / eps`` per case is appended to
``scan_key_bounds.jsonl`` in the temporary directory.
"""

from __future__ import annotations

import json
import tempfile
import zlib
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_RAGGED = 128 * 133 + 5   # several tiles per CTA and a ragged last tile


@pytest.fixture(scope="module")
def rl():
    import torch

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import raglite_b200

    return raglite_b200


def _record(name: str, payload: dict) -> None:
    with (Path(tempfile.gettempdir()) / "scan_key_bounds.jsonl").open("a") as f:
        f.write(json.dumps({"test": name, **payload}) + "\n")


# ---- corpora and queries (seeded, made on the device) ------------------------------------------------------------
def _corpus(kind: str, n: int, d: int, seed: int, Q):  # noqa: ANN001, ANN202
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    E = torch.randn((n, d), generator=g, device="cuda")
    if kind == "unit":
        E /= E.norm(dim=1, keepdim=True)
    elif kind == "gauss":
        E *= 1.5
    elif kind == "zero_row":          # one all-zero row: the cosine scan scales rows in the loader
        E /= E.norm(dim=1, keepdim=True)
        E[n // 3] = 0.0
    elif kind == "norm03":            # one row of norm 0.3: same loader
        E /= E.norm(dim=1, keepdim=True)
        E[n // 2] *= 0.3
    elif kind in ("subnormal_unit", "subnormal"):
        # magnitudes log-uniform over nine decades: after scaling, most small elements are fp16 subnormals (or flush)
        E *= torch.pow(10.0, -9.0 * torch.rand((n, d), generator=g, device="cuda"))
        if kind == "subnormal_unit":
            E /= E.norm(dim=1, keepdim=True)
    elif kind == "outlier":           # one row 1000x the rest: the global power-of-two scale pushes the others down
        E[n // 2] *= 1000.0
    elif kind == "cancel":            # e ~ -q: the key is near 0 while |e||q| is not
        E /= E.norm(dim=1, keepdim=True)
        m = min(n, Q.shape[0])
        E[:m] = -Q[:m] + 1e-3 * E[:m]
    else:
        raise AssertionError(kind)
    return E


def _queries(kind: str, B: int, d: int, seed: int):  # noqa: ANN202
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed + 1000)
    Q = torch.randn((B, d), generator=g, device="cuda")
    Q /= Q.norm(dim=1, keepdim=True)
    if kind == "norms":               # queries of norm 1e-3 and 1e3
        Q[0::2] *= 1e-3
        Q[1::2] *= 1e3
    return Q.contiguous()


def _exact_keys(E, Q, metric: str):  # noqa: ANN001, ANN202
    """Float64 keys [B, n] as the comment above ``sim_floor_to_thr_kernel`` defines them.  A zero row has inv_norm 0
    in the index, so its cosine key is 0."""
    Ed, Qd = E.double(), Q.double()
    G = Qd @ Ed.T
    if metric == "dot":
        return G
    ne2 = (Ed * Ed).sum(dim=1)
    if metric == "l2":
        return 2.0 * G - ne2[None, :]
    ne, nq = ne2.sqrt(), Qd.norm(dim=1)
    inv_e = (1.0 / ne).nan_to_num(posinf=0.0)
    return G * inv_e[None, :] / nq[:, None]


def _build(rl, E, storage: str, tombstones: bool):  # noqa: ANN001, ANN202
    n = int(E.shape[0])
    ids = [f"c{i}" for i in range(n)]
    if storage == "fp16":
        E = E.half()
    idx = rl.CorpusIndex(E, vecs_per_chunk=1, chunk_ids=ids, storage=storage)
    dead = np.arange(5, n, 97) if tombstones and n > 5 else np.zeros(0, np.int64)
    if len(dead):
        idx.delete_chunks([ids[i] for i in dead])
    return idx, dead


# (id naming the path it exists for, metric, storage, d, n_rows, B, corpus, queries, tombstones)
CASES = [
    # fp32 storage, fast loader (d % 64 == 0, even number of 64-wide K slices, no per-row scale)
    ("fast_cos_d128", "cosine", "fp32", 128, N_RAGGED, 129, "unit", "unit", True),
    ("fast_cos_d384", "cosine", "fp32", 384, 129, 1100, "unit", "unit", False),
    ("fast_cos_d1024", "cosine", "fp32", 1024, N_RAGGED, 17, "unit", "unit", False),
    ("fast_dot_d128", "dot", "fp32", 128, N_RAGGED, 128, "gauss", "unit", False),
    ("fast_dot_d1024", "dot", "fp32", 1024, 129, 1024, "gauss", "unit", True),
    ("fast_l2_d384", "l2", "fp32", 384, N_RAGGED, 1025, "gauss", "unit", False),
    ("fast_l2_d1024", "l2", "fp32", 1024, 1, 1, "gauss", "unit", False),
    # fp32 storage, generic loader: one K slice (d <= 64), an odd number of slices, K tails (d % 64 != 0)
    ("generic_cos_d4", "cosine", "fp32", 4, N_RAGGED, 129, "unit", "unit", False),
    ("generic_dot_d60", "dot", "fp32", 60, 129, 17, "gauss", "unit", False),
    ("generic_l2_d64", "l2", "fp32", 64, N_RAGGED, 128, "gauss", "unit", True),
    ("generic_cos_d72", "cosine", "fp32", 72, 129, 1025, "unit", "unit", False),
    ("generic_dot_d192", "dot", "fp32", 192, N_RAGGED, 1, "gauss", "unit", False),
    ("generic_l2_d200", "l2", "fp32", 200, N_RAGGED, 17, "gauss", "unit", False),
    # cosine with per-row scaling in the loader (a row of norm < 0.5 or an all-zero row)
    ("scaled_cos_zero_row_d128", "cosine", "fp32", 128, N_RAGGED, 129, "zero_row", "unit", False),
    ("scaled_cos_norm03_d384", "cosine", "fp32", 384, N_RAGGED, 128, "norm03", "unit", True),
    ("scaled_cos_norm03_d200", "cosine", "fp32", 200, 129, 17, "norm03", "unit", False),
    # fp16 storage through the TMA tensor map
    ("fp16_cos_d8", "cosine", "fp16", 8, N_RAGGED, 129, "unit", "unit", False),
    ("fp16_dot_d72", "dot", "fp16", 72, 129, 1100, "gauss", "unit", False),
    ("fp16_l2_d1024", "l2", "fp16", 1024, N_RAGGED, 128, "gauss", "unit", True),
    ("fp16_cos_d1024", "cosine", "fp16", 1024, 1, 1025, "unit", "unit", False),
    # accumulation length
    ("fast_cos_d4096", "cosine", "fp32", 4096, N_RAGGED, 17, "unit", "unit", False),
    ("fast_dot_d4096", "dot", "fp32", 4096, 129, 129, "gauss", "unit", False),
    # adversarial values
    ("subnormal_cos_d384", "cosine", "fp32", 384, N_RAGGED, 128, "subnormal_unit", "unit", False),
    ("subnormal_dot_d256", "dot", "fp32", 256, N_RAGGED, 129, "subnormal", "unit", False),
    ("subnormal_l2_d200", "l2", "fp32", 200, N_RAGGED, 17, "subnormal", "unit", False),
    ("subnormal_fp16_cos_d384", "cosine", "fp16", 384, N_RAGGED, 128, "subnormal_unit", "unit", False),
    ("subnormal_fp16_dot_d128", "dot", "fp16", 128, N_RAGGED, 17, "subnormal", "unit", False),
    ("outlier_dot_d384", "dot", "fp32", 384, N_RAGGED, 129, "outlier", "unit", False),
    ("outlier_l2_d384", "l2", "fp32", 384, N_RAGGED, 128, "outlier", "unit", True),
    ("outlier_l2_d72", "l2", "fp32", 72, N_RAGGED, 17, "outlier", "unit", False),
    ("qnorms_cos_d128", "cosine", "fp32", 128, N_RAGGED, 129, "unit", "norms", False),
    ("qnorms_dot_d128", "dot", "fp32", 128, N_RAGGED, 128, "gauss", "norms", False),
    ("qnorms_l2_d200", "l2", "fp32", 200, N_RAGGED, 129, "gauss", "norms", False),
    ("qnorms_fp16_l2_d128", "l2", "fp16", 128, N_RAGGED, 17, "gauss", "norms", False),
    ("cancel_cos_d384", "cosine", "fp32", 384, N_RAGGED, 128, "cancel", "unit", False),
    ("cancel_dot_d384", "dot", "fp32", 384, N_RAGGED, 129, "cancel", "unit", False),
    ("cancel_l2_d384", "l2", "fp32", 384, N_RAGGED, 128, "cancel", "unit", False),
    ("cancel_fp16_dot_d1024", "dot", "fp16", 1024, N_RAGGED, 129, "cancel", "unit", False),
]


def _params():
    out = []
    for c in CASES:
        for algo in ("tcgen05", "fp32"):
            if algo == "fp32" and c[2] == "fp16":
                continue   # float16 storage only has the tensor-core scan
            out.append(pytest.param(c, algo, id=f"{c[0]}-{algo}"))
    return out


@pytest.mark.parametrize(("case", "algo"), _params())
def test_coarse_keys_within_kernel_eps(rl, case, algo):
    import torch

    name, metric, storage, d, n, B, ckind, qkind, tomb = case
    seed = zlib.crc32(name.encode()) % (1 << 30)
    Q = _queries(qkind, B, d, seed)
    E = _corpus(ckind, n, d, seed, Q)
    idx, dead = _build(rl, E, storage, tomb)
    idx.scan(Q, k=1, num_hits=1, metric=metric, algo=algo, sample_stride=1)
    st = idx.scan_stats()
    assert st["algo"] == (2 if algo == "tcgen05" else 1) and st["sample_stride"] == 1
    dump, eps = idx.debug_dump(), idx.debug_eps()
    torch.cuda.synchronize()
    n_pad = (n + 127) // 128 * 128
    assert tuple(dump.shape) == (B, n_pad)
    assert bool(torch.all(eps > 0)) and bool(torch.all(torch.isfinite(eps)))
    assert bool(torch.all(dump[:, n:] == float("-inf"))), "positions past n_rows must be -inf"
    dead_t = torch.as_tensor(dead, dtype=torch.long, device="cuda")
    if len(dead):
        assert bool(torch.all(dump[:, dead_t] == float("-inf"))), "tombstoned rows must be -inf"
    exact = _exact_keys(idx.E, Q, metric)                  # the values the scan reads (fp16 storage: the fp16 values)
    alive = torch.ones(n, dtype=torch.bool, device="cuda")
    alive[dead_t] = False
    key = dump[:, :n].double()
    assert bool(torch.all(torch.isfinite(key[:, alive])))
    err = (key - exact).abs()[:, alive]
    ratio = err / eps.double()[:, None]
    worst = float(ratio.max())
    b, r = divmod(int(ratio.argmax()), int(alive.sum()))
    _record(name, {"algo": algo, "metric": metric, "storage": storage, "d": d, "n_rows": n, "B": B,
                   "max_err_over_eps": worst, "max_abs_err": float(err.max()),
                   "eps_min": float(eps.min()), "eps_max": float(eps.max())})
    assert worst <= 1.0, (name, algo, worst, "query", b, "live row", r, float(eps[b]))


# ---- emit path against the dump ---------------------------------------------------------------------------------
def _floor_for_key(T: np.ndarray, metric: str, q_sq: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """Similarity floor whose key threshold (``sim_floor_to_thr_kernel``, bound 0) is near T, and that threshold
    as the kernel computes it from the float32 floor."""
    if metric == "cosine":
        f = T.astype(np.float32)
        return f, f
    if metric == "dot":
        f = (T + 1.0).astype(np.float32)
        return f, (f - np.float32(1.0)).astype(np.float32)
    f = (1.0 - np.sqrt(q_sq - T)).astype(np.float32)
    dist = 1.0 - f.astype(np.float64)
    return f, (q_sq - dist * dist).astype(np.float32)


@pytest.mark.parametrize("algo", ["tcgen05", "fp32"])
@pytest.mark.parametrize("metric", ["cosine", "dot", "l2"])
def test_count_at_least_matches_dump(rl, metric, algo):
    """The emit-mode epilogue and the per-group / per-launch offsets (B = 1100: a second launch with a ragged last
    group), which the dump does not go through: ``count_at_least(bound=0)`` must count exactly the dump keys at or
    above the threshold.  Each floor sits in the middle of a wide gap between consecutive sorted dump keys, so the
    float32 floor -> key conversion cannot move a row across it."""
    import torch

    n, d, B = N_RAGGED, 128, 1100
    Q = _queries("unit", B, d, 7)
    E = _corpus("unit" if metric == "cosine" else "gauss", n, d, 8, Q)
    idx, dead = _build(rl, E, "fp32", True)
    idx.scan(Q, k=1, num_hits=1, metric=metric, algo=algo, sample_stride=1)
    keys = idx.debug_dump()[:, :n]
    srt = torch.sort(keys, dim=1, descending=True).values.double()
    n_live = n - len(dead)
    gaps = srt[:, :-1] - srt[:, 1:]
    q_sq = (Q.double() ** 2).sum(dim=1).cpu().numpy()
    checked = 0
    for lo, hi in ((0, 8), (50, 200), (n_live // 2 - 500, n_live // 2 + 500)):
        i = gaps[:, lo:hi].argmax(dim=1) + lo                       # widest gap in this rank window, per query
        above = srt.gather(1, i[:, None])[:, 0].cpu().numpy()
        below = srt.gather(1, (i + 1)[:, None])[:, 0].cpu().numpy()
        floor, thr = _floor_for_key(0.5 * (above + below), metric, q_sq)
        inside = (thr > below + 0.25 * (above - below)) & (thr < above - 0.25 * (above - below))
        assert inside.mean() > 0.99, (lo, hi, inside.mean())
        ok = torch.from_numpy(inside).cuda()
        want = (keys.double() >= torch.from_numpy(thr.astype(np.float64)).cuda()[:, None]).sum(dim=1).to(torch.int32)
        assert torch.equal(want[ok], (i[ok] + 1).to(torch.int32))     # the gap holds: rows of rank <= i and no others
        got = idx.count_at_least(Q, torch.from_numpy(floor).cuda(), k=1, num_hits=1, metric=metric, algo=algo, bound=0)
        assert torch.equal(got[ok], want[ok]), (lo, hi, int((got[ok] != want[ok]).sum()))
        checked += int(inside.sum())
    assert checked > 3 * B * 0.99
