"""Query adapter: apply (hot path) and fit (SURVEY.md section 8f-4, the caller that produces ``A``).

Apply -- ``(A @ q).astype(q.dtype)`` (reference ``_search.py:58-62``) -- runs in ``rl_adapter_apply``
via ``CorpusIndex.apply_adapter``.  The fit follows ``raglite/_query_adapter.py:141-219``: for every
eval, embed the question, retrieve the top chunks *without* the adapter, take each chunk's best
vector for the query (MaxSim ``argmax(E_c @ q)``, ``:172-183``) as a positive or negative, solve the
bounded least squares for the target ``t`` (``:21-38``), then ``M = T^T Q / n`` (+ null-space
completion) and the orthogonal Procrustes / Frobenius-scaled solution (``:193-205``).

On a single-GPU index the whole fit runs on the device, batched over the evals: retrieval through the scan
(``vector_search_batch``), the MaxSim picks in ``rl_best_vectors``, every eval's bounded least squares in ONE
launch of ``rl_adapter_targets`` (active-set NNLS in float64, ``csrc/adapter_fit.cu``), and the final d x d algebra
(normalisation, ``T^T Q``, rank test, null-space completion, SVD) as float64 ``torch.linalg`` calls on the GPU.
A sharded corpus keeps the picks per shard (summed over ranks) and solves with SciPy as the reference does.
"""

from __future__ import annotations

from collections.abc import Sequence
from dataclasses import replace
from typing import Any

import numpy as np
import torch
from scipy.optimize import lsq_linear

from ._config import RAGLiteConfig
from ._index import CorpusIndex, get_index
from ._search import vector_search_batch


def _optimize_query_target(q: np.ndarray, P: np.ndarray, N: np.ndarray, *, alpha: float = 0.05) -> np.ndarray:
    """Dual of ``min ||t - q||`` s.t. every positive beats every negative by a margin (``:21-38``)."""
    dtype = q.dtype
    q64, P64, N64 = q.astype(np.float64), P.astype(np.float64), N.astype(np.float64)
    D = (P64[:, None, :] - (1.0 + alpha) * N64[None, :, :]).reshape(-1, P64.shape[1])
    mu = lsq_linear(D.T, -q64, bounds=(0.0, np.inf), tol=np.finfo(np.float64).eps).x
    return (q64 + D.T @ mu).astype(dtype)


def _best_vectors(index: Any, chunks: Sequence[int], q: np.ndarray) -> np.ndarray:
    """Row ``argmax(E_c @ q)`` of every chunk in ``chunks`` (GLOBAL chunk indices, as ``vector_search_batch``
    returns them): one gather + one matvec on the device.  On a sharded corpus every rank resolves the
    chunks it owns and the rows are summed over the shards (each chunk lives on exactly one)."""
    local: CorpusIndex = getattr(index, "local", index)
    off, base = local.chunk_off, local.chunk_base
    out = torch.zeros((len(chunks), local.d), dtype=torch.float32, device=local.device)
    mine = [(i, int(c) - base) for i, c in enumerate(chunks) if base <= int(c) < base + local.n_chunks]
    if mine:
        rows = np.concatenate([np.arange(off[c], off[c + 1]) for _, c in mine])
        seg = np.cumsum([0] + [int(off[c + 1] - off[c]) for _, c in mine])
        E = local.E[torch.from_numpy(rows).to(local.device)].float()
        s = (E @ torch.from_numpy(q.astype(np.float32)).to(local.device)).cpu().numpy()
        best = [rows[seg[j] + int(np.argmax(s[seg[j]:seg[j + 1]]))] for j in range(len(mine))]
        out[torch.tensor([i for i, _ in mine], device=local.device)] = \
            local.E[torch.from_numpy(np.asarray(best)).to(local.device)].float()
    elif not hasattr(index, "sum_over_shards") or getattr(index, "world", 1) == 1:
        raise ValueError("retrieved chunks are not in this index (chunk_base mismatch)")
    return index.sum_over_shards(out).cpu().numpy()


def _fit_on_device(local: CorpusIndex, evals: Sequence[tuple[np.ndarray, Sequence[int]]], Qm: np.ndarray, ids: np.ndarray,
                   counts: np.ndarray, alpha: float, metric: str) -> np.ndarray:
    """The fit for a device-resident shard (``_query_adapter.py:160-205``), batched over the evals."""
    from . import _lib

    lib = _lib.load()
    dev = local.device
    n, top_k = ids.shape
    kind = np.full((n, top_k), 2, dtype=np.uint8)     # 1 relevant, 0 irrelevant, 2 unused
    for e, (_, relevant) in enumerate(evals):
        rel = {int(r) for r in relevant}
        for j in range(int(counts[e])):
            kind[e, j] = 1 if int(ids[e, j]) in rel else 0
    chunks = np.where(np.arange(top_k)[None, :] < counts[:, None], ids - local.chunk_base, -1).astype(np.int64)
    with local._lock, torch.cuda.device(dev):
        Qd = torch.from_numpy(np.ascontiguousarray(Qm, dtype=np.float32)).to(dev)
        off = torch.from_numpy(local.chunk_off).to(dev)
        ch = torch.from_numpy(chunks).to(dev)
        kd = torch.from_numpy(kind).to(dev)
        best = torch.empty((n, top_k, local.d), dtype=torch.float32, device=dev)
        best_row = torch.empty((n, top_k), dtype=torch.int64, device=dev)
        stream = torch.cuda.current_stream().cuda_stream
        _lib.check(lib.rl_best_vectors(local.E.data_ptr(), 1 if local.storage == "fp16" else 0, local.d, local.d, off.data_ptr(),
                                       ch.data_ptr(), n, top_k, Qd.data_ptr(), best.data_ptr(), best_row.data_ptr(), stream),
                   "rl_best_vectors")
        T = torch.empty((n, local.d), dtype=torch.float64, device=dev)
        ok = torch.empty((n,), dtype=torch.int32, device=dev)
        iters = torch.empty((n,), dtype=torch.int32, device=dev)
        _lib.check(lib.rl_adapter_targets(best.data_ptr(), kd.data_ptr(), n, top_k, local.d, Qd.data_ptr(), float(alpha), T.data_ptr(),
                                          ok.data_ptr(), iters.data_ptr(), stream), "rl_adapter_targets")
        keep = ok == 1
        if not bool(keep.any()):
            raise ValueError("No eval had both relevant and irrelevant chunks among the retrieved ones.")
        # the reference casts every target back to its query's dtype (q_star.astype(q_dtype), :37) before stacking
        half = torch.tensor([np.ravel(q).dtype == np.float16 for q, _ in evals], device=dev)
        T = torch.where(half[:, None], T.to(torch.float16).to(torch.float64), T.to(torch.float32).to(torch.float64))
        Q64 = torch.from_numpy(np.ascontiguousarray(Qm)).to(dev).to(torch.float64)[keep]
        T64 = T[keep]
        Q64 = Q64 / torch.linalg.norm(Q64, dim=1, keepdim=True)
        if metric == "cosine":
            T64 = T64 / torch.linalg.norm(T64, dim=1, keepdim=True)
        m, d = Q64.shape
        M = (1 / m) * T64.T @ Q64
        if m < d or int(torch.linalg.matrix_rank(Q64)) < d:
            M = M + torch.eye(d, dtype=torch.float64, device=dev) - Q64.T @ torch.linalg.pinv(Q64 @ Q64.T) @ Q64
        if metric == "dot":
            A = M / torch.linalg.norm(M, ord="fro") * np.sqrt(d)
        else:
            U, _, VT = torch.linalg.svd(M, full_matrices=False)
            A = U @ VT
        return A.cpu().numpy()


def update_query_adapter(  # noqa: PLR0913
    evals: Sequence[tuple[np.ndarray, Sequence[int]]],
    *,
    max_evals: int = 4096,
    optimize_top_k: int = 40,
    optimize_gap: float = 0.05,
    config: RAGLiteConfig | None = None,
    index: Any | None = None,
    solver: str = "device",
) -> np.ndarray:
    """Compute the optimal query adapter and attach it to the index.

    ``evals`` are ``(question_embedding, relevant_chunk_indices)`` pairs -- what the reference reads from
    its ``Eval`` table and ``embed_strings`` (``_query_adapter.py:151-160``).

    ``solver="device"`` (default on a single-GPU index) solves every eval's bounded least squares on the
    device (the projection to ~1e-15 relative; with examples 1e-7 apart or closer, to ~1e-8).  ``solver="scipy"`` calls
    ``scipy.optimize.lsq_linear`` per eval as the reference does: identical to the device answer to ~1e-8 on small
    instances, but SciPy's trust-region iteration stops up to ~1e-3 short of the optimum on the larger rank-deficient
    ones (20 x 20 positives x negatives), so choose it only to reproduce the reference's iterate.
    """
    config = config or RAGLiteConfig()
    index = index if index is not None else get_index(config)
    local: CorpusIndex = getattr(index, "local", index)
    if local is None or local.n_rows == 0:
        raise ValueError("First insert documents (the index is empty).")
    if len(evals) == 0:
        raise ValueError("First generate evals.")
    metric = config.vector_search_distance_metric
    if metric not in ("cosine", "dot"):
        raise ValueError(f"Unsupported metric: {metric}")
    cfg_no_adapter = replace(config, vector_search_query_adapter=False)
    evals = list(evals)[:max_evals]
    Qm = np.stack([np.ravel(q) for q, _ in evals])
    ids, _, counts = vector_search_batch(Qm, num_results=optimize_top_k, config=cfg_no_adapter, index=index)
    if solver not in ("device", "scipy"):
        raise ValueError("solver must be 'device' or 'scipy'")
    if solver == "device" and not hasattr(index, "group") and optimize_top_k <= 64:
        A_star = _fit_on_device(local, evals, Qm, ids, counts, optimize_gap, metric)
        local.set_query_adapter(A_star)
        return A_star
    Qs, Ts = [], []
    for e, (q, relevant) in enumerate(evals):
        retrieved = [int(c) for c in ids[e, : counts[e]]]
        is_rel = np.array([c in set(int(r) for r in relevant) for c in retrieved], dtype=bool)
        if not is_rel.any() or is_rel.all():
            continue
        q = np.ravel(q)
        best = _best_vectors(index, retrieved, q)
        t = _optimize_query_target(q, best[is_rel], best[~is_rel], alpha=optimize_gap)
        Qs.append(q.astype(np.float64))
        Ts.append(t.astype(np.float64))
    if not Qs:
        raise ValueError("No eval had both relevant and irrelevant chunks among the retrieved ones.")
    Q, T = np.vstack(Qs), np.vstack(Ts)
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    if metric == "cosine":
        T /= np.linalg.norm(T, axis=1, keepdims=True)
    n, d = Q.shape
    M = (1 / n) * T.T @ Q
    if n < d or np.linalg.matrix_rank(Q) < d:
        M += np.eye(d) - Q.T @ np.linalg.pinv(Q @ Q.T) @ Q
    if metric == "dot":
        A_star = M / np.linalg.norm(M, ord="fro") * np.sqrt(d)
    else:
        U, _, VT = np.linalg.svd(M, full_matrices=False)
        A_star = U @ VT
    local.set_query_adapter(A_star)
    return A_star
