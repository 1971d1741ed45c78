"""NumPy restatement of ``vector_search`` under the ``l1`` metric (TEST INFRASTRUCTURE), beside ``oracle.vector_search``,
whose cosine / dot / l2 restatements it reuses for everything after the distance.

PARITY UNPINNED: ``l1`` exists only on the reference's PostgreSQL branch, where pgvector evaluates ``embedding <+> query``
on ``halfvec`` columns; pgvector is not part of the reference tree.  What is restated here is recalled, not read:
pgvector is recalled to sum ``fabsf(HalfToFloat4(a[i]) - HalfToFloat4(b[i]))`` over i in float32, in ascending i, and
to return the sum widened to double, and to parse each element of a bound ``halfvec`` with ``strtof`` and round it to
binary16 (round to nearest even), refusing a value outside the binary16 range ("infinite value not allowed").
"""

from __future__ import annotations

from collections.abc import Callable, Iterable

import numpy as np

from oracle import vector_search as ovs


def halfvec_query(q: np.ndarray) -> np.ndarray:
    """The query as pgvector holds it after ``PostgresHalfVec.bind_processor`` (``_typing.py:157-163``) bound it as the
    text ``str(x)`` of each element: ``strtof`` then binary16, round to nearest even, returned as float32.  A float64
    element is rounded twice, to float32 first (the float ``strtof`` makes of its shortest decimal) and then to binary16;
    float32 / float16 elements once / not at all.  An element that rounds to +-inf (or is NaN) raises ``ValueError``."""
    q = np.asarray(q)
    if q.dtype != np.float16:
        q = q.astype(np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        h = q.astype(np.float16)
    if not np.isfinite(h).all():
        raise ValueError("infinite value not allowed in halfvec")
    return h.astype(np.float32)


def l1_distances(E: np.ndarray, q: np.ndarray) -> np.ndarray:
    """``<+>`` as pgvector computes it (recalled): a float32 running sum of ``|e_i - q_i|`` in ascending i, as float64."""
    E = np.asarray(E, dtype=np.float32)
    q = np.ravel(q).astype(np.float32)
    acc = np.zeros(E.shape[0], np.float32)
    for i in range(E.shape[1]):
        acc += np.abs(E[:, i] - q[i])
    return acc.astype(np.float64)


def l1_distances_f64(E: np.ndarray, q: np.ndarray) -> np.ndarray:
    """``sum |e - q|`` in float64 (the exact rescoring's quantity)."""
    return np.abs(np.asarray(E, np.float64) - np.ravel(q).astype(np.float64)[None, :]).sum(1)


def l1_search_sql(  # noqa: PLR0913
    E: np.ndarray, chunk_off: np.ndarray, q: np.ndarray, *, num_results: int = 3, oversample: int = 4,
    chunk_max_size: int = 2048, allowed_chunks: np.ndarray | None = None, f64: bool = True, f32_ties: bool = True,
    filter_first_max: int = 100_000, rank_first_limit: int = 1_000_000, row_chunk: np.ndarray | None = None,
) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """``ovs.vector_search_sql`` with the ``l1`` distance: the same ``num_hits`` rule, ``ORDER BY dist LIMIT num_hits``,
    both metadata branches and ``GROUP BY chunk max(sim)``; ties by row / chunk index.  With ``f64`` and ``f32_ties``
    the float64 distance is rounded to the FLOAT the SQL returns before ordering, so ``sim = 1 - float(dist)``."""
    E = np.asarray(E)
    if E.shape[0] == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.float32), np.zeros(0, np.int64)
    num_hits = ovs.num_hits_rule(num_results, oversample, chunk_max_size)
    dist = l1_distances_f64(E, q) if f64 else l1_distances(E, q)
    if f64 and f32_ties:
        dist = ovs.float_distance_of_f64(dist, "l1")
    r2c = ovs.row_to_chunk(chunk_off, E.shape[0]) if row_chunk is None else np.asarray(row_chunk, dtype=np.int64)
    rows = np.arange(E.shape[0])
    if allowed_chunks is not None:
        row_ok = np.asarray(allowed_chunks, dtype=bool)[r2c]
        if int(row_ok.sum()) <= filter_first_max:
            rows = rows[row_ok]
        else:
            nearest = np.argsort(dist, kind="stable")[:rank_first_limit]
            rows = np.sort(nearest[row_ok[nearest]])
    order = rows[np.argsort(dist[rows], kind="stable")][:num_hits]
    ids, sims = ovs.group_hits(dist[order], r2c[order], num_results)
    return ids, sims, order.astype(np.int64)


def l1_maxsim_topk(E: np.ndarray, chunk_off: np.ndarray, q: np.ndarray, k: int) -> tuple[np.ndarray, np.ndarray]:
    """Exact per-chunk MaxSim under ``l1``: per chunk the largest ``1 - float(dist)`` (float32), ties by chunk index."""
    dist = ovs.float_distance_of_f64(l1_distances_f64(E, q), "l1")
    sim = np.float32(1.0) - dist
    s = np.maximum.reduceat(sim, np.asarray(chunk_off, np.int64)[:-1])
    rank = np.lexsort((np.arange(len(s)), -s.astype(np.float64)))[:k]
    return rank.astype(np.int64), s[rank]


def l1_topn_rows_blocked(blocks: Iterable[tuple[int, np.ndarray]], Q: np.ndarray, n_keep: int, *, f32_ties: bool = True,
                         row_ok: Callable[[int, int], np.ndarray] | None = None) -> list[tuple[np.ndarray, np.ndarray]]:
    """``ORDER BY dist LIMIT n_keep`` under ``l1`` over a table handed over block by block (``(first_row, E_block)`` in
    row order, e.g. slices copied back from the device).  There is no GEMM shortcut for L1: each block's distances are
    summed directly, in float64 (with ``f32_ties`` rounded to FLOAT); ties by row index, as the unblocked restatement.
    Returns, per query, ``(rows int64, dist)`` ascending."""
    Q64 = np.asarray(Q, dtype=np.float64)
    B = Q64.shape[0]
    keep_d = [np.zeros(0, np.float32 if f32_ties else np.float64) for _ in range(B)]
    keep_r = [np.zeros(0, np.int64) for _ in range(B)]
    for row0, Eb in blocks:
        E64 = np.asarray(Eb, dtype=np.float64)
        n = E64.shape[0]
        if n == 0:
            continue
        idx_all = np.arange(n) if row_ok is None else np.nonzero(np.asarray(row_ok(row0, n), dtype=bool))[0]
        for b in range(B):
            d = np.abs(E64[idx_all] - Q64[b][None, :]).sum(1)
            if f32_ties:
                d = ovs.float_distance_of_f64(d, "l1")
            cd = np.concatenate([keep_d[b], d])
            cr = np.concatenate([keep_r[b], idx_all.astype(np.int64) + int(row0)])
            if len(cd) > n_keep:
                v = np.partition(cd, n_keep - 1)[n_keep - 1]
                sel = cd <= v
                cd, cr = cd[sel], cr[sel]
            keep_d[b], keep_r[b] = cd, cr
    out = []
    for b in range(B):
        o = np.lexsort((keep_r[b], keep_d[b]))[:n_keep]
        out.append((keep_r[b][o], keep_d[b][o]))
    return out
