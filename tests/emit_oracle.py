"""NumPy restatement of what the scan's emission must hand to finalize (TEST INFRASTRUCTURE).

A scan with sample stride S > 1 dumps the keys of every S-th block of 128 rows (the sample), ``select_kernel`` turns
them into one emission threshold ``thr[b]`` per query and joins the sample rows at or above it to the candidate list,
and the main pass emits the rows of the other blocks whose key reaches the query's threshold -- a threshold the
tensor-core scan raises while it runs (online refinement, ``scan_wgmma.cu``).  Finalize then selects the ``sel_count``-th
best key ``T'`` of the list and rescores only the band ``[T' - 2 eps, inf)``; a row missing from that band is lost.

Let ``K_sel`` be the ``sel_count``-th best key over the valid rows of the shard (ties counted with multiplicity, as the
kernels' histograms count them).  Every row of exact similarity within reach of the top ``sel_count`` has a key of at
least ``K_sel - 2 eps`` (each key is within ``eps`` of its exact value), so the list must hold

    the required set  R = {valid rows: key >= K_sel - 2 eps}        (float64, from the float32 keys and eps),

and it can only hold

    the allowed set   A = {valid rows: key >= thr}                  (thr: the select kernel's threshold),

because no threshold the scan uses lies below ``thr``.  R is a subset of A whenever ``thr <= K_sel - 2 eps``, which the
select kernel's lower bound guarantees.  The keys come from a ``sample_stride=1`` dump of the same rows and queries:
at stride 1 every block is a sample block, and dump and emission share the epilogue's key arithmetic, so a candidate's
key equals its dump key bit for bit.

``cnt_all`` (``RL_FLAG_COUNT_UNFILTERED``) counts the rows of the main blocks that the filter masks out but that are
alive, at the threshold in force when their tile was scanned: at least those with key >= ``K_sel - 2 eps`` (no
threshold exceeds it), at most those with key >= ``thr``.

``hist_bin`` and ``refresh_edge`` restate the refinement's float32 arithmetic (``common.cuh``, ``scan_wgmma.cu``).
"""

from __future__ import annotations

import numpy as np

BLOCK_ROWS = 128        # kBlockRows
HIST_BINS = 16          # kHistBins
F32 = np.float32


def sel_count(*, k: int, num_hits: int, max_vecs: int) -> int:
    """The order statistic the emission must reach: ``num_hits`` (SQL semantics) or ``(k - 1) * max_vecs + 1``
    (exact MaxSim: the k best chunks own at most that many of the best vectors)."""
    return num_hits if num_hits > 0 else (k - 1) * max_vecs + 1


def auto_stride(n_rows: int, *, k: int, num_hits: int, max_vecs: int) -> int:
    """The sample stride ``make_layout`` picks for ``sample_stride=0`` (api.cu)."""
    sel_k = num_hits if num_hits > 0 else k
    rows_per_sel = 1.0 if num_hits > 0 else float(max_vecs)
    f = np.sqrt(sel_k * rows_per_sel * 16.0 / (max(n_rows, 1) * 4.0))
    x, S = (4.0 / f if f > 0 else 1.0), 1
    while S * 2 <= x:
        S *= 2
    S = min(S, 256)
    nb = n_blocks(n_rows)
    while S > 1 and (nb // S) * BLOCK_ROWS < 8 * sel_k * rows_per_sel:
        S //= 2
    return 1 if nb < 64 else max(S, 1)


def n_blocks(n_rows: int) -> int:
    return (n_rows + BLOCK_ROWS - 1) // BLOCK_ROWS


def sample_blocks(n_rows: int, S: int) -> np.ndarray:
    """Blocks the sample pass dumps: every S-th, starting at 0."""
    return np.arange(0, n_blocks(n_rows), S, dtype=np.int64)


def main_block_index(ord_: np.ndarray | int, S: int) -> np.ndarray:
    """``main_block_index`` (common.cuh): the ord-th block that is not a sample block."""
    o = np.asarray(ord_, np.int64)
    return o if S <= 1 else o + o // (S - 1) + 1


def main_blocks(n_rows: int, S: int) -> np.ndarray:
    nb = n_blocks(n_rows)
    n_main = nb - (nb + S - 1) // S
    return main_block_index(np.arange(n_main, dtype=np.int64), S)


def sample_rows(n_sample_rows: int, S: int) -> np.ndarray:
    """Row of each dump position p: ``(p / 128) * S * 128 + p % 128`` (``sample_row_of``)."""
    p = np.arange(n_sample_rows, dtype=np.int64)
    return (p // BLOCK_ROWS) * S * BLOCK_ROWS + p % BLOCK_ROWS


def block_rows(blocks: np.ndarray, n_rows: int) -> np.ndarray:
    """The rows of the given blocks that exist."""
    r = (np.asarray(blocks, np.int64)[:, None] * BLOCK_ROWS + np.arange(BLOCK_ROWS)[None, :]).ravel()
    return r[r < n_rows]


def kth_key(keys: np.ndarray, valid: np.ndarray, sel: int) -> np.ndarray:
    """``K_sel`` per query: the sel-th largest valid key (ties with multiplicity), -inf when fewer valid rows."""
    k = np.where(valid, keys, -np.inf).astype(np.float32)
    n = k.shape[1]
    if sel > n:
        return np.full(k.shape[0], -np.inf, np.float32)
    return -np.partition(-k, sel - 1, axis=1)[:, sel - 1]


def required(keys: np.ndarray, valid: np.ndarray, sel: int, eps: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """``(R [B, n] bool, K_sel [B])``: the valid rows with key >= K_sel - 2 eps, in float64."""
    ks = kth_key(keys, valid, sel)
    lim = ks.astype(np.float64) - 2.0 * np.asarray(eps, np.float64)
    return valid & (keys.astype(np.float64) >= lim[:, None]), ks


def allowed(keys: np.ndarray, valid: np.ndarray, thr: np.ndarray) -> np.ndarray:
    """A [B, n]: the valid rows with key >= thr (the float32 comparison of the epilogues)."""
    return valid & (keys >= np.asarray(thr, np.float32)[:, None])


def cnt_all_bounds(keys: np.ndarray, masked_alive: np.ndarray, main: np.ndarray, ksel: np.ndarray, eps: np.ndarray,
                   thr: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """Bounds of ``cnt_all`` per query.  ``keys`` [B, n] hold the key of every alive row (masked or not); ``masked_alive``
    [n] the rows the filter removes that are alive; ``main`` [n] the rows of main-pass blocks."""
    rows = masked_alive & main
    lim = ksel.astype(np.float64) - 2.0 * np.asarray(eps, np.float64)
    lo = (rows[None, :] & (keys.astype(np.float64) >= lim[:, None])).sum(1)
    hi = (rows[None, :] & (keys >= np.asarray(thr, np.float32)[:, None])).sum(1)
    return lo, hi


# ---- the refinement's float32 arithmetic ---------------------------------------------------------------------------
def hist_bin(key, thr0, inv_w) -> np.ndarray:
    """``hist_bin`` (common.cuh) in float32: ``(int)((key - thr0) * inv_w)`` clamped to [0, 15]."""
    x = (F32(key) - F32(thr0)) * F32(inv_w)
    b = np.where(x > 0, np.trunc(np.minimum(x, HIST_BINS)), 0).astype(np.int64)
    return np.minimum(b, HIST_BINS - 1)


def naive_edge(thr0, inv_w, best: int) -> np.float32:
    """The lower edge of bin ``best`` as ``thr0 + best / inv_w`` in float32 (the refresh before it was made safe)."""
    return F32(F32(thr0) + F32(F32(best) / F32(inv_w)))


def refresh_edge(thr0, inv_w, best: int) -> np.float32:
    """The refresh's edge: ``naive_edge`` lowered by ``2^-21 (g + |edge|)``, ``g = best / inv_w``, so that every key the
    histogram counts at or above ``best`` is at or above the edge."""
    g = F32(F32(best) / F32(inv_w))
    e0 = F32(F32(thr0) + g)
    return F32(e0 - F32(F32(g + np.abs(e0)) * F32(2.0**-21)))


def least_key_in_bin(thr0, inv_w, best: int) -> np.float32:
    """The least float32 key that ``hist_bin`` puts in a bin >= best: a bisection over the order-preserving integer
    image of float32 (``hist_bin`` is monotone in the key)."""
    def of(o: int) -> np.float32:    # ord2f
        u = np.uint32(o & 0x7FFFFFFF) if o & 0x80000000 else np.uint32(~o & 0xFFFFFFFF)
        return u.view(F32)
    lo, hi = 0x00800000, 0xFF7FFFFF          # -max finite .. +max finite
    assert hist_bin(of(hi), thr0, inv_w) >= best
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if hist_bin(of(mid), thr0, inv_w) >= best:
            hi = mid
        else:
            lo = mid
    return of(hi)


def refreshed_threshold(thr0, inv_w, eps, best: int) -> np.float32:
    """``edge - 2 eps`` in float32: the threshold a refresh that found ``best`` raises the query to."""
    return F32(refresh_edge(thr0, inv_w, best) - F32(F32(2.0) * F32(eps)))
