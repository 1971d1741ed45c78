"""Batches at the tensor-core scan's 256-query group width.

On a float32 corpus with d > 960, a batch of more than 128 queries is scanned in groups of 256: one CTA per lane
converts each corpus tile once for all 256 queries.  These are more inputs for two existing checks: the coarse-key
contract of ``test_gpu_scan_keys`` (every key within the kernel's own eps of the float64 key) and the block-boundary
search of ``test_gpu_search``.  They cover one full group on the fast loader, a full group followed by a second group
of 127, the generic loader (a K tail; per-row cosine scaling) at 256-wide groups, fp16 storage at B = 256 (which keeps
groups of 128), and batches of 256 and 384 on both sides of a 128-row block edge.
"""

from __future__ import annotations

import pytest
import test_gpu_scan_keys as keys
from parity import check_sql_semantics
from synth import make_corpus, make_queries
from test_gpu_search import ALGOS, _algo_ok

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rl():
    import torch

    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import raglite_b200

    return raglite_b200


# (id, metric, storage, d, n_rows, B, corpus, queries, tombstones), as test_gpu_scan_keys.CASES
CASES = [
    ("fast_cos_d1024_b256", "cosine", "fp32", 1024, keys.N_RAGGED, 256, "unit", "unit", False),
    ("fast_dot_d1024_b383", "dot", "fp32", 1024, keys.N_RAGGED, 383, "gauss", "unit", True),
    ("generic_l2_d1000_b256", "l2", "fp32", 1000, keys.N_RAGGED, 256, "gauss", "unit", False),
    ("scaled_cos_norm03_d1024_b300", "cosine", "fp32", 1024, keys.N_RAGGED, 300, "norm03", "unit", False),
    ("fp16_cos_d1024_b256", "cosine", "fp16", 1024, keys.N_RAGGED, 256, "unit", "unit", False),
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
def test_coarse_keys_within_kernel_eps_256_groups(rl, case, algo):
    keys.test_coarse_keys_within_kernel_eps(rl, case, algo)


@pytest.mark.parametrize("algo", ALGOS)
def test_block_boundaries_256_groups(rl, algo):
    """As test_block_boundaries_and_batch_groups, at d = 1024 with batches of 256 (one full group) and 384 (a full
    group and a second of 128)."""
    _algo_ok(rl, algo, 1024)
    for n_rows in (128, 129, 256 * 3):
        E, off = make_corpus(n_rows, 1, 1024, seed=n_rows)
        idx = rl.CorpusIndex(E, off)
        for B in (256, 384):
            Q = make_queries(E, B, seed=B)
            ids, sims, counts = rl.vector_search_batch(Q, num_results=3, config=rl.RAGLiteConfig(reranker=None), index=idx, algo=algo)
            for b in (0, 127, 128, B - 1):
                check_sql_semantics(E, off, Q[b], ids[b, :counts[b]], sims[b, :counts[b]], k=3)
