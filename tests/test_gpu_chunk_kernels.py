"""The chunk kernels at the C-ABI: ``rl_chunklet_partition`` and ``rl_chunk_partition`` bit for bit against the
restated loops of ``chunks_oracle`` (one launch of thousands of documents, each with its own max_size, dyadic costs
that tie everywhere, infinite windows, windows wider than 32 and 512 items, documents past the grid stride; seeded
non-dyadic costs; statement counts of 0; length prefixes past 2^31), and
``rl_chunk_similarities`` within ``chunks_oracle.chunk_cost_bound`` of float64.  Sentinels guard every output slice.
The largest similarity error as a fraction of the bound goes to ``chunk_errors.jsonl`` in the temporary directory."""

from __future__ import annotations

import json
import tempfile
from pathlib import Path

import chunks_oracle as co
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
SENT = -7


def _lib():
    from raglite_b200 import _lib

    return _lib.load()


def _dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _stream():
    import torch

    return torch.cuda.current_stream().cuda_stream


def _docs(rng, D: int):
    """Per document: lengths, max_size.  Mixed shapes: short documents, wide windows (> 32, > 512 items), sentences
    longer than max_size (infinite windows), one-item documents."""
    docs = []
    for k in range(D):
        kind = k % 10
        if k % 100 == 0:
            n, lens, mx = 700, rng.integers(1, 4, size=700), 2000          # windows of 500-2000 items
        elif kind in (0, 1):
            n = int(rng.integers(40, 120))
            lens, mx = rng.integers(1, 5, size=n), 120                      # windows of 30-120 items
        elif kind == 2:
            n = int(rng.integers(5, 30))
            lens = rng.integers(1, 30, size=n)
            lens[rng.integers(0, n, size=2)] = 200                          # longer than max_size
            mx = 64
        elif kind == 3:
            n, lens, mx = 1, rng.integers(1, 10, size=1), 5
        else:
            n = int(rng.integers(2, 40))
            lens, mx = rng.integers(1, 60, size=n), int(rng.integers(40, 400))
        docs.append((lens.astype(np.int32), int(mx)))
    return docs


def _run_partition(kind: str, docs, values):
    import torch

    lib = _lib()
    D = len(docs)
    off = np.zeros(D + 1, np.int64)
    np.cumsum([len(x) for x, _ in docs], out=off[1:])
    N = int(off[-1])
    lens = np.concatenate([x for x, _ in docs])
    mx = np.array([m for _, m in docs], np.int32)
    cuts = torch.full((N + 64,), SENT, dtype=torch.int32, device="cuda")
    cs = torch.full((2 * D + 64,), SENT, dtype=torch.int32, device="cuda")
    counts, status = cs[:D], cs[D + 32:2 * D + 32]
    ws = torch.empty(int(lib.rl_chunk_partition_workspace_bytes(N, D)), dtype=torch.uint8, device="cuda")
    a = [_dev(v) for v in values]
    d_len, d_off, d_mx = _dev(lens), _dev(off), _dev(mx)
    if kind == "chunklet":
        rc = lib.rl_chunklet_partition(a[0].data_ptr(), a[1].data_ptr(), d_len.data_ptr(), d_off.data_ptr(),
                                       d_mx.data_ptr(), D, N, cuts.data_ptr(), counts.data_ptr(), status.data_ptr(),
                                       ws.data_ptr(), ws.numel(), _stream())
    else:
        rc = lib.rl_chunk_partition(a[0].data_ptr(), d_len.data_ptr(), d_off.data_ptr(), d_mx.data_ptr(), D, N,
                                    cuts.data_ptr(), counts.data_ptr(), status.data_ptr(), ws.data_ptr(), ws.numel(),
                                    _stream())
    assert rc == 0
    h, c = cuts.cpu().numpy(), cs.cpu().numpy()
    assert (h[N:] == SENT).all() and (c[D:D + 32] == SENT).all() and (c[2 * D + 32:] == SENT).all()
    return off, h, c[:D], c[D + 32:2 * D + 32]


def test_chunklet_partition_bit_for_bit():
    rng = np.random.default_rng(1)
    docs = _docs(rng, 9000)                               # 9000 warps: past the 8192-document grid stride
    # dyadic inputs: every cost is exact and ties are everywhere
    p = [rng.choice([0.0, 0.25, 0.5, 0.75, 1.0], size=len(x)) for x, _ in docs]
    st = [rng.choice([0.25, 0.5, 0.75, 1.0, 1.5], size=len(x)) for x, _ in docs]
    off, h, counts, status = _run_partition("chunklet", docs, [np.concatenate(p), np.concatenate(st)])
    assert (status == 0).all()
    for i, (lens, mx) in enumerate(docs):
        want = co.chunklet_cuts(p[i], st[i], lens, mx)
        n = len(lens)
        got = h[off[i]:off[i] + counts[i]].tolist()
        assert got == want, i
        assert (h[off[i] + counts[i]:off[i] + n] == SENT).all(), i
    # seeded non-dyadic values through the same launch shape
    p2 = [rng.random(len(x)) for x, _ in docs[:600]]
    st2 = [rng.random(len(x)) * 2 for x, _ in docs[:600]]
    off, h, counts, _ = _run_partition("chunklet", docs[:600], [np.concatenate(p2), np.concatenate(st2)])
    for i, (lens, mx) in enumerate(docs[:600]):
        assert h[off[i]:off[i] + counts[i]].tolist() == co.chunklet_cuts(p2[i], st2[i], lens, mx), i


def test_chunklet_partition_empty_document_status():
    docs = [(np.array([3, 4], np.int32), 5), (np.zeros(0, np.int32), 5), (np.array([9], np.int32), 5)]
    _, _, counts, status = _run_partition("chunklet", docs, [np.full(3, 0.5), np.full(3, 1.0)])
    assert status.tolist() == [0, 1, 0] and counts.tolist() == [1, 0, 0]


def test_chunk_partition_bit_for_bit():
    rng = np.random.default_rng(2)
    docs = _docs(rng, 9000)
    costs = [rng.choice(np.float32([0.25, 0.5, 0.75, 1.0]), size=len(x)) for x, _ in docs]
    costs = [np.where(np.arange(len(c)) == len(c) - 1, np.float32(np.nan), c).astype(np.float32) for c in costs]
    off, h, counts, status = _run_partition("chunk", docs, [np.concatenate(costs)])
    for i, (lens, mx) in enumerate(docs):
        if (lens > mx).any():
            assert status[i] == 1 and counts[i] == 0, i
            continue
        assert status[i] == 0, i
        assert h[off[i]:off[i] + counts[i]].tolist() == co.chunk_cuts(costs[i][:-1], lens, mx), i
        assert (h[off[i] + counts[i]:off[i] + len(lens)] == SENT).all(), i
    assert (status == 1).sum() > 100


def _record(payload: dict) -> None:
    with (Path(tempfile.gettempdir()) / "chunk_errors.jsonl").open("a") as f:
        f.write(json.dumps(payload) + "\n")


@pytest.mark.parametrize(("dtype", "dim"), [(np.float16, 64), (np.float16, 1024), (np.float32, 384), (np.float32, 8192)])
def test_chunk_similarities_within_bound(dtype, dim):
    import torch

    lib = _lib()
    rng = np.random.default_rng(dim)
    D = 300 if dim < 8192 else 60
    docs = []
    for k in range(D):
        n = int(rng.integers(1, 60)) if k % 7 else 3
        centers = rng.standard_normal((3, dim))
        X = centers[rng.integers(0, 3, size=n)] + rng.standard_normal((n, dim))
        if k % 50 == 5:
            X[:] = X[0]                                   # identical rows: every projection is zero, skipped
        sizes = rng.integers(10, 400, size=n)
        head = rng.random(n) < 0.2
        if k % 50 == 7:
            sizes[:] = 1000                                   # q15 == q85: every row selected
        docs.append((X.astype(dtype), sizes, head))
    zero_doc = 11
    docs[zero_doc][0][min(1, len(docs[zero_doc][0]) - 1)] = 0
    off = np.zeros(D + 1, np.int64)
    np.cumsum([len(x) for x, _, _ in docs], out=off[1:])
    N = int(off[-1])
    ld = dim + 8                                          # a row stride wider than the row
    Xa = np.zeros((N, ld), dtype)
    Xa[:, :dim] = np.concatenate([x for x, _, _ in docs])
    non = np.concatenate([co.nonoutlying(s) for _, s, _ in docs])
    head = np.concatenate([h for _, _, h in docs])
    costs = torch.full((N + 64,), float("nan"), dtype=torch.float32, device="cuda")
    status = torch.full((D + 32,), SENT, dtype=torch.int32, device="cuda")
    ws = torch.empty(int(lib.rl_chunk_similarities_workspace_bytes(N)), dtype=torch.uint8, device="cuda")
    d_x, d_off, d_non, d_head = _dev(Xa), _dev(off), _dev(non.view(np.uint8)), _dev(head.view(np.uint8))
    assert lib.rl_chunk_similarities(d_x.data_ptr(), 1 if dtype == np.float16 else 0, ld, dim, d_off.data_ptr(), D, N,
                                     d_non.data_ptr(), d_head.data_ptr(), costs.data_ptr(), status.data_ptr(),
                                     ws.data_ptr(), ws.numel(), _stream()) == 0
    got, st = costs.cpu().numpy(), status.cpu().numpy()
    assert np.isnan(got[N:]).all() and (st[D:] == SENT).all()
    worst, zero_proj = 0.0, 0
    for i, (X, sizes, h) in enumerate(docs):
        g = got[off[i]:off[i + 1]]
        assert np.isnan(g[-1]), i                          # the last row's slot is not written
        if i == zero_doc:
            assert st[i] == 1 and np.isnan(g).all()
            continue
        assert st[i] == 0, i
        keep = co.nonoutlying(sizes)
        want, info = co.chunk_costs_f64(X, keep, h)
        if keep.any():
            # away from the projection test's edge: either a row's exact projection is zero (identical rows, or the one
            # row a three-chunklet document selects; then it is skipped) or every projection is clearly above eps
            pmin = float(info["pn_all"].min())
            assert pmin < 1e-9 or pmin > 1e-4, (i, pmin)
            zero_proj += pmin < 1e-9
        bound = co.chunk_cost_bound(dim, int(keep.sum()), info)
        err = np.abs(g[:-1].astype(np.float64) - want)
        assert (err <= bound).all(), (i, float((err / bound).max()))
        if len(err):
            worst = max(worst, float((err / bound).max()))
    assert zero_proj >= 2
    _record({"dtype": np.dtype(dtype).name, "dim": dim, "docs": D, "zero_projection_docs": zero_proj,
             "max_err_over_bound": worst})


@pytest.mark.parametrize("dtype", [np.float16, np.float32])
def test_chunk_similarities_skip_exact_zero_projection(dtype):
    """Identical rows whose every step is exact (a basis vector): the mean is the row, every projection is exactly 0,
    so the projection is skipped in any arithmetic and every cost is (1 + 1) / 2 = 1 (then the heading rule); a second
    document of distinct rows, in the same launch, keeps its projection."""
    import torch

    lib = _lib()
    dim = 32
    same = np.zeros((6, dim), dtype)
    same[:, 3] = 2
    rng = np.random.default_rng(9)
    other = rng.standard_normal((5, dim)).astype(dtype)
    X = np.concatenate([same, other])
    off = np.array([0, 6, 11], np.int64)
    non = np.ones(11, np.uint8)
    head = np.zeros(11, np.uint8)
    head[2] = 1
    costs = torch.full((16,), float("nan"), dtype=torch.float32, device="cuda")
    status = torch.full((2,), SENT, dtype=torch.int32, device="cuda")
    ws = torch.empty(int(lib.rl_chunk_similarities_workspace_bytes(11)), dtype=torch.uint8, device="cuda")
    d_x, d_off, d_non, d_head = _dev(X), _dev(off), _dev(non), _dev(head)
    assert lib.rl_chunk_similarities(d_x.data_ptr(), 1 if dtype == np.float16 else 0, dim, dim, d_off.data_ptr(), 2, 11,
                                     d_non.data_ptr(), d_head.data_ptr(), costs.data_ptr(), status.data_ptr(),
                                     ws.data_ptr(), ws.numel(), _stream()) == 0
    got = costs.cpu().numpy()
    assert status.cpu().tolist() == [0, 0]
    assert got[:5].tolist() == [1.0, 0.25, 1.0, 1.0, 1.0]        # the cut before the heading divided by 4
    want, info = co.chunk_costs_f64(other, np.ones(5, bool), np.zeros(5, bool))
    assert info["proj"] and (np.abs(got[6:10] - want) <= co.chunk_cost_bound(dim, 5, info)).all()


def test_chunk_partition_non_dyadic_costs():
    """Seeded float32 costs that round in the sums: random values, sqrt(eps), 1.0, the quarters the heading rule makes
    and values repeated across different cuts of a document, in one launch of 9000 documents."""
    rng = np.random.default_rng(3)
    docs = _docs(rng, 9000)
    special = np.float32([co.SQRT_EPS32, co.SQRT_EPS32 / 4, 1.0, 0.25])
    costs = []
    for lens, _ in docs:
        c = rng.random(len(lens)).astype(np.float32) * np.float32(0.999) + co.SQRT_EPS32
        c = np.where(rng.random(len(c)) < 0.2, c / np.float32(4), c)
        c = np.where(rng.random(len(c)) < 0.15, rng.choice(special, size=len(c)), c)
        c = np.where(rng.random(len(c)) < 0.2, c[0], c)                  # equal costs at different j
        c[-1] = np.nan
        costs.append(c.astype(np.float32))
    off, h, counts, status = _run_partition("chunk", docs, [np.concatenate(costs)])
    nontrivial = 0
    for i, (lens, mx) in enumerate(docs):
        if (lens > mx).any():
            assert status[i] == 1 and counts[i] == 0, i
            continue
        assert status[i] == 0, i
        want = co.chunk_cuts(costs[i][:-1], lens, mx)
        assert h[off[i]:off[i] + counts[i]].tolist() == want, i
        assert (h[off[i] + counts[i]:off[i] + len(lens)] == SENT).all(), i
        nontrivial += len(want) > 1
    assert nontrivial > 1000


def test_chunklet_partition_zero_statements():
    """Statement counts of 0 in every document, so a window of no statements takes sqrt(max(s, 1e-6)); non-dyadic
    probabilities."""
    rng = np.random.default_rng(4)
    docs = _docs(rng, 2000)
    p = [rng.random(len(x)) for x, _ in docs]
    st = [np.where(rng.random(len(x)) < 0.5, 0.0, rng.choice([0.5, 1.0, 2.0, 3.0], size=len(x))) for x, _ in docs]
    off, h, counts, status = _run_partition("chunklet", docs, [np.concatenate(p), np.concatenate(st)])
    assert (status == 0).all()
    empty_windows = 0
    for i, (lens, mx) in enumerate(docs):
        want = co.chunklet_cuts(p[i], st[i], lens, mx)
        assert h[off[i]:off[i] + counts[i]].tolist() == want, i
        edges = [0, *want, len(lens)]
        empty_windows += sum(st[i][a:b].sum() == 0 for a, b in zip(edges[:-1], edges[1:]))
    assert empty_windows > 100                              # chunklets without statements are chosen, not only tried


def test_partitions_past_2_31_characters():
    """Documents of lengths near 2^30 with max_size near 2^31 - 1: the length prefixes pass 2^31 (a 32-bit prefix
    wraps), and a window holds one to three items."""
    rng = np.random.default_rng(5)
    docs = []
    for _ in range(64):
        n = int(rng.integers(6, 24))
        lens = rng.integers(2**28, 2**30 + 1, size=n).astype(np.int32)
        docs.append((lens, int(rng.integers(2**31 - 2**28, 2**31))))
    assert max(int(x.astype(np.int64).sum()) for x, _ in docs) > 2**33
    costs = [rng.random(len(x)).astype(np.float32) for x, _ in docs]
    off, h, counts, status = _run_partition("chunk", docs, [np.concatenate(costs)])
    p = [rng.random(len(x)) for x, _ in docs]
    st = [rng.choice([0.0, 1.0, 2.0, 4.0], size=len(x)) for x, _ in docs]
    off2, h2, counts2, status2 = _run_partition("chunklet", docs, [np.concatenate(p), np.concatenate(st)])
    assert (status == 0).all() and (status2 == 0).all()
    multi = 0
    for i, (lens, mx) in enumerate(docs):
        want = co.chunk_cuts(costs[i][:-1], lens, mx)
        assert h[off[i]:off[i] + counts[i]].tolist() == want, i
        assert h2[off2[i]:off2[i] + counts2[i]].tolist() == co.chunklet_cuts(p[i], st[i], lens, mx), i
        multi += len(want) < len(lens) - 1                  # some chunk holds more than one item
    assert multi > 10
