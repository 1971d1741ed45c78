"""BM25 keyword search throughput (``keyword_search_batch``: ``rl_bm25_topk_global`` over the device postings) on one GPU,
next to the NumPy port of DuckDB's FTS tables and ``match_bm25`` (tests/keyword_oracle.py) on the host cores.

Corpus: seeded, ``--chunks`` bodies (default 1.25 M, the chunk count of the headline shard) of 0-600 words drawn from a
Zipf distribution over a generated vocabulary.  Queries: ``--batch`` queries of 3-12 words from the same distribution,
top ``--k`` (256 x top-64: what ``hybrid_search`` asks for under ``search_and_rerank_chunks``' defaults, 2 x 4 x 8).
Prints one JSON line: index build time (device analysis and its split into host encoding, device work and the dictionary
round trip / device postings / statistics), the host analyzer (``Analyzer.analyze``) timed on the same bodies and
``analysis_match`` (the device-built dictionary and postings identical to the host analysis), queries/s end to end, CUDA-event
time of the top-k launch, per-kernel device times (torch.profiler), algorithmic bytes over kernel time against the
H100's 3.35 TB/s, the port's queries/s for ``--oracle-queries`` queries, and how many of those the device matched.
At the default size the host stages dominate the run (generating 375 M words, analysing them for the index and again for
the port): about ten minutes on a 16-thread host; ``--chunks 250000`` takes about three.
``--shards 1`` adds the sharded path on one GPU: ``ShardedIndex(group=None)`` over the same index against the bare index
(per-batch medians, alternating), and ``rl_bm25_merge_packed`` alone on synthetic full lists at R = 2, 8 and k = 64, 4096
(B = 256).
``--dialect postgresql`` measures the PostgreSQL branch instead (``ts_rank``, ``rl_tsrank_topk_global``): the same corpus
and queries, each body's ``to_tsvector('simple', body)::text`` synthesised on the host (the ``simple`` configuration keeps
every word, lower-cased, with its positions: the bodies here are lower-case words separated by spaces), the index built
from that text with ``add_tsvector_rows``, then the batch end to end, the kernels, and the NumPy port of ``calc_rank_or``
(tests/tsrank_oracle.py) on ``--oracle-queries`` queries, checked bit for bit."""
import argparse, json, operator, subprocess, sys, time
from pathlib import Path
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
import numpy as np, torch

HBM_TBPS = 3.35   # H100 SXM data sheet

ap = argparse.ArgumentParser()
ap.add_argument("--chunks", type=int, default=1_250_000)
ap.add_argument("--vocab", type=int, default=100_000)
ap.add_argument("--max-words", type=int, default=600)
ap.add_argument("--batch", type=int, default=256)
ap.add_argument("--k", type=int, default=64)
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--oracle-queries", type=int, default=16)
ap.add_argument("--seed", type=int, default=0)
ap.add_argument("--shards", type=int, default=0,
                help="1: also time the sharded path (ShardedIndex(group=None)) against the bare index, alternating, "
                     "and the merge alone at R = 2, 8 and k = 64, 4096")
ap.add_argument("--accents", type=float, default=0.0,
                help="a seeded fraction of the vocabulary words get one accented vowel and capitals, so that the "
                     "analyzers' non-ASCII paths are measured too")
ap.add_argument("--dialect", choices=["duckdb", "postgresql"], default="duckdb",
                help="postgresql: ts_rank over synthesised tsvectors instead of BM25")
args = ap.parse_args()
if args.shards not in (0, 1):
    sys.exit("--shards: only 1 (one GPU) is implemented; a multi-GPU run under torchrun is not")
T0 = time.perf_counter()


def stage(name):   # progress on stderr, so that a slow stage shows itself
    print(f"[{time.perf_counter() - T0:7.1f}s] {name}", file=sys.stderr, flush=True)

import keyword_oracle as ko
import raglite_b200 as rl
from raglite_b200._fts import Analyzer
from synth import make_corpus

rng = np.random.default_rng(args.seed)
vocab = ko.make_vocab(args.vocab, args.seed + 1)
if args.accents > 0:   # one vowel accented, the word capitalised or upper-cased
    acc_rng = np.random.default_rng(args.seed + 2)
    accented = dict(zip("aeiou", "áéíóú"))
    for i in np.flatnonzero(acc_rng.random(len(vocab)) < args.accents):
        w = vocab[i]
        at = [j for j, ch in enumerate(w) if ch in accented]
        if at:
            j = at[int(acc_rng.integers(0, len(at)))]
            w = w[:j] + accented[w[j]] + w[j + 1:]
        vocab[i] = w.upper() if acc_rng.random() < 0.5 else w.capitalize()
p = 1.0 / np.arange(1, len(vocab) + 1) ** 1.07
p /= p.sum()
words_sp = [w + " " for w in vocab]
lens = rng.integers(0, args.max_words + 1, size=args.chunks)
bodies: list[str] = []
t0 = time.perf_counter()
step = 50_000
for c0 in range(0, args.chunks, step):
    ln = lens[c0:c0 + step]
    ids = rng.choice(len(vocab), size=int(ln.sum()), p=p)
    cuts = np.concatenate([[0], np.cumsum(ln)])
    for a, b in zip(cuts[:-1], cuts[1:]):
        bodies.append("" if a == b else "".join(operator.itemgetter(*ids[a:b])(words_sp)) if b - a > 1 else words_sp[ids[a]])
gen_s = time.perf_counter() - t0
stage("corpus generated")
queries = [" ".join(vocab[i] for i in rng.choice(len(vocab), size=int(rng.integers(3, 13)), p=p)) for _ in range(args.batch)]


def card_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30, check=False).stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name()


def postgresql_bench():
    import tsrank_oracle as to
    from raglite_b200 import _lib

    t0 = time.perf_counter()
    rows = []
    for c, body in enumerate(bodies):
        held: dict[str, list[int]] = {}
        for i, w in enumerate(body.split(), 1):
            held.setdefault(w, []).append(min(i, 16383))
        rows.append((str(c), " ".join(f"'{w}':" + ",".join(map(str, ps[:256])) for w, ps in sorted(held.items()))))
    tsv_s = time.perf_counter() - t0
    stage("tsvector text synthesised")
    E, off = make_corpus(args.chunks, 1, 16, seed=args.seed)
    idx = rl.CorpusIndex(E, off, chunk_ids=[str(c) for c in range(args.chunks)])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    idx.add_tsvector_rows(rows)
    build_s = time.perf_counter() - t0
    ts = idx._tsrank
    stage("ts_rank index built")
    cfg = rl.RAGLiteConfig(db_url="postgresql://bench/raglite")
    for _ in range(2):
        rl.keyword_search_batch(queries, num_results=args.k, config=cfg, index=idx)
    wall = []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        ids_, scores_, counts_ = rl.keyword_search_batch(queries, num_results=args.k, config=cfg, index=idx)
        wall.append(time.perf_counter() - t0)
    stage("end-to-end timed")
    from raglite_b200._keyword import tsrank_plan

    B, C, k = len(queries), args.chunks, args.k
    q_off, q_terms = tsrank_plan(queries, ts.lexeme_ids)
    qd = torch.from_numpy(np.concatenate([q_off, q_terms])).cuda()
    group = max(1, min(B, (1 << 30) // (8 * C)))
    need = int(ts.lib.rl_bm25_workspace_bytes(C, group))
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    packed = torch.empty(int(ts.lib.rl_bm25_packed_bytes(B, k)), dtype=torch.uint8, device="cuda")

    def launch():
        _lib.check(ts.lib.rl_tsrank_topk_global(ts.term_off.data_ptr(), ts.doc.data_ptr(), ts.npos.data_ptr(), ts.n_terms, C,
                                                None, qd.data_ptr(), qd.data_ptr() + 4 * (B + 1), B, k, 0, packed.data_ptr(),
                                                ws.data_ptr(), need, torch.cuda.current_stream().cuda_stream),
                   "rl_tsrank_topk_global")

    launch()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(args.reps):
        launch()
    ev[1].record()
    torch.cuda.synchronize()
    kernel_ms = ev[0].elapsed_time(ev[1]) / args.reps
    per_kernel = {}
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        launch()
        torch.cuda.synchronize()
    for e in prof.key_averages():
        if "tsrank_score" in e.key or "bm25_select" in e.key:
            name = "score" if "score" in e.key else "select"
            per_kernel[name] = per_kernel.get(name, 0.0) + getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3
    stage("kernels timed")
    df = np.diff(ts.term_off.cpu().numpy())
    postings = int(sum(int(df[t]) for t in q_terms if t >= 0))
    alg_bytes = postings * 8 + B * C * 8 * 2   # postings (doc, npos) + dense keys written and read once
    # the NumPy port on the host cores over the same CSR: calc_rank_or per query, then the (score desc, chunk asc) top k
    nq = min(args.oracle_queries, B)
    csr = (ts.term_off.cpu().numpy(), ts.doc.cpu().numpy(), ts.npos.cpu().numpy())
    t0 = time.perf_counter()
    scores, matched = to.tsrank_csr_scores(*csr, q_off[: nq + 1], q_terms[: q_off[nq]], C)
    w_ids, w_sc, w_cnt = to.tsrank_topk(scores, matched, None, k)
    port_s = time.perf_counter() - t0
    ok = sum(int(np.array_equal(ids_[b], w_ids[b]) and np.array_equal(scores_[b].view(np.int64), w_sc[b].view(np.int64))
                 and counts_[b] == w_cnt[b]) for b in range(nq))
    print(json.dumps({
        "metric": f"ts_rank keyword_search queries/sec ({B} queries x top-{k}, {C} chunks)", "card": card_name(),
        "chunks": C, "tokens": int(lens.sum()), "lexemes": ts.n_terms, "postings": int(ts.doc.numel()),
        "corpus_gen_s": gen_s, "tsvector_text_s": tsv_s, "build_from_tsvector_text_s": build_s,
        "build_parse_s": ts.build_seconds["parse"], "build_device_postings_s": ts.build_seconds["postings"],
        "queries_per_s": B / float(np.median(wall)), "batch_wall_ms_median": 1e3 * float(np.median(wall)),
        "batch_wall_ms_min": 1e3 * float(np.min(wall)), "topk_kernel_ms": kernel_ms, "kernel_ms": per_kernel,
        "query_groups": -(-B // group), "algorithmic_gb": alg_bytes / 1e9,
        "algorithmic_tb_per_s": alg_bytes / (kernel_ms * 1e-3) / 1e12,
        "share_of_hbm": alg_bytes / (kernel_ms * 1e-3) / 1e12 / HBM_TBPS,
        "port_numpy_queries_per_s": nq / port_s, "port_queries": nq, "cpu_threads": torch.get_num_threads(),
        "oracle_match_bitwise": f"{ok}/{nq}",
    }))


if args.dialect == "postgresql":
    postgresql_bench()
    sys.exit(0)

E, off = make_corpus(args.chunks, 1, 16, seed=args.seed)
chunks = [rl.Chunk(id=str(c), body=b) for c, b in enumerate(bodies)]
idx = rl.CorpusIndex(E, off, chunk_ids=[c.id for c in chunks], chunks=chunks)
stage("corpus index built")
torch.cuda.synchronize()
t0 = time.perf_counter()
kw = idx.keyword_index()
build_s = time.perf_counter() - t0
t0 = time.perf_counter()
kw.refresh(idx._chunk_alive)
stats_s = time.perf_counter() - t0

stage("keyword index built")
for _ in range(2):
    rl.keyword_search_batch(queries, num_results=args.k, index=idx)
wall = []
for _ in range(args.reps):
    t0 = time.perf_counter()
    ids_, scores_, counts_ = rl.keyword_search_batch(queries, num_results=args.k, index=idx)
    wall.append(time.perf_counter() - t0)

stage("end-to-end timed")
# device time of the top-k launch alone: the plan and its statistics built as KeywordIndex.topk_to_host builds them for
# a CorpusIndex and uploaded once, CUDA events around rl_bm25_topk_global
from raglite_b200 import _lib
from raglite_b200._keyword import B_PARAM, K1

B, C, k = len(queries), kw.n_chunks, args.k
qids = [kw.analyzer.query_ids(q) for q in queries]
q_off = np.concatenate([[0], np.cumsum([len(x) for x in qids])]).astype(np.int32)
ids = np.concatenate(qids).astype(np.int32)
stats_d = torch.from_numpy(np.concatenate([[kw.n_live, kw.sum_len], kw.df_host[ids]]).astype(np.int64)).cuda()
qd = torch.from_numpy(np.concatenate([q_off, ids])).cuda()
group = max(1, min(B, (1 << 30) // (8 * C)))
need = int(kw.lib.rl_bm25_workspace_bytes(C, group))
ws = torch.empty(need, dtype=torch.uint8, device="cuda")
packed = torch.empty(int(kw.lib.rl_bm25_packed_bytes(B, k)), dtype=torch.uint8, device="cuda")


def launch():
    _lib.check(kw.lib.rl_bm25_topk_global(kw.term_off.data_ptr(), kw.doc.data_ptr(), kw.tf.data_ptr(), kw.doc_len.data_ptr(),
                                          stats_d.data_ptr(), kw.n_terms, C, None, qd.data_ptr(), qd.data_ptr() + 4 * (B + 1),
                                          B, k, K1, B_PARAM, 0, packed.data_ptr(), ws.data_ptr(), need,
                                          torch.cuda.current_stream().cuda_stream), "rl_bm25_topk_global")


launch()
ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
ev[0].record()
for _ in range(args.reps):
    launch()
ev[1].record()
torch.cuda.synchronize()
kernel_ms = ev[0].elapsed_time(ev[1]) / args.reps
per_kernel = {}
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    launch()
    torch.cuda.synchronize()
for e in prof.key_averages():
    if "bm25" in e.key:
        name = "score" if "score" in e.key else "select" if "select" in e.key else e.key
        per_kernel[name] = per_kernel.get(name, 0.0) + getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3
stage("kernels timed")
df_post = np.diff(kw.term_off.cpu().numpy())
postings = int(sum(int(df_post[x].sum()) for x in qids))
alg_bytes = postings * 12 + B * C * 8 * 2 + B * C   # postings (doc, tf, doc_len) + dense keys written and read once + mask

# the NumPy port on the host cores: FTS tables from an independent analysis pass, then match_bm25 per query
t0 = time.perf_counter()
an = Analyzer()
terms, owners, dlen = an.analyze(bodies)
host_analysis_s = time.perf_counter() - t0
pairs, pair_tf = np.unique((terms.astype(np.int64) << 32) | owners, return_counts=True)
ix = ko.FTSIndex(an.term_ids, dlen.astype(np.int64), np.ones(C, bool), owners.astype(np.int64), terms.astype(np.int64),
                 float(C), float(dlen.sum()) / C, np.bincount(pairs >> 32, minlength=len(an.term_ids)).astype(np.int64))
oracle_build_s = time.perf_counter() - t0
# the device analysis against the host's: the dictionary, ids included, and the postings it produced
analysis_match = bool(
    list(kw.analyzer.term_ids.items()) == list(an.term_ids.items())
    and np.array_equal(kw.term_off.cpu().numpy(), np.searchsorted(pairs >> 32, np.arange(len(an.term_ids) + 1)))
    and np.array_equal(kw.doc.cpu().numpy(), (pairs & 0xFFFFFFFF).astype(np.int32))
    and np.array_equal(kw.tf.cpu().numpy(), pair_tf) and np.array_equal(kw.doc_len.cpu().numpy(), dlen))
stage("port tables built")
nq = min(args.oracle_queries, B)
t0 = time.perf_counter()
want = [ko.keyword_search(ix, q, num_results=k, term_order=kw.analyzer.term_ids) for q in queries[:nq]]
oracle_s = time.perf_counter() - t0
stage("port queries done")
ok = 0
for b in range(nq):
    n = int(counts_[b])
    w_ids, w_sc = want[b]
    ok += int(n == len(w_ids) and np.allclose(scores_[b, :n], w_sc, rtol=1e-12, atol=0) and list(ids_[b, :n]) == w_ids)
sharded = {}
if args.shards == 1:
    from raglite_b200._dist import ShardedIndex

    sh = ShardedIndex(idx)
    s_ids, s_sc, s_cnt = rl.keyword_search_batch(queries, num_results=k, index=sh)
    sharded["sharded_same_counts"] = bool(np.array_equal(s_cnt, counts_))
    n_ok = [np.allclose(s_sc[b, :counts_[b]], scores_[b, :counts_[b]], rtol=1e-12, atol=0) for b in range(B)]
    sharded["sharded_scores_within_1e-12"] = f"{sum(n_ok)}/{B}"
    t_bare, t_sh = [], []
    for _ in range(args.reps):   # alternate the two paths so that drift on a shared host hits both alike
        t0 = time.perf_counter()
        rl.keyword_search_batch(queries, num_results=k, index=idx)
        t_bare.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        rl.keyword_search_batch(queries, num_results=k, index=sh)
        t_sh.append(time.perf_counter() - t0)
    sharded["bare_batch_ms_median"] = 1e3 * float(np.median(t_bare))
    sharded["sharded_r1_batch_ms_median"] = 1e3 * float(np.median(t_sh))
    st = torch.cuda.current_stream().cuda_stream

    def merge(src, R, Bm, km, dst):
        _lib.check(kw.lib.rl_bm25_merge_packed(src.data_ptr(), R, Bm, km, dst.data_ptr(), dst.data_ptr() + Bm * km * 8,
                                               dst.data_ptr() + Bm * km * 16, st), "rl_bm25_merge_packed")

    def event_ms(fn):
        fn()
        e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        e[0].record()
        for _ in range(args.reps):
            fn()
        e[1].record()
        torch.cuda.synchronize()
        return e[0].elapsed_time(e[1]) / args.reps

    # the merge alone on synthetic full lists: R shards x B queries x k entries, sorted, unique global chunks
    for R in (2, 8):
        for km in (64, 4096):
            Bm = 256
            g = torch.empty(R * int(kw.lib.rl_bm25_packed_bytes(Bm, km)), dtype=torch.uint8, device="cuda")
            per = g.view(R, -1)
            for r in range(R):
                sc = torch.sort(torch.rand(Bm, km, dtype=torch.float64, device="cuda") * 20, dim=1, descending=True).values
                ch = (r << 40) + torch.arange(km, dtype=torch.int64, device="cuda").expand(Bm, km)
                per[r, : Bm * km * 8].copy_(ch.contiguous().view(torch.uint8).reshape(-1))
                per[r, Bm * km * 8: Bm * km * 16].copy_(sc.contiguous().view(torch.uint8).reshape(-1))
                per[r, Bm * km * 16: Bm * km * 16 + Bm * 4].copy_(
                    torch.full((Bm,), km, dtype=torch.int32, device="cuda").view(torch.uint8))
            dst = torch.empty(int(kw.lib.rl_bm25_packed_bytes(Bm, km)), dtype=torch.uint8, device="cuda")
            sharded[f"merge_r{R}_k{km}_b{Bm}_ms"] = event_ms(lambda g=g, R=R, Bm=Bm, km=km, dst=dst: merge(g, R, Bm, km, dst))
    stage("sharded path timed")
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True, timeout=30, check=False).stdout.strip().splitlines()[0]
except Exception:  # noqa: BLE001
    card = torch.cuda.get_device_name()
print(json.dumps({
    "metric": f"BM25 keyword_search queries/sec ({B} queries x top-{k}, {C} chunks)", "card": card,
    "chunks": C, "tokens": int(lens.sum()), "terms": kw.n_terms, "postings": int(kw.doc.numel()), "corpus_gen_s": gen_s,
    "build_s": build_s, "build_device_analysis_s": kw.build_seconds["analysis"],
    "build_device_analysis_split_s": kw.analysis_seconds, "host_analysis_s": host_analysis_s,
    "analysis_speedup": host_analysis_s / kw.build_seconds["analysis"], "analysis_match": analysis_match,
    "build_device_postings_s": kw.build_seconds["postings"], "accents": args.accents,
    "stats_s": stats_s, "queries_per_s": B / float(np.median(wall)), "batch_wall_ms_median": 1e3 * float(np.median(wall)),
    "topk_kernel_ms": kernel_ms, "kernel_ms": per_kernel, "query_groups": -(-B // group),
    "algorithmic_gb": alg_bytes / 1e9, "algorithmic_tb_per_s": alg_bytes / (kernel_ms * 1e-3) / 1e12,
    "share_of_hbm": alg_bytes / (kernel_ms * 1e-3) / 1e12 / HBM_TBPS,
    "port_numpy_queries_per_s": nq / oracle_s, "port_build_s": oracle_build_s, "port_queries": nq,
    "cpu_threads": torch.get_num_threads(), "oracle_match": f"{ok}/{nq}", **sharded,
}))
