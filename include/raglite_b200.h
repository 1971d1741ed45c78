/* raglite_b200 -- C-ABI of the H100-native (sm_90a) RAGLite retrieval hot path.
 *
 * Every entry point takes plain device/host pointers, sizes and a CUDA stream handle
 * (`void* stream` == cudaStream_t); there are no torch / C++ types in any signature.
 * Return value: 0 on success, a negative RL_E* code on failure; rl_last_error() gives the
 * message of the last failure on the calling thread.  No entry point allocates device memory:
 * the caller passes a workspace sized by the matching *_workspace_bytes() query.  All calls are
 * asynchronous on `stream` and re-entrant (no global mutable state), so several host threads may
 * drive different streams concurrently (reference callers use thread pools: _rag.py:317,
 * _eval.py:178).
 *
 * The reference (superlinear-ai/raglite @ 2069f8d) is pure Python and has no FFI; each entry point
 * cites the Python code whose arithmetic it replaces.  INTEGRATION.md shows the ctypes binding a
 * RAGLite maintainer would add.
 */
#ifndef RAGLITE_B200_H_
#define RAGLITE_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RL_OK 0
#define RL_EINVAL (-1)    /* bad argument (null pointer, unsupported size/metric, misalignment) */
#define RL_ECUDA (-2)     /* a CUDA runtime call failed */
#define RL_ENOSPACE (-3)  /* workspace too small */
#define RL_EUNSUPPORTED (-4)

/* Distance metric: RAGLiteConfig.vector_search_distance_metric (_config.py:69), rendered per
 * dialect at _typing.py:110-134.  sim = 1 - dist (_search.py:72). */
#define RL_METRIC_COSINE 0 /* dist = 1 - <e,q>/sqrt(|e|^2 |q|^2)  (array_cosine_distance)        */
#define RL_METRIC_DOT 1    /* dist = -<e,q>                        (array_negative_inner_product) */
#define RL_METRIC_L2 2     /* dist = |e - q|_2                     (array_distance)               */
#define RL_METRIC_L1 3     /* dist = sum_i |e_i - q_i|             (PostgreSQL only: pgvector `<+>`, HNSW
                              index halfvec_l1_ops; _typing.py:110-120, _database.py:573-578).  Runs the
                              CUDA-core L1 scan under RL_ALGO_AUTO and RL_ALGO_FP32; RL_ALGO_TCGEN05 is refused. */

/* Scan kernel selection. */
#define RL_ALGO_AUTO 0
#define RL_ALGO_FP32 1    /* exact fp32 CUDA-core scan (any d) */
#define RL_ALGO_TCGEN05 2 /* fp16-input tensor-core (wgmma) coarse scan + exact rescoring (d % 4 == 0) */

/* rl_maxsim_topk flags. */
#define RL_FLAG_REUSE_THRESHOLDS 1u /* skip the sample pass; use thresholds left in the workspace */
#define RL_FLAG_TIME_KERNELS 2u     /* record CUDA events around each stage (see rl_maxsim_kernel_times) */
#define RL_FLAG_COUNT_UNFILTERED 4u /* also count, per query, the rows that pass the emission threshold but are masked
                                       out by row_allowed (and alive per row_alive): rl_maxsim_unfiltered_bound */

/* Per-query status bits written by rl_maxsim_topk. */
#define RL_STATUS_CAND_OVERFLOW 1 /* candidate list overflowed: call again with REUSE_THRESHOLDS */
#define RL_STATUS_TIE_OVERFLOW 2  /* reserved (never set since v101: more than RL_MAX_SURVIVORS rows inside the error
                                     band of the cut are rescored by a streaming pass over the candidate list) */
#define RL_STATUS_QUERY_NONFINITE 4 /* RL_METRIC_L1 only: the query has an infinite or NaN element (pgvector refuses
                                       such a halfvec); the hits of that query are meaningless */

#define RL_MAX_SURVIVORS 4096

int rl_version(void);
const char* rl_last_error(void);

/* Number of SMs etc. of the current device (diagnostics for bench.py). */
int rl_device_info(int* sm_count, int* cc_major, int* cc_minor, size_t* l2_bytes);

/* ---- Index build -------------------------------------------------------------------------
 * Per-row statistics of the embedding matrix E[n_rows, d] (row stride ld floats): inv_norm[j] =
 * 1/|e_j| (0 for a zero row), sq_norm[j] = |e_j|^2, and four global statistics used to scale rows for
 * the fp16 scan (stats[4], device floats, zeroed by the caller once -- the kernel folds maxima in, so
 * appended rows (insert_documents flushes, _insert.py:247-255) only need a call over the new rows): [0] max row norm, [1] max
 * |element|, [2] max 1/|e_j| over non-zero rows, [3] 1 if any row is all-zero.  Replaces nothing in the reference (DuckDB recomputes norms per query inside
 * array_cosine_distance); it is the device-side part of building the resident index from the
 * chunk_embedding table (_database.py:403-430). */
int rl_row_stats(const float* E, int64_t n_rows, int d, int64_t ld, float* inv_norm, float* sq_norm,
                 float* stats, void* stream);
/* Same for an embedding matrix stored as float16 (rl_scan_params.e_dtype == 1). */
int rl_row_stats_f16(const void* E, int64_t n_rows, int d, int64_t ld, float* inv_norm, float* sq_norm,
                     float* stats, void* stream);

/* row_chunk[j] = c for chunk_off[c] <= j < chunk_off[c+1]  (CSR -> per-row owner; the
 * chunk_embedding.chunk_id column, _database.py:421). */
int rl_chunk_row_map(const int64_t* chunk_off, int64_t n_chunks, int32_t* row_chunk, void* stream);

/* Per-row byte mask for rl_scan_params.row_allowed: out[j] = chunk_ok[row_chunk[j]] AND alive[j].
 * chunk_ok (uint8 [n_chunks], or NULL = every chunk) is the metadata filter resolved per chunk (the JSON
 * containment tests of _search.py:82-95), alive (uint8 [n_rows], or NULL) the tombstones of deleted
 * chunks (_delete.py:146-152).  row_chunk, alive and out must be 16-byte aligned. */
int rl_row_mask(const uint8_t* chunk_ok, const int32_t* row_chunk, const uint8_t* alive, int64_t n_rows,
                uint8_t* out, void* stream);

/* ---- Query adapter apply: _search.py:58-62 -------------------------------------------------
 * Q_out[b,:] = round_to(A @ Q_in[b,:]) with A[d,d] float64 row-major exactly as the reference
 * stores it (_query_adapter.py:211), accumulated in float64; round_mode 0 = keep float32,
 * 1 = round through float16 (the reference casts back to the query dtype, fp16 for string
 * queries, _embed.py:140). */
int rl_adapter_apply(const double* A, const float* Q_in, float* Q_out, int B, int d, int round_mode,
                     void* stream);

/* ---- MaxSim scan + top-k: _search.py:65-79, 143-153 -----------------------------------------
 * One shard of the corpus, a batch of B queries.
 *   E[n_rows,d] float32 row-major (ld = row stride in floats), inv_norm/sq_norm from
 *   rl_row_stats, row_chunk from rl_chunk_row_map, chunk_base = global index of this shard's
 *   first chunk, max_vecs_per_chunk = max CSR segment length, row_stats = stats from rl_row_stats.
 *   row_allowed: optional uint8[n_rows], or NULL: rows with a zero byte do not take part -- the metadata
 *     filter (_search.py:82-121) and the tombstones of deleted chunks (_delete.py:146-152), ANDed by the caller.
 *   Q[B,d] float32 (already adapter-applied).
 *   num_hits > 0: reference SQL semantics -- the num_hits vectors with smallest distance
 *     (_search.py:75-79); hits are those vectors, ascending distance.
 *   num_hits == 0: exact per-chunk MaxSim -- hits are the best k chunks.
 * Outputs (H = num_hits ? num_hits : k):
 *   hit_sim[B,H] float32 (sim = 1 - dist), hit_chunk[B,H] int64 global chunk index,
 *   hit_count[B] int32, status[B] int32 (RL_STATUS_* bits).
 * Feed the hit lists of all shards to rl_topk_merge for the GROUP BY / ORDER BY / LIMIT. */
typedef struct rl_scan_params {
  const float* E;
  const float* inv_norm;
  const float* sq_norm;
  const int32_t* row_chunk;
  const float* row_stats;
  const uint8_t* row_allowed;
  int64_t n_rows;
  int64_t ld;
  int64_t chunk_base;
  int32_t d;
  int32_t max_vecs_per_chunk;
  const float* Q;
  int32_t B;
  int32_t metric;
  int32_t k;
  int32_t num_hits;
  int32_t algo;
  uint32_t flags;
  int32_t sample_stride; /* 0 = auto */
  int32_t cand_cap;      /* 0 = auto */
  int32_t e_dtype;       /* storage of E: 0 = float32, 1 = float16 (E then points to IEEE binary16; needs
                            d % 8 == 0, ld % 8 == 0 and 16-byte aligned E, and then RL_ALGO_TCGEN05 with rows that
                            need no per-row scaling for cosine / dot / l2, the L1 scan for RL_METRIC_L1) */
  int32_t rows_unit_scale; /* 1: the caller guarantees (from the rl_row_stats statistics: max 1/|e| <= 2, max |e_ij| <= 1024,
                            no all-zero row -- true for normalised embeddings) that rows can enter the fp16 scan unscaled,
                            which lets the cosine scan use the two-tiles-per-query-slice kernel.  0: unknown (always valid) */
  const uint8_t* row_alive; /* optional uint8[n_rows] (NULL = all): rows that exist at all -- the tombstone mask without
                            the metadata filter (only read with RL_FLAG_COUNT_UNFILTERED) */
} rl_scan_params;

size_t rl_maxsim_workspace_bytes(const rl_scan_params* p);
int rl_maxsim_topk(const rl_scan_params* p, float* hit_sim, int64_t* hit_chunk, int32_t* hit_count,
                   int32_t* status, void* workspace, size_t workspace_bytes, void* stream);

/* Counters of the last rl_maxsim_topk call on this workspace (device->host copy, synchronises the
 * stream): kernel launches issued, and per-call totals of emitted candidates / survivors. */
typedef struct rl_scan_stats {
  int32_t launches;
  int32_t sample_stride;
  int32_t cand_cap;
  int32_t algo;
  int64_t n_sample_rows;
  int64_t cand_total;
  int64_t cand_max;
  int64_t survivors_total;
  int64_t survivors_max; /* largest per-query survivor count (> RL_MAX_SURVIVORS: that query took the streaming path) */
} rl_scan_stats;
int rl_maxsim_stats(const rl_scan_params* p, const void* workspace, rl_scan_stats* out, void* stream);

/* Fused bound for the rank-then-filter metadata branch (_search.py:122-143).  After an rl_maxsim_topk call made
 * with RL_FLAG_COUNT_UNFILTERED on a FILTERED scan (row_allowed set), bound[b] (device int64 [B]) is an UPPER bound
 * of the number of live rows of the shard -- filtered or not -- that are at least as near to query b as the worst
 * of its num_hits filtered hits: every emission threshold the scan ever used lies at or below that hit's key, so
 * the rows counted against the thresholds (allowed ones = the candidate count, masked ones = the extra counter)
 * plus the whole sample are a superset.  bound <= 1 000 000 proves that the filter-first answer is also the
 * rank-then-filter answer, without the second pass over the corpus rl_maxsim_count_at_least needs.  The
 * tensor-core scan and the L1 scan count; bound[b] is -1 when the last call did not count (fp32 scan of cosine / dot /
 * l2, flag not set).  An empty shard (p->n_rows == 0)
 * gets bound 0 without the workspace being read: rl_maxsim_topk writes nothing there for it. */
int rl_maxsim_unfiltered_bound(const rl_scan_params* p, const void* workspace, int64_t* bound, void* stream);

/* Rank probe for the reference's rank-then-filter metadata branch (_search.py:122-143, which keeps the
 * 1 000 000 nearest vectors before it applies the filter): counts[b] = number of rows of the shard
 * (p->row_allowed honoured, normally the tombstone mask only) whose similarity to query b is at least
 * sim_floor[b] (device float32 [B], in the units vector_search returns: 1 - dist).  The scan compares
 * approximate keys, so `bound` picks the side of the bracket: +1 counts every row whose exact
 * similarity can reach the floor (upper bound), -1 only rows that certainly do (lower bound), 0 the raw
 * key comparison.  One pass over the corpus, nothing stored; p is the same struct rl_maxsim_topk takes
 * and the workspace the same size.  counts is device int32 [B]. */
int rl_maxsim_count_at_least(const rl_scan_params* p, const float* sim_floor, int bound, int32_t* counts,
                             void* workspace, size_t workspace_bytes, void* stream);

/* Device time in ms of the stages of the rl_maxsim_topk calls made with RL_FLAG_TIME_KERNELS on this
 * workspace since the previous read (average over up to 32 calls): ms[0] = prep, ms[1] = sample scan (dump), ms[2] = select, ms[3] = main scan (emit),
 * ms[4] = finalize.  CUDA events are recorded on the launching stream; the call synchronises on the
 * last one.  Diagnostics for bench.py's roofline figure. */
int rl_maxsim_kernel_times(const void* workspace, float* ms);

/* Releases the timing events tied to a workspace pointer (created on the first RL_FLAG_TIME_KERNELS call);
 * call before freeing the workspace.  No-op for a workspace that was never timed. */
int rl_maxsim_release(const void* workspace);

/* Debug/test hook: copy the sampled approximate keys of the last call (float32 [B, n_sample_rows],
 * sample position p <-> row (p / 128) * sample_stride * 128 + p % 128) into dst (device memory);
 * *n_sample_rows receives the row count.  dst may be NULL to query the size only. */
int rl_maxsim_copy_dump(const rl_scan_params* p, const void* workspace, float* dst, int64_t* n_sample_rows,
                        void* stream);

/* Debug/test hook: copy the per-query error bound of the approximate key that the last call used
 * (float32 [B], key units: |approximate key - exact key| <= eps[b] for every row) into dst (device memory). */
int rl_maxsim_copy_eps(const rl_scan_params* p, const void* workspace, float* dst, void* stream);

/* Debug/test hook: copy the candidate list of the last call into device memory: key float32 [B, cap] and
 * row int32 [B, cap] (the first min(cand_cnt[b], cap) entries of query b are the emitted candidates, in no
 * particular order), cand_cnt int32 [B] (the number emitted, > cap on overflow), the emission threshold the
 * select kernel handed to the main scan (thr float32 [B]) and the reciprocal bin width of the online
 * refinement's histogram (hist_inv_w float32 [B]).  cap is the candidate capacity of the call
 * (rl_maxsim_stats).  Any output pointer may be NULL.  When more than RL_MAX_SURVIVORS rows of a query survive,
 * finalize rescores them in place: that query's keys then hold the order-preserving bits of exact similarities
 * (0 for rows outside the band), not the emitted keys. */
int rl_maxsim_copy_candidates(const rl_scan_params* p, const void* workspace, float* key, int32_t* row, int32_t* cand_cnt,
                              float* thr, float* hist_inv_w, void* stream);

/* ---- Shard merge + GROUP BY chunk + top-k: _search.py:143-150 --------------------------------
 * hit_*[R,B,H] are the per-shard outputs of rl_maxsim_topk (all-gathered).  num_hits > 0: keep
 * the num_hits best vectors overall, group by chunk (max sim), order desc, limit k.  num_hits == 0:
 * merge the per-shard chunk lists, limit k.  Outputs out_sim[B,k], out_chunk[B,k] (-1 padded),
 * out_count[B]. */
int rl_topk_merge(const float* hit_sim, const int64_t* hit_chunk, const int32_t* hit_count, int R,
                  int B, int H, int num_hits, int k, float* out_sim, int64_t* out_chunk,
                  int32_t* out_count, void* stream);

/* Packed per-shard hit list, the unit the single all-gather of the sharded path moves (NCCL over NVLink):
 *   chunk int64 [B, H] | sim float32 [B, H] | count int32 [B] | (status int32 [B])   -- padded to 16 bytes.
 * rl_maxsim_topk can write straight into such a buffer (its four output pointers are the four sections),
 * so nothing is re-packed before the collective, and rl_topk_merge_packed reads the R gathered buffers in
 * place (rank_stride_bytes apart), so nothing is unpacked after it. */
size_t rl_hits_packed_bytes(int B, int H, int with_status);
int rl_topk_merge_packed(const void* packed, int64_t rank_stride_bytes, int R, int B, int H, int num_hits, int k,
                         float* out_sim, int64_t* out_chunk, int32_t* out_count, void* stream);

/* ---- Query-adapter fit: _query_adapter.py:21-38, 172-183 ---------------------------------------------------
 * rl_best_vectors: for every eval e and retrieved chunk chunks[e, slot] (shard-local chunk index, -1 = unused), the
 * vector of that chunk with the largest inner product with the eval's query Q[e, :] -- argmax(embedding_matrix @ q),
 * first maximum on ties -- written to best[e, slot, :] (float32; zeros for unused slots) and its row to best_row.
 * E: the corpus (e_dtype 0 = float32, 1 = float16), chunk_off the CSR offsets (device int64 [n_chunks + 1]). */
int rl_best_vectors(const void* E, int e_dtype, int64_t ld, int d, const int64_t* chunk_off, const int64_t* chunks,
                    int n_evals, int n_slots, const float* Q, float* best, int64_t* best_row, void* stream);
/* rl_adapter_targets: _optimize_query_target for every eval at once.  kind[e, slot] = 1 for a relevant chunk's vector
 * (P), 0 for an irrelevant one (N), anything else = unused.  T[e, :] (float64) = q + D^T mu* with
 * D = {p_i - (1 + alpha) n_j} and mu* = argmin_{mu >= 0} |q + D^T mu|^2 (active-set NNLS in float64 on the Gram
 * form, see csrc/adapter_fit.cu); ok[e] = 0 when the eval has no relevant or no irrelevant chunk (T = q then, the
 * reference skips such evals), iters[e] = outer iterations.  n_slots <= 64, |P| |N| <= 1024. */
int rl_adapter_targets(const float* best, const uint8_t* kind, int n_evals, int n_slots, int d, const float* Q, double alpha,
                       double* T, int32_t* ok, int32_t* iters, void* stream);

/* ---- Fusion and span collation on device chunk indices: _search.py:233-280, 323-360 ------------------------
 * rl_rrf_fuse: Reciprocal Rank Fusion of R rankings per query.  ids[B, R, L] int64 chunk indices (-1 padded at
 * the tail of a ranking), weights[R] float64 (device), k the RRF constant (60 in the reference).
 * score(c) = sum_r weights[r] / (k + position of c in ranking r), float64 summed ranking by ranking exactly as the
 * reference's dict does; output ordered by descending score, ties in first-appearance order (ranking 0 first) --
 * Python's stable sort.  out_ids[B, K] (-1 padded), out_score[B, K] float64, out_count[B].  R * L <= 4096. */
int rl_rrf_fuse(const int64_t* ids, const double* weights, int B, int R, int L, double k, int K, int64_t* out_ids,
                double* out_score, int32_t* out_count, void* stream);

/* rl_span_collate: the ranking half of retrieve_chunk_spans (_search.py:323-360) for B lists of M retrieved chunk
 * indices (ranked[B, M], -1 padded).  Index tables (device): chunk_doc[c] = ordinal of the chunk's document in
 * ascending document_id order, chunk_pos[c] = Chunk.index, chunk_alive[c] (or NULL), and the lookup
 * (doc << 32 | pos) -> chunk as two arrays of n_chunks entries sorted by key (ranked indices outside [0, n_chunks) are
 * skipped, so the lookup covers every chunk; deleted ones are turned away through chunk_alive).  Every retrieved
 * chunk is joined by its neighbours at the given position offsets inside its document (neighbors[n_neighbors], e.g. {-1, +1}), duplicates are dropped,
 * members are ordered by (document, position) and cut into runs of consecutive positions; a run's score is the
 * sum of 1 / (rank + 1) over its retrieved members (float64, compensated as Python's sum() is since 3.12), runs
 * are ordered by descending score (stable).
 * Outputs, cap = M * (1 + n_neighbors) per query: out_member[B, cap] chunk indices in document order (-1 padded),
 * out_span_start / out_span_len[B, cap] (offsets into the member row, in final span order), out_span_score[B, cap],
 * out_n_span[B], out_n_member[B].  cap <= 4096. */
int rl_span_collate(const int64_t* ranked, int B, int M, const int32_t* chunk_doc, const int32_t* chunk_pos,
                    const uint8_t* chunk_alive, const uint64_t* sorted_key, const int64_t* sorted_chunk, int64_t n_chunks,
                    const int32_t* neighbors, int n_neighbors, int64_t* out_member, int32_t* out_span_start,
                    int32_t* out_span_len, double* out_span_score, int32_t* out_n_span, int32_t* out_n_member, void* stream);

/* ---- Late-chunking pool: _embed.py:129-140 (and the simple pool :154-164) ---------------------
 * X[T,d] token embeddings (float32, row stride ld); sentence s averages rows
 * [row_begin[s], row_end[s]) (host computes them with the largest-remainder rule, _embed.py:122-128;
 * preamble sentences are simply not listed), then optional L2 normalisation (normalize: 0 = off,
 * 1 = divide by the norm as _embed.py:139, 2 = eps-guarded as _embed.py:161-163) and a cast to
 * float16 (out[S,d], IEEE binary16 bit patterns).  Accumulation is float64 like NumPy's. */
int rl_segment_mean_pool(const float* X, int64_t ld, int d, const int32_t* row_begin,
                         const int32_t* row_end, int S, int normalize, uint16_t* out, void* stream);

/* ---- Standard embedding type's chunk rows: _insert.py:132-145 -------------------------------------
 * out[r] = alpha * X[r] + one_minus_alpha * F[chunk(r)] with NumPy's float16 arithmetic: each product and the
 * sum computed in float32 and rounded to float16 (round to nearest even).  X[n_rows, d] chunklet rows (fp16, row
 * stride ldx), F[n_chunks, d] full-chunk rows (fp16, dense), chunk_off[n_chunks + 1] the CSR of chunk rows over
 * [0, n_rows] (chunk(r) = the c with chunk_off[c] <= r < chunk_off[c + 1]), alpha / one_minus_alpha fp16 bit
 * patterns, out[n_rows, d] fp16 (dense).  d and ldx multiples of 8, X / F / out 16-byte aligned. */
int rl_chunk_embedding_blend(const uint16_t* X, int64_t ldx, const uint16_t* F, const int64_t* chunk_off,
                             int64_t n_chunks, int64_t n_rows, int d, uint16_t alpha, uint16_t one_minus_alpha,
                             uint16_t* out, void* stream);

/* ---- Cross-encoder scoring: _search.py:364-397 (reranker.rank -> FlashRank -> onnxruntime) --------
 * BERT / XLM-RoBERTa cross-encoder forward (ms-marco-MiniLM-L-12-v2 architecture and wider:
 * LayerNorm(word+pos+type) -> n_layers x [self-attention, dense+residual+LN, dense+GELU(erf),
 * dense+residual+LN] -> pooler (dense+tanh on the first token) -> classifier (1 or 2 logits)), fp16
 * storage / fp32 accumulate.  XLM-RoBERTa's classifier.dense / classifier.out_proj fill the pooler /
 * classifier slots.  Linear layers are pre-packed once with rl_xenc_pack_linear into the swizzled fp16
 * image the tensor-core kernel bulk-copies.  All pointers are device pointers except `layers` (host
 * array). */
typedef struct rl_xenc_layer {
  const void* qkv_img;   /* packed [3H, H]  (Q | K | V rows) */
  const float* qkv_bias; /* [3H] */
  const void* o_img;     /* packed [H, H] */
  const float* o_bias;
  const float* ln1_g;
  const float* ln1_b;
  const void* up_img;    /* packed [F, H] */
  const float* up_bias;
  const void* down_img;  /* packed [H, F] */
  const float* down_bias;
  const float* ln2_g;
  const float* ln2_b;
  /* Image type of each linear (appended: every earlier field keeps its offset; a zero-initialised tail is the fp16
   * images of rl_xenc_pack_linear): RL_XENC_IMAGE_F16 or RL_XENC_IMAGE_QUANT (rl_xenc_pack_qlinear /
   * rl_xenc_concat_qlinear, K % 128 == 0, N <= 8192).  rl_xenc_encode and rl_xenc_score refuse any other type
   * (RL_EINVAL) and a quantized linear of another shape (RL_EUNSUPPORTED) before any CUDA call. */
  int32_t qkv_type, o_type, up_type, down_type;
} rl_xenc_layer;
#define RL_XENC_IMAGE_F16 0
#define RL_XENC_IMAGE_QUANT 1

typedef struct rl_xenc_weights {
  int32_t n_layers, hidden, n_heads, ffn, vocab, max_pos, type_vocab;
  float ln_eps;
  const void* word_emb; /* fp16 [vocab, H] */
  const void* pos_emb;  /* fp16 [max_pos, H] */
  const void* type_emb; /* fp16 [type_vocab, H] */
  const float* emb_ln_g;
  const float* emb_ln_b;
  const rl_xenc_layer* layers; /* HOST array of n_layers entries */
  const float* pooler_w; /* fp32 [H, H] */
  const float* pooler_b;
  const float* cls_w;    /* fp32 [n_labels, H] */
  const float* cls_b;    /* fp32 [n_labels] */
  int32_t n_labels;      /* 1 or 2; 0 is read as 1 (appended: every earlier field keeps its offset) */
} rl_xenc_weights;

size_t rl_xenc_linear_image_bytes(int N, int K);
/* W[N, K] float32 row-major (torch nn.Linear.weight) -> packed fp16 image. */
int rl_xenc_pack_linear(const float* W, int N, int K, void* image, void* stream);
/* Y[T, N] (fp16) = act(X[T, K] (fp16) W^T + bias); act 0 = identity, 1 = GELU(erf).  N % 32 == 0,
 * K % 8 == 0, bias 16-byte aligned. */
int rl_xenc_linear(const void* X, const void* image, const float* bias, void* Y, int T, int N, int K, int act,
                   void* stream);
/* GGUF-quantized weights, by GGML type id: Q8_0 = 8, Q4_K = 12, Q6_K = 14.  `blocks` (device) holds W[N, K] as GGUF
 * stores it: row n's K / block_elems blocks at n * (K / block_elems) * block_bytes (Q8_0 32 elements in 34 bytes, Q4_K
 * and Q6_K 256 in 144 and 210).  Values are ggml's formulas in float32 without contraction -- Q8_0 d q, Q4_K
 * (d sc) q - (dmin m), Q6_K (d sc) (q - 32) -- rounded once to fp16 to nearest even. */
/* rows x K elements to fp16 out[rows, K]. */
int rl_dequant_rows_f16(int type, const void* blocks, int64_t rows, int K, void* out, void* stream);
/* Quantized linear image: the blocks reordered per 128-row pass and 128-element K slice, at most 1.06x the GGUF bytes
 * plus a 2 KB header holding each pass's type.  N % 32 == 0, N <= 8192, K % 128 == 0 and whole blocks per row; 0 bytes
 * for any other shape. */
size_t rl_xenc_qlinear_image_bytes(int type, int N, int K);
int rl_xenc_pack_qlinear(int type, const void* blocks, int N, int K, void* image, void* stream);
/* The image of the row-wise concatenation of n_parts images (one K; every part but the last N % 128 == 0), for parts of
 * different types, e.g. Q | K | V.  image holds at least the sum of the parts' sizes.  Reads the parts' headers with a
 * synchronous copy on `stream`. */
int rl_xenc_concat_qlinear(const void* const* parts, int n_parts, void* image, void* stream);
/* Debug/test hook: rl_xenc_linear on a quantized image (the launch rl_xenc_encode makes for RL_XENC_IMAGE_QUANT); equal
 * bit for bit to rl_xenc_linear on rl_xenc_pack_linear of the dequantized weights.  N and K must be the image's. */
int rl_xenc_linear_q(const void* X, const void* image, const float* bias, void* Y, int T, int N, int K, int act,
                     void* stream);
size_t rl_xenc_workspace_bytes(const rl_xenc_weights* w, int T);
/* Packed variable-length batch: input_ids/type_ids/pos_ids [T], cu_seqlens [P+1]; max_len = longest
 * sequence.  out_logit [P, n_labels] row-major ([P] at one label); out_score [P] is FlashRank's score:
 * sigmoid(logit) at one label, softmax(logits)[1] = 1 / (1 + exp(l0 - l1)) at two.
 * Shapes: either head_dim (hidden / n_heads) 32 with hidden % 32 == 0, hidden <= 512 and
 * 0 < max_len <= max_pos (bounded by the attention kernel's shared memory: about 1280 tokens), or
 * everything rl_xenc_encode takes (head_dim 32 or 64, hidden % 32 == 0 and <= 1024, n_layers >= 1,
 * 0 < max_len <= min(512, max_pos)); ffn % 32 == 0, n_labels 0, 1 or 2, P <= T, workspace >=
 * rl_xenc_workspace_bytes(w, T).  Anything else is refused with RL_EUNSUPPORTED / RL_EINVAL /
 * RL_ENOSPACE before any CUDA call. */
int rl_xenc_score(const rl_xenc_weights* w, const int32_t* input_ids, const int32_t* type_ids, const int32_t* pos_ids,
                  const int32_t* cu_seqlens, int P, int T, int max_len, float* out_logit, float* out_score,
                  void* workspace, size_t workspace_bytes, void* stream);
/* Debug/test hook: the attention step of rl_xenc_score on its own.  qkv [T, 3*hidden] fp16 (Q | K | V), ctx [T, hidden]
 * fp16, cu_seqlens [P+1] (device), max_len = longest sequence; head_dim 32.  workspace: >= 4*P bytes (the
 * length-sorted order), 16-byte aligned. */
int rl_xenc_attention(const void* qkv, const int32_t* cu_seqlens, int P, int T, int max_len, int hidden, int n_heads,
                      void* ctx, void* workspace, size_t workspace_bytes, void* stream);
/* Token encoder (BERT / XLM-RoBERTa, e.g. bge-m3): the embeddings and layers of rl_xenc_score without its head.
 * out_hidden [T, H] float32 = the last layer's output LayerNorm for every token.  pooler_* and cls_* may be null.
 * head_dim (hidden / n_heads) 32 or 64, hidden % 32 == 0 and <= 1024, ffn % 32 == 0, n_layers >= 1,
 * 0 < max_len <= min(512, max_pos), P <= T; workspace >= rl_xenc_workspace_bytes(w, T), 16-byte aligned.  Anything
 * else is refused with RL_EUNSUPPORTED / RL_EINVAL / RL_ENOSPACE before any CUDA call. */
int rl_xenc_encode(const rl_xenc_weights* w, const int32_t* input_ids, const int32_t* type_ids, const int32_t* pos_ids,
                   const int32_t* cu_seqlens, int P, int T, int max_len, float* out_hidden, void* workspace,
                   size_t workspace_bytes, void* stream);
/* Debug/test hook: the attention step of rl_xenc_encode on its own (arguments as rl_xenc_attention; head_dim 32 or 64,
 * hidden <= 1024, max_len <= 512). */
int rl_xenc_encode_attention(const void* qkv, const int32_t* cu_seqlens, int P, int T, int max_len, int hidden, int n_heads,
                             void* ctx, void* workspace, size_t workspace_bytes, void* stream);
/* Debug/test hook: the embeddings + LayerNorm step of rl_xenc_score / rl_xenc_encode on its own (same launch): out_f16
 * [T, hidden] fp16 from w's word / position / token-type tables, emb_ln_g / emb_ln_b and ln_eps.  ids / type_ids /
 * pos_ids [T] (device) index the tables (clamped to them).  hidden % 32 == 0 and <= 1024. */
int rl_xenc_embed_ln(const rl_xenc_weights* w, const int32_t* ids, const int32_t* type_ids, const int32_t* pos_ids, int T,
                     void* out_f16, void* stream);
/* Debug/test hook: the residual + LayerNorm step of the encoder on its own (same launch): out [T, H] =
 * LayerNorm(x + res) * gamma + beta with variance eps, x and res fp16 [T, H], out fp16 (out_f32 = 0) or fp32
 * (out_f32 = 1, the last layer of rl_xenc_encode).  H % 32 == 0 and <= 1024, every pointer 16-byte aligned; out may be
 * res (the encoder normalises in place). */
int rl_xenc_add_ln(const void* x, const void* res, const float* gamma, const float* beta, float eps, int T, int H,
                   int out_f32, void* out, void* stream);
/* Debug/test hook: the pooler + classifier + score step of rl_xenc_score on its own (same launch): out_logit
 * [P, n_labels] and out_score [P] from the fp16 rows hidden_f16 [T, hidden], the [CLS] row of sequence s at
 * cu_seqlens[s] (device).  w's pooler_* / cls_* / n_labels (0 read as 1) and hidden (% 32 == 0, <= 1024). */
int rl_xenc_cls_head(const rl_xenc_weights* w, const void* hidden_f16, const int32_t* cu_seqlens, int P, float* out_logit,
                     float* out_score, void* stream);

/* ---- BM25 keyword search: _search.py:203-225 (DuckDB fts match_bm25 at its defaults) -------------------------------
 * Inverted index over the chunk bodies (device arrays): term_off int64 [n_terms + 1], a term-major postings CSR whose
 * doc int32 / tf int32 [P] are sorted by chunk within each term; doc_len int32 [n_chunks] = terms left after stop-word
 * removal.  chunk_alive / chunk_mask: uint8 [n_chunks] or NULL (= every chunk).
 *
 * rl_bm25_stats: over the chunks with chunk_alive set, df[t] (int32 [n_terms]) = number of such chunks that contain t,
 * corpus (float64 [3]) = {N, sum of doc_len, avgdl = sum / N}.  Every double is rounded as the SQL expression reads (no
 * contraction). */
int rl_bm25_stats(const int64_t* term_off, const int32_t* doc, const int32_t* doc_len, const uint8_t* chunk_alive,
                  int64_t n_terms, int64_t n_chunks, int32_t* df, double* corpus, void* stream);
/* Workspace that lets rl_bm25_topk_global score `group` queries at a time: group * n_chunks * 8 bytes. */
size_t rl_bm25_workspace_bytes(int64_t n_chunks, int group);
/* Bytes of one packed top-k buffer: chunk int64 [B, k] | score float64 [B, k] | count int32 [B], padded to a multiple of
 * 16 (0 when B or k is not positive). */
size_t rl_bm25_packed_bytes(int B, int k);
/* rl_bm25_topk_global: B queries, query b = the entries q_off[b] .. q_off[b+1] (device int32), q_terms[j] the term id of
 * entry j or -1 (a term this index does not hold; skipped), distinct within a query.  The per-chunk sum runs in entry
 * order.  stats (device int64
 * [2 + J]) = {N, sum of doc_len, df of entry 0 .. J-1}: on a single index its own live counts, on a ShardedIndex their
 * sums over the shards (integers, so exact on every rank).  avgdl = sum / N, idf_j = log10((N - df_j + 0.5) / (df_j +
 * 0.5) + 1), score(d) = sum over the entries j with a term in d of idf_j * (tf * (k1 + 1) / (tf + k1 * (1 - b + b *
 * (doc_len[d] / avgdl)))), float64, rounded as written.  A chunk is a result when it contains an entry's term and
 * chunk_mask allows it (tombstones AND the metadata filter: the mask changes nothing in the statistics).  Output: one
 * rl_bm25_packed_bytes(B, k) buffer (16-byte aligned), best first by (score desc, chunk asc), chunk_base added to every
 * chunk: chunk -1 padded, score -inf padded, padding zeroed.  1 <= k <= 4096 (RL_MAX_SURVIVORS), k1 >= 0, 0 <= b <= 1;
 * the queries are scored in groups of as many as the workspace holds (at least one, else RL_ENOSPACE).
 * n_chunks == 0 (an empty shard) is valid: every count is 0 and workspace may be NULL. */
int rl_bm25_topk_global(const int64_t* term_off, const int32_t* doc, const int32_t* tf, const int32_t* doc_len,
                        const int64_t* stats, int64_t n_terms, int64_t n_chunks, const uint8_t* chunk_mask,
                        const int32_t* q_off, const int32_t* q_terms, int B, int k, double k1, double b, int64_t chunk_base,
                        void* out_packed, void* workspace, size_t workspace_bytes, void* stream);
/* rl_bm25_merge_packed: gathered = R packed buffers of rl_bm25_packed_bytes(B, k) bytes end to end (16-byte aligned);
 * per query, the top k of the R lists by (score desc, chunk asc) -- exact, chunks being unique across the shards.
 * Outputs, best first: out_chunk int64 [B, k] (-1 padded), out_score float64 [B, k] (-inf padded), out_count int32 [B].
 * 1 <= R <= 64, 1 <= k <= 4096; one CTA per query, no global atomics. */
int rl_bm25_merge_packed(const void* gathered, int R, int B, int k, int64_t* out_chunk, double* out_score,
                         int32_t* out_count, void* stream);

/* ---- ts_rank keyword search: _search.py:176-201 (PostgreSQL, ts_rank over to_tsvector('simple', body)) -------------
 * rl_tsrank_topk_global: the top k of B queries by PostgreSQL's ts_rank(tsvector, tsquery) at the default weights and
 * normalization 0, every position of weight D.  Index: term_off int64 [n_terms + 1], a lexeme-major CSR whose doc int32
 * [P] is sorted by chunk within each lexeme and npos int32 [P] is the number of positions the chunk's tsvector lists for
 * it (1 for a lexeme without positions; values outside [1, 256] are clamped to it).  Query b = the entries q_off[b] ..
 * q_off[b+1] (device int32): its distinct lexemes in ascending UTF-8 byte order, q_terms[j] the lexeme id of entry j or -1
 * (a lexeme this index does not hold: it matches nothing but still counts in the divisor).  Per chunk, in entry order,
 * res = (float)((double)res + c[npos]) with c[n] = (double)((0.1f + sum_{j<n} 0.1f / (float)((j+1)^2)) - 0.1f) /
 * 1.64493406685 (float steps, ascending j), then score = res / (float)(number of entries): calc_rank_or, every step
 * rounded to nearest in its C type, no contraction.  A chunk is a result when it holds an entry and chunk_mask allows it.
 * Output as rl_bm25_topk_global: one rl_bm25_packed_bytes(B, k) buffer, best first by (score desc, chunk asc), the
 * float32 score widened to double, chunk_base added, -1 / -inf padded, padding zeroed; 1 <= k <= 4096; workspace sized by
 * rl_bm25_workspace_bytes (query groups, RL_ENOSPACE below one query); n_chunks == 0 valid.  The table c[1..256] is
 * computed on the device by the first call on each device, which waits for it once. */
int rl_tsrank_topk_global(const int64_t* term_off, const int32_t* doc, const int32_t* npos, int64_t n_terms,
                          int64_t n_chunks, const uint8_t* chunk_mask, const int32_t* q_off, const int32_t* q_terms, int B,
                          int k, int64_t chunk_base, void* out_packed, void* workspace, size_t workspace_bytes,
                          void* stream);

/* ---- sentence splitting (SaT boundary probabilities + the reference's sentence partition) ---------------------------
 * logits[r, l] = hidden[r, :] . W[l, :] + bias[l] for rows r < rows (float32; W [n_labels, hidden_size] row-major,
 * 1 <= n_labels <= 16).  Runs on the output of rl_xenc_encode, one call at a time. */
int rl_sat_token_logits(const float* hidden, int64_t rows, int hidden_size, const float* W, const float* bias,
                        int n_labels, float* logits, void* stream);
size_t rl_sat_workspace_bytes(int64_t n_tokens, int n_docs, int n_labels);
/* One float32 probability per character of n_docs documents (probas [n_chars], document d at
 * doc_char_off[d] .. doc_char_off[d + 1]; its tokens at doc_tok_off[d] .. doc_tok_off[d + 1]; both [n_docs + 1],
 * ascending from 0).  Document d's blocks are blk_off[d] .. blk_off[d + 1]: each holds doc_block[d] = B tokens from
 * document-relative token blk_start[b] (ascending), whose in-block position k is logits row blk_row[b] + k.
 *  1. stitched[t, l] = sum_b hat[B (B - 1) / 2 + k] logits[blk_row[b] + k, l] / sum_b hat[..] over the blocks b that
 *     cover token t, ascending b (k = t - blk_start[b]; float32, one rounding per operation);
 *  2. every character of document d = min over its stitched logits (all tokens, all labels; -inf when it has none);
 *  3. probas[tok_char[t]] = stitched[t, 0] for every token with tok_char[t] >= 0 (global character index, at most one
 *     token per character);
 *  4. probas = 1 / (1 + exp(-probas)); then, when known is not null, probas[c] = known[c] wherever known[c] is not NaN;
 *  5. when is_space is not null: for each run of is_space characters inside a document, from the non-space character i
 *     before it to the first non-space j after it, probas[i .. j-2] = min(probas[i .. j-1]), probas[j-1] = max(..).
 * No atomics: results do not depend on the grouping of documents.  workspace >= rl_sat_workspace_bytes(n_tokens,
 * n_docs, n_labels). */
int rl_sat_char_probas(const float* logits, int n_labels, const int64_t* doc_tok_off, const int64_t* doc_char_off,
                       const int32_t* doc_block, int n_docs, int64_t n_tokens, int64_t n_chars, const int64_t* blk_off,
                       const int32_t* blk_start, const int64_t* blk_row, const float* hat, const int64_t* tok_char,
                       const float* known, const uint8_t* is_space, float* probas, void* workspace,
                       size_t workspace_bytes, void* stream);
size_t rl_sentence_partition_workspace_bytes(int64_t n_chars);
/* raglite's split_sentences partition per document d (probas[doc_off[d] .. + doc_len[d]], disjoint ranges inside
 * [0, n_chars)): the dynamic program with no maximum length over the whole document, then, when max_len[d] > 0, the
 * deque program with max_len[d] over every resulting sentence longer than max_len[d].  score = p - 0.25f in float32,
 * dp in float64 (one rounded addition per step, strict comparisons).  Writes the partition indices (a sentence ends
 * before each) ascending to cuts[doc_off[d] ..], their number to counts[d], and status[d] = 0, or 1 when no split
 * satisfies the constraints (the reference's ValueError).  One thread per document; workspace >=
 * rl_sentence_partition_workspace_bytes(n_chars) (dp, back, the deque's index ring and the stage-1 boundaries). */
int rl_sentence_partition(const float* probas, const int64_t* doc_off, const int32_t* doc_len, const int32_t* min_len,
                          const int32_t* max_len, int n_docs, int64_t n_chars, int32_t* cuts, int32_t* counts,
                          int32_t* status, void* workspace, size_t workspace_bytes, void* stream);

/* ---- chunklets and chunks (the reference's split_chunklets dynamic program and split_chunks' partition) -------------
 * Both partitions are one windowed dynamic program, one warp per document: dp[0] = 0 and, for i = 1 .. n,
 * dp[i] = min over j of dp[j] + cost(j, i) (one rounded float64 addition) over the window j = i-1, i-2, ... while
 * lens[j] + .. + lens[i-1] <= max_size[d]; the minimum of (dp[j] + cost, j) lexicographically (the smallest j of the
 * smallest cost, inf included), dp[i] = inf and back[i] = -1 when the window is empty.  The cuts are read back from
 * back[n] down to the first back <= 0 and written ascending to cuts[doc_off[d] ..] (the first item of each piece but the
 * first), their number to counts[d].  Document d owns items doc_off[d] .. doc_off[d + 1] (doc_off [n_docs + 1], ascending
 * from 0).  The workspace holds n + 1 entries per document of dp, back and the prefix sums. */
size_t rl_chunklet_partition_workspace_bytes(int64_t n_sentences, int n_docs);
/* split_chunklets with its default costs, per sentence: the Markdown boundary probability, the statement count (both
 * float64, as markdown_chunklet_boundaries / compute_num_statements give them) and the length in characters.
 * cost(j, i) = ((1 - p[j]) + (PB[i] - PB[j+1])) + (s - 3)(s - 3) / sqrt(max(s, 1e-6)) / 2, s = PS[i] - PS[j], every
 * step one rounded float64 operation, PB / PS the sequential prefix sums from 0.  status[d] = 0, or 1 for a document
 * without sentences (the reference refuses it).  A sentence longer than max_size[d] is kept as the reference keeps it:
 * dp stays inf past it and later windows take their smallest j. */
int rl_chunklet_partition(const double* boundary_probas, const double* num_statements, const int32_t* lens,
                          const int64_t* doc_off, const int32_t* max_size, int n_docs, int64_t n_sentences,
                          int32_t* cuts, int32_t* counts, int32_t* status, void* workspace, size_t workspace_bytes,
                          void* stream);
size_t rl_chunk_similarities_workspace_bytes(int64_t n_rows);
/* split_chunks' cut costs, one CTA per document: rows doc_off[d] .. doc_off[d + 1] of X (x_dtype 0: float32,
 * 1: float16; row stride ld elements, 1 <= dim <= 8192) are normalised in float32; the mean of the rows nonoutlying[]
 * selects, normalised, is the discourse vector (float64, from the float32 normalised rows); when some row is selected
 * and no row's projection x - (x . disc) disc has norm <= FLT_EPSILON (x . disc and the norm in float64), the
 * normalised projections replace the rows (float32, x . disc, the norm and disc rounded to float32).
 * costs[doc_off[d] + i] = max((x_i . x_{i+1} + 1) / 2, sqrt(FLT_EPSILON)) in float32 for i < n - 1; then, i ascending
 * over i < n - 1 with the first chunklet counted as preceded by a heading, a heading i (is_heading[]) sets
 * costs[i] = 1 and divides costs[i - 1] by 4 when chunklet i - 1 is not a heading.  The slot of each document's last
 * row is not written.  status[d] = 0, or 1 when a row has zero norm (then no cost of d is written).  A documented
 * bound from float64, not the reference's bits. */
int rl_chunk_similarities(const void* X, int x_dtype, int64_t ld, int dim, const int64_t* doc_off, int n_docs,
                          int64_t n_rows, const uint8_t* nonoutlying, const uint8_t* is_heading, float* costs,
                          int32_t* status, void* workspace, size_t workspace_bytes, void* stream);
size_t rl_chunk_partition_workspace_bytes(int64_t n_chunklets, int n_docs);
/* split_chunks' partition: cost(j, i) = costs[doc_off[d] + j - 1] widened to float64 for j > 0, 0 for j = 0 (a chunk
 * starting at j pays for the cut before it), lens the chunklet lengths.  This is the optimum of the reference's integer
 * program.  status[d] = 0, or 1 when a chunklet is longer than max_size[d] (no partition; counts[d] = 0). */
int rl_chunk_partition(const float* costs, const int32_t* lens, const int64_t* doc_off, const int32_t* max_size,
                       int n_docs, int64_t n_chunklets, int32_t* cuts, int32_t* counts, int32_t* status,
                       void* workspace, size_t workspace_bytes, void* stream);

/* ---- text analysis of the BM25 index: DuckDB fts's tokenizer, english stop list and Snowball porter stemmer ----------
 * The host analyzer (raglite_b200/_fts.py, Analyzer.analyze) bit for bit, in four steps around two host round trips:
 * rl_fts_mark finds the words, rl_fts_stem stems them, rl_fts_verify and rl_fts_stem_bytes settle the distinct stems
 * exactly, rl_fts_term_keys turns the term id of each distinct stem into postings keys.  No global atomics: every
 * output is the same run to run.
 *
 * rl_fts_mark: text = n_bytes of UTF-8 (bodies joined by a separator byte, so that no word spans two bodies).
 * class_table uint8 [0x110000] (device) classifies each code point as lower(strip_accents(chr(cp))) does: 1..26 the
 * letter a..z, 0xFF dropped (it vanishes: combining marks and what decomposes into marks only), anything else a
 * separator.  '\' is a separator that, with the dropped code points removed, swallows the letter right after a run of
 * backslashes of odd length (the `\\.` of the tokenizer's regular expression).  Writes mark uint8 [n_bytes]: at the
 * lead byte of each kept letter the letter, upper case when it starts a word, lower case otherwise; 0 at every other
 * byte.  A parallel scan of the tokenizer's three-state automaton, exact for runs of any length.  workspace >=
 * rl_fts_workspace_bytes(n_bytes); n_bytes == 0 is valid and launches nothing. */
size_t rl_fts_workspace_bytes(int64_t n_bytes);
int rl_fts_mark(const uint8_t* text, int64_t n_bytes, const uint8_t* class_table, uint8_t* mark, void* workspace,
                size_t workspace_bytes, void* stream);
/* rl_fts_stem: word w = letters[word_off[w] .. word_off[w + 1]) (letters uint8 'a'..'z', word_off int64 [n_words + 1],
 * both device).  stop (device uint64 [n_stop][2]): the stop list, each entry zero-padded to 16 bytes and read as two
 * big-endian uint64 (hi, lo), sorted ascending.  A word equal to an entry gets keep[w] = -1.  Any other word is stemmed
 * by Snowball's porter: its stem is letters word_off[w] .. word_off[w] + keep[w] followed by the nonzero bytes of
 * tail[w], low byte first (at most 8), and hash[w] is a 64-bit hash of the stem cut to its low hash_bits bits
 * (1 <= hash_bits <= 64; fewer bits only make collisions, which rl_fts_verify detects). */
int rl_fts_stem(const uint8_t* letters, const int64_t* word_off, int64_t n_words, const uint64_t* stop, int n_stop,
                int hash_bits, int32_t* keep, uint64_t* tail, int64_t* hash, void* stream);
/* rl_fts_verify: differ[t] = 1 when the stems of the words word_a[t] and word_b[t] differ byte for byte, else 0
 * (word_a, word_b int64 [n]; stems as rl_fts_stem left them, of words with keep >= 0). */
int rl_fts_verify(const uint8_t* letters, const int64_t* word_off, const int32_t* keep, const uint64_t* tail,
                  const int64_t* word_a, const int64_t* word_b, int64_t n, uint8_t* differ, void* stream);
/* rl_fts_stem_bytes: the stems of words[0 .. n) as a bytes CSR: stem u at out[out_off[u] .. out_off[u + 1]) (out_off
 * int64 [n + 1], each length keep + the number of tail letters). */
int rl_fts_stem_bytes(const uint8_t* letters, const int64_t* word_off, const int32_t* keep, const uint64_t* tail,
                      const int64_t* words, int64_t n, const int64_t* out_off, uint8_t* out, void* stream);
/* rl_fts_term_keys: the postings keys of n tokens, key[t] = stem_term[tok_stem[t]] << 32 | (chunk_base + owner[t])
 * (tok_stem, owner int64 [n]; stem_term int32, the term id of each distinct stem; chunk_base >= 0). */
int rl_fts_term_keys(const int64_t* tok_stem, const int64_t* owner, int64_t n, const int32_t* stem_term,
                     int64_t chunk_base, int64_t* key, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RAGLITE_B200_H_ */
