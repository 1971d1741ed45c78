// BM25 keyword search over a resident inverted index: the arithmetic of DuckDB's fts `match_bm25` macro, which the
// reference's keyword_search runs at its defaults (reference _search.py:203-225).
//
//   rl_bm25_stats         df(t) over live chunks, N, sum of len and avgdl (refreshed after every change to the index)
//   rl_bm25_topk_global   per query, the k best chunks by (score desc, chunk asc), with idf and avgdl computed from the
//                         integers N, sum of len and the df of each query entry; chunk_base added; one packed buffer out
//   rl_bm25_merge_packed  the top k of R gathered buffers (a ShardedIndex of R > 1 shards, DESIGN.md section 3.7)
//
// Index layout (include/raglite_b200.h): term-major postings CSR term_off [V + 1], doc / tf [P] sorted by chunk within a
// term, doc_len [C].  Every double is rounded exactly as the SQL expression reads (explicit _rn intrinsics: no FMA
// contraction), so a score differs from a float64 NumPy restatement only through log10 in idf.
//
// rl_bm25_topk_global processes the batch in groups of G queries, G set by the workspace (G * C keys of 8 bytes):
//   score kernel   one CTA per (query, tile of kTile chunks); float64 accumulators in shared memory; for each query
//                  entry in the given order, the term's postings inside the tile are found by binary search and each
//                  adds its contribution (a term touches a chunk at most once; a barrier separates the entries, so a
//                  chunk's sum runs in entry order and nothing races).  Output: an order-preserving 64-bit key per
//                  chunk, 0 where the chunk is unmatched or masked.
//   select kernel  one CTA per query: MSB-first radix select over the 96-bit composite (key, ~chunk) -- unique per
//                  chunk, so the k-th largest composite is the exact cut of (score desc, chunk asc) -- then the k
//                  survivors are sorted in shared memory.
// Nothing depends on launch order and no global atomics are used; the shared-memory histogram counts are integers.
//
// rl_tsrank_topk_global ranks the same way by PostgreSQL's ts_rank (calc_rank_or at the default weights, normalization 0)
// over a lexeme-major CSR whose value is npos, the number of positions a chunk's tsvector lists for the lexeme: its own
// score kernel (float32 accumulators, DESIGN.md section 3.9), then the select kernel above, unchanged.
#include <cuda_runtime.h>

#include <algorithm>
#include <mutex>

#include "common.cuh"

namespace rl {
namespace {

constexpr int kTile = 4096;            // chunks per score CTA (32 KB of float64 accumulators)
constexpr int kScoreThreads = 512;
constexpr int kSelectThreads = 1024;
constexpr int kBm25MaxK = 4096;        // RL_MAX_SURVIVORS: the num_hits cap of the vector path
constexpr int kSelBins = 2048;        // 11-bit digits
constexpr uint64_t kSign = 1ull << 63;

// ---- corpus statistics -> BM25 weights -----------------------------------------------------------------------------
__device__ __forceinline__ double bm25_avgdl(double n, double sum_len) {
  return __ddiv_rn(sum_len, n);   // AVG(len); NaN for an empty corpus (nothing is scored then)
}
__device__ __forceinline__ double bm25_idf(double N, double df) {
  const double ratio = __ddiv_rn(__dadd_rn(__dsub_rn(N, df), 0.5), __dadd_rn(df, 0.5));
  return log10(__dadd_rn(ratio, 1.0));
}

// ---- rl_bm25_stats ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) bm25_corpus_kernel(const int32_t* __restrict__ doc_len, const uint8_t* __restrict__ alive,
                                                           int64_t n_chunks, double* __restrict__ corpus) {
  __shared__ long long s_n[32], s_len[32];
  long long n = 0, len = 0;
  for (int64_t c = threadIdx.x; c < n_chunks; c += blockDim.x) {
    if (alive == nullptr || alive[c]) {
      ++n;
      len += doc_len[c];
    }
  }
  for (int off = 16; off > 0; off >>= 1) {
    n += __shfl_down_sync(0xffffffffu, n, off);
    len += __shfl_down_sync(0xffffffffu, len, off);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { s_n[warp] = n; s_len[warp] = len; }
  __syncthreads();
  if (threadIdx.x == 0) {
    long long tn = 0, tl = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { tn += s_n[w]; tl += s_len[w]; }
    corpus[0] = (double)tn;
    corpus[1] = (double)tl;
    corpus[2] = bm25_avgdl((double)tn, (double)tl);
  }
}

__global__ void __launch_bounds__(256) bm25_df_kernel(const int64_t* __restrict__ term_off, const int32_t* __restrict__ doc,
                                                      const uint8_t* __restrict__ alive, int64_t n_terms,
                                                      int32_t* __restrict__ df_out) {
  __shared__ int s_part[8];
  for (int64_t t = blockIdx.x; t < n_terms; t += gridDim.x) {
    const int64_t p0 = term_off[t], p1 = term_off[t + 1];
    int cnt = 0;
    for (int64_t p = p0 + threadIdx.x; p < p1; p += blockDim.x) cnt += (alive == nullptr || alive[doc[p]]) ? 1 : 0;
    for (int off = 16; off > 0; off >>= 1) cnt += __shfl_down_sync(0xffffffffu, cnt, off);
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
      int df = 0;
      for (int w = 0; w < 8; ++w) df += s_part[w];
      df_out[t] = df;
    }
    __syncthreads();
  }
}

// ---- rl_bm25_topk_global: scores of one (query, tile) ------------------------------------------------------------------
// The weights come from the integers stats = {N, sum of doc_len, df of entry 0, 1, ...}: avgdl once per CTA, the idf of
// entry j where the term is met -- the expressions of DuckDB's stats / dict tables, rounded alike on every shard.
__global__ void __launch_bounds__(kScoreThreads) bm25_score_kernel(
    const int64_t* __restrict__ term_off, const int32_t* __restrict__ doc, const int32_t* __restrict__ tf,
    const int32_t* __restrict__ doc_len, const int64_t* __restrict__ stats, int64_t n_terms, int64_t n_chunks,
    const uint8_t* __restrict__ mask, const int32_t* __restrict__ q_off, const int32_t* __restrict__ q_terms, int q0,
    double k1, double b, uint64_t* __restrict__ keys) {
  __shared__ double acc[kTile];
  __shared__ int64_t range[2];
  const int q = q0 + (int)blockIdx.y;
  const int64_t c0 = (int64_t)blockIdx.x * kTile;
  const int n = (int)min((int64_t)kTile, n_chunks - c0);
  for (int i = threadIdx.x; i < n; i += blockDim.x) acc[i] = 0.0;
  const double avgdl = bm25_avgdl((double)stats[0], (double)stats[1]);
  const double k1p1 = __dadd_rn(k1, 1.0), one_minus_b = __dsub_rn(1.0, b);
  const int j0 = q_off[q], j1 = q_off[q + 1];
  for (int j = j0; j < j1; ++j) {
    const int t = q_terms[j];
    if (t < 0 || (int64_t)t >= n_terms) continue;   // uniform over the CTA
    __syncthreads();   // the previous term's additions (and the zeroing) are done; range[] is free
    if (threadIdx.x < 2) {   // lower_bound of the tile's first chunk (thread 0) and of the next tile's (thread 1)
      int64_t lo = term_off[t], hi = term_off[t + 1];
      const int64_t target = c0 + (threadIdx.x ? n : 0);
      while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if ((int64_t)doc[mid] < target) lo = mid + 1; else hi = mid;
      }
      range[threadIdx.x] = lo;
    }
    __syncthreads();
    const int64_t p0 = range[0], p1 = range[1];
    const double w = bm25_idf((double)stats[0], (double)stats[2 + j]);
    for (int64_t p = p0 + threadIdx.x; p < p1; p += blockDim.x) {
      const int c = doc[p];
      const double f = (double)tf[p];
      const double norm = __dadd_rn(one_minus_b, __dmul_rn(b, __ddiv_rn((double)doc_len[c], avgdl)));
      const double sub = __dmul_rn(w, __ddiv_rn(__dmul_rn(f, k1p1), __dadd_rn(f, __dmul_rn(k1, norm))));
      acc[c - c0] = __dadd_rn(acc[c - c0], sub);
    }
  }
  __syncthreads();
  uint64_t* out = keys + (int64_t)blockIdx.y * n_chunks + c0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const double s = acc[i];
    const bool ok = s > 0.0 && (mask == nullptr || mask[c0 + i]);
    out[i] = ok ? ((uint64_t)__double_as_longlong(s) | kSign) : 0ull;   // positive doubles order as their bits
  }
}

// ---- rl_tsrank_topk_global: ts_rank of one (query, tile) --------------------------------------------------------------
// tsrank.c's calc_rank_or with every position of weight D (w = 0.1f, so the maximum weight is at j = 0): an entry held
// n times adds contrib[n - 1] = (double)t / 1.64493406685 with t = (0.1f + resj) - 0.1f / 1 and resj = sum over j < n of
// 0.1f / (float)((j + 1)^2), float sums in ascending j -- the C expressions in their own types.  The 256 values (npos is
// capped at MAXNUMPOS = 256) are built once per device by tsrank_table_kernel.
constexpr int kTsMaxPos = 256;

__device__ double g_tsrank_contrib[kTsMaxPos];

__global__ void __launch_bounds__(kTsMaxPos) tsrank_table_kernel() {
  __shared__ float term[kTsMaxPos], resj[kTsMaxPos];
  const int j = threadIdx.x;
  term[j] = __fdiv_rn(0.1f, (float)((j + 1) * (j + 1)));
  __syncthreads();
  if (j == 0) {   // a sequential float sum: its rounding depends on the order
    float r = 0.0f;
    for (int i = 0; i < kTsMaxPos; ++i) {
      r = __fadd_rn(r, term[i]);
      resj[i] = r;
    }
  }
  __syncthreads();
  const float t = __fsub_rn(__fadd_rn(0.1f, resj[j]), __fdiv_rn(0.1f, 1.0f));
  g_tsrank_contrib[j] = __ddiv_rn((double)t, 1.64493406685);
}

// Per chunk res = (float)((double)res + contrib) over the query's entries in the given order (the plan's byte order, that
// of SortAndUniqItems), then res / (float)size with size = every entry of the query, known to this index or not.  A
// chunk matches when it holds an entry (every contribution is > 0, so exactly when res > 0).
__global__ void __launch_bounds__(kScoreThreads) tsrank_score_kernel(
    const int64_t* __restrict__ term_off, const int32_t* __restrict__ doc, const int32_t* __restrict__ npos,
    int64_t n_terms, int64_t n_chunks, const uint8_t* __restrict__ mask, const int32_t* __restrict__ q_off,
    const int32_t* __restrict__ q_terms, int q0, uint64_t* __restrict__ keys) {
  __shared__ float acc[kTile];
  __shared__ double contrib[kTsMaxPos];
  __shared__ int64_t range[2];
  const int q = q0 + (int)blockIdx.y;
  const int64_t c0 = (int64_t)blockIdx.x * kTile;
  const int n = (int)min((int64_t)kTile, n_chunks - c0);
  for (int i = threadIdx.x; i < n; i += blockDim.x) acc[i] = 0.0f;
  for (int i = threadIdx.x; i < kTsMaxPos; i += blockDim.x) contrib[i] = g_tsrank_contrib[i];
  const int j0 = q_off[q], j1 = q_off[q + 1];
  for (int j = j0; j < j1; ++j) {
    const int t = q_terms[j];
    if (t < 0 || (int64_t)t >= n_terms) continue;   // uniform over the CTA; still counted in size
    __syncthreads();   // the previous entry's additions (and the zeroing, the table) are done; range[] is free
    if (threadIdx.x < 2) {
      int64_t lo = term_off[t], hi = term_off[t + 1];
      const int64_t target = c0 + (threadIdx.x ? n : 0);
      while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if ((int64_t)doc[mid] < target) lo = mid + 1; else hi = mid;
      }
      range[threadIdx.x] = lo;
    }
    __syncthreads();
    const int64_t p0 = range[0], p1 = range[1];
    for (int64_t p = p0 + threadIdx.x; p < p1; p += blockDim.x) {
      const int c = doc[p];
      const int np = min(max(npos[p], 1), kTsMaxPos);
      acc[c - c0] = __double2float_rn(__dadd_rn((double)acc[c - c0], contrib[np - 1]));
    }
  }
  __syncthreads();
  const float size = (float)(j1 - j0);
  uint64_t* out = keys + (int64_t)blockIdx.y * n_chunks + c0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float s = acc[i];
    const bool ok = s > 0.0f && (mask == nullptr || mask[c0 + i]);
    out[i] = ok ? ((uint64_t)__double_as_longlong((double)__fdiv_rn(s, size)) | kSign) : 0ull;
  }
}

// ---- rl_bm25_topk_global: top k of one query -----------------------------------------------------------------------------
// Radix digits of the composite (key: bits 95..32, ~chunk: bits 31..0), most significant first.
struct Digit {
  int8_t part;   // 1: key, 0: ~chunk
  int8_t shift;
  int8_t width;
};
__constant__ Digit kDigits[9] = {{1, 53, 11}, {1, 42, 11}, {1, 31, 11}, {1, 20, 11}, {1, 9, 11}, {1, 0, 9},
                                 {0, 21, 11}, {0, 10, 11}, {0, 0, 10}};

__device__ __forceinline__ bool ge_prefix(uint64_t key, uint32_t lo, uint64_t m_hi, uint32_t m_lo, uint64_t p_hi, uint32_t p_lo) {
  const uint64_t a = key & m_hi;
  return a > p_hi || (a == p_hi && (lo & m_lo) >= p_lo);
}

// out_chunk holds chunk_base + chunk (the shard's global numbering).  With n_chunks == 0 (an empty shard) nothing is read
// and every row comes out empty.
__global__ void __launch_bounds__(kSelectThreads) bm25_select_kernel(const uint64_t* __restrict__ keys, int64_t n_chunks, int q0,
                                                                     int k, int64_t chunk_base, int64_t* __restrict__ out_chunk,
                                                                     double* __restrict__ out_score,
                                                                     int32_t* __restrict__ out_count) {
  extern __shared__ __align__(16) unsigned char smem[];
  uint64_t* s_key = reinterpret_cast<uint64_t*>(smem);              // [kBm25MaxK]
  int32_t* s_chunk = reinterpret_cast<int32_t*>(s_key + kBm25MaxK);  // [kBm25MaxK]
  uint32_t* hist = reinterpret_cast<uint32_t*>(s_chunk + kBm25MaxK); // [kSelBins]
  __shared__ uint64_t s_phi, s_mhi;
  __shared__ uint32_t s_plo, s_mlo;
  __shared__ int s_rank, s_want, s_done, s_n;
  const uint64_t* row = keys + (int64_t)blockIdx.x * n_chunks;
  const int q = q0 + (int)blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) { s_phi = 0; s_mhi = 0; s_plo = 0; s_mlo = 0; s_rank = 0; s_want = -1; s_done = 0; s_n = 0; }
  __syncthreads();
  for (int pass = 0; pass < 9; ++pass) {
    const Digit dg = kDigits[pass];
    const uint32_t nb = 1u << dg.width;
    for (uint32_t i = tid; i < nb; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    const uint64_t p_hi = s_phi, m_hi = s_mhi;
    const uint32_t p_lo = s_plo, m_lo = s_mlo;
    for (int64_t base = 0; base < n_chunks; base += blockDim.x) {
      const int64_t c = base + tid;
      bool in = false;
      uint32_t bin = 0;
      if (c < n_chunks) {
        const uint64_t key = row[c];
        const uint32_t lo = ~(uint32_t)c;
        in = (key & m_hi) == p_hi && (lo & m_lo) == p_lo;
        bin = (uint32_t)(((dg.part ? key : (uint64_t)lo) >> dg.shift) & (nb - 1));
      }
      const unsigned active = __ballot_sync(0xffffffffu, in);
      if (in) {   // warp-aggregated: all-zero keys and a shared exponent would otherwise pile onto one bin
        const unsigned peers = __match_any_sync(active, bin);
        if (lane == __ffs(peers) - 1) atomicAdd(&hist[bin], (uint32_t)__popc(peers));
      }
    }
    __syncthreads();
    if (warp == 0) {
      const uint32_t per = nb / 32;
      uint32_t sum = 0;
      for (uint32_t i = 0; i < per; ++i) sum += hist[lane * per + i];
      uint32_t x = sum;   // inclusive suffix sum over lanes (higher bins first)
      for (int off = 1; off < 32; off <<= 1) {
        const uint32_t v = __shfl_down_sync(0xffffffffu, x, off);
        if (lane + off < 32) x += v;
      }
      const uint32_t excl = x - sum;
      int rank = s_rank;
      bool stop = false;
      if (pass == 0) {   // keys with the top bit set are the matched chunks (bins 1024..2047)
        const int valid = (int)__shfl_sync(0xffffffffu, x, 16);
        const int want = min(k, valid);
        if (lane == 0) { s_want = want; s_rank = want; }
        rank = want;
        stop = want == 0 || want == valid;   // nothing, or every matched chunk: no cut needed (prefix/mask stay 0)
        if (stop && lane == 0) s_done = 1;
        __syncwarp();   // lane 0's s_rank lands before the cut lane's
      }
      if (!stop && excl < (uint32_t)rank && (uint32_t)rank <= excl + sum) {   // exactly one lane holds the cut
        uint32_t cum = excl;
        uint32_t d = lane * per + per - 1;
        for (;; --d) {
          if (cum + hist[d] >= (uint32_t)rank) break;
          cum += hist[d];
        }
        const int r = rank - (int)cum;
        if (dg.part) {
          s_phi = p_hi | ((uint64_t)d << dg.shift);
          s_mhi = m_hi | ((uint64_t)(nb - 1) << dg.shift);
        } else {
          s_plo = p_lo | (d << dg.shift);
          s_mlo = m_lo | ((nb - 1) << dg.shift);
        }
        s_rank = r;
        if (hist[d] == (uint32_t)r) s_done = 1;   // the whole bin is taken: the prefix is the cut
      }
    }
    __syncthreads();
    if (s_done) break;
  }
  const int want = s_want;
  // Gather: every matched composite at or above the cut (exactly `want` of them: composites are unique).
  if (want > 0) {
    const uint64_t p_hi = s_phi, m_hi = s_mhi;
    const uint32_t p_lo = s_plo, m_lo = s_mlo;
    for (int64_t base = 0; base < n_chunks; base += blockDim.x) {
      const int64_t c = base + tid;
      if (c < n_chunks) {
        const uint64_t key = row[c];
        if (key != 0 && ge_prefix(key, ~(uint32_t)c, m_hi, m_lo, p_hi, p_lo)) {
          const int pos = atomicAdd(&s_n, 1);
          if (pos < kBm25MaxK) { s_key[pos] = key; s_chunk[pos] = (int32_t)c; }
        }
      }
    }
  }
  __syncthreads();
  const int m = min(want, kBm25MaxK);
  int npow2 = 1;
  while (npow2 < m) npow2 <<= 1;
  for (int i = m + tid; i < npow2; i += blockDim.x) { s_key[i] = 0; s_chunk[i] = 0x7fffffff; }
  __syncthreads();
  // bitonic sort: (key desc, chunk asc) first
  for (int size = 2; size <= npow2; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = tid; i < npow2; i += blockDim.x) {
        const int j = i ^ stride;
        if (j > i) {
          const bool up = (i & size) == 0;
          const uint64_t ki = s_key[i], kj = s_key[j];
          const int32_t ci = s_chunk[i], cj = s_chunk[j];
          const bool j_first = kj > ki || (kj == ki && cj < ci);
          if (j_first == up) {
            s_key[i] = kj; s_key[j] = ki;
            s_chunk[i] = cj; s_chunk[j] = ci;
          }
        }
      }
      __syncthreads();
    }
  }
  int64_t* oc = out_chunk + (int64_t)q * k;
  double* os = out_score + (int64_t)q * k;
  for (int i = tid; i < k; i += blockDim.x) {
    if (i < m) {
      oc[i] = chunk_base + s_chunk[i];
      os[i] = __longlong_as_double((long long)(s_key[i] & ~kSign));
    } else {
      oc[i] = -1;
      os[i] = -__builtin_huge_val();
    }
  }
  if (tid == 0) out_count[q] = m;
}

// ---- rl_bm25_merge_packed ----------------------------------------------------------------------------------------------
// One CTA per query merges the R sorted lists of the gathered per-shard buffers (rl_bm25_packed_bytes each) into the top
// k by (score desc, global chunk asc).  Global chunks are unique, so that order is total and every entry has one rank.
//   cut     how many entries of each list make the top want = min(k, sum of counts): a binary search over the list's
//           positions whose predicate "rank of the entry <= want" costs one lower-bound search per list (ranks are
//           counted in shared-memory integer atomics); every list halves its window each round, 13 rounds at k = 4096.
//   place   the survivors, at most k, are staged in shared memory by list; each one's output position is its index in
//           its own list plus the number of better survivors of every other list (binary searches in shared memory).
constexpr int kMergeThreads = 512;
constexpr int kMergeMaxR = 64;

struct PackedList {   // one shard's row of one query inside a gathered buffer
  const int64_t* chunk;
  const double* score;
  int n;
};

// Entries of a sorted run (score, chunk)[0, n) that come before (s, c) or are (s, c) itself.
__device__ __forceinline__ int count_at_or_before(const double* score, const int64_t* chunk, int n, double s, int64_t c) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const double sm = score[mid];
    const int64_t cm = chunk[mid];
    if (sm > s || (sm == s && cm <= c)) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ PackedList packed_list(const unsigned char* gathered, size_t stride, int r, int B, int k, int q) {
  const unsigned char* base = gathered + (size_t)r * stride;
  const size_t bk = (size_t)B * k;
  PackedList L;
  L.chunk = reinterpret_cast<const int64_t*>(base) + (size_t)q * k;
  L.score = reinterpret_cast<const double*>(base + bk * 8) + (size_t)q * k;
  L.n = min(max(reinterpret_cast<const int32_t*>(base + bk * 16)[q], 0), k);
  return L;
}

__global__ void __launch_bounds__(kMergeThreads) bm25_merge_kernel(const unsigned char* __restrict__ gathered, size_t stride,
                                                                    int R, int B, int k, int64_t* __restrict__ out_chunk,
                                                                    double* __restrict__ out_score,
                                                                    int32_t* __restrict__ out_count) {
  extern __shared__ __align__(16) unsigned char smem[];
  double* s_score = reinterpret_cast<double*>(smem);                  // [k]
  int64_t* s_chunk = reinterpret_cast<int64_t*>(s_score + k);         // [k]
  __shared__ int s_lo[kMergeMaxR], s_hi[kMergeMaxR], s_rank[kMergeMaxR], s_off[kMergeMaxR + 1];
  __shared__ int s_want;
  const int q = blockIdx.x, tid = threadIdx.x;
  if (tid < R) {
    s_lo[tid] = 0;
    s_hi[tid] = packed_list(gathered, stride, tid, B, k, q).n;
    s_rank[tid] = 0;
  }
  __syncthreads();
  if (tid == 0) {
    int total = 0;
    for (int r = 0; r < R; ++r) total += s_hi[r];
    s_want = min(total, k);
  }
  __syncthreads();
  const int want = s_want;
  // cut: afterwards s_lo[r] = the number of list r's entries among the best `want`
  for (;;) {
    const bool open = tid < R && s_lo[tid] < s_hi[tid];
    if (!__syncthreads_or(open)) break;
    for (int p = tid; p < R * R; p += blockDim.x) {
      const int r = p / R, o = p - r * R;
      const int lo = s_lo[r], hi = s_hi[r];
      if (lo >= hi) continue;
      const int mid = (lo + hi) >> 1;
      const PackedList a = packed_list(gathered, stride, r, B, k, q);
      const PackedList other = packed_list(gathered, stride, o, B, k, q);
      const int c = o == r ? mid + 1 : count_at_or_before(other.score, other.chunk, other.n, a.score[mid], a.chunk[mid]);
      atomicAdd(&s_rank[r], c);
    }
    __syncthreads();
    if (tid < R && s_lo[tid] < s_hi[tid]) {
      const int mid = (s_lo[tid] + s_hi[tid]) >> 1;
      if (s_rank[tid] <= want) s_lo[tid] = mid + 1; else s_hi[tid] = mid;
      s_rank[tid] = 0;
    }
  }
  if (tid == 0) {
    s_off[0] = 0;
    for (int r = 0; r < R; ++r) s_off[r + 1] = s_off[r] + s_lo[r];
  }
  __syncthreads();
  // place: stage the survivors list by list, then scatter each to its rank
  for (int r = 0; r < R; ++r) {
    const PackedList a = packed_list(gathered, stride, r, B, k, q);
    for (int i = tid; i < s_lo[r]; i += blockDim.x) {
      s_score[s_off[r] + i] = a.score[i];
      s_chunk[s_off[r] + i] = a.chunk[i];
    }
  }
  __syncthreads();
  int64_t* oc = out_chunk + (int64_t)q * k;
  double* os = out_score + (int64_t)q * k;
  for (int i = tid; i < want; i += blockDim.x) {
    int r = 0;
    while (s_off[r + 1] <= i) ++r;
    const double s = s_score[i];
    const int64_t c = s_chunk[i];
    int pos = i - s_off[r];
    for (int o = 0; o < R; ++o) {
      if (o != r) pos += count_at_or_before(s_score + s_off[o], s_chunk + s_off[o], s_off[o + 1] - s_off[o], s, c);
    }
    oc[pos] = c;
    os[pos] = s;
  }
  for (int i = want + tid; i < k; i += blockDim.x) {
    oc[i] = -1;
    os[i] = -__builtin_huge_val();
  }
  if (tid == 0) out_count[q] = want;
}

// ---- the query-group loop shared by rl_bm25_topk_global and rl_tsrank_topk_global ---------------------------------------
// Called once the arguments are checked and B > 0: the queries are scored in groups of as many as the workspace holds
// (G * n_chunks keys), each group by score(q0, g, keys) and then the select kernel into the packed output.  prepare()
// runs first when there is a chunk to score.
template <typename Prepare, typename ScoreLaunch>
int topk_by_groups(const char* who, int B, int k, int64_t n_chunks, int64_t chunk_base, void* out_packed, void* workspace,
                   size_t workspace_bytes, cudaStream_t st, Prepare prepare, ScoreLaunch score) {
  int group = std::min(B, 65535);
  if (n_chunks > 0) {
    const int64_t group64 = (int64_t)(workspace_bytes / ((size_t)n_chunks * sizeof(uint64_t)));
    RL_REQUIRE(group64 >= 1, RL_ENOSPACE, "%s: workspace of %zu bytes holds no query (needs %zu)", who, workspace_bytes,
               (size_t)n_chunks * sizeof(uint64_t));
    group = (int)std::min<int64_t>(group64, group);
    const int rc = prepare();
    if (rc != RL_OK) return rc;
  }
  unsigned char* out = static_cast<unsigned char*>(out_packed);
  const size_t bk = (size_t)B * k;
  int64_t* out_chunk = reinterpret_cast<int64_t*>(out);
  double* out_score = reinterpret_cast<double*>(out + bk * 8);
  int32_t* out_count = reinterpret_cast<int32_t*>(out + bk * 16);
  const size_t used = bk * 16 + (size_t)B * 4, total = ((used + 15) & ~(size_t)15);
  if (total > used) RL_CUDA_CHECK(cudaMemsetAsync(out + used, 0, total - used, st));   // the padding travels too
  const size_t sel_smem = (size_t)kBm25MaxK * (sizeof(uint64_t) + sizeof(int32_t)) + kSelBins * sizeof(uint32_t);
  RL_CUDA_CHECK(cudaFuncSetAttribute(bm25_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sel_smem));
  uint64_t* keys = static_cast<uint64_t*>(workspace);
  for (int q0 = 0; q0 < B; q0 += group) {
    const int g = min(group, B - q0);
    if (n_chunks > 0) {
      score(q0, g, keys);
      RL_CUDA_CHECK(cudaGetLastError());
    }
    bm25_select_kernel<<<g, kSelectThreads, sel_smem, st>>>(keys, n_chunks, q0, k, chunk_base, out_chunk, out_score,
                                                            out_count);
    RL_CUDA_CHECK(cudaGetLastError());
  }
  return RL_OK;
}

// g_tsrank_contrib of the current device, built on the first call that needs it.  That call waits for the table kernel
// (once per device and process), so every later call on any stream finds the table complete.
int ensure_tsrank_table(cudaStream_t st) {
  constexpr int kMaxDevices = 256;
  static std::mutex mu;
  static bool built[kMaxDevices] = {};
  int dev = 0;
  RL_CUDA_CHECK(cudaGetDevice(&dev));
  RL_REQUIRE(dev >= 0 && dev < kMaxDevices, RL_EINVAL, "rl_tsrank_topk_global: device %d out of range", dev);
  std::lock_guard<std::mutex> lock(mu);
  if (!built[dev]) {
    tsrank_table_kernel<<<1, kTsMaxPos, 0, st>>>();
    RL_CUDA_CHECK(cudaGetLastError());
    RL_CUDA_CHECK(cudaStreamSynchronize(st));
    built[dev] = true;
  }
  return RL_OK;
}

}  // namespace
}  // namespace rl

using namespace rl;

extern "C" int rl_bm25_stats(const int64_t* term_off, const int32_t* doc, const int32_t* doc_len, const uint8_t* chunk_alive,
                             int64_t n_terms, int64_t n_chunks, int32_t* df, double* corpus, void* stream) {
  RL_REQUIRE(n_terms >= 0 && n_chunks >= 0 && n_chunks <= INT32_MAX, RL_EINVAL, "rl_bm25_stats: bad sizes");
  RL_REQUIRE(term_off && corpus && (n_chunks == 0 || doc_len) && (n_terms == 0 || (doc && df)), RL_EINVAL,
             "rl_bm25_stats: null pointer");
  bm25_corpus_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(doc_len, chunk_alive, n_chunks, corpus);
  RL_CUDA_CHECK(cudaGetLastError());
  if (n_terms > 0) {
    const int grid = (int)std::min<int64_t>(n_terms, 1 << 16);
    bm25_df_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(term_off, doc, chunk_alive, n_terms, df);
    RL_CUDA_CHECK(cudaGetLastError());
  }
  return RL_OK;
}

extern "C" size_t rl_bm25_workspace_bytes(int64_t n_chunks, int group) {
  if (n_chunks <= 0 || group <= 0) return 0;
  return (size_t)group * (size_t)n_chunks * sizeof(uint64_t);
}

extern "C" size_t rl_bm25_packed_bytes(int B, int k) {
  if (B <= 0 || k <= 0) return 0;
  const size_t raw = (size_t)B * (size_t)k * 16 + (size_t)B * 4;
  return (raw + 15) & ~(size_t)15;
}

extern "C" int rl_bm25_topk_global(const int64_t* term_off, const int32_t* doc, const int32_t* tf, const int32_t* doc_len,
                                   const int64_t* stats, int64_t n_terms, int64_t n_chunks, const uint8_t* chunk_mask,
                                   const int32_t* q_off, const int32_t* q_terms, int B, int k, double k1, double b,
                                   int64_t chunk_base, void* out_packed, void* workspace, size_t workspace_bytes,
                                   void* stream) {
  RL_REQUIRE(B >= 0 && n_terms >= 0 && n_chunks >= 0 && n_chunks <= INT32_MAX && chunk_base >= 0, RL_EINVAL,
             "rl_bm25_topk_global: bad sizes");
  RL_REQUIRE(k >= 1 && k <= kBm25MaxK, RL_EINVAL, "rl_bm25_topk_global: k=%d outside [1, %d]", k, kBm25MaxK);
  RL_REQUIRE(k1 >= 0.0 && b >= 0.0 && b <= 1.0, RL_EINVAL, "rl_bm25_topk_global: k1 must be >= 0 and b in [0, 1]");
  if (B == 0) return RL_OK;
  RL_REQUIRE(term_off && stats && q_off && out_packed && (n_chunks == 0 || (doc_len && workspace)) &&
                 (n_terms == 0 || n_chunks == 0 || (doc && tf)),
             RL_EINVAL, "rl_bm25_topk_global: null pointer");
  RL_REQUIRE(((uintptr_t)out_packed & 15) == 0 && ((uintptr_t)workspace & 7) == 0, RL_EINVAL,
             "rl_bm25_topk_global: out_packed must be 16-byte and workspace 8-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned n_tiles = (unsigned)((n_chunks + kTile - 1) / kTile);
  return topk_by_groups("rl_bm25_topk_global", B, k, n_chunks, chunk_base, out_packed, workspace, workspace_bytes, st,
                        [] { return (int)RL_OK; }, [&](int q0, int g, uint64_t* keys) {
                          bm25_score_kernel<<<dim3(n_tiles, g), kScoreThreads, 0, st>>>(
                              term_off, doc, tf, doc_len, stats, n_terms, n_chunks, chunk_mask, q_off, q_terms, q0, k1, b,
                              keys);
                        });
}

extern "C" int rl_tsrank_topk_global(const int64_t* term_off, const int32_t* doc, const int32_t* npos, int64_t n_terms,
                                     int64_t n_chunks, const uint8_t* chunk_mask, const int32_t* q_off,
                                     const int32_t* q_terms, int B, int k, int64_t chunk_base, void* out_packed,
                                     void* workspace, size_t workspace_bytes, void* stream) {
  RL_REQUIRE(B >= 0 && n_terms >= 0 && n_chunks >= 0 && n_chunks <= INT32_MAX && chunk_base >= 0, RL_EINVAL,
             "rl_tsrank_topk_global: bad sizes");
  RL_REQUIRE(k >= 1 && k <= kBm25MaxK, RL_EINVAL, "rl_tsrank_topk_global: k=%d outside [1, %d]", k, kBm25MaxK);
  if (B == 0) return RL_OK;
  RL_REQUIRE(term_off && q_off && out_packed && (n_chunks == 0 || workspace) &&
                 (n_terms == 0 || n_chunks == 0 || (doc && npos)),
             RL_EINVAL, "rl_tsrank_topk_global: null pointer");
  RL_REQUIRE(((uintptr_t)out_packed & 15) == 0 && ((uintptr_t)workspace & 7) == 0, RL_EINVAL,
             "rl_tsrank_topk_global: out_packed must be 16-byte and workspace 8-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned n_tiles = (unsigned)((n_chunks + kTile - 1) / kTile);
  return topk_by_groups("rl_tsrank_topk_global", B, k, n_chunks, chunk_base, out_packed, workspace, workspace_bytes, st,
                        [&] { return ensure_tsrank_table(st); }, [&](int q0, int g, uint64_t* keys) {
                          tsrank_score_kernel<<<dim3(n_tiles, g), kScoreThreads, 0, st>>>(
                              term_off, doc, npos, n_terms, n_chunks, chunk_mask, q_off, q_terms, q0, keys);
                        });
}

extern "C" int rl_bm25_merge_packed(const void* gathered, int R, int B, int k, int64_t* out_chunk, double* out_score,
                                    int32_t* out_count, void* stream) {
  RL_REQUIRE(R >= 1 && R <= kMergeMaxR && B >= 0, RL_EINVAL, "rl_bm25_merge_packed: R=%d outside [1, %d] or B < 0", R,
             kMergeMaxR);
  RL_REQUIRE(k >= 1 && k <= kBm25MaxK, RL_EINVAL, "rl_bm25_merge_packed: k=%d outside [1, %d]", k, kBm25MaxK);
  if (B == 0) return RL_OK;
  RL_REQUIRE(gathered && out_chunk && out_score && out_count, RL_EINVAL, "rl_bm25_merge_packed: null pointer");
  RL_REQUIRE(((uintptr_t)gathered & 15) == 0, RL_EINVAL, "rl_bm25_merge_packed: gathered must be 16-byte aligned");
  const size_t smem = (size_t)k * (sizeof(double) + sizeof(int64_t));
  RL_CUDA_CHECK(cudaFuncSetAttribute(bm25_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaStream_t st = (cudaStream_t)stream;
  const size_t stride = rl_bm25_packed_bytes(B, k);
  bm25_merge_kernel<<<B, kMergeThreads, smem, st>>>(static_cast<const unsigned char*>(gathered), stride, R, B, k, out_chunk,
                                                    out_score, out_count);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}
