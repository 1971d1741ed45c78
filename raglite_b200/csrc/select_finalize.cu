// Selection side of the MaxSim scan (sm_90a): query prep, the radix select that turns the sampled
// scores into per-query emission thresholds, the finalize pass (radix select over the candidate
// list, exact float64 rescoring with warp-shuffle reductions, bitonic sort, GROUP BY chunk) and the
// cross-shard merge.
//
// Reference semantics restated here: _search.py:75-79 (ORDER BY dist LIMIT num_hits) and
// _search.py:143-150 (GROUP BY chunk_id, max(sim), ORDER BY sim DESC LIMIT num_results).
#include <cuda_fp16.h>

#include "select_finalize.cuh"

namespace rl {

constexpr int kSelThreads = 512;
constexpr int kBins = 4096;

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- block-cooperative order statistic ---------------------------------------------------------
// Warp 0: find the histogram bin holding the K-th largest element (counting from the top bin).
// Returns through shared memory: res[0] = bin (or -1 if fewer than K elements), res[1] = count above.
__device__ void find_bin_from_top(const uint32_t* hist, int K, int* res) {
  if (threadIdx.x >= 32) return;
  const int lane = threadIdx.x;
  constexpr int kPer = kBins / 32;
  uint32_t lane_sum = 0;
  for (int i = 0; i < kPer; ++i) lane_sum += hist[lane * kPer + i];
  // inclusive suffix sum over lanes (lane 31 holds the top bins)
  uint32_t suf = lane_sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t v = __shfl_down_sync(0xffffffffu, suf, o);
    if (lane + o < 32) suf += v;
  }
  const uint32_t above_lane = suf - lane_sum;  // elements in lanes above this one
  const bool mine = (above_lane < (uint32_t)K) && (suf >= (uint32_t)K);
  const uint32_t vote = __ballot_sync(0xffffffffu, mine);
  if (vote == 0) {
    if (lane == 0) { res[0] = -1; res[1] = 0; }
    return;
  }
  if (mine) {
    uint32_t above = above_lane;
    int bin = lane * kPer + kPer - 1;
    for (; bin >= lane * kPer; --bin) {
      const uint32_t h = hist[bin];
      if (above + h >= (uint32_t)K) break;
      above += h;
    }
    res[0] = bin;
    res[1] = (int)above;
  }
}

// Narrow n 64-bit composites -- larger = better, 0 = absent, the non-zero ones all distinct -- to the K best plus at
// most (window - K) more, by a radix select over the composite from the top digit down (12 bits per pass; at full
// resolution a digit holds one composite, so the loop always ends inside the window), and gather ~composite (an
// ascending sort key) into out[0 .. *count).  All threads of the block must call it; comp_of(i) may read global memory.
template <class Comp>
__device__ void block_gather_top(int n, int K, int window, Comp comp_of, uint64_t* out, uint32_t* hist, int* res, int* count) {
  uint64_t prefix = 0;      // value of the top `bits` bits of the K-th largest composite
  int bits = 0, need = K;
  while (bits < 64) {
    const int w = min(12, 64 - bits);
    const int shift = 64 - bits - w;
    for (int i = threadIdx.x; i < kBins; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const uint64_t c = comp_of(i);
      if (c != 0ull && (bits == 0 || (c >> (64 - bits)) == prefix)) atomicAdd(&hist[(uint32_t)(c >> shift) & ((1u << w) - 1u)], 1u);
    }
    __syncthreads();
    find_bin_from_top(hist, need, res);
    __syncthreads();
    const int bin = res[0] < 0 ? 0 : res[0];     // < 0: fewer than `need` composites left -> take everything
    const int above = res[0] < 0 ? 0 : res[1];
    const int in_bin = (int)hist[bin];
    const bool all = res[0] < 0;
    __syncthreads();
    prefix = (prefix << w) | (uint64_t)bin;
    bits += w;
    need -= above;
    // composites with top bits > prefix number K - need; those == prefix number in_bin
    if (all || (K - need) + in_bin <= window) break;
  }
  if (threadIdx.x == 0) *count = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const uint64_t c = comp_of(i);
    if (c != 0ull && (c >> (64 - bits)) >= prefix) {
      const int pos = atomicAdd(count, 1);
      if (pos < window) out[pos] = ~c;
    }
  }
  __syncthreads();
}

// Lower bound (24-bit bin edge, i.e. within 2^-15 relative) of the K-th largest of get(0..n).
// -inf when fewer than K finite values exist.  All threads of the block must call it.
template <class Get>
__device__ float block_kth_largest_lb(int64_t n, int K, Get get, uint32_t* hist, int* res) {
  for (int i = threadIdx.x; i < kBins; i += blockDim.x) hist[i] = 0;
  __syncthreads();
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) atomicAdd(&hist[f2ord(get(i)) >> 20], 1u);
  __syncthreads();
  find_bin_from_top(hist, K, res);
  __syncthreads();
  const int bin1 = res[0];
  const int above1 = res[1];
  __syncthreads();
  if (bin1 <= 7) return kNegInf;  // bins 0..7 hold -inf / negative NaN patterns only
  for (int i = threadIdx.x; i < kBins; i += blockDim.x) hist[i] = 0;
  __syncthreads();
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const uint32_t o = f2ord(get(i));
    if ((int)(o >> 20) == bin1) atomicAdd(&hist[(o >> 8) & 0xFFFu], 1u);
  }
  __syncthreads();
  find_bin_from_top(hist, K - above1, res);
  __syncthreads();
  const int bin2 = res[0] < 0 ? 0 : res[0];
  __syncthreads();
  return ord2f(((uint32_t)bin1 << 20) | ((uint32_t)bin2 << 8));
}

// Ascending bitonic sort of n (power of two) keys in shared memory.
template <class K>
__device__ void bitonic_sort(K* keys, int n) {
  for (int k = 2; k <= n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const K x = keys[i], y = keys[ixj];
          const bool up = (i & k) == 0;
          if ((x > y) == up) { keys[i] = y; keys[ixj] = x; }
        }
      }
      __syncthreads();
    }
  }
}
__device__ void bitonic_sort_u64(uint64_t* keys, int n) { bitonic_sort<uint64_t>(keys, n); }

// Cheap lower bound of the K-th largest of a value stream: every thread keeps the T largest values
// it is handed in registers (one streaming pass, no atomics), the blockDim*T kept values are sorted in
// shared memory and the K-th largest of that subset is returned (a subset's order statistic never
// exceeds the full set's).  -inf if K > blockDim*T.  `for_each(cb)` must call cb(value) for every
// value exactly once across the block.  scratch: blockDim*T words.
template <int T, class ForEach>
__device__ float block_topk_lower_bound(ForEach for_each, int K, uint32_t* scratch) {
  float top[T];
#pragma unroll
  for (int i = 0; i < T; ++i) top[i] = kNegInf;
  for_each([&](float x) {
    if (x > top[T - 1]) {
      top[T - 1] = x;
#pragma unroll
      for (int j = T - 1; j > 0; --j) {
        if (top[j] > top[j - 1]) { const float tmp = top[j]; top[j] = top[j - 1]; top[j - 1] = tmp; }
      }
    }
  });
  const int total = (int)blockDim.x * T;
#pragma unroll
  for (int i = 0; i < T; ++i) scratch[threadIdx.x * T + i] = f2ord(top[i]);
  __syncthreads();
  bitonic_sort<uint32_t>(scratch, total);   // total is a power of two (512 * {1,4,8})
  const float lb = K <= total ? ord2f(scratch[total - K]) : kNegInf;
  __syncthreads();
  return lb;
}
template <class ForEach>
__device__ float block_topk_lower_bound_any(ForEach for_each, int K, uint32_t* scratch) {
  if (K <= kSelThreads) return block_topk_lower_bound<1>(for_each, K, scratch);
  if (K <= 4 * kSelThreads) return block_topk_lower_bound<4>(for_each, K, scratch);
  return block_topk_lower_bound<8>(for_each, K, scratch);
}

// ---- query prep ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) query_prep_kernel(const float* __restrict__ Q, int B, int d, int metric,
                                                         int algo, const float* __restrict__ row_stats,
                                                         double* __restrict__ q_sq, float* __restrict__ q_inv,
                                                         float* __restrict__ eps) {
  __shared__ double red[4], red1[4];
  const int b = blockIdx.x;
  double s = 0.0, s1 = 0.0;
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    const double v = Q[(size_t)b * d + c];
    s += v * v;
    s1 += fabs(v);
  }
  s = warp_sum_d(s);
  s1 = warp_sum_d(s1);
  if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5] = s; red1[threadIdx.x >> 5] = s1; }
  __syncthreads();
  if (threadIdx.x == 0 && metric == RL_METRIC_L1) {
    // L1 scan: each key is -fl(sum_i |fl(e_i - q_i)|), summed sequentially in float32 (scan_l1.cu), so
    // |key + sum |e - q|| <= gamma_d * sum |e - q| <= d u (1 + O(d u)) (sum |e| + sum |q|), u = 2^-24; the fp16 -> fp32
    // row conversion is exact.  sum |e| <= min(sqrt(d) max |e|_2, d max |e_ij|) from row_stats.  The same
    // (d + 8) 2^-23 factor as the fp32 scan leaves a factor 2 of slack.
    const double sum_q = red1[0] + red1[1] + red1[2] + red1[3];
    const double sum_e = fmin(sqrt((double)d) * (double)row_stats[0], (double)d * (double)row_stats[1]);
    q_sq[b] = red[0] + red[1] + red[2] + red[3];
    q_inv[b] = 0.f;
    eps[b] = (float)((double)(d + 8) * 1.1920928955078125e-7 * (sum_q + sum_e));
    return;
  }
  if (threadIdx.x == 0) {
    const double nq = red[0] + red[1] + red[2] + red[3];
    q_sq[b] = nq;
    const float qn = (float)sqrt(nq);
    q_inv[b] = nq > 0.0 ? (float)(1.0 / sqrt(nq)) : 0.f;
    const float max_norm = row_stats ? row_stats[0] : 1.f;
    // Worst-case error of the approximate key in key units.  fp32 scan: accumulation error
    // <= d * 2^-24 * |q||e| (doubled for slack); fp16-input tensor-core scan: inputs rounded to 11 bits
    // => 2^-10 (1 + 2^-11) |q||e| plus fp32 accumulation plus fp16 subnormal absolute terms.
    const float base = algo == RL_ALGO_TCGEN05 ? (1.25e-3f + (float)(d + 8) * 1.1920929e-7f)
                                               : (float)(d + 8) * 1.1920929e-7f;
    float e;
    if (metric == RL_METRIC_COSINE) e = base;
    else if (metric == RL_METRIC_DOT) e = base * qn * max_norm;
    else e = base * (2.f * qn * max_norm + max_norm * max_norm);
    eps[b] = e;
  }
}

// ---- sample select + emit from the dump -----------------------------------------------------------
constexpr int kSelListCap = 8192;

__device__ __forceinline__ int32_t sample_row_of(int64_t p, int S) {
  return (int32_t)((p / kBlockRows) * S * kBlockRows + (p % kBlockRows));
}

// Walk the sampled keys of one query: cb(p, v, sv) with v = the row's approximate key and sv = the
// value that takes part in the order statistic -- v itself (SQL semantics) or, for exact MaxSim, the
// max over the run of sample rows one chunk owns, reported once at the head of the run (-inf
// elsewhere).  A warp owns 32 consecutive sample rows (coalesced loads of keys and owners, kU segments
// in flight); the run max is a segmented suffix max over the warp (shuffles).  A sampled row is a head
// exactly when it is the first row of its chunk, whether or not the row before it was sampled: with
// S > 1 a chunk that spans two sampled blocks would otherwise be counted once in each and lift the
// statistic above the shard's sel_k-th chunk maximum.  Runs are cut at 32-row segment and sampled
// block boundaries; a continuation is not a head, so a chunk is counted at most once and a partial
// max only lowers the statistic (it must be a lower bound).
template <class CB>
__device__ void for_each_sample(const SelectArgs& a, const float* __restrict__ dump, int64_t n, CB cb) {
  constexpr int kU = 4;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int64_t n_seg = n / 32;  // n is a multiple of kBlockRows
  for (int64_t seg0 = (int64_t)warp * kU; seg0 < n_seg; seg0 += (int64_t)nw * kU) {
    float v[kU];
    int32_t c[kU], cprev0[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const int64_t p = (seg0 + u) * 32 + lane;
      v[u] = seg0 + u < n_seg ? dump[p] : kNegInf;
      c[u] = -1 - lane;
      cprev0[u] = -100;
      if (!a.mode_sql && seg0 + u < n_seg) {
        const int64_t row = sample_row_of(p, a.S);
        if (row < a.n_rows) {
          c[u] = a.row_chunk[row];
          // Owner of the row before lane 0 (sampled or not): lane 0 is a head only at its chunk's first row.
          if (lane == 0 && row > 0) cprev0[u] = a.row_chunk[row - 1];
        }
      }
    }
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      if (seg0 + u >= n_seg) break;
      const int64_t p = (seg0 + u) * 32 + lane;
      if (a.mode_sql) {
        cb(p, v[u], v[u]);
      } else {
        int32_t cp = __shfl_up_sync(0xffffffffu, c[u], 1);
        if (lane == 0) cp = cprev0[u];
        const bool head = c[u] >= 0 && c[u] != cp;
        float m = v[u];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const float m2 = __shfl_down_sync(0xffffffffu, m, o);
          const int32_t c2 = __shfl_down_sync(0xffffffffu, c[u], o);
          if (lane + o < 32 && c2 == c[u]) m = fmaxf(m, m2);
        }
        cb(p, v[u], head ? m : kNegInf);
      }
    }
  }
}

__global__ void __launch_bounds__(kSelThreads) select_kernel(const SelectArgs a) {
  extern __shared__ __align__(16) unsigned char sel_smem[];
  uint32_t* hist = reinterpret_cast<uint32_t*>(sel_smem);                   // [kBins] / top-T scratch [4096]
  Cand* elist = reinterpret_cast<Cand*>(hist + kBins);                      // [kSelListCap] sample rows >= LB - 2 eps
  float* slist = reinterpret_cast<float*>(elist + kSelListCap);             // [kSelListCap] selection values >= LB
  __shared__ int res[2];
  __shared__ int n_e, n_s, n_out;
  const int b = blockIdx.x;
  const float* dump = a.dump + (size_t)b * a.n_sample_rows;
  const int64_t n = a.n_sample_rows;
  const float eps2 = 2.f * a.eps[b];

  // Per-position fallback spelling of the selection value (only used on degenerate inputs).
  auto sel_value_slow = [&](int64_t p) -> float {
    if (a.mode_sql) return dump[p];
    const int r_in = (int)(p % kBlockRows);
    const int64_t row = sample_row_of(p, a.S);
    if (row >= a.n_rows) return kNegInf;
    const int32_t c = a.row_chunk[row];
    if (row > 0 && a.row_chunk[row - 1] == c) return kNegInf;  // not the first row of its chunk
    float m = dump[p];
    for (int j = 1; (r_in + j < kBlockRows || a.S == 1) && p + j < n && row + j < a.n_rows && a.row_chunk[row + j] == c; ++j)
      m = fmaxf(m, dump[p + j]);
    return m;
  };

  if (threadIdx.x == 0) { n_e = 0; n_s = 0; n_out = 0; }
  __syncthreads();
  float thr;
  float inv_w = eps2 > 0.f ? 1.f / (2.f * eps2) : 0.f;   // default bin width 4 eps
  bool listed = false;   // elist holds every sample row >= thr
  if (a.reuse_thr) {
    thr = a.thr[b];
    if (threadIdx.x == 0) a.hist_inv_w[b] = inv_w;
  } else {
    // 1) cheap lower bound LB of the sel_k-th largest selection value
    const float LB = block_topk_lower_bound_any(
        [&](auto push) { for_each_sample(a, dump, n, [&](int64_t, float, float sv) { push(sv); }); }, a.sel_k, hist);
    // 2) one more streaming pass collects the few values at or above the bound
    const float lo = LB - eps2;
    for_each_sample(a, dump, n, [&](int64_t p, float v, float sv) {
      if (v >= lo && v > kNegInf) {
        const int i = atomicAdd(&n_e, 1);
        if (i < kSelListCap) elist[i] = Cand{v, sample_row_of(p, a.S)};
      }
      if (!a.mode_sql && sv >= LB && sv > kNegInf) {
        const int i = atomicAdd(&n_s, 1);
        if (i < kSelListCap) slist[i] = sv;
      }
    });
    __syncthreads();
    float T;
    if (LB > kNegInf && n_e <= kSelListCap && n_s <= kSelListCap) {
      // 3) order statistic over the short list in shared memory
      if (a.mode_sql) {
        T = block_kth_largest_lb(n_e, a.sel_k, [&](int64_t i) { const float v = elist[i].key; return v >= LB ? v : kNegInf; }, hist, res);
      } else {
        T = block_kth_largest_lb(n_s, a.sel_k, [&](int64_t i) { return slist[i]; }, hist, res);
      }
      listed = true;
    } else {  // degenerate distributions (massive ties, tiny samples): full streaming radix select
      T = block_kth_largest_lb(n, a.sel_k, sel_value_slow, hist, res);
    }
    thr = T - eps2;
    // Histogram bin width for the online refinement.  The tail of the score distribution is roughly
    // exponential: with T2 = the (sel_k/4)-th largest sample value, (T2 - T) / ln 4 estimates its decay
    // length, and the shard-wide sel_k-th largest sits about ln(S) decay lengths above T.  Spread the
    // bins over 1.5x that distance (an outlier-proof estimate: single planted neighbours do not move it).
    float w = 2.f * eps2;   // 4 eps
    if (listed && a.S > 1) {
      const int k2 = max(1, a.sel_k / 4);
      float T2;
      if (a.mode_sql) {
        T2 = block_kth_largest_lb(n_e, k2, [&](int64_t i) { return elist[i].key; }, hist, res);
      } else {
        T2 = block_kth_largest_lb(n_s, k2, [&](int64_t i) { return slist[i]; }, hist, res);
      }
      if (T2 > T) {
        const float gap = (T2 - T) * (__logf((float)a.S) / __logf((float)(a.sel_k >= 4 ? 4 : a.sel_k + 1)));
        w = fmaxf(w, 1.5f * gap / (float)(kHistBins - 1));
      }
    }
    inv_w = w > 0.f ? 1.f / w : 0.f;
    if (threadIdx.x == 0) {
      a.thr[b] = thr;
      a.hist_inv_w[b] = inv_w;
    }
  }
  // Sample rows that pass the threshold join the candidate list like any emitted row.  Nothing else
  // writes this query's list before the main scan starts, so slots are handed out block-locally.
  Cand* out = a.cand + (size_t)b * a.cap;
  int32_t* gh = a.ghist + (size_t)b * kHistBins;
  if (listed) {
    const int ne = n_e;
    for (int i = threadIdx.x; i < ne; i += blockDim.x) {
      const Cand c = elist[i];
      if (c.key >= thr) {
        const int slot = atomicAdd(&n_out, 1);
        if (slot < a.cap) out[slot] = c;
        atomicAdd(gh + hist_bin(c.key, thr, inv_w), 1);
      }
    }
  } else {
    for (int64_t p = threadIdx.x; p < n; p += blockDim.x) {
      const float v = dump[p];
      if (v >= thr && v > kNegInf) {
        const int slot = atomicAdd(&n_out, 1);
        if (slot < a.cap) out[slot] = Cand{v, sample_row_of(p, a.S)};
        atomicAdd(gh + hist_bin(v, thr, inv_w), 1);
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) a.cand_cnt[b] = n_out;
}

// ---- finalize --------------------------------------------------------------------------------------
// d2 = sum (e - q)^2, accumulated directly: ne + nq - 2 dot cancels to its rounding error for a row that (nearly)
// duplicates a query of large norm.  For l1 the last argument is d1 = sum |e - q| instead.
__device__ __forceinline__ float exact_sim(int metric, double dot, double ne, double nq, double d2) {
  if (metric == RL_METRIC_L1) return 1.0f - (float)d2;   // the FLOAT the SQL returns, then sim = 1 - dist
  if (metric == RL_METRIC_COSINE) {
    double s = dot / sqrt(ne * nq);
    s = fmin(1.0, fmax(-1.0, s));
    const float dist = 1.0f - (float)s;  // array_cosine_distance returns FLOAT
    return 1.0f - dist;                  // sim = 1 - dist (_search.py:72)
  }
  if (metric == RL_METRIC_DOT) return 1.0f - (float)(-dot);
  return 1.0f - (float)sqrt(d2);
}

// flags[i] = 1 when no j < i has the same group id.  O(n^2 / threads); n is a few hundred.
template <class T>
__device__ void first_occurrence(const T* ids, int n, uint8_t* flags) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const T c = ids[i];
    uint8_t f = 1;
    for (int j = 0; j < i; ++j)
      if (ids[j] == c) { f = 0; break; }
    flags[i] = f;
  }
  __syncthreads();
}

// Ordered compaction positions: pos[i] = number of set flags before i.  Single-warp scan (n small).
__device__ void exclusive_scan_flags(const uint8_t* flags, int n, int* pos) {
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += blockDim.x) {
    const int i = base + threadIdx.x;
    const int f = (i < n) ? flags[i] : 0;
    // block-wide inclusive scan via warp scans
    __shared__ int wsum[32];
    int v = f;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += t;
    }
    if (lane == 31) wsum[w] = v;
    __syncthreads();
    if (w == 0) {
      int s = (lane < (int)(blockDim.x >> 5)) ? wsum[lane] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, s, o);
        if (lane >= o) s += t;
      }
      wsum[lane] = s;
    }
    __syncthreads();
    const int before = carry + (w > 0 ? wsum[w - 1] : 0) + v - f;
    if (i < n) pos[i] = before;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry = before + f;
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kSelThreads) finalize_kernel(const FinalizeArgs f) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint64_t* keys = reinterpret_cast<uint64_t*>(smem_raw);                      // [RL_MAX_SURVIVORS]
  int32_t* rows = reinterpret_cast<int32_t*>(keys + RL_MAX_SURVIVORS);         // [RL_MAX_SURVIVORS] (later: chunk ids)
  uint32_t* hist = reinterpret_cast<uint32_t*>(rows + RL_MAX_SURVIVORS);       // kFinalizeScratch bytes
  float* qv = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(hist) + kFinalizeScratch);  // [d]
  __shared__ int res[2];
  __shared__ int s_count;

  const int b = blockIdx.x;
  if (b == 0 && threadIdx.x == 0 && f.header != nullptr) {
    f.header->launches = f.launches;
    f.header->sample_stride = f.S;
    f.header->cand_cap = f.cap;
    f.header->algo = f.algo;
    f.header->n_sample_rows = f.n_sample_rows;
    f.header->counted_unfiltered = f.counted_unfiltered;
  }
  const int cnt = f.cand_cnt[b];
  const int n = min(cnt, f.cap);
  int st = cnt > f.cap ? RL_STATUS_CAND_OVERFLOW : 0;
  if (f.metric == RL_METRIC_L1 && !isfinite(f.q_sq[b])) st |= RL_STATUS_QUERY_NONFINITE;   // (q_sq is finite for finite q)
  const Cand* cand = f.cand + (size_t)b * f.cap;

  __shared__ int s_coll;
  const float eps2 = 2.f * f.eps[b];
  if (threadIdx.x == 0) { s_count = 0; s_coll = 0; }
  for (int c = threadIdx.x; c < f.d; c += blockDim.x) qv[c] = f.Q[(size_t)b * f.d + c];
  // 1) cheap lower bound of the sel_k-th largest approximate key (per-thread top-T, no atomics)
  auto key_of = [&](int64_t i) { return cand[i].key; };
  auto for_each_cand = [&](auto cb) {   // 4 independent 8-byte loads in flight per thread
    constexpr int kU = 4;
    for (int i0 = threadIdx.x; i0 < n; i0 += blockDim.x * kU) {
      Cand c[kU];
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int i = i0 + u * blockDim.x;
        c[u] = i < n ? cand[i] : Cand{kNegInf, 0};
      }
#pragma unroll
      for (int u = 0; u < kU; ++u)
        if (i0 + u * (int)blockDim.x < n) cb(c[u]);
    }
  };
  const float LB = block_topk_lower_bound_any([&](auto push) { for_each_cand([&](const Cand& c) { push(c.key); }); },
                                              f.sel_k, hist);
  // 2) collect the candidates at or above it; the order statistic then runs on that short list
  const float lo = LB - eps2;
  for_each_cand([&](const Cand& c) {
    if (c.key >= lo) {
      const int pos = atomicAdd(&s_coll, 1);
      if (pos < RL_MAX_SURVIVORS) keys[pos] = ((uint64_t)f2ord(c.key) << 32) | (uint32_t)c.row;
    }
  });
  __syncthreads();
  const int n_coll = s_coll;
  float cut;
  if (LB > kNegInf && n_coll <= RL_MAX_SURVIVORS) {
    const float T = block_kth_largest_lb(n_coll, f.sel_k, [&](int64_t i) {
      const float v = ord2f((uint32_t)(keys[i] >> 32));
      return v >= LB ? v : kNegInf; }, hist, res);
    cut = T - eps2;
    for (int i = threadIdx.x; i < n_coll; i += blockDim.x) {
      const uint64_t kk = keys[i];
      if (ord2f((uint32_t)(kk >> 32)) >= cut) {
        const int pos = atomicAdd(&s_count, 1);
        rows[pos] = (int32_t)(uint32_t)kk;   // pos < n_coll <= RL_MAX_SURVIVORS
      }
    }
  } else {  // degenerate (massive ties / fewer than sel_k candidates): streaming radix select
    const float T = block_kth_largest_lb(n, f.sel_k, key_of, hist, res);
    cut = T - eps2;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const Cand c = cand[i];
      if (c.key >= cut) {
        const int pos = atomicAdd(&s_count, 1);
        if (pos < RL_MAX_SURVIVORS) rows[pos] = c.row;
      }
    }
  }
  if (threadIdx.x == 0) f.thr_out[b] = cut;
  __syncthreads();
  const int ns_all = s_count;
  int ns = min(ns_all, RL_MAX_SURVIVORS);

  // Exact rescoring of one row by one warp: float64 dot / norm, warp-shuffle reduction.
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const double nq = f.q_sq[b];
  const bool vec = (f.d % 4 == 0) && (f.ld % 4 == 0) && ((reinterpret_cast<uintptr_t>(f.E) & 15) == 0);
  // l2 needs only d2 = sum (e - q)^2, cosine and dot only dot and ne: one loop each, chosen once per row (the metric
  // is uniform per launch), so the cosine / dot loop is the one it always was.
  const bool l2 = f.metric == RL_METRIC_L2;
  const bool l1 = f.metric == RL_METRIC_L1;
  auto exact_row_sim = [&](int32_t row) -> float {   // all 32 lanes call it; every lane gets the result
    const float* e = f.E + (int64_t)row * f.ld;
    double dot = 0.0, ne = 0.0, d2 = 0.0;
    if (l1) {   // d1 = sum |e - q| in float64, the loop layout of the l2 one
      double d1 = 0.0;
      if (f.e_f16) {
        const __half* eh = reinterpret_cast<const __half*>(f.E) + (int64_t)row * f.ld;
        for (int c = lane * 8; c < f.d; c += 256) {
          const uint4 v = __ldg(reinterpret_cast<const uint4*>(eh + c));
          const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
          for (int k2 = 0; k2 < 4; ++k2) {
            const float2 ev = __half22float2(h[k2]);
            d1 += fabs((double)ev.x - qv[c + 2 * k2]) + fabs((double)ev.y - qv[c + 2 * k2 + 1]);
          }
        }
      } else if (vec) {
        for (int c = lane * 4; c < f.d; c += 128) {
          const float4 ev = __ldg(reinterpret_cast<const float4*>(e + c));
          const float4 qq = *reinterpret_cast<const float4*>(qv + c);
          d1 += fabs((double)ev.x - qq.x) + fabs((double)ev.y - qq.y) + fabs((double)ev.z - qq.z) + fabs((double)ev.w - qq.w);
        }
      } else {
        for (int c = lane; c < f.d; c += 32) d1 += fabs((double)__ldg(e + c) - qv[c]);
      }
      d1 = warp_sum_d(d1);
      return exact_sim(f.metric, dot, ne, nq, d1);
    }
    if (l2) {
      if (f.e_f16) {
        const __half* eh = reinterpret_cast<const __half*>(f.E) + (int64_t)row * f.ld;
        for (int c = lane * 8; c < f.d; c += 256) {
          const uint4 v = __ldg(reinterpret_cast<const uint4*>(eh + c));
          const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
          for (int k2 = 0; k2 < 4; ++k2) {
            const float2 ev = __half22float2(h[k2]);
            const double tx = (double)ev.x - qv[c + 2 * k2], ty = (double)ev.y - qv[c + 2 * k2 + 1];
            d2 += tx * tx + ty * ty;
          }
        }
      } else if (vec) {
        for (int c = lane * 4; c < f.d; c += 128) {
          const float4 ev = __ldg(reinterpret_cast<const float4*>(e + c));
          const float4 qq = *reinterpret_cast<const float4*>(qv + c);
          const double tx = (double)ev.x - qq.x, ty = (double)ev.y - qq.y, tz = (double)ev.z - qq.z, tw = (double)ev.w - qq.w;
          d2 += tx * tx + ty * ty + tz * tz + tw * tw;
        }
      } else {
        for (int c = lane; c < f.d; c += 32) {
          const double t = (double)__ldg(e + c) - qv[c];
          d2 += t * t;
        }
      }
      d2 = warp_sum_d(d2);
      return exact_sim(f.metric, dot, ne, nq, d2);
    }
    if (f.e_f16) {   // float16 storage: 8 halves per 16-byte load (d % 8 == 0)
      const __half* eh = reinterpret_cast<const __half*>(f.E) + (int64_t)row * f.ld;
      for (int c = lane * 8; c < f.d; c += 256) {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(eh + c));
        const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
        for (int k2 = 0; k2 < 4; ++k2) {
          const float2 ev = __half22float2(h[k2]);
          dot += (double)ev.x * qv[c + 2 * k2] + (double)ev.y * qv[c + 2 * k2 + 1];
          ne += (double)ev.x * ev.x + (double)ev.y * ev.y;
        }
      }
    } else if (vec) {
      for (int c = lane * 4; c < f.d; c += 128) {
        const float4 ev = __ldg(reinterpret_cast<const float4*>(e + c));
        const float4 qq = *reinterpret_cast<const float4*>(qv + c);
        dot += (double)ev.x * qq.x + (double)ev.y * qq.y + (double)ev.z * qq.z + (double)ev.w * qq.w;
        ne += (double)ev.x * ev.x + (double)ev.y * ev.y + (double)ev.z * ev.z + (double)ev.w * ev.w;
      }
    } else {
      for (int c = lane; c < f.d; c += 32) {
        const double ev = __ldg(e + c);
        dot += ev * qv[c];
        ne += ev * ev;
      }
    }
    dot = warp_sum_d(dot);
    ne = warp_sum_d(ne);
    return exact_sim(f.metric, dot, ne, nq, d2);
  };

  if (ns_all <= RL_MAX_SURVIVORS) {
    for (int s = warp; s < ns; s += nwarps) {
      const int32_t row = rows[s];
      const float sim = exact_row_sim(row);
      if (lane == 0) keys[s] = ((uint64_t)(~f2ord(sim)) << 32) | (uint32_t)row;  // ascending: sim desc, row asc
    }
  } else {
    // More rows than the shared-memory window sit inside the coarse key's error band of the cut (tight
    // clusters / near-duplicates: thousands of vectors within 2 eps of each other).  Stream instead:
    // (1) every survivor in the global candidate list is rescored exactly and its record overwritten
    //     with the order-preserving bits of the exact similarity (0 = not a survivor),
    // (2) a radix select over the 64-bit composite (sim desc, row asc) -- all composites are distinct --
    //     narrows the list to the sel_k best plus at most a window's worth of ties in the last digit,
    // (3) those are gathered into the window and take the normal sort / GROUP BY path below.
    Cand* wc = f.cand_rw + (size_t)b * f.cap;
    for (int i = warp; i < n; i += nwarps) {
      const Cand c = wc[i];                      // same address for the whole warp: one broadcast load
      uint32_t o = 0u;
      if (c.key >= cut) o = f2ord(exact_row_sim(c.row));
      if (lane == 0) wc[i].key = __uint_as_float(o);
    }
    __syncthreads();
    auto comp_of = [&](int i) -> uint64_t {      // larger = better; 0 for non-survivors
      const Cand c = wc[i];
      const uint32_t o = __float_as_uint(c.key);
      return o == 0u ? 0ull : (((uint64_t)o << 32) | (uint32_t)(~(uint32_t)c.row));
    };
    block_gather_top(n, f.sel_k, RL_MAX_SURVIVORS, comp_of, keys, hist, res, &s_count);
    ns = min(s_count, RL_MAX_SURVIVORS);
  }
  int npow2 = 1;
  while (npow2 < ns) npow2 <<= 1;
  for (int i = ns + threadIdx.x; i < npow2; i += blockDim.x) keys[i] = ~0ull;
  __syncthreads();
  bitonic_sort_u64(keys, npow2);

  float* out_sim = f.hit_sim + (size_t)b * f.H;
  int64_t* out_chunk = f.hit_chunk + (size_t)b * f.H;
  int n_out;
  if (f.mode_sql) {
    n_out = min(ns, f.H);
    for (int i = threadIdx.x; i < n_out; i += blockDim.x) {
      const uint64_t kk = keys[i];
      out_sim[i] = ord2f(~(uint32_t)(kk >> 32));
      out_chunk[i] = f.chunk_base + f.row_chunk[(uint32_t)kk];
    }
  } else {
    // exact MaxSim: GROUP BY chunk -> the first occurrence in descending-sim order carries the max.
    int32_t* chunk = rows;
    uint8_t* flags = reinterpret_cast<uint8_t*>(hist);
    int* pos = reinterpret_cast<int*>(hist) + RL_MAX_SURVIVORS / 4;
    for (int i = threadIdx.x; i < ns; i += blockDim.x) chunk[i] = f.row_chunk[(uint32_t)keys[i]];
    __syncthreads();
    first_occurrence(chunk, ns, flags);
    exclusive_scan_flags(flags, ns, pos);
    for (int i = threadIdx.x; i < ns; i += blockDim.x) {
      if (flags[i] && pos[i] < f.H) {
        out_sim[pos[i]] = ord2f(~(uint32_t)(keys[i] >> 32));
        out_chunk[pos[i]] = f.chunk_base + chunk[i];
      }
    }
    __syncthreads();
    n_out = ns > 0 ? min(f.H, pos[ns - 1] + (int)flags[ns - 1]) : 0;
  }
  for (int i = n_out + threadIdx.x; i < f.H; i += blockDim.x) {
    out_sim[i] = kNegInf;
    out_chunk[i] = -1;
  }
  if (threadIdx.x == 0) {
    f.hit_count[b] = n_out;
    f.status[b] = st;
    f.n_surv[b] = ns_all;
  }
}

// ---- cross-shard merge + GROUP BY + LIMIT ------------------------------------------------------------
constexpr int kMergeMax = 8192;

__global__ void __launch_bounds__(kSelThreads) merge_kernel(const MergeArgs m) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int win = m.win;   // power of two >= R * H (<= kMergeMax): the arrays are sized by the actual problem
  uint64_t* keys = reinterpret_cast<uint64_t*>(smem_raw);      // [win]
  int64_t* chunk = reinterpret_cast<int64_t*>(keys + win);     // [win]
  int* pos = reinterpret_cast<int*>(chunk + win);              // [win]
  uint8_t* flags = reinterpret_cast<uint8_t*>(pos + win);      // [win]
  __shared__ int s_n;
  const int b = blockIdx.x;
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  const int64_t sim_rs = m.sim_rs ? m.sim_rs : (int64_t)m.B * m.H;
  const int64_t chunk_rs = m.chunk_rs ? m.chunk_rs : (int64_t)m.B * m.H;
  const int64_t count_rs = m.count_rs ? m.count_rs : (int64_t)m.B;
  if (m.prefilter) {
    // More gathered hits than the shared-memory window (R * H > 8192: many shards x a large num_hits): only the
    // num_hits best overall can matter, so select them straight from global memory -- a radix select over the
    // composite (sim desc, shard-major position asc; all distinct) -- and sort just those.
    uint32_t* hist = reinterpret_cast<uint32_t*>(flags + win);   // [kBins]
    __shared__ int res[2];
    auto comp_of = [&](int idx) -> uint64_t {
      const int r = idx / m.H, i = idx % m.H;
      if (i >= min(m.hit_count[(size_t)r * count_rs + b], m.H)) return 0ull;
      const uint32_t o = f2ord(m.hit_sim[(size_t)r * sim_rs + (size_t)b * m.H + i]);
      return o == 0u ? 0ull : (((uint64_t)o << 32) | (uint32_t)(~(uint32_t)idx));
    };
    block_gather_top(m.R * m.H, m.num_hits, win, comp_of, keys, hist, res, &s_n);
    if (threadIdx.x == 0 && s_n > win) s_n = win;
    __syncthreads();
  } else {
    for (int r = 0; r < m.R; ++r) {
      const int cnt = min(m.hit_count[(size_t)r * count_rs + b], m.H);
      __shared__ int base;
      if (threadIdx.x == 0) { base = s_n; s_n += cnt; }
      __syncthreads();
      for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
        const size_t e = (size_t)r * sim_rs + (size_t)b * m.H + i;
        keys[base + i] = ((uint64_t)(~f2ord(m.hit_sim[e])) << 32) | (uint32_t)(r * m.H + i);
      }
      __syncthreads();
    }
  }
  const int n = s_n;
  int npow2 = 1;
  while (npow2 < n) npow2 <<= 1;
  for (int i = n + threadIdx.x; i < npow2; i += blockDim.x) keys[i] = ~0ull;
  __syncthreads();
  bitonic_sort_u64(keys, npow2);
  const int n_keep = m.num_hits > 0 ? min(n, m.num_hits) : n;
  for (int i = threadIdx.x; i < n_keep; i += blockDim.x) {
    const uint32_t e = (uint32_t)keys[i];
    const int r = e / m.H, j = e % m.H;
    chunk[i] = m.hit_chunk[(size_t)r * chunk_rs + (size_t)b * m.H + j];
  }
  __syncthreads();
  first_occurrence(chunk, n_keep, flags);
  exclusive_scan_flags(flags, n_keep, pos);
  float* out_sim = m.out_sim + (size_t)b * m.k;
  int64_t* out_chunk = m.out_chunk + (size_t)b * m.k;
  for (int i = threadIdx.x; i < n_keep; i += blockDim.x) {
    if (flags[i] && pos[i] < m.k) {
      out_sim[pos[i]] = ord2f(~(uint32_t)(keys[i] >> 32));
      out_chunk[pos[i]] = chunk[i];
    }
  }
  __syncthreads();
  const int n_out = n_keep > 0 ? min(m.k, pos[n_keep - 1] + (int)flags[n_keep - 1]) : 0;
  for (int i = n_out + threadIdx.x; i < m.k; i += blockDim.x) {
    out_sim[i] = kNegInf;
    out_chunk[i] = -1;
  }
  if (threadIdx.x == 0) m.out_count[b] = n_out;
}

// ---- launchers ---------------------------------------------------------------------------------------
// ---- similarity floor -> key threshold (rl_maxsim_count_at_least) ------------------------------------
// The scan compares approximate keys: cosine -> the similarity itself, dot -> <e,q> = sim - 1, l1 -> -sum |e - q| = sim - 1,
// l2 -> 2<e,q> - |e|^2 = |q|^2 - dist^2 with dist = 1 - sim.  `bound` moves the threshold by the key's
// error bound so that the count brackets the exact one (+1: no exact match is missed, -1: none is extra).
__global__ void sim_floor_to_thr_kernel(const float* __restrict__ sim_floor, const double* __restrict__ q_sq,
                                        const float* __restrict__ eps, int metric, int bound, int B,
                                        float* __restrict__ thr) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const float f = sim_floor[b];
  float key;
  if (metric == RL_METRIC_COSINE) key = f;
  else if (metric == RL_METRIC_DOT || metric == RL_METRIC_L1) key = f - 1.f;   // l1: -sum |e - q| = sim - 1
  else {
    const double dist = 1.0 - (double)f;
    key = dist < 0.0 ? __builtin_huge_valf() : (float)(q_sq[b] - dist * dist);
  }
  thr[b] = key - (float)bound * eps[b] * 1.0001f;
}

int launch_sim_floor_to_thr(const float* sim_floor, const double* q_sq, const float* eps, int metric, int bound, int B,
                            float* thr, cudaStream_t stream) {
  sim_floor_to_thr_kernel<<<(B + 127) / 128, 128, 0, stream>>>(sim_floor, q_sq, eps, metric, bound, B, thr);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

int launch_query_prep(const float* Q, int B, int d, int metric, int algo, const float* row_stats, double* q_sq,
                      float* q_inv, float* eps, cudaStream_t stream) {
  query_prep_kernel<<<B, 128, 0, stream>>>(Q, B, d, metric, algo, row_stats, q_sq, q_inv, eps);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

int launch_select(const SelectArgs& a, int B, cudaStream_t stream) {
  const size_t smem = (size_t)kBins * 4 + (size_t)kSelListCap * (sizeof(Cand) + sizeof(float));
  RL_CUDA_CHECK(cudaFuncSetAttribute(select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  select_kernel<<<B, kSelThreads, smem, stream>>>(a);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

size_t finalize_smem_bytes(int d) {
  return (size_t)RL_MAX_SURVIVORS * (8 + 4) + (size_t)kFinalizeScratch + (size_t)d * 4;
}

int launch_finalize(const FinalizeArgs& f, int B, cudaStream_t stream) {
  static_assert(kFinalizeScratch >= kBins * 4 && kFinalizeScratch >= RL_MAX_SURVIVORS * 5, "scratch reuse");
  const size_t smem = finalize_smem_bytes(f.d);
  RL_REQUIRE(smem <= 220 * 1024, RL_EUNSUPPORTED, "finalize: d=%d too large", f.d);
  RL_CUDA_CHECK(cudaFuncSetAttribute(finalize_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  finalize_kernel<<<B, kSelThreads, smem, stream>>>(f);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

int launch_merge(const MergeArgs& m_in, cudaStream_t stream) {
  MergeArgs m = m_in;
  const int64_t total = (int64_t)m.R * m.H;
  m.prefilter = total > kMergeMax ? 1 : 0;
  RL_REQUIRE(!m.prefilter || (m.num_hits > 0 && m.num_hits <= kMergeMax && total < (1ll << 31)), RL_EUNSUPPORTED,
             "rl_topk_merge: R*H=%lld exceeds %d (supported beyond that only with 0 < num_hits <= %d)", (long long)total,
             kMergeMax, kMergeMax);
  int win = 32;
  while (win < (m.prefilter ? m.num_hits : total)) win <<= 1;
  m.win = win;
  // sized by the problem, not by the cap: R*H = 3200 -> 86 KB -> two CTAs per SM, a 256-query batch is one wave
  const size_t smem = (size_t)win * (8 + 8 + 4 + 1) + (m.prefilter ? (size_t)kBins * 4 : 0);
  RL_CUDA_CHECK(cudaFuncSetAttribute(merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  merge_kernel<<<m.B, kSelThreads, smem, stream>>>(m);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

}  // namespace rl
