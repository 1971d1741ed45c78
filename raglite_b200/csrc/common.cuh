// Shared helpers for the raglite_b200 CUDA sources (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdio>
#include <cstring>

#include "../../include/raglite_b200.h"

namespace rl {

// ---- error plumbing ---------------------------------------------------------------------------
void set_error(const char* fmt, ...);
#define RL_CUDA_CHECK(expr)                                                                \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess) {                                                               \
      rl::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return RL_ECUDA;                                                                     \
    }                                                                                      \
  } while (0)
#define RL_REQUIRE(cond, code, ...) \
  do {                              \
    if (!(cond)) {                  \
      rl::set_error(__VA_ARGS__);   \
      return (code);                \
    }                               \
  } while (0)

constexpr int kBlockRows = 128;  // rows per scan block (tile of the corpus; also the sampling unit)
constexpr float kNegInf = -__builtin_huge_valf();

// ---- order-preserving float <-> uint32 ---------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t f2ord(float f) {
#ifdef __CUDA_ARCH__
  uint32_t u = __float_as_uint(f);
#else
  uint32_t u;
  memcpy(&u, &f, 4);
#endif
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float ord2f(uint32_t o) {
  uint32_t u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  float f;
  memcpy(&f, &u, 4);
  return f;
#endif
}

// Online threshold refinement: every emitted candidate is also counted in a small per-query
// histogram of (key - thr0) in bins of 4 eps; once the count at or above a bin edge reaches the
// selection size, that edge (minus the 2 eps guard band) is a valid, tighter emission threshold.
constexpr int kHistBins = 16;
__host__ __device__ __forceinline__ int hist_bin(float key, float thr0, float inv_w) {
  const float x = (key - thr0) * inv_w;
  const int b = x > 0.f ? (int)x : 0;
  return b < kHistBins - 1 ? b : kHistBins - 1;
}

// Candidate record emitted by the scan: approximate key + shard-local row.
struct __align__(8) Cand {
  float key;
  int32_t row;
};

// Non-sample block ordinal -> block index (blocks with t % S == 0 are the sample).
__host__ __device__ __forceinline__ int64_t main_block_index(int64_t ord, int S) {
  return S <= 1 ? ord : ord + ord / (S - 1) + 1;
}

// ---- workspace layout ---------------------------------------------------------------------------
struct Layout {
  int algo;
  int mode_sql;          // 1: top-num_hits vectors (reference SQL semantics), 0: exact MaxSim
  int S;                 // sample stride in blocks
  int cap;               // candidate capacity per query
  int sel_k;             // order statistic the sample select looks for
  int H;                 // hits per query
  int64_t n_blocks, n_sample_blocks, n_main_blocks, n_sample_rows;
  int d_pad;             // d rounded up to 64 (fp16 query image)
  int b_pad;             // B rounded up to 16
  // byte offsets
  size_t off_hdr, off_dump, off_cand, off_cnt, off_thr, off_thr_out, off_eps, off_qinv, off_qsq,
      off_qscale, off_qimg, off_nsurv, off_hist, off_histw, off_cntall, total;
};
int make_layout(const rl_scan_params* p, int sm_count, Layout* L);

struct Header {  // first bytes of the workspace
  int32_t launches, sample_stride, cand_cap, algo;
  int64_t n_sample_rows;
  int32_t counted_unfiltered, pad_;   // 1: off_cntall holds the counters of the last call
};

}  // namespace rl
