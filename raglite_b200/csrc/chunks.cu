// Chunklets and chunks on the GPU: the reference's chunklet dynamic program (raglite/_split_chunklets.py, its default
// O(1) cost path), the chunk partition costs of raglite/_split_chunks.py (normalise, remove the discourse vector, adjacent
// similarities, the heading rule) and the chunk partition itself.
//
// split_chunks solves an integer program whose constraint row i asks for a cut among the chunklets that fit in max_size
// from chunklet i.  Those rows say exactly that every chunk is at most max_size characters, and the matrix is an interval
// matrix, so the program's optimum is the minimum-cost segmentation with cost costs[a - 1] for a chunk starting at a > 0.
// Both partitions are therefore one windowed dynamic program, run by one warp per document (partition_warp), with two
// cost functors.
#include <cuda_fp16.h>

#include "common.cuh"

namespace rl {
namespace {

constexpr int kPartThreads = 128;        // 4 documents per block
constexpr int kPartMaxBlocks = 2048;     // the document loop strides past 8192 documents
constexpr int kSimThreads = 256;
constexpr int kSimMaxBlocks = 4096;
constexpr int kSimMaxDim = 8192;         // the float64 discourse vector lives in shared memory (64 KB at 8192)
constexpr double kInf = __builtin_huge_val();

__host__ __device__ __forceinline__ int64_t align256(int64_t b) { return (b + 255) / 256 * 256; }

// Per-document scratch of the partition: n + 1 entries of each array, document d's at doc_off[d] + d.
struct PartScratch {
  double* dp;
  double* pb;     // prefix sums of the boundary probabilities (chunklets only)
  double* ps;     // prefix sums of the statement counts (chunklets only)
  int64_t* pl;    // prefix sums of the lengths
  int* back;
};

__host__ __device__ __forceinline__ PartScratch part_scratch(void* ws, int64_t entries) {
  char* p = (char*)ws;
  const int64_t s8 = align256(entries * 8);
  return PartScratch{(double*)p, (double*)(p + s8), (double*)(p + 2 * s8), (int64_t*)(p + 3 * s8),
                     (int*)(p + 4 * s8)};
}

size_t part_workspace_bytes(int64_t n_items, int n_docs) {
  if (n_items < 0 || n_docs < 0) return 0;
  const int64_t e = n_items + n_docs;
  return (size_t)(4 * align256(e * 8) + align256(e * 4));
}

// (cost, j) pairs ordered lexicographically; j < 0 is "no candidate".  The reference walks j downwards and keeps a
// candidate when cost <= the best so far, so it ends on the smallest j of the smallest cost (inf included: inf <= inf).
__device__ __forceinline__ bool better(double c, int j, double bc, int bj) {
  return j >= 0 && (bj < 0 || c < bc || (c == bc && j < bj));
}

// dp[i] = min over the window j of dp[j] + cost(j, i), for i = 1 .. n, with dp[0] = 0; the window is j = i-1, i-2, ...
// while the lengths of items j .. i-1 sum to at most max_size.  An empty window leaves dp[i] = inf, back[i] = -1.  The
// lanes split the window and reduce to the lexicographic minimum of (cost, j), so the result does not depend on how the
// lanes are assigned.  Lane 0 then walks back from n, stops at the first back <= 0 and writes the cuts ascending.
// Returns the number of cuts (valid in lane 0).
template <class Cost>
__device__ int partition_warp(int n, int64_t max_size, const int64_t* __restrict__ pl, double* __restrict__ dp,
                              int* __restrict__ back, const Cost& cost, int* __restrict__ cuts) {
  const int lane = threadIdx.x & 31;
  if (lane == 0) {
    dp[0] = 0.0;
    back[0] = -1;
  }
  __syncwarp();
  int lo = 0;   // the smallest j with pl[i] - pl[j] <= max_size; nondecreasing in i
  for (int i = 1; i <= n; ++i) {
    while (lo < i && pl[i] - pl[lo] > max_size) ++lo;
    double bc = kInf;
    int bj = -1;
    for (int j = i - 1 - lane; j >= lo; j -= 32) {
      const double c = __dadd_rn(dp[j], cost(j, i));
      if (better(c, j, bc, bj)) {
        bc = c;
        bj = j;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double oc = __shfl_xor_sync(0xffffffffu, bc, o);
      const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
      if (better(oc, oj, bc, bj)) {
        bc = oc;
        bj = oj;
      }
    }
    if (lane == 0) {
      dp[i] = bc;
      back[i] = bj;
    }
    __syncwarp();
  }
  int k = 0;
  if (lane == 0) {
    for (int i = back[n]; i > 0; i = back[i]) ++k;
    int m = k;
    for (int i = back[n]; i > 0; i = back[i]) cuts[--m] = i;
  }
  return k;
}

// split_chunklets' chunklet cost of sentences j .. i-1: ((1 - p[j]) + (PB[i] - PB[j+1])) + (s - 3)^2 / sqrt(max(s,
// 1e-6)) / 2 with s = PS[i] - PS[j], every step one rounded float64 operation.  The square is d * d; the reference's
// NumPy scalar power goes through pow (DESIGN.md section 5).
struct ChunkletCost {
  const double* p;
  const double* pb;
  const double* ps;
  __device__ __forceinline__ double operator()(int j, int i) const {
    const double b = __dadd_rn(__dsub_rn(1.0, p[j]), __dsub_rn(pb[i], pb[j + 1]));
    const double s = __dsub_rn(ps[i], ps[j]);
    const double d = __dsub_rn(s, 3.0);
    const double sc = __ddiv_rn(__ddiv_rn(__dmul_rn(d, d), __dsqrt_rn(fmax(s, 1e-6))), 2.0);
    return __dadd_rn(b, sc);
  }
};

// split_chunks' cost of a chunk starting at chunklet j: the cost of the cut before it, none for the first chunk.
struct ChunkCost {
  const float* c;
  __device__ __forceinline__ double operator()(int j, int) const { return j > 0 ? (double)c[j - 1] : 0.0; }
};

__global__ void chunklet_partition_kernel(const double* __restrict__ probas, const double* __restrict__ statements,
                                          const int32_t* __restrict__ lens, const int64_t* __restrict__ doc_off,
                                          const int32_t* __restrict__ max_size, int n_docs, PartScratch ws,
                                          int32_t* __restrict__ cuts, int32_t* __restrict__ counts,
                                          int32_t* __restrict__ status) {
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int d = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); d < n_docs; d += warps) {
    const int64_t o = doc_off[d], s0 = o + d;
    const int n = (int)(doc_off[d + 1] - o);
    if (n == 0) {
      if (lane == 0) {
        counts[d] = 0;
        status[d] = 1;
      }
      continue;
    }
    // np.cumsum is sequential: the prefix sums are too, from 0
    if (lane == 0) {
      double b = 0.0, s = 0.0;
      int64_t l = 0;
      ws.pb[s0] = 0.0;
      ws.ps[s0] = 0.0;
      ws.pl[s0] = 0;
      for (int k = 0; k < n; ++k) {
        b = k == 0 ? probas[o] : __dadd_rn(b, probas[o + k]);
        s = k == 0 ? statements[o] : __dadd_rn(s, statements[o + k]);
        l += lens[o + k];
        ws.pb[s0 + k + 1] = b;
        ws.ps[s0 + k + 1] = s;
        ws.pl[s0 + k + 1] = l;
      }
    }
    __syncwarp();
    const int k = partition_warp(n, max_size[d], ws.pl + s0, ws.dp + s0, ws.back + s0,
                                 ChunkletCost{probas + o, ws.pb + s0, ws.ps + s0}, cuts + o);
    if (lane == 0) {
      counts[d] = k;
      status[d] = 0;
    }
    __syncwarp();
  }
}

__global__ void chunk_partition_kernel(const float* __restrict__ costs, const int32_t* __restrict__ lens,
                                       const int64_t* __restrict__ doc_off, const int32_t* __restrict__ max_size,
                                       int n_docs, PartScratch ws, int32_t* __restrict__ cuts,
                                       int32_t* __restrict__ counts, int32_t* __restrict__ status) {
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int d = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); d < n_docs; d += warps) {
    const int64_t o = doc_off[d], s0 = o + d;
    const int n = (int)(doc_off[d + 1] - o);
    if (lane == 0) {
      int64_t l = 0;
      ws.pl[s0] = 0;
      for (int k = 0; k < n; ++k) ws.pl[s0 + k + 1] = l += lens[o + k];
    }
    __syncwarp();
    const int k = partition_warp(n, max_size[d], ws.pl + s0, ws.dp + s0, ws.back + s0, ChunkCost{costs + o}, cuts + o);
    if (lane == 0) {
      const bool ok = ws.dp[s0 + n] < kInf;   // inf: a chunklet longer than max_size, no partition exists
      counts[d] = ok ? k : 0;
      status[d] = ok ? 0 : 1;
    }
    __syncwarp();
  }
}

// ---- the chunk partition costs ---------------------------------------------------------------------------------------
template <bool F16>
__device__ __forceinline__ float load_x(const void* X, int64_t i) {
  if constexpr (F16) return __half2float(((const __half*)X)[i]);
  else return ((const float*)X)[i];
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// One CTA per document of n rows (rows doc_off[d] .. doc_off[d + 1] of X, row stride ld):
//  1. |x_r| per row in float32 (status 1 and nothing else when one is 0); xn_r = x_r / |x_r| in float32;
//  2. the discourse vector in float64 from the float32 xn_r: the mean over the rows nonoutlying[r] selects, divided by
//     its norm (only when some row is selected);
//  3. the projection y_r = xn_r - (xn_r . disc) disc in float64, kept (and y_r / |y_r| used) only if no
//     |y_r| <= FLT_EPSILON.  In float32 the decision would follow rounding where the exact projection is zero (the one
//     row a three-chunklet document selects, identical rows): the float32 residual there is a few u, the same order as
//     eps = 2u.  In float64, from float32 rows, such a residual is of the order of 2^-53 and the decision is the exact
//     one; c_r and |y_r| are rounded to float32 for step 4;
//  4. costs[i] = max((y_i . y_{i+1} + 1) / 2, sqrt(FLT_EPSILON)) for i < n - 1, in float32 (disc rounded to float32);
//  5. the heading rule of _split_chunks.py:74-83, serially in thread 0.
template <bool F16>
__global__ void __launch_bounds__(kSimThreads, 1) chunk_similarity_kernel(
    const void* __restrict__ X, int64_t ld, int dim, const int64_t* __restrict__ doc_off, int n_docs,
    const uint8_t* __restrict__ nonoutlying, const uint8_t* __restrict__ is_heading, float* __restrict__ costs,
    int32_t* __restrict__ status, float* __restrict__ nrm, float* __restrict__ dot, float* __restrict__ pnrm) {
  extern __shared__ double disc[];
  __shared__ double red[kSimThreads / 32];
  __shared__ int flags;   // bit 0: a zero row, bit 1: a projected row at most eps
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = kSimThreads / 32;
  const float kEps = 1.1920928955078125e-7f, kSqrtEps = 3.4526698300124390840e-4f;   // float32 eps, sqrt(eps) rounded
  for (int d = blockIdx.x; d < n_docs; d += gridDim.x) {
    const int64_t o = doc_off[d];
    const int n = (int)(doc_off[d + 1] - o);
    if (threadIdx.x == 0) flags = 0;
    __syncthreads();
    for (int r = warp; r < n; r += nw) {
      const int64_t row = (o + r) * ld;
      float ss = 0.f;
      for (int k = lane; k < dim; k += 32) {
        const float x = load_x<F16>(X, row + k);
        ss = __fmaf_rn(x, x, ss);
      }
      const float v = __fsqrt_rn(warp_sum(ss));
      if (lane == 0) {
        nrm[o + r] = v;
        if (v == 0.f) atomicOr(&flags, 1);
      }
    }
    __syncthreads();
    if (flags & 1) {
      if (threadIdx.x == 0) status[d] = 1;
      __syncthreads();
      continue;
    }
    // discourse vector
    int m = 0;
    for (int r = 0; r < n; ++r) m += nonoutlying[o + r] != 0;
    double part = 0.0;
    for (int k = threadIdx.x; k < dim; k += kSimThreads) {
      double mu = 0.0;
      for (int r = 0; r < n; ++r)
        if (nonoutlying[o + r]) mu = __dadd_rn(mu, (double)__fdiv_rn(load_x<F16>(X, (o + r) * ld + k), nrm[o + r]));
      mu = m > 0 ? __ddiv_rn(mu, (double)m) : 0.0;
      disc[k] = mu;
      part = __fma_rn(mu, mu, part);
    }
    part = warp_sum(part);
    if (lane == 0) red[warp] = part;
    __syncthreads();
    double dn = 0.0;
    for (int w = 0; w < nw; ++w) dn = __dadd_rn(dn, red[w]);
    dn = __dsqrt_rn(dn);
    for (int k = threadIdx.x; k < dim; k += kSimThreads) disc[k] = __ddiv_rn(disc[k], dn);
    __syncthreads();
    // projection off the discourse vector
    if (m > 0) {
      for (int r = warp; r < n; r += nw) {
        const int64_t row = (o + r) * ld;
        const float nr = nrm[o + r];
        double c = 0.0;
        for (int k = lane; k < dim; k += 32) c = __fma_rn((double)__fdiv_rn(load_x<F16>(X, row + k), nr), disc[k], c);
        c = warp_sum(c);
        double ss = 0.0;
        for (int k = lane; k < dim; k += 32) {
          const double y = __fma_rn(-c, disc[k], (double)__fdiv_rn(load_x<F16>(X, row + k), nr));
          ss = __fma_rn(y, y, ss);
        }
        ss = warp_sum(ss);
        const double pn = __dsqrt_rn(ss);
        if (lane == 0) {
          dot[o + r] = (float)c;
          pnrm[o + r] = (float)pn;
          if (pn <= (double)kEps) atomicOr(&flags, 2);
        }
      }
    }
    __syncthreads();
    const bool proj = m > 0 && !(flags & 2);
    for (int i = warp; i < n - 1; i += nw) {
      const int64_t ra = (o + i) * ld, rb = ra + ld;
      const float na = nrm[o + i], nb = nrm[o + i + 1];
      float ca = 0.f, cb = 0.f, pa = 1.f, pb = 1.f;
      if (proj) {
        ca = dot[o + i];
        cb = dot[o + i + 1];
        pa = pnrm[o + i];
        pb = pnrm[o + i + 1];
      }
      float s = 0.f;
      for (int k = lane; k < dim; k += 32) {
        float a = __fdiv_rn(load_x<F16>(X, ra + k), na), b = __fdiv_rn(load_x<F16>(X, rb + k), nb);
        if (proj) {
          const float dk = (float)disc[k];
          a = __fdiv_rn(__fsub_rn(a, __fmul_rn(ca, dk)), pa);
          b = __fdiv_rn(__fsub_rn(b, __fmul_rn(cb, dk)), pb);
        }
        s = __fmaf_rn(a, b, s);
      }
      s = warp_sum(s);
      if (lane == 0) {
        const float v = __fmul_rn(__fadd_rn(s, 1.f), 0.5f);
        costs[o + i] = v < kSqrtEps ? kSqrtEps : v;   // np.maximum: NaN stays NaN
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      bool prev = true;   // the first chunklet counts as preceded by a heading
      for (int i = 0; i < n - 1; ++i) {
        const bool h = is_heading[o + i] != 0;
        if (h) {
          if (!prev) costs[o + i - 1] = __fdiv_rn(costs[o + i - 1], 4.f);
          costs[o + i] = 1.f;
        }
        prev = h;
      }
      status[d] = 0;
    }
    __syncthreads();
  }
}

}  // namespace
}  // namespace rl

using namespace rl;

extern "C" size_t rl_chunklet_partition_workspace_bytes(int64_t n_sentences, int n_docs) {
  return part_workspace_bytes(n_sentences, n_docs);
}

extern "C" int rl_chunklet_partition(const double* boundary_probas, const double* num_statements, const int32_t* lens,
                                     const int64_t* doc_off, const int32_t* max_size, int n_docs, int64_t n_sentences,
                                     int32_t* cuts, int32_t* counts, int32_t* status, void* workspace,
                                     size_t workspace_bytes, void* stream) {
  RL_REQUIRE(n_docs >= 0 && n_sentences >= 0, RL_EINVAL, "rl_chunklet_partition: n_docs, n_sentences >= 0");
  if (n_docs == 0) return RL_OK;
  RL_REQUIRE(doc_off && max_size && counts && status && workspace, RL_EINVAL, "rl_chunklet_partition: null pointer");
  RL_REQUIRE(n_sentences == 0 || (boundary_probas && num_statements && lens && cuts), RL_EINVAL,
             "rl_chunklet_partition: null pointer");
  RL_REQUIRE(workspace_bytes >= part_workspace_bytes(n_sentences, n_docs), RL_ENOSPACE,
             "rl_chunklet_partition: workspace too small");
  const int64_t blocks = ((int64_t)n_docs + kPartThreads / 32 - 1) / (kPartThreads / 32);
  chunklet_partition_kernel<<<(int)(blocks < kPartMaxBlocks ? blocks : kPartMaxBlocks), kPartThreads, 0,
                              (cudaStream_t)stream>>>(boundary_probas, num_statements, lens, doc_off, max_size, n_docs,
                                                      part_scratch(workspace, n_sentences + n_docs), cuts, counts,
                                                      status);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" size_t rl_chunk_similarities_workspace_bytes(int64_t n_rows) {
  if (n_rows < 0) return 0;
  return (size_t)(3 * align256(n_rows * 4));
}

extern "C" int rl_chunk_similarities(const void* X, int x_dtype, int64_t ld, int dim, const int64_t* doc_off,
                                     int n_docs, int64_t n_rows, const uint8_t* nonoutlying, const uint8_t* is_heading,
                                     float* costs, int32_t* status, void* workspace, size_t workspace_bytes,
                                     void* stream) {
  RL_REQUIRE(n_docs >= 0 && n_rows >= 0 && (x_dtype == 0 || x_dtype == 1), RL_EINVAL,
             "rl_chunk_similarities: n_docs, n_rows >= 0 and x_dtype 0 (float32) or 1 (float16)");
  RL_REQUIRE(dim >= 1 && dim <= kSimMaxDim && ld >= dim, RL_EINVAL,
             "rl_chunk_similarities: 1 <= dim <= %d and ld >= dim", kSimMaxDim);
  if (n_docs == 0) return RL_OK;
  RL_REQUIRE(doc_off && status && workspace, RL_EINVAL, "rl_chunk_similarities: null pointer");
  RL_REQUIRE(n_rows == 0 || (X && nonoutlying && is_heading && costs), RL_EINVAL, "rl_chunk_similarities: null pointer");
  RL_REQUIRE(workspace_bytes >= rl_chunk_similarities_workspace_bytes(n_rows), RL_ENOSPACE,
             "rl_chunk_similarities: workspace too small");
  float* nrm = (float*)workspace;
  float* dot = (float*)((char*)workspace + align256(n_rows * 4));
  float* pnrm = (float*)((char*)workspace + 2 * align256(n_rows * 4));
  const int grid = n_docs < kSimMaxBlocks ? n_docs : kSimMaxBlocks;
  const size_t smem = (size_t)dim * 8;
  cudaStream_t st = (cudaStream_t)stream;
  if (smem > 48 * 1024) {
    RL_CUDA_CHECK(cudaFuncSetAttribute(chunk_similarity_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem));
    RL_CUDA_CHECK(cudaFuncSetAttribute(chunk_similarity_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem));
  }
  if (x_dtype == 1)
    chunk_similarity_kernel<true><<<grid, kSimThreads, smem, st>>>(X, ld, dim, doc_off, n_docs, nonoutlying, is_heading,
                                                                   costs, status, nrm, dot, pnrm);
  else
    chunk_similarity_kernel<false><<<grid, kSimThreads, smem, st>>>(X, ld, dim, doc_off, n_docs, nonoutlying,
                                                                    is_heading, costs, status, nrm, dot, pnrm);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" size_t rl_chunk_partition_workspace_bytes(int64_t n_chunklets, int n_docs) {
  return part_workspace_bytes(n_chunklets, n_docs);
}

extern "C" int rl_chunk_partition(const float* costs, const int32_t* lens, const int64_t* doc_off,
                                  const int32_t* max_size, int n_docs, int64_t n_chunklets, int32_t* cuts,
                                  int32_t* counts, int32_t* status, void* workspace, size_t workspace_bytes,
                                  void* stream) {
  RL_REQUIRE(n_docs >= 0 && n_chunklets >= 0, RL_EINVAL, "rl_chunk_partition: n_docs, n_chunklets >= 0");
  if (n_docs == 0) return RL_OK;
  RL_REQUIRE(doc_off && max_size && counts && status && workspace, RL_EINVAL, "rl_chunk_partition: null pointer");
  RL_REQUIRE(n_chunklets == 0 || (costs && lens && cuts), RL_EINVAL, "rl_chunk_partition: null pointer");
  RL_REQUIRE(workspace_bytes >= part_workspace_bytes(n_chunklets, n_docs), RL_ENOSPACE,
             "rl_chunk_partition: workspace too small");
  const int64_t blocks = ((int64_t)n_docs + kPartThreads / 32 - 1) / (kPartThreads / 32);
  chunk_partition_kernel<<<(int)(blocks < kPartMaxBlocks ? blocks : kPartMaxBlocks), kPartThreads, 0,
                           (cudaStream_t)stream>>>(costs, lens, doc_off, max_size, n_docs,
                                                   part_scratch(workspace, n_chunklets + n_docs), cuts, counts, status);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}
