// Index-build kernels, query-adapter apply and the late-chunking pool (sm_90a).
//
//   rl_row_stats         -- per-row norms of the resident embedding matrix
//   rl_chunk_row_map     -- CSR chunk offsets -> per-row owner
//   rl_adapter_apply     -- reference _search.py:58-62  (float64 matvec, cast to query dtype)
//   rl_segment_mean_pool -- reference _embed.py:129-140 / :154-164 (mean pool, L2, fp16)
//   rl_chunk_embedding_blend -- reference _insert.py:132-145 (α-blend of chunklet and full-chunk rows, fp16)
#include <cuda_fp16.h>

#include "common.cuh"

namespace rl {

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// One warp per row; float64 accumulation so that inv_norm is the correctly rounded 1/|e|.
__global__ void __launch_bounds__(256) row_stats_kernel(const float* __restrict__ E, int64_t n_rows, int d,
                                                        int64_t ld, float* __restrict__ inv_norm,
                                                        float* __restrict__ sq_norm, float* __restrict__ stats) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t n_warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const bool vec = (d % 4 == 0) && (ld % 4 == 0) && ((reinterpret_cast<uintptr_t>(E) & 15) == 0);
  float max_norm = 0.f, max_abs = 0.f, max_inv = 0.f;
  bool zero_row = false;
  for (int64_t r = warp; r < n_rows; r += n_warps) {
    const float* row = E + r * ld;
    double s = 0.0;
    float ma = 0.f;
    if (vec) {
      for (int c = lane * 4; c < d; c += 128) {
        float4 v = __ldg(reinterpret_cast<const float4*>(row + c));
        s += (double)v.x * v.x + (double)v.y * v.y + (double)v.z * v.z + (double)v.w * v.w;
        ma = fmaxf(ma, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
      }
    } else {
      for (int c = lane; c < d; c += 32) {
        float v = __ldg(row + c);
        s += (double)v * v;
        ma = fmaxf(ma, fabsf(v));
      }
    }
    s = warp_sum(s);
    ma = warp_max(ma);
    if (lane == 0) {
      float nrm = (float)sqrt(s);
      inv_norm[r] = s > 0.0 ? (float)(1.0 / sqrt(s)) : 0.f;
      sq_norm[r] = (float)s;
      max_norm = fmaxf(max_norm, nrm);
      max_abs = fmaxf(max_abs, ma);
      if (s > 0.0) max_inv = fmaxf(max_inv, (float)(1.0 / sqrt(s)));
      else zero_row = true;
    }
  }
  if (lane == 0 && stats != nullptr) {  // non-negative floats order like their int bit patterns
    atomicMax(reinterpret_cast<int*>(stats + 0), __float_as_int(max_norm));
    atomicMax(reinterpret_cast<int*>(stats + 1), __float_as_int(max_abs));
    atomicMax(reinterpret_cast<int*>(stats + 2), __float_as_int(max_inv));
    if (zero_row) atomicMax(reinterpret_cast<int*>(stats + 3), __float_as_int(1.f));
  }
}

// Same statistics for a float16 matrix (8 halves per 16-byte load).
__global__ void __launch_bounds__(256) row_stats_f16_kernel(const __half* __restrict__ E, int64_t n_rows, int d,
                                                            int64_t ld, float* __restrict__ inv_norm,
                                                            float* __restrict__ sq_norm, float* __restrict__ stats) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t n_warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  float max_norm = 0.f, max_abs = 0.f, max_inv = 0.f;
  bool zero_row = false;
  for (int64_t r = warp; r < n_rows; r += n_warps) {
    const __half* row = E + r * ld;
    double s = 0.0;
    float ma = 0.f;
    for (int c = lane * 8; c < d; c += 256) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(row + c));
      const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(h[e]);
        s += (double)f.x * f.x + (double)f.y * f.y;
        ma = fmaxf(ma, fmaxf(fabsf(f.x), fabsf(f.y)));
      }
    }
    s = warp_sum(s);
    ma = warp_max(ma);
    if (lane == 0) {
      inv_norm[r] = s > 0.0 ? (float)(1.0 / sqrt(s)) : 0.f;
      sq_norm[r] = (float)s;
      max_norm = fmaxf(max_norm, (float)sqrt(s));
      max_abs = fmaxf(max_abs, ma);
      if (s > 0.0) max_inv = fmaxf(max_inv, (float)(1.0 / sqrt(s)));
      else zero_row = true;
    }
  }
  if (lane == 0 && stats != nullptr) {
    atomicMax(reinterpret_cast<int*>(stats + 0), __float_as_int(max_norm));
    atomicMax(reinterpret_cast<int*>(stats + 1), __float_as_int(max_abs));
    atomicMax(reinterpret_cast<int*>(stats + 2), __float_as_int(max_inv));
    if (zero_row) atomicMax(reinterpret_cast<int*>(stats + 3), __float_as_int(1.f));
  }
}

__global__ void chunk_row_map_kernel(const int64_t* __restrict__ chunk_off, int64_t n_chunks,
                                     int32_t* __restrict__ row_chunk) {
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks;
       c += (int64_t)gridDim.x * blockDim.x) {
    const int64_t lo = chunk_off[c], hi = chunk_off[c + 1];
    for (int64_t r = lo; r < hi; ++r) row_chunk[r] = (int32_t)c;
  }
}

// out[b, i] = round( sum_j A[i, j] * q[b, j] ), float64 accumulate.  One warp per output row i, a
// block shares kQB queries through shared memory so each A row is read once per kQB queries.
constexpr int kQB = 8;
__global__ void __launch_bounds__(256) adapter_apply_kernel(const double* __restrict__ A,
                                                            const float* __restrict__ Qin, float* __restrict__ Qout,
                                                            int B, int d, int round_mode) {
  extern __shared__ float qs[];  // [kQB][d]
  const int b0 = blockIdx.y * kQB;
  const int nb = min(kQB, B - b0);
  for (int idx = threadIdx.x; idx < kQB * d; idx += blockDim.x) {
    const int qb = idx / d, j = idx - qb * d;
    qs[idx] = qb < nb ? Qin[(size_t)(b0 + qb) * d + j] : 0.f;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= d) return;
  double acc[kQB];
#pragma unroll
  for (int qb = 0; qb < kQB; ++qb) acc[qb] = 0.0;
  const double* arow = A + (size_t)i * d;
  for (int j = lane; j < d; j += 32) {
    const double a = __ldg(arow + j);
#pragma unroll
    for (int qb = 0; qb < kQB; ++qb) acc[qb] = fma(a, (double)qs[qb * d + j], acc[qb]);
  }
#pragma unroll
  for (int qb = 0; qb < kQB; ++qb) {
    const double s = warp_sum(acc[qb]);
    if (lane == 0 && qb < nb) {
      // The reference casts the float64 product straight to the query dtype (one rounding).
      const float o = round_mode == 1 ? __half2float(__double2half(s)) : (float)s;
      Qout[(size_t)(b0 + qb) * d + i] = o;
    }
  }
}

// One block per output sentence: sequential float64 row sum per column (NumPy's axis-0 order),
// mean, optional L2 normalisation over the row, cast to fp16.
__global__ void __launch_bounds__(256) segment_mean_pool_kernel(const float* __restrict__ X, int64_t ld, int d,
                                                                const int32_t* __restrict__ row_begin,
                                                                const int32_t* __restrict__ row_end,
                                                                int normalize, __half* __restrict__ out) {
  extern __shared__ double mean_s[];  // [d]
  __shared__ double red[8];
  const int s = blockIdx.x;
  const int r0 = row_begin[s], r1 = row_end[s];
  double sq = 0.0;
  const bool vec = (d % 4 == 0) && (ld % 4 == 0) && ((reinterpret_cast<uintptr_t>(X) & 15) == 0);
  if (vec) {
    // Four adjacent columns per thread (one 16-byte load per row), four rows of loads in flight; the adds
    // stay in row order per column, so the sum is the one NumPy's axis-0 reduction produces.
    for (int c = threadIdx.x * 4; c < d; c += blockDim.x * 4) {
      double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
      const float* p = X + (int64_t)r0 * ld + c;
      int r = r0;
      for (; r + 4 <= r1; r += 4) {
        const float4 v0 = __ldg(reinterpret_cast<const float4*>(p));
        const float4 v1 = __ldg(reinterpret_cast<const float4*>(p + ld));
        const float4 v2 = __ldg(reinterpret_cast<const float4*>(p + 2 * ld));
        const float4 v3 = __ldg(reinterpret_cast<const float4*>(p + 3 * ld));
        a0 += (double)v0.x; a1 += (double)v0.y; a2 += (double)v0.z; a3 += (double)v0.w;
        a0 += (double)v1.x; a1 += (double)v1.y; a2 += (double)v1.z; a3 += (double)v1.w;
        a0 += (double)v2.x; a1 += (double)v2.y; a2 += (double)v2.z; a3 += (double)v2.w;
        a0 += (double)v3.x; a1 += (double)v3.y; a2 += (double)v3.z; a3 += (double)v3.w;
        p += 4 * ld;
      }
      for (; r < r1; ++r) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(p));
        a0 += (double)v.x; a1 += (double)v.y; a2 += (double)v.z; a3 += (double)v.w;
        p += ld;
      }
      const double n = (double)(r1 - r0);   // 0/0 = NaN for an empty sentence, like np.mean
      const double m0 = a0 / n, m1 = a1 / n, m2 = a2 / n, m3 = a3 / n;
      mean_s[c] = m0; mean_s[c + 1] = m1; mean_s[c + 2] = m2; mean_s[c + 3] = m3;
      sq += m0 * m0;
      sq += m1 * m1;
      sq += m2 * m2;
      sq += m3 * m3;
    }
  } else {
    for (int c = threadIdx.x; c < d; c += blockDim.x) {
      double acc = 0.0;
      for (int r = r0; r < r1; ++r) acc += (double)__ldg(X + (int64_t)r * ld + c);
      const double m = acc / (double)(r1 - r0);  // 0/0 = NaN for an empty sentence, like np.mean
      mean_s[c] = m;
      sq += m * m;
    }
  }
  sq = warp_sum(sq);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sq;
  __syncthreads();
  double tot = 0.0;
#pragma unroll
  for (int w = 0; w < 8; ++w) tot += red[w];
  double nrm = sqrt(tot);
  if (normalize == 2) nrm = fmax(nrm, 2.220446049250313e-16);
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    const double v = normalize ? mean_s[c] / nrm : mean_s[c];
    out[(size_t)s * d + c] = __double2half(v);
  }
}

// NumPy's float16 a * x (one rounding: the product of two halves is exact in float32).
__device__ __forceinline__ float blend_term(float a, float x) { return __half2float(__float2half_rn(__fmul_rn(a, x))); }

// One warp per row, grid-stride: the row's chunk by binary search over the CSR, then 8 halves per lane and
// 16-byte load.  out = fp16(fp16(a x) + fp16(b f)), as NumPy evaluates α * e + (1 - α) * f on float16 rows with
// weak Python scalars; __fmul_rn / __fadd_rn keep the compiler from contracting the float32 steps into an FMA.
__global__ void __launch_bounds__(256) chunk_embedding_blend_kernel(const __half* __restrict__ X, int64_t ldx,
                                                                    const __half* __restrict__ F,
                                                                    const int64_t* __restrict__ chunk_off,
                                                                    int64_t n_chunks, int64_t n_rows, int d,
                                                                    float a, float b, __half* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t n_warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t r = warp; r < n_rows; r += n_warps) {
    int64_t lo = 0, hi = n_chunks;  // chunk_off[lo] <= r < chunk_off[hi]
    while (hi - lo > 1) {
      const int64_t mid = (lo + hi) >> 1;
      if (__ldg(chunk_off + mid) <= r) lo = mid;
      else hi = mid;
    }
    const __half* x = X + r * ldx;
    const __half* f = F + lo * d;
    __half* o = out + r * d;
    for (int c = lane * 8; c < d; c += 256) {
      const uint4 xv = __ldg(reinterpret_cast<const uint4*>(x + c));
      const uint4 fv = __ldg(reinterpret_cast<const uint4*>(f + c));
      const __half2* xh = reinterpret_cast<const __half2*>(&xv);
      const __half2* fh = reinterpret_cast<const __half2*>(&fv);
      uint4 ov;
      __half2* oh = reinterpret_cast<__half2*>(&ov);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 xf = __half22float2(xh[e]), ff = __half22float2(fh[e]);
        oh[e] = __halves2half2(__float2half_rn(__fadd_rn(blend_term(a, xf.x), blend_term(b, ff.x))),
                               __float2half_rn(__fadd_rn(blend_term(a, xf.y), blend_term(b, ff.y))));
      }
      *reinterpret_cast<uint4*>(o + c) = ov;
    }
  }
}

// out[row] = chunk_ok[row_chunk[row]] (all-ones when chunk_ok is null) AND alive[row] (when given): the
// per-row byte mask the scan epilogue reads.  chunk_ok is the metadata filter resolved per chunk
// (reference _search.py:82-95), alive the tombstones of deleted chunks (_delete.py:146-152).
// 16 rows per thread: four int4 loads of owners, one 16-byte load of tombstones, one 16-byte store.
__global__ void __launch_bounds__(256) row_mask_kernel(const uint8_t* __restrict__ chunk_ok,
                                                       const int32_t* __restrict__ row_chunk,
                                                       const uint8_t* __restrict__ alive, int64_t n_rows,
                                                       uint8_t* __restrict__ out) {
  const int64_t n16 = n_rows / 16;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (int64_t)gridDim.x * blockDim.x) {
    uint32_t w[4] = {0x01010101u, 0x01010101u, 0x01010101u, 0x01010101u};
    if (chunk_ok != nullptr) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int4 c = __ldg(reinterpret_cast<const int4*>(row_chunk) + i * 4 + q);
        w[q] = (uint32_t)(chunk_ok[c.x] != 0) | ((uint32_t)(chunk_ok[c.y] != 0) << 8) |
               ((uint32_t)(chunk_ok[c.z] != 0) << 16) | ((uint32_t)(chunk_ok[c.w] != 0) << 24);
      }
    }
    if (alive != nullptr) {
      const uint4 a = __ldg(reinterpret_cast<const uint4*>(alive) + i);
      // any non-zero tombstone byte counts as alive: normalise each byte to 0/1 before the AND
      auto norm = [](uint32_t x) { return ((x | (x >> 1) | (x >> 2) | (x >> 3) | (x >> 4) | (x >> 5) | (x >> 6) | (x >> 7)) & 0x01010101u); };
      w[0] &= norm(a.x); w[1] &= norm(a.y); w[2] &= norm(a.z); w[3] &= norm(a.w);
    }
    reinterpret_cast<uint4*>(out)[i] = make_uint4(w[0], w[1], w[2], w[3]);
  }
  // ragged tail (n_rows % 16 rows)
  const int64_t t0 = n16 * 16;
  for (int64_t r = t0 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n_rows; r += (int64_t)gridDim.x * blockDim.x) {
    uint8_t v = chunk_ok != nullptr ? (uint8_t)(chunk_ok[row_chunk[r]] != 0) : (uint8_t)1;
    if (alive != nullptr && alive[r] == 0) v = 0;
    out[r] = v;
  }
}

}  // namespace rl

using namespace rl;

extern "C" int rl_row_stats(const float* E, int64_t n_rows, int d, int64_t ld, float* inv_norm, float* sq_norm,
                            float* stats, void* stream) {
  RL_REQUIRE(n_rows >= 0 && d > 0 && ld >= d, RL_EINVAL, "rl_row_stats: bad shape");
  if (n_rows == 0) return RL_OK;
  RL_REQUIRE(E && inv_norm && sq_norm, RL_EINVAL, "rl_row_stats: null pointer");
  const int64_t blocks = (n_rows + 7) / 8;
  const int grid = (int)(blocks < 132 * 16 ? blocks : 132 * 16);
  row_stats_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(E, n_rows, d, ld, inv_norm, sq_norm, stats);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" int rl_row_stats_f16(const void* E, int64_t n_rows, int d, int64_t ld, float* inv_norm, float* sq_norm,
                                float* stats, void* stream) {
  RL_REQUIRE(n_rows >= 0 && d > 0 && ld >= d, RL_EINVAL, "rl_row_stats_f16: bad shape");
  RL_REQUIRE(d % 8 == 0 && ld % 8 == 0 && (reinterpret_cast<uintptr_t>(E) & 15) == 0, RL_EUNSUPPORTED,
             "rl_row_stats_f16: d and ld must be multiples of 8 and E 16-byte aligned");
  if (n_rows == 0) return RL_OK;
  RL_REQUIRE(E && inv_norm && sq_norm, RL_EINVAL, "rl_row_stats_f16: null pointer");
  const int64_t blocks = (n_rows + 7) / 8;
  const int grid = (int)(blocks < 132 * 16 ? blocks : 132 * 16);
  row_stats_f16_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const __half*>(E), n_rows, d, ld, inv_norm,
                                                               sq_norm, stats);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" int rl_chunk_row_map(const int64_t* chunk_off, int64_t n_chunks, int32_t* row_chunk, void* stream) {
  RL_REQUIRE(n_chunks >= 0, RL_EINVAL, "rl_chunk_row_map: bad n_chunks");
  if (n_chunks == 0) return RL_OK;
  RL_REQUIRE(chunk_off && row_chunk, RL_EINVAL, "rl_chunk_row_map: null pointer");
  const int64_t blocks = (n_chunks + 255) / 256;
  const int grid = (int)(blocks < 132 * 8 ? blocks : 132 * 8);
  chunk_row_map_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(chunk_off, n_chunks, row_chunk);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" int rl_adapter_apply(const double* A, const float* Q_in, float* Q_out, int B, int d, int round_mode,
                                void* stream) {
  RL_REQUIRE(B >= 0 && d > 0, RL_EINVAL, "rl_adapter_apply: bad shape");
  if (B == 0) return RL_OK;
  RL_REQUIRE(A && Q_in && Q_out && Q_in != Q_out, RL_EINVAL, "rl_adapter_apply: null or aliased pointer");
  RL_REQUIRE(round_mode == 0 || round_mode == 1, RL_EINVAL, "rl_adapter_apply: round_mode must be 0 or 1");
  const size_t smem = (size_t)kQB * d * sizeof(float);
  RL_REQUIRE(smem <= 200 * 1024, RL_EUNSUPPORTED, "rl_adapter_apply: d=%d too large", d);
  RL_CUDA_CHECK(cudaFuncSetAttribute(adapter_apply_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid((d + 7) / 8, (B + kQB - 1) / kQB);
  adapter_apply_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>(A, Q_in, Q_out, B, d, round_mode);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" int rl_segment_mean_pool(const float* X, int64_t ld, int d, const int32_t* row_begin,
                                    const int32_t* row_end, int S, int normalize, uint16_t* out, void* stream) {
  RL_REQUIRE(S >= 0 && d > 0 && ld >= d, RL_EINVAL, "rl_segment_mean_pool: bad shape");
  if (S == 0) return RL_OK;
  RL_REQUIRE(X && row_begin && row_end && out, RL_EINVAL, "rl_segment_mean_pool: null pointer");
  RL_REQUIRE(normalize >= 0 && normalize <= 2, RL_EINVAL, "rl_segment_mean_pool: normalize must be 0..2");
  const size_t smem = (size_t)d * sizeof(double);
  RL_REQUIRE(smem <= 200 * 1024, RL_EUNSUPPORTED, "rl_segment_mean_pool: d=%d too large", d);
  RL_CUDA_CHECK(cudaFuncSetAttribute(segment_mean_pool_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  segment_mean_pool_kernel<<<S, 256, smem, (cudaStream_t)stream>>>(X, ld, d, row_begin, row_end, normalize,
                                                                     reinterpret_cast<__half*>(out));
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" int rl_chunk_embedding_blend(const uint16_t* X, int64_t ldx, const uint16_t* F, const int64_t* chunk_off,
                                        int64_t n_chunks, int64_t n_rows, int d, uint16_t alpha,
                                        uint16_t one_minus_alpha, uint16_t* out, void* stream) {
  RL_REQUIRE(n_rows >= 0 && n_chunks >= 0 && d > 0 && ldx >= d && (n_rows == 0 || n_chunks > 0), RL_EINVAL,
             "rl_chunk_embedding_blend: bad shape");
  RL_REQUIRE(d % 8 == 0 && ldx % 8 == 0 && ((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(F) |
                                             reinterpret_cast<uintptr_t>(out)) & 15) == 0,
             RL_EUNSUPPORTED, "rl_chunk_embedding_blend: d and ldx must be multiples of 8 and X, F, out 16-byte aligned");
  if (n_rows == 0) return RL_OK;
  RL_REQUIRE(X && F && chunk_off && out, RL_EINVAL, "rl_chunk_embedding_blend: null pointer");
  const __half_raw ra{alpha}, rb{one_minus_alpha};
  const int64_t blocks = (n_rows + 7) / 8;
  const int grid = (int)(blocks < 132 * 16 ? blocks : 132 * 16);
  chunk_embedding_blend_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const __half*>(X), ldx, reinterpret_cast<const __half*>(F), chunk_off, n_chunks, n_rows, d,
      __half2float(__half(ra)), __half2float(__half(rb)), reinterpret_cast<__half*>(out));
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" int rl_row_mask(const uint8_t* chunk_ok, const int32_t* row_chunk, const uint8_t* alive, int64_t n_rows,
                           uint8_t* out, void* stream) {
  RL_REQUIRE(n_rows >= 0, RL_EINVAL, "rl_row_mask: bad n_rows");
  if (n_rows == 0) return RL_OK;
  RL_REQUIRE(out && (chunk_ok == nullptr || row_chunk != nullptr), RL_EINVAL, "rl_row_mask: null pointer");
  RL_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0 && (reinterpret_cast<uintptr_t>(row_chunk) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(alive) & 15) == 0,
             RL_EINVAL, "rl_row_mask: row_chunk, alive and out must be 16-byte aligned");
  const int64_t blocks = (n_rows / 16 + 255) / 256 + 1;
  const int grid = (int)(blocks < 132 * 8 ? blocks : 132 * 8);
  row_mask_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(chunk_ok, row_chunk, alive, n_rows, out);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}
