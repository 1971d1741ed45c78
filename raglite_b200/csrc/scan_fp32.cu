// Exact fp32 CUDA-core scan (RL_ALGO_FP32): S = Q E^T tile by tile with a fused key / threshold /
// emit epilogue.  General shapes (any d, any alignment); the wgmma scan is the fast path.
//
// Replaces the per-row distance expression DuckDB evaluates for vector_search
// (reference _search.py:69-79, _typing.py:123-134).
#include "scan_common.cuh"

namespace rl {

constexpr int kBM = 128;  // rows per block (== kBlockRows)
constexpr int kBN = 64;   // queries per block
constexpr int kBK = 16;
constexpr int kPad = 4;

__device__ __forceinline__ float make_key(int metric, float acc, float inv_e, float sq_e, float inv_q) {
  if (metric == RL_METRIC_COSINE) return acc * inv_e * inv_q;
  if (metric == RL_METRIC_DOT) return acc;
  return 2.f * acc - sq_e;  // l2: monotone in -|e - q|^2 (+ |q|^2, constant per query)
}

__global__ void __launch_bounds__(256) scan_fp32_kernel(const ScanArgs a) {
  __shared__ float Es[kBK][kBM + kPad];
  __shared__ float Qs[kBK][kBN + kPad];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int64_t ord = blockIdx.x;
  const int64_t blk = mode_block_index(a, ord);
  const int64_t row0 = blk * kBM;
  const int q0 = blockIdx.y * kBN;
  const bool vec = (a.d % 4 == 0) && (a.ld % 4 == 0) && ((reinterpret_cast<uintptr_t>(a.E) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(a.Q) & 15) == 0);

  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  // Loader coordinates: E tile 128 x 16 (two float4 per thread), Q tile 64 x 16 (one float4).
  const int e_row = tid >> 1, e_k = (tid & 1) * 8;
  const int q_row = tid >> 2, q_k = (tid & 3) * 4;
  const int64_t e_grow = row0 + e_row;
  const int q_gcol = q0 + q_row;

  for (int k0 = 0; k0 < a.d; k0 += kBK) {
    float ev[8], qv[4];
#pragma unroll
    for (int i = 0; i < 8; ++i) ev[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) qv[i] = 0.f;
    if (e_grow < a.n_rows) {
      const float* src = a.E + e_grow * a.ld + k0 + e_k;
      if (vec) {
        if (k0 + e_k < a.d) { float4 v = __ldg(reinterpret_cast<const float4*>(src)); ev[0] = v.x; ev[1] = v.y; ev[2] = v.z; ev[3] = v.w; }
        if (k0 + e_k + 4 < a.d) { float4 v = __ldg(reinterpret_cast<const float4*>(src + 4)); ev[4] = v.x; ev[5] = v.y; ev[6] = v.z; ev[7] = v.w; }
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) if (k0 + e_k + i < a.d) ev[i] = __ldg(src + i);
      }
    }
    if (q_gcol < a.B) {
      const float* src = a.Q + (size_t)q_gcol * a.d + k0 + q_k;
      if (vec) {
        if (k0 + q_k < a.d) { float4 v = __ldg(reinterpret_cast<const float4*>(src)); qv[0] = v.x; qv[1] = v.y; qv[2] = v.z; qv[3] = v.w; }
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) if (k0 + q_k + i < a.d) qv[i] = __ldg(src + i);
      }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 8; ++i) Es[e_k + i][e_row] = ev[i];
#pragma unroll
    for (int i = 0; i < 4; ++i) Qs[q_k + i][q_row] = qv[i];
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kBK; ++kk) {
      float er[8], qr[4];
      const float4 e0 = *reinterpret_cast<const float4*>(&Es[kk][ty * 8]);
      const float4 e1 = *reinterpret_cast<const float4*>(&Es[kk][ty * 8 + 4]);
      const float4 qq = *reinterpret_cast<const float4*>(&Qs[kk][tx * 4]);
      er[0] = e0.x; er[1] = e0.y; er[2] = e0.z; er[3] = e0.w; er[4] = e1.x; er[5] = e1.y; er[6] = e1.z; er[7] = e1.w;
      qr[0] = qq.x; qr[1] = qq.y; qr[2] = qq.z; qr[3] = qq.w;
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(er[i], qr[j], acc[i][j]);
    }
  }

  // Epilogue: key, then dump (sample blocks) or threshold + emit (the rest).
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r_in = ty * 8 + i;
    const int64_t row = row0 + r_in;
    bool valid = row < a.n_rows;
    if (valid && a.row_allowed != nullptr) valid = a.row_allowed[row] != 0;
    const float inv_e = valid ? a.inv_norm[row] : 0.f;
    const float sq_e = valid ? a.sq_norm[row] : 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int col = q0 + tx * 4 + j;
      if (col >= a.B) continue;
      const float key = make_key(a.metric, acc[i][j], inv_e, sq_e, a.q_inv_norm[col]);
      if (a.dump_mode) {
        a.dump[(size_t)col * a.n_sample_rows + ord * kBM + r_in] = valid ? key : kNegInf;
      } else if (valid && key >= a.thr[col]) {
        emit_candidate(a, col, key, (int32_t)row);
      }
    }
  }
}

int launch_scan_fp32(const ScanArgs& a, cudaStream_t stream) {
  if (a.n_mode_blocks == 0 || a.B == 0) return RL_OK;
  RL_REQUIRE(a.n_mode_blocks < (1ll << 31), RL_EUNSUPPORTED, "scan_fp32: too many blocks");
  dim3 grid((unsigned)a.n_mode_blocks, (unsigned)((a.B + kBN - 1) / kBN));
  scan_fp32_kernel<<<grid, 256, 0, stream>>>(a);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

}  // namespace rl
