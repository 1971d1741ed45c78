// Exact L1 scan (RL_METRIC_L1, pgvector's `<+>` on halfvec): key = -sum_i |e_i - q_i| = sim - 1, tile by tile, with
// the fp32 scan's dump / threshold / emit epilogue.  There is no GEMM form of the L1 distance, so this is a CUDA-core
// kernel: rows enter shared memory as fp32 once per CTA and K slice (the fp16 -> fp32 conversion is exact), every
// thread keeps a register tile of TR rows x TQ queries, and the inner step is two FP32 instructions per element --
// FADD for e - q and FADD with the |.| operand modifier for the accumulation.  Each accumulator sums its d terms in
// ascending k, so the key's error is that of a sequential float32 sum (query_prep_kernel's eps, DESIGN section 3.8).
//
// Replaces the per-row `embedding <+> query` PostgreSQL evaluates for vector_search (reference _typing.py:110-120).
#include <cuda_fp16.h>

#include "scan_common.cuh"

namespace rl {
namespace {

constexpr int kL1BK = 32;            // K slice
constexpr int kL1Pitch = kL1BK + 2;  // floats per shared row: 8-byte aligned, conflict-free 64-bit accesses

enum L1Storage { kF32Scalar = 0, kF32Vec4 = 1, kF16 = 2 };

// The tile: NT threads; RT = 128 / TR row threads x QT = NT / RT query threads.  Thread (rt, qt) owns rows
// rt + RT * i and queries qt + QT * j (strided, so a half-warp's 64-bit shared loads hit distinct banks).
template <int ST, int TR, int TQ, int NT>
__global__ void __launch_bounds__(NT) scan_l1_kernel(const ScanArgs a) {
  constexpr int RT = kBlockRows / TR;
  constexpr int QT = NT / RT;
  constexpr int CQ = QT * TQ;  // queries per CTA
  static_assert(RT * QT == NT, "tile");
  // Per-thread share of one K slice of rows: 16-byte chunks (8 halves / 4 floats) or single floats.
  constexpr int kRowItems = ST == kF16 ? kBlockRows * kL1BK / 8 / NT : ST == kF32Vec4 ? kBlockRows * kL1BK / 4 / NT
                                                                                      : kBlockRows * kL1BK / NT;
  constexpr int kQItems = (CQ * kL1BK + NT - 1) / NT;
  __shared__ __align__(16) float Es[kBlockRows * kL1Pitch];
  __shared__ __align__(16) float Qs[CQ * kL1Pitch];

  const int tid = threadIdx.x;
  const int qt = tid % QT, rt = tid / QT;
  const int64_t n_qg = (a.B + CQ - 1) / CQ;
  const int64_t ord = (int64_t)blockIdx.x / n_qg;   // query groups of one row block are neighbours: L2 reuse
  const int q0 = (int)((int64_t)blockIdx.x % n_qg) * CQ;
  const int64_t row0 = mode_block_index(a, ord) * kBlockRows;

  float acc[TR][TQ];
#pragma unroll
  for (int i = 0; i < TR; ++i)
#pragma unroll
    for (int j = 0; j < TQ; ++j) acc[i][j] = 0.f;

  uint4 er16[ST == kF16 ? kRowItems : 1];
  float4 er4[ST == kF32Vec4 ? kRowItems : 1];
  float er1[ST == kF32Scalar ? kRowItems : 1];
  float qr[kQItems];

  // Global -> registers for the slice at k0 (zeros past n_rows, d and B: |0 - 0| adds nothing).  Item t of a thread is
  // row (tid / kPer) + t * (NT / kPer) at the same column offset for every t, so one base pointer serves them all.
  constexpr int kPer = ST == kF16 ? kL1BK / 8 : ST == kF32Vec4 ? kL1BK / 4 : kL1BK;   // items per row and slice
  constexpr int kElems = kL1BK / kPer;                                                 // elements per item
  const int my_r = tid / kPer, my_k = (tid % kPer) * kElems;
  const int n_my_rows = a.n_rows - row0 < kBlockRows ? (int)(a.n_rows - row0) : kBlockRows;   // rows of the block that exist
  const int64_t row_step = (int64_t)(NT / kPer) * a.ld;
  const float* e_base = ST == kF16 ? reinterpret_cast<const float*>(reinterpret_cast<const __half*>(a.E) + (row0 + my_r) * a.ld + my_k)
                                   : a.E + (row0 + my_r) * a.ld + my_k;
  const int my_qi = tid / kL1BK, my_qk = tid % kL1BK;
  const float* q_base = a.Q + (size_t)(q0 + my_qi) * a.d + my_qk;
  auto load = [&](int k0) {
    const bool k_in = k0 + my_k < a.d;
#pragma unroll
    for (int t = 0; t < kRowItems; ++t) {
      const bool in = k_in && my_r + t * (NT / kPer) < n_my_rows;
      if constexpr (ST == kF16) {
        const __half* src = reinterpret_cast<const __half*>(e_base) + t * row_step + k0;
        er16[t] = in ? __ldg(reinterpret_cast<const uint4*>(src)) : make_uint4(0u, 0u, 0u, 0u);
      } else if constexpr (ST == kF32Vec4) {
        er4[t] = in ? __ldg(reinterpret_cast<const float4*>(e_base + t * row_step + k0)) : make_float4(0.f, 0.f, 0.f, 0.f);
      } else {
        er1[t] = in ? __ldg(e_base + t * row_step + k0) : 0.f;
      }
    }
    const bool qk_in = k0 + my_qk < a.d;
#pragma unroll
    for (int t = 0; t < kQItems; ++t) {
      const int qi = my_qi + t * (NT / kL1BK);
      qr[t] = (qi < CQ && q0 + qi < a.B && qk_in) ? __ldg(q_base + (size_t)t * (NT / kL1BK) * a.d + k0) : 0.f;
    }
  };
  // Registers -> shared memory, rows as fp32.
  auto store = [&]() {
#pragma unroll
    for (int t = 0; t < kRowItems; ++t) {
      const int c = tid + t * NT;
      if constexpr (ST == kF16) {
        float* dst = Es + (c >> 2) * kL1Pitch + (c & 3) * 8;
        const __half2* h = reinterpret_cast<const __half2*>(&er16[t]);
#pragma unroll
        for (int m = 0; m < 4; ++m) *reinterpret_cast<float2*>(dst + 2 * m) = __half22float2(h[m]);
      } else if constexpr (ST == kF32Vec4) {
        float* dst = Es + (c >> 3) * kL1Pitch + (c & 7) * 4;
        *reinterpret_cast<float2*>(dst) = make_float2(er4[t].x, er4[t].y);
        *reinterpret_cast<float2*>(dst + 2) = make_float2(er4[t].z, er4[t].w);
      } else {
        Es[(c >> 5) * kL1Pitch + (c & 31)] = er1[t];
      }
    }
#pragma unroll
    for (int t = 0; t < kQItems; ++t) {
      const int c = tid + t * NT;
      if (c < CQ * kL1BK) Qs[(c >> 5) * kL1Pitch + (c & 31)] = qr[t];
    }
  };

  load(0);
  for (int k0 = 0; k0 < a.d; k0 += kL1BK) {
    __syncthreads();
    store();
    __syncthreads();
    if (k0 + kL1BK < a.d) load(k0 + kL1BK);   // next slice in flight while this one is summed
#pragma unroll
    for (int kk = 0; kk < kL1BK; kk += 2) {
      float2 e[TR], q[TQ];
#pragma unroll
      for (int i = 0; i < TR; ++i) e[i] = *reinterpret_cast<const float2*>(Es + (rt + RT * i) * kL1Pitch + kk);
#pragma unroll
      for (int j = 0; j < TQ; ++j) q[j] = *reinterpret_cast<const float2*>(Qs + (qt + QT * j) * kL1Pitch + kk);
#pragma unroll
      for (int i = 0; i < TR; ++i)
#pragma unroll
        for (int j = 0; j < TQ; ++j) acc[i][j] += fabsf(e[i].x - q[j].x);
#pragma unroll
      for (int i = 0; i < TR; ++i)
#pragma unroll
        for (int j = 0; j < TQ; ++j) acc[i][j] += fabsf(e[i].y - q[j].y);
    }
  }

  // Epilogue (scan_fp32_kernel's, plus the masked-row count of RL_FLAG_COUNT_UNFILTERED): dump (sample blocks)
  // or threshold + emit (the rest).
  float thr[TQ];
#pragma unroll
  for (int j = 0; j < TQ; ++j) {
    const int col = q0 + qt + QT * j;
    thr[j] = (!a.dump_mode && col < a.B) ? a.thr[col] : 0.f;
  }
#pragma unroll
  for (int i = 0; i < TR; ++i) {
    const int r_in = rt + RT * i;
    const int64_t row = row0 + r_in;
    bool valid = row < a.n_rows, masked_alive = false;
    if (valid && a.row_allowed != nullptr) {
      valid = a.row_allowed[row] != 0;
      if (!valid && a.cnt_all != nullptr) masked_alive = a.row_alive == nullptr || a.row_alive[row] != 0;
    }
#pragma unroll
    for (int j = 0; j < TQ; ++j) {
      const int col = q0 + qt + QT * j;
      if (col >= a.B) continue;
      const float key = -acc[i][j];
      if (a.dump_mode) {
        a.dump[(size_t)col * a.n_sample_rows + ord * kBlockRows + r_in] = valid ? key : kNegInf;
      } else if (key >= thr[j]) {
        if (valid) emit_candidate(a, col, key, (int32_t)row);
        else if (masked_alive) atomicAdd(a.cnt_all + col, 1);
      }
    }
  }
}

template <int TR, int TQ, int NT>
int launch_l1_tile(const ScanArgs& a, int storage, cudaStream_t stream) {
  constexpr int CQ = NT / (kBlockRows / TR) * TQ;
  const int64_t n_ctas = a.n_mode_blocks * ((a.B + CQ - 1) / CQ);
  RL_REQUIRE(n_ctas < (1ll << 31), RL_EUNSUPPORTED, "scan_l1: too many blocks");
  if (storage == kF16) scan_l1_kernel<kF16, TR, TQ, NT><<<(unsigned)n_ctas, NT, 0, stream>>>(a);
  else if (storage == kF32Vec4) scan_l1_kernel<kF32Vec4, TR, TQ, NT><<<(unsigned)n_ctas, NT, 0, stream>>>(a);
  else scan_l1_kernel<kF32Scalar, TR, TQ, NT><<<(unsigned)n_ctas, NT, 0, stream>>>(a);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

}  // namespace

int launch_scan_l1(const ScanArgs& a, bool e_f16, cudaStream_t stream) {
  if (a.n_mode_blocks == 0 || a.B == 0) return RL_OK;
  const bool vec = (a.d % 4 == 0) && (a.ld % 4 == 0) && ((reinterpret_cast<uintptr_t>(a.E) & 15) == 0);
  const int storage = e_f16 ? kF16 : vec ? kF32Vec4 : kF32Scalar;
  // The tile follows B.  Up to 8 queries, one thread per row and every query of the batch in its registers: the
  // scan reads the corpus once and stays near the HBM bound.  Beyond, 8 rows x 4 or 8 queries per thread (64- or
  // 128-query CTAs, whichever pads B less): 16 or 32 FADD pairs per four 64-bit shared loads, near the FP32 issue
  // bound.
  if (a.B == 1) return launch_l1_tile<1, 1, 128>(a, storage, stream);
  if (a.B == 2) return launch_l1_tile<1, 2, 128>(a, storage, stream);
  if (a.B <= 4) return launch_l1_tile<1, 4, 128>(a, storage, stream);
  if (a.B <= 8) return launch_l1_tile<1, 8, 128>(a, storage, stream);
  if ((a.B + 127) / 128 * 128 <= (a.B + 63) / 64 * 64) return launch_l1_tile<8, 8, 256>(a, storage, stream);
  return launch_l1_tile<8, 4, 256>(a, storage, stream);
}

}  // namespace rl
