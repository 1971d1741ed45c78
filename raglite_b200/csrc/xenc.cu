// BERT cross-encoder forward (ms-marco-MiniLM-L-12 architecture) for sm_90a: the arithmetic behind
// rerank_chunks (reference _search.py:364-397 -> rerankers FlashRankRanker -> onnxruntime, all
// third-party).  Variable-length packed batches (no padding): tokens [T, H], cu_seqlens [P + 1].
//
//   embed_ln_kernel      word + position + token-type embeddings, LayerNorm          (fp32 math, fp16 out)
//   linear_wgmma_kernel  Y = act(X W^T + b): wgmma (M=128 tokens, N<=128 outputs per pass, K
//                        sliced by 64), X through a TMA tensor map into 128B-swizzled smem, W as a
//                        pre-swizzled fp16 image fetched with cp.async.bulk, fp32 accumulate in
//                        registers, bias / GELU(erf) fused in the epilogue
//   attention2_kernel    softmax(Q K^T / sqrt(dh)) V per (sequence, head) at head_dim 32, fp32 math
//                        (attention64_kernel: head_dim 64, the token encoder of rl_xenc_encode)
//   add_ln_kernel        LayerNorm(x + residual)
//   cls_head_kernel      pooler (dense + tanh on [CLS]) -> classifier -> 1 or 2 logits, FlashRank's score
//                        (BERT's pooler + classifier; XLM-RoBERTa's classifier.dense + out_proj is the same head)
#include <cuda.h>
#include <cuda_fp16.h>

#include <type_traits>

#include "common.cuh"
#include "hopper_ptx.cuh"
#include "qimg.cuh"

namespace rl {
namespace {

using namespace tc;

constexpr int kTileM = 128;          // tokens per tile (two consumer warpgroups of M = 64)
constexpr int kSliceK = 64;          // fp16 elements per K slice = one 128-byte swizzle row
constexpr int kPassN = 128;          // output columns per pass (wgmma N)
constexpr int kLinConsumerWarps = 8;
constexpr int kLinProdWarp = 8;
constexpr int kLinThreads = (kLinConsumerWarps + 1) * 32;
constexpr int kMaxStages = 8;
constexpr int kABytes = kTileM * 128;
// Activations + weight slice: 32 KB.  The wgmma always reads kPassN weight rows; the short last pass of a layer
// copies only its nb rows, so the rest of the stage's weight region holds stale rows.  They stay inside the stage and
// only feed accumulator columns >= nb, which the epilogue never stores.
constexpr uint32_t kLinStageBytes = kABytes + kPassN * 128u;
constexpr uint32_t kEpiPitch = kPassN * 2 + 16;                 // bytes per staged row: 256 B of fp16 + pad (conflict-free)
constexpr uint32_t kEpiBytes = kTileM * kEpiPitch;
constexpr uint32_t kSmemBudget = 227 * 1024;

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}
__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// GELU(x) = x/2 (1 + erf(x / sqrt 2)) with erfc from Abramowitz & Stegun 7.1.28,
// 1 - erf(z) = (1 + a1 z + ... + a6 z^6)^-16 (|error| <= 3e-7; 8e-7 on the GELU value in float32, far
// below the fp16 rounding of the stored activation): 6 FMAs, 4 squarings and ONE special-function op.
// The epilogue is bound by the ALU / MUFU pipes, so the instruction count per element is what counts.
__device__ __forceinline__ float gelu_erf(float x) {
  const float z = fabsf(x) * 0.70710678118654752f;
  float p = fmaf(0.0000430638f, z, 0.0002765672f);
  p = fmaf(p, z, 0.0001520143f);
  p = fmaf(p, z, 0.0092705272f);
  p = fmaf(p, z, 0.0422820123f);
  p = fmaf(p, z, 0.0705230784f);
  p = fmaf(p, z, 1.f);
  p *= p; p *= p; p *= p; p *= p;   // p^16 (overflows to +inf for huge z: the tail is then exactly 0)
  float tail;                       // 1 - erf(z), z >= 0
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(tail) : "f"(p));
  const float half_x = 0.5f * x;
  // x >= 0: x/2 (2 - tail);  x < 0: x/2 tail
  return half_x * (x >= 0.f ? 2.f - tail : tail);
}

// ---- weight image: W[N, K] fp32 row-major -> per (pass, k-slice) swizzled fp16 wgmma B tiles -------------
// A pass is kPassN output columns; the last pass may be shorter (its slices have that pitch).
__host__ __device__ inline int pass_rows(int N, int pass) {
  const int rem = N - pass * kPassN;
  return rem < kPassN ? rem : kPassN;
}
__host__ __device__ inline size_t pass_offset_halves(int K, int pass) {
  const int n_ks = (K + kSliceK - 1) / kSliceK;
  return (size_t)pass * kPassN * n_ks * kSliceK;  // full passes precede; only the last pass is short
}

__global__ void pack_linear_kernel(const float* __restrict__ W, int N, int K, __half* __restrict__ img) {
  const int n_ks = (K + kSliceK - 1) / kSliceK;
  const int64_t total = (int64_t)((N + 15) / 16 * 16) * n_ks * kSliceK;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int n = (int)(idx / (n_ks * kSliceK));
    const int kk = (int)(idx % (n_ks * kSliceK));
    const int pass = n / kPassN, r = n % kPassN;
    const int nb = (pass_rows(N, pass) + 15) / 16 * 16;
    const int ks = kk / kSliceK, e = kk % kSliceK;
    const float v = (n < N && kk < K) ? W[(size_t)n * K + kk] : 0.f;
    const size_t off = pass_offset_halves(K, pass) + ((size_t)ks * nb + r) * kSliceK +
                       (size_t)((((e >> 3) ^ (r & 7)) << 3) + (e & 7));
    img[off] = __float2half_rn(v);
  }
}

// ---- wgmma linear layer ---------------------------------------------------------------------------------
// Y[T, N] = act(X W^T + b).  A work item is one (128-token tile, kPassN-column pass); CTA c takes items c, c + grid, ...
// (passes fastest, so the CTAs working at the same time share their activation tiles in L2).  Per K slice the
// producer thread issues one TMA tensor-map copy of the activations (box 64 x 128, SWIZZLE_128B: rows past T and
// columns past K arrive as zeros) and one bulk copy of the pre-swizzled weight slice into a stage; two consumer
// warpgroups (64 tokens each) run wgmma.m64n128k16 on it and, after the last slice, add the bias, apply the
// activation, round to fp16 and stage the tile in shared memory so that it leaves as 16-byte row-contiguous stores.
// Epilogue of one work item, run by each consumer warpgroup on its 64 tokens: + bias -> activation -> fp16 -> shared
// staging (columns >= nb belong to no output: skipped) -> 16-byte row-contiguous stores.
__device__ __forceinline__ void linear_epilogue(const float (&acc)[64], const float* __restrict__ bias, __half* __restrict__ Y,
                                                int ldy, int T, int N, int act, int m_tile, int pass, int wg,
                                                unsigned char* stg) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wt = threadIdx.x & 127;
  const int r_lo = (warp & 3) * 16 + (lane >> 2);   // rows r_lo and r_lo + 8 of this warpgroup's 64
  const int c_lane = 2 * (lane & 3);
  const int nb = pass_rows(N, pass);
  const int n0 = pass * kPassN;
#pragma unroll
  for (int c8 = 0; c8 < kPassN / 8; ++c8) {
    if (8 * c8 >= nb) break;
    const int c = 8 * c8 + c_lane;
    const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + n0 + c));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float x0 = acc[4 * c8 + 2 * h] + bb.x, x1 = acc[4 * c8 + 2 * h + 1] + bb.y;
      if (act == 1) { x0 = gelu_erf(x0); x1 = gelu_erf(x1); }
      *reinterpret_cast<uint32_t*>(stg + (uint32_t)(r_lo + 8 * h) * kEpiPitch + (uint32_t)c * 2u) = pack_half2(x0, x1);
    }
  }
  named_bar_sync(2 + wg, 128);
  const int row_chunks = nb / 8;   // 16-byte chunks per row (nb is a multiple of 32)
  const int row_base = m_tile * kTileM + wg * 64;
  for (int idx = wt; idx < 64 * row_chunks; idx += 128) {
    const int rr = idx / row_chunks, ch = idx - rr * row_chunks;
    const int grow = row_base + rr;
    if (grow < T)
      *reinterpret_cast<uint4*>(Y + (size_t)grow * ldy + n0 + ch * 8) =
          *reinterpret_cast<const uint4*>(stg + (uint32_t)rr * kEpiPitch + (uint32_t)ch * 16u);
  }
  named_bar_sync(2 + wg, 128);   // the staging buffer is free for the next item
}

struct LinArgs {
  const __half* img;   // packed weights
  const float* bias;   // [N]
  __half* Y;           // [T, ldy]
  int ldy, T, N, K, act;    // act: 0 none, 1 GELU(erf)
  int n_pass, n_ks, stages;
};

__global__ void __launch_bounds__(kLinThreads, 1) linear_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const LinArgs t) {
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* base = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
  uint64_t* full = reinterpret_cast<uint64_t*>(base + (size_t)t.stages * kLinStageBytes);
  uint64_t* empty = full + kMaxStages;
  unsigned char* epi = reinterpret_cast<unsigned char*>(empty + kMaxStages);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_tiles = (t.T + kTileM - 1) / kTileM;
  const int64_t n_items = (int64_t)m_tiles * t.n_pass;
  const int64_t first = blockIdx.x, stride = gridDim.x;
  const int64_t my_items = first < n_items ? (n_items - first + stride - 1) / stride : 0;

  if (threadIdx.x == 0) {
    for (int i = 0; i < t.stages; ++i) {
      mbar_init(&full[i], 1);                    // the producer's expect_tx
      mbar_init(&empty[i], kLinConsumerWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kLinProdWarp) {
    if (lane == 0 && my_items > 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
      int stage = 0;
      uint32_t phase = 0;
      for (int64_t it = 0; it < my_items; ++it) {
        const int64_t item = first + it * stride;
        const int m_tile = (int)(item / t.n_pass), pass = (int)(item % t.n_pass);
        const int nb = (pass_rows(t.N, pass) + 15) / 16 * 16;
        const uint32_t wbytes = (uint32_t)nb * 128u;
        const __half* src = t.img + pass_offset_halves(t.K, pass);
        for (int ks = 0; ks < t.n_ks; ++ks) {
          mbar_wait(&empty[stage], phase ^ 1u);
          unsigned char* st = base + (size_t)stage * kLinStageBytes;
          mbar_arrive_expect_tx(&full[stage], (uint32_t)kABytes + wbytes);
          tma_load_2d(st, &tmA, ks * kSliceK, m_tile * kTileM, &full[stage]);
          bulk_g2s(st + kABytes, src + (size_t)ks * nb * kSliceK, wbytes, &full[stage]);
          if (++stage == t.stages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else if (warp < kLinConsumerWarps) {
    const int wg = warp >> 2;
    unsigned char* stg = epi + (size_t)wg * 64 * kEpiPitch;
    int stage = 0;
    uint32_t phase = 0;
    float acc[64];
    for (int64_t it = 0; it < my_items; ++it) {
      const int64_t item = first + it * stride;
      const int m_tile = (int)(item / t.n_pass), pass = (int)(item % t.n_pass);
      int prev = -1;
      for (int ks = 0; ks < t.n_ks; ++ks) {
        mbar_wait(&full[stage], phase);
        const uint32_t st_addr = smem_u32(base + (size_t)stage * kLinStageBytes);
        wgmma_fence();
        wgmma_slice(acc, make_kmajor_sw128_desc(st_addr + (uint32_t)wg * (64u * 128u)), make_kmajor_sw128_desc(st_addr + kABytes),
                    ks > 0);
        wgmma_commit();
        if (prev >= 0) {
          wgmma_wait<1>();
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[prev]);
        }
        prev = stage;
        if (++stage == t.stages) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[prev]);
      linear_epilogue(acc, t.bias, t.Y, t.ldy, t.T, t.N, t.act, m_tile, pass, wg, stg);
    }
  }
}

// ---- GGUF-quantized weights (types and image layout: qimg.cuh) -----------------------------------------
// The small integer u (< 2^23) as float without a conversion instruction: its bits under 2^23's exponent, minus 2^23 +
// `bias`.  Exact, so (float)(u - bias) either way.
__device__ __forceinline__ float small_int_f(uint32_t u, float bias) {
  return __fsub_rn(__uint_as_float(0x4B000000u | u), 8388608.f + bias);
}
__device__ __forceinline__ float ld_half(const unsigned char* p) {
  return __half2float(__ushort_as_half(*reinterpret_cast<const unsigned short*>(p)));
}
// rows x K elements from GGUF blocks (row r's blocks at r * K / block_elems) to fp16: one thread per element.
__global__ void dequant_rows_kernel(int type, const unsigned char* __restrict__ blocks, int64_t rows, int K,
                                    __half* __restrict__ out) {
  const int be = q_block_elems(type), bb = q_block_bytes(type);
  const int64_t total = rows * K;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx / K;
    const int k = (int)(idx - r * K);
    const unsigned char* b = blocks + (r * (K / be) + k / be) * bb;
    const int e = k % be;
    float y;
    if (type == kGgmlQ8_0) {
      y = __fmul_rn(ld_half(b), (float)(int8_t)b[2 + e]);
    } else if (type == kGgmlQ4_K) {
      // ggml walks 64 elements at a time: 32 low nibbles (sub-block 2 j64), then the same 32 bytes' high nibbles
      const int j64 = e / 64, hi = (e % 64) / 32, l = e % 32;
      int sc, m;
      q4k_scale_min(2 * j64 + hi, b + 4, sc, m);
      const int q = (b[16 + 32 * j64 + l] >> (4 * hi)) & 0xF;
      y = __fsub_rn(__fmul_rn(__fmul_rn(ld_half(b), (float)sc), (float)q), __fmul_rn(ld_half(b + 2), (float)m));
    } else {
      // 128 elements at a time (n): four groups g of 32 from ql[64 n ..], qh[32 n ..], scales[8 n ..]
      const int n = e / 128, g = (e % 128) / 32, l = e % 32;
      const unsigned char* ql = b + 64 * n;
      const unsigned char* qh = b + 128 + 32 * n;
      const int8_t* sc = reinterpret_cast<const int8_t*>(b + 192 + 8 * n);
      const int q = ((ql[l + 32 * (g & 1)] >> (4 * (g >> 1))) & 0xF) | (((qh[l] >> (2 * g)) & 3) << 4);
      y = __fmul_rn(__fmul_rn(ld_half(b + 208), (float)sc[l / 16 + 2 * g]), (float)(q - 32));
    }
    out[idx] = __float2half_rn(y);
  }
}

// ---- quantized weight image (layout: qimg.cuh) -----------------------------------------------------
static_assert(kPassN == kQPassRows, "a wgmma pass is one image pass");
inline size_t q_pass_bytes(int type, int N, int K, int pass) {
  const int nb16 = (pass_rows(N, pass) + 15) / 16 * 16;
  return (size_t)(K / kQSliceK) * nb16 * q_row_bytes(type);
}

// One thread per (pass, K slice, row): reorders the row's GGUF bytes of that slice into the image.
__global__ void pack_qlinear_kernel(int type, const unsigned char* __restrict__ blocks, int N, int K, unsigned char* __restrict__ img) {
  const int n_qs = K / kQSliceK, n_pass = (N + kPassN - 1) / kPassN;
  const uint32_t rb = q_row_bytes(type);
  const int be = q_block_elems(type), bb = q_block_bytes(type);
  const int64_t total = (int64_t)n_pass * n_qs * kPassN;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(idx % kPassN);
    const int s = (int)((idx / kPassN) % n_qs);
    const int pass = (int)(idx / ((int64_t)kPassN * n_qs));
    const int nb16 = (pass_rows(N, pass) + 15) / 16 * 16;
    if (r >= nb16) continue;
    const int n = pass * kPassN + r;
    unsigned char* o = img + kQImgData + (size_t)pass * kPassN * n_qs * rb + ((size_t)s * nb16 + r) * rb;
    if (n >= N) {
      for (uint32_t i = 0; i < rb; ++i) o[i] = 0;
      continue;
    }
    const unsigned char* row = blocks + (size_t)n * (K / be) * bb;
    const int k0 = s * kQSliceK;
    if (type == kGgmlQ8_0) {
      for (int i = 0; i < 4; ++i) {
        const unsigned char* b = row + (size_t)(k0 / 32 + i) * bb;
        o[2 * i] = b[0];
        o[2 * i + 1] = b[1];
        for (int l = 0; l < 32; ++l) o[8 + 32 * i + l] = b[2 + l];
      }
    } else if (type == kGgmlQ4_K) {
      const unsigned char* b = row + (size_t)(k0 / 256) * bb;
      const int h = (k0 / 128) & 1;
      for (int i = 0; i < 4; ++i) o[i] = b[i];
      for (int i = 0; i < 4; ++i) {
        int sc, m;
        q4k_scale_min(4 * h + i, b + 4, sc, m);
        o[4 + i] = (unsigned char)sc;
        o[8 + i] = (unsigned char)m;
      }
      for (int i = 0; i < 64; ++i) o[12 + i] = b[16 + 64 * h + i];
    } else {
      const unsigned char* b = row + (size_t)(k0 / 256) * bb;
      const int h = (k0 / 128) & 1;
      for (int i = 0; i < 64; ++i) o[i] = b[64 * h + i];
      for (int i = 0; i < 32; ++i) o[64 + i] = b[128 + 32 * h + i];
      for (int i = 0; i < 8; ++i) o[96 + i] = b[192 + 8 * h + i];
      o[104] = b[208];
      o[105] = b[209];
      o[106] = o[107] = 0;
    }
  }
}

// Four fp16 values from the four bytes of w (each < 2^23 after `bias` is added back), as two half2 words:
// y_i = mul(scale, byte_i - bias) - sub.
template <bool SUB>
__device__ __forceinline__ uint2 dq4(uint32_t w, float bias, float scale, float sub) {
  float y[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float q = small_int_f(__byte_perm(w, 0u, 0x4440u + i), bias);
    y[i] = SUB ? __fsub_rn(__fmul_rn(scale, q), sub) : __fmul_rn(scale, q);
  }
  return make_uint2(pack_half2(y[0], y[1]), pack_half2(y[2], y[3]));
}

// Dequantize one image row's half slice (64 elements: B slice `half` of the stage) into the 128B-swizzled fp16 rows the
// wgmma reads: chunk c (elements 8c .. 8c + 7) of row r lands at r * 128 + ((c ^ (r & 7)) * 16).
__device__ __forceinline__ void dequant_row_half(int type, const unsigned char* __restrict__ src, int half, int r,
                                                 unsigned char* __restrict__ dst) {
  unsigned char* drow = dst + (uint32_t)r * 128u;
  auto put = [&](int c, uint2 lo, uint2 hi) {
    *reinterpret_cast<uint4*>(drow + ((c ^ (r & 7)) << 4)) = make_uint4(lo.x, lo.y, hi.x, hi.y);
  };
  if (type == kGgmlQ8_0) {
    const uint32_t* q = reinterpret_cast<const uint32_t*>(src + 8 + 64 * half);
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      const float d = ld_half(src + 2 * (2 * half + b));
#pragma unroll
      for (int c = 0; c < 4; ++c)   // int8 q + 128 = the byte with its top bit flipped
        put(4 * b + c, dq4<false>(q[8 * b + 2 * c] ^ 0x80808080u, 128.f, d, 0.f),
            dq4<false>(q[8 * b + 2 * c + 1] ^ 0x80808080u, 128.f, d, 0.f));
    }
  } else if (type == kGgmlQ4_K) {
    const float d = ld_half(src), dmin = ld_half(src + 2);
    const uint32_t* q = reinterpret_cast<const uint32_t*>(src + 12 + 32 * half);
#pragma unroll
    for (int sub = 0; sub < 2; ++sub) {   // low nibbles: sub-block 2 half, high nibbles: 2 half + 1
      const float d1 = __fmul_rn(d, (float)src[4 + 2 * half + sub]);
      const float m1 = __fmul_rn(dmin, (float)src[8 + 2 * half + sub]);
#pragma unroll
      for (int c = 0; c < 4; ++c)
        put(4 * sub + c, dq4<true>((q[2 * c] >> (4 * sub)) & 0x0F0F0F0Fu, 0.f, d1, m1),
            dq4<true>((q[2 * c + 1] >> (4 * sub)) & 0x0F0F0F0Fu, 0.f, d1, m1));
    }
  } else {
    const float d = ld_half(src + 104);
    const int8_t* sc = reinterpret_cast<const int8_t*>(src + 96);
    const uint32_t* qh = reinterpret_cast<const uint32_t*>(src + 64);
#pragma unroll
    for (int gg = 0; gg < 2; ++gg) {   // group g = 2 half + gg: ql bytes 32 (g & 1) on, nibble g >> 1, qh bits 2 g
      const int g = 2 * half + gg;
      const uint32_t* ql = reinterpret_cast<const uint32_t*>(src + 32 * (g & 1));
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const float ds = __fmul_rn(d, (float)sc[c / 2 + 2 * g]);
        uint2 v[2];
#pragma unroll
        for (int w = 0; w < 2; ++w) {
          const int i = 2 * c + w;
          const uint32_t q = ((ql[i] >> (4 * half)) & 0x0F0F0F0Fu) | (((qh[i] >> (2 * g)) & 0x03030303u) << 4);
          v[w] = dq4<false>(q, 32.f, ds, 0.f);
        }
        put(4 * gg + c, v[0], v[1]);
      }
    }
  }
}

// ---- wgmma linear layer on a quantized image ----------------------------------------------------------------
// linear_wgmma_kernel's work items, wgmma sequence (slices of 64 in ascending K) and epilogue.  A stage spans 128 K: the
// producer issues two TMA copies of the activations and one bulk copy of the slice's quantized rows; eight dequantizer
// warps (a thread per row and 64-element half) expand them into the stage's two swizzled fp16 B tiles, fence them for
// the async proxy and arrive on the stage's full barrier beside the activations' transaction count.
constexpr int kDqWarps = 8;
constexpr int kQLinDqWarp0 = kLinProdWarp + 1;
constexpr int kQLinThreads = (kLinConsumerWarps + 1 + kDqWarps) * 32;
constexpr uint32_t kQABytes = 2 * kABytes;                     // two 64-wide activation slices
constexpr uint32_t kQBBytes = 2 * kPassN * 128u;               // two swizzled fp16 weight slices
constexpr uint32_t kQRawBytes = kPassN * kQMaxRowBytes;        // quantized rows as they arrive
constexpr uint32_t kQStageBytes = kQABytes + kQBBytes + kQRawBytes;   // 81 KB, a multiple of 1024
constexpr int kQMaxStages = 4;

struct QLinArgs {
  const unsigned char* img;   // quantized image
  const float* bias;          // [N]
  __half* Y;                  // [T, ldy]
  int ldy, T, N, K, act;
  int n_pass, n_qs, stages;
};

__global__ void __launch_bounds__(kQLinThreads, 1) linear_q_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const QLinArgs t) {
  extern __shared__ unsigned char smem_dyn[];
  unsigned char* base = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
  uint64_t* full = reinterpret_cast<uint64_t*>(base + (size_t)t.stages * kQStageBytes);
  uint64_t* raw = full + kQMaxStages;
  uint64_t* empty = raw + kQMaxStages;
  unsigned char* epi = reinterpret_cast<unsigned char*>(empty + kQMaxStages);
  const QImgPass* passes = reinterpret_cast<const QImgPass*>(t.img + sizeof(QImgHead));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_tiles = (t.T + kTileM - 1) / kTileM;
  const int64_t n_items = (int64_t)m_tiles * t.n_pass;
  const int64_t first = blockIdx.x, stride = gridDim.x;
  const int64_t my_items = first < n_items ? (n_items - first + stride - 1) / stride : 0;

  if (threadIdx.x == 0) {
    for (int i = 0; i < t.stages; ++i) {
      mbar_init(&full[i], 1 + kDqWarps);         // the producer's expect_tx + one arrival per dequantizer warp
      mbar_init(&raw[i], 1);
      mbar_init(&empty[i], kLinConsumerWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kLinProdWarp) {
    if (lane == 0 && my_items > 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
      int stage = 0;
      uint32_t phase = 0;
      for (int64_t it = 0; it < my_items; ++it) {
        const int64_t item = first + it * stride;
        const int m_tile = (int)(item / t.n_pass), pass = (int)(item % t.n_pass);
        const QImgPass pp = passes[pass];
        const uint32_t qbytes = (uint32_t)((pass_rows(t.N, pass) + 15) / 16 * 16) * (uint32_t)pp.row_bytes;
        const unsigned char* src = t.img + pp.offset;
        for (int qs = 0; qs < t.n_qs; ++qs) {
          mbar_wait(&empty[stage], phase ^ 1u);
          unsigned char* st = base + (size_t)stage * kQStageBytes;
          mbar_arrive_expect_tx(&full[stage], kQABytes);
          tma_load_2d(st, &tmA, 2 * qs * kSliceK, m_tile * kTileM, &full[stage]);
          tma_load_2d(st + kABytes, &tmA, (2 * qs + 1) * kSliceK, m_tile * kTileM, &full[stage]);
          mbar_arrive_expect_tx(&raw[stage], qbytes);
          bulk_g2s(st + kQABytes + kQBBytes, src + (size_t)qs * qbytes, qbytes, &raw[stage]);
          if (++stage == t.stages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else if (warp >= kQLinDqWarp0) {
    const int dt = threadIdx.x - kQLinDqWarp0 * 32;
    const int r = dt & (kPassN - 1), half = dt / kPassN;
    int stage = 0;
    uint32_t phase = 0;
    for (int64_t it = 0; it < my_items; ++it) {
      const int64_t item = first + it * stride;
      const int pass = (int)(item % t.n_pass);
      const QImgPass pp = passes[pass];
      const bool live = r < pass_rows(t.N, pass);   // the rest of the B rows feed no stored column: left stale
      for (int qs = 0; qs < t.n_qs; ++qs) {
        mbar_wait(&raw[stage], phase);
        unsigned char* st = base + (size_t)stage * kQStageBytes;
        if (live)
          dequant_row_half(pp.type, st + kQABytes + kQBBytes + (uint32_t)r * (uint32_t)pp.row_bytes, half, r,
                           st + kQABytes + (uint32_t)half * (kPassN * 128u));
        fence_proxy_async();   // the generic-proxy stores become visible to the consumers' wgmma
        __syncwarp();
        if (lane == 0) mbar_arrive(&full[stage]);
        if (++stage == t.stages) { stage = 0; phase ^= 1u; }
      }
    }
  } else {
    const int wg = warp >> 2;
    unsigned char* stg = epi + (size_t)wg * 64 * kEpiPitch;
    int stage = 0;
    uint32_t phase = 0;
    float acc[64];
    for (int64_t it = 0; it < my_items; ++it) {
      const int64_t item = first + it * stride;
      const int m_tile = (int)(item / t.n_pass), pass = (int)(item % t.n_pass);
      int prev = -1;
      for (int qs = 0; qs < t.n_qs; ++qs) {
        mbar_wait(&full[stage], phase);
        const uint32_t st_addr = smem_u32(base + (size_t)stage * kQStageBytes);
        wgmma_fence();
#pragma unroll
        for (int h = 0; h < 2; ++h)
          wgmma_slice(acc, make_kmajor_sw128_desc(st_addr + (uint32_t)h * kABytes + (uint32_t)wg * (64u * 128u)),
                      make_kmajor_sw128_desc(st_addr + kQABytes + (uint32_t)h * (kPassN * 128u)), qs > 0 || h > 0);
        wgmma_commit();
        if (prev >= 0) {
          wgmma_wait<1>();
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[prev]);
        }
        prev = stage;
        if (++stage == t.stages) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[prev]);
      linear_epilogue(acc, t.bias, t.Y, t.ldy, t.T, t.N, t.act, m_tile, pass, wg, stg);
    }
  }
}

// 16-byte asynchronous global -> shared copy (zero-fills when src_bytes == 0).
__device__ __forceinline__ void cp_async_16(uint32_t dst_smem, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst_smem), "l"(src), "r"(src_bytes) : "memory");
}


// ---- embeddings + LayerNorm: one warp per token ----------------------------------------------------------
// NC columns per lane: H <= 32 NC (16 for the cross-encoder's H <= 512, 32 for H <= 1024).
template <int NC>
__global__ void __launch_bounds__(256) embed_ln_kernel(const int32_t* __restrict__ ids, const int32_t* __restrict__ type_ids,
                                                       const int32_t* __restrict__ pos_ids, const __half* __restrict__ word,
                                                       const __half* __restrict__ pos, const __half* __restrict__ type,
                                                       const float* __restrict__ g, const float* __restrict__ bta, float eps,
                                                       int T, int H, int vocab, int max_pos, int type_vocab,
                                                       __half* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int tok = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (tok >= T) return;
  // ids are validated on the host (_xenc.py); the clamp only keeps a bad caller from reading out of bounds
  const __half* w = word + (size_t)min(max(ids[tok], 0), vocab - 1) * H;
  const __half* p = pos + (size_t)min(max(pos_ids[tok], 0), max_pos - 1) * H;
  const __half* ty = type + (size_t)min(max(type_ids[tok], 0), type_vocab - 1) * H;
  float x[NC];  // H <= 32 NC
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NC; ++i) {
    const int c = lane + 32 * i;
    x[i] = c < H ? __half2float(w[c]) + __half2float(p[c]) + __half2float(ty[c]) : 0.f;
    s += x[i];
  }
  const float mean = warp_sum_f(s) / (float)H;
  float var = 0.f;
#pragma unroll
  for (int i = 0; i < NC; ++i) {
    const int c = lane + 32 * i;
    if (c < H) var += (x[i] - mean) * (x[i] - mean);
  }
  const float rstd = rsqrtf(warp_sum_f(var) / (float)H + eps);
#pragma unroll
  for (int i = 0; i < NC; ++i) {
    const int c = lane + 32 * i;
    if (c < H) out[(size_t)tok * H + c] = __float2half_rn((x[i] - mean) * rstd * g[c] + bta[c]);
  }
}

// Four consecutive LayerNorm outputs: fp16 rows (8 bytes) inside the encoder, fp32 rows (16 bytes) for the last
// layer of rl_xenc_encode.
__device__ __forceinline__ void store4(__half* row, int piece, float a, float b, float c, float d) {
  uint2 o;
  o.x = pack_half2(a, b);
  o.y = pack_half2(c, d);
  reinterpret_cast<uint2*>(row)[piece] = o;
}
__device__ __forceinline__ void store4(float* row, int piece, float a, float b, float c, float d) {
  reinterpret_cast<float4*>(row)[piece] = make_float4(a, b, c, d);
}
__device__ __forceinline__ void store1(__half* p, float a) { *p = __float2half_rn(a); }
__device__ __forceinline__ void store1(float* p, float a) { *p = a; }

// out = LayerNorm(x + res), one warp per token.  H % 128 == 0 (384 for MiniLM): a lane owns the columns
// lane * 4 + 128 i, so every load / store instruction of the warp covers 256 contiguous bytes (8-byte pieces)
// rather than 2 bytes per lane and instruction.  NC columns per lane: H <= 32 NC.  OutT: __half, or float for
// the fp32 rows rl_xenc_encode returns.
template <bool VEC, int NC = 16, typename OutT = __half>
__global__ void __launch_bounds__(256) add_ln_kernel(const __half* __restrict__ xin, const __half* __restrict__ res,
                                                     const float* __restrict__ g, const float* __restrict__ bta, float eps,
                                                     int T, int H, OutT* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int tok = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (tok >= T) return;
  float x[NC];   // H <= 32 NC
  float s = 0.f;
  if (VEC) {
    const uint2* xi = reinterpret_cast<const uint2*>(xin + (size_t)tok * H);
    const uint2* ri = reinterpret_cast<const uint2*>(res + (size_t)tok * H);
#pragma unroll
    for (int i = 0; i < NC / 4; ++i) {
      if (i * 128 < H) {
        const uint2 a = __ldg(xi + lane + 32 * i), r = __ldg(ri + lane + 32 * i);
        const float2 a0 = __half22float2(*reinterpret_cast<const __half2*>(&a.x)), a1 = __half22float2(*reinterpret_cast<const __half2*>(&a.y));
        const float2 r0 = __half22float2(*reinterpret_cast<const __half2*>(&r.x)), r1 = __half22float2(*reinterpret_cast<const __half2*>(&r.y));
        x[4 * i] = a0.x + r0.x; x[4 * i + 1] = a0.y + r0.y; x[4 * i + 2] = a1.x + r1.x; x[4 * i + 3] = a1.y + r1.y;
        s += (x[4 * i] + x[4 * i + 1]) + (x[4 * i + 2] + x[4 * i + 3]);
      } else {
        x[4 * i] = x[4 * i + 1] = x[4 * i + 2] = x[4 * i + 3] = 0.f;
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      const int c = lane + 32 * i;
      x[i] = c < H ? __half2float(xin[(size_t)tok * H + c]) + __half2float(res[(size_t)tok * H + c]) : 0.f;
      s += x[i];
    }
  }
  const float mean = warp_sum_f(s) / (float)H;
  float var = 0.f;
#pragma unroll
  for (int i = 0; i < NC; ++i) {
    const int c = VEC ? (i >> 2) * 128 : lane + 32 * i;   // (VEC: all four values of a piece are in or out together)
    if (c < H) var += (x[i] - mean) * (x[i] - mean);
  }
  const float rstd = rsqrtf(warp_sum_f(var) / (float)H + eps);
  if (VEC) {
    OutT* oo = out + (size_t)tok * H;
#pragma unroll
    for (int i = 0; i < NC / 4; ++i) {
      if (i * 128 < H) {
        const float4 gg = __ldg(reinterpret_cast<const float4*>(g) + lane + 32 * i);
        const float4 bb = __ldg(reinterpret_cast<const float4*>(bta) + lane + 32 * i);
        store4(oo, lane + 32 * i, (x[4 * i] - mean) * rstd * gg.x + bb.x,
               (x[4 * i + 1] - mean) * rstd * gg.y + bb.y, (x[4 * i + 2] - mean) * rstd * gg.z + bb.z,
               (x[4 * i + 3] - mean) * rstd * gg.w + bb.w);
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      const int c = lane + 32 * i;
      if (c < H) store1(out + (size_t)tok * H + c, (x[i] - mean) * rstd * g[c] + bta[c]);
    }
  }
}

// ---- attention: one block per (sequence, head), flash-style on mma.sync tensor cores ---------------------
// qkv [T, 3H] (Q | K | V), ctx [T, H].  head_dim must be 32 (MiniLM-L12-H384: 12 heads x 32).
// K and V of the head sit in shared memory (80-byte row pitch: conflict-free ldmatrix): S = Q K^T with
// m16n8k16 (fp16 in, fp32 acc), online softmax in the exp2 domain, O += P V with P re-packed from the S
// accumulators as the A operand.  The running maxima are kept scaled (m = max(S) * scale); the scale itself
// is folded into the exponent's FMA, so a score costs one FMNMX, one FFMA, one ex2 and one FADD.
constexpr int kAttPitch = 40;  // halves

__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldsm_x4_trans(uint32_t (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(p)));
}

__device__ __forceinline__ float ex2_approx(float x) {   // 2^x, one MUFU op; ex2(-inf) = +0
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Sequence indices of a call sorted by length, longest first (counting sort over the lengths; equal lengths in any
// order).  One CTA, once per forward.
constexpr int kMaxSeqLenBins = 2048;
__global__ void __launch_bounds__(1024) seq_order_kernel(const int32_t* __restrict__ cu, int P, int32_t* __restrict__ order) {
  __shared__ int cnt[kMaxSeqLenBins + 1];
  for (int i = threadIdx.x; i <= kMaxSeqLenBins; i += blockDim.x) cnt[i] = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < P; i += blockDim.x) atomicAdd(&cnt[min(cu[i + 1] - cu[i], kMaxSeqLenBins)], 1);
  __syncthreads();
  if (threadIdx.x == 0) {   // exclusive prefix from the longest bin down: cnt[L] becomes the first slot of length L
    int run = 0;
    for (int b = kMaxSeqLenBins; b >= 0; --b) { const int c = cnt[b]; cnt[b] = run; run += c; }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < P; i += blockDim.x) order[atomicAdd(&cnt[min(cu[i + 1] - cu[i], kMaxSeqLenBins)], 1)] = i;
}

// Two 16-query tiles per warp and key block: the K / V fragments are fetched from shared memory once and feed both
// tiles' MMAs, and the two tiles' softmax chains (max -> ex2 -> sum -> pack) interleave: with one tile per warp and
// three CTAs = 12 warps per SM, the dependent chain of that tile, not a pipe's throughput, sets the pace.
//
// Launch order: one CTA per (sequence, head), heads fastest, the sequences walked longest first (`order`, built once per call by
// seq_order_kernel).  A CTA's work grows with L^2 and the lengths of a call spread over an order of magnitude; in
// arrival order a long sequence that starts in the last wave leaves most SMs idle while it finishes.  Longest first
// the last wave holds the shortest sequences.  The last key block is 32 keys wide when no more than 32 are left.
__global__ void __launch_bounds__(128, 3) attention2_kernel(const __half* __restrict__ qkv, const int32_t* __restrict__ cu,
                                                         const int32_t* __restrict__ order, int H, int n_heads,
                                                         float scale_log2e, __half* __restrict__ ctx) {
  extern __shared__ __align__(16) unsigned char att_smem[];
  // CTA -> (sequence slot, head), heads fastest: the twelve CTAs of a sequence run together and read the same qkv rows.
  const int head = (int)(blockIdx.x % (unsigned)n_heads);
  const int seq = order[(int)(blockIdx.x / (unsigned)n_heads)];
  const int t0 = cu[seq], L = cu[seq + 1] - t0;
  const int Lp = (L + 63) / 64 * 64;
  __half* Ks = reinterpret_cast<__half*>(att_smem);
  __half* Vs = Ks + (size_t)Lp * kAttPitch;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t ld = (size_t)3 * H;
  // K / V of the head: global -> shared memory with cp.async (16 bytes each, zero-filled past the sequence), no
  // registers in between; the first Q fragments are requested below while these copies are in flight.
#pragma unroll 4
  for (int idx = threadIdx.x; idx < Lp * 4; idx += blockDim.x) {
    const int j = idx >> 2, c = idx & 3;
    const __half* base = qkv + (size_t)(t0 + (j < L ? j : L - 1)) * ld + head * 32 + c * 8;
    const uint32_t nbytes = j < L ? 16u : 0u;
    cp_async_16(smem_u32(Ks + (size_t)j * kAttPitch + c * 8), base + H, nbytes);
    cp_async_16(smem_u32(Vs + (size_t)j * kAttPitch + c * 8), base + 2 * H, nbytes);
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  const int r = lane >> 2, cp = (lane & 3) * 2;
  auto load_q = [&](int qb, uint32_t (&a)[2][4]) {   // A fragments of S = Q K^T for one 16-query tile (rows >= L read as zero)
    const int q0 = qb * 16 + r, q1 = q0 + 8;
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      const __half* p0 = qkv + (size_t)(t0 + q0) * ld + head * 32 + ks * 16 + cp;
      const __half* p1 = qkv + (size_t)(t0 + q1) * ld + head * 32 + ks * 16 + cp;
      a[ks][0] = q0 < L ? __ldg(reinterpret_cast<const uint32_t*>(p0)) : 0u;
      a[ks][1] = q1 < L ? __ldg(reinterpret_cast<const uint32_t*>(p1)) : 0u;
      a[ks][2] = q0 < L ? __ldg(reinterpret_cast<const uint32_t*>(p0 + 8)) : 0u;
      a[ks][3] = q1 < L ? __ldg(reinterpret_cast<const uint32_t*>(p1 + 8)) : 0u;
    }
  };
  // Q fragments of the warp's first pair of tiles: global loads that overlap the K / V staging above.
  uint32_t a[2][2][4];
  load_q(2 * warp, a[0]);
  load_q(2 * warp + 1, a[1]);
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();
  for (int pb = warp; pb * 32 < L; pb += 4) {   // this warp's pair of tiles: queries [32 pb, 32 pb + 32)
    float m[2][2], l[2][2], O[2][4][4];
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      m[t][0] = m[t][1] = -INFINITY;
      l[t][0] = l[t][1] = 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e) O[t][i][e] = 0.f;
    }
    // One block of NKK k-steps (16 keys each) starting at key kb: NKK = 4 for a full 64-key block, 1..3 for the tail of
    // the sequence.  NKK is a compile-time constant so that every loop unrolls without guards (run-time guards inside
    // the unrolled body keep the compiler from interleaving the MMAs with the softmax).
    auto block = [&](auto nkk_tag, int kb) {
      constexpr int NKK = decltype(nkk_tag)::value;
      constexpr int NJ = 2 * NKK;   // 8-key score tiles
      float S[2][NJ][4];
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        uint32_t b[4];
        ldsm_x4(b, Ks + (size_t)(kb + j * 8 + (lane & 7)) * kAttPitch + (lane >> 3) * 8);
#pragma unroll
        for (int t = 0; t < 2; ++t) {
#pragma unroll
          for (int e = 0; e < 4; ++e) S[t][j][e] = 0.f;
          mma16816(S[t][j], a[t][0], b[0], b[1]);
          mma16816(S[t][j], a[t][1], b[2], b[3]);
        }
      }
      if (kb + NJ * 8 > L) {   // only the last key block holds padding keys
#pragma unroll
        for (int t = 0; t < 2; ++t)
#pragma unroll
          for (int j = 0; j < NJ; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e)
              if (kb + j * 8 + cp + (e & 1) >= L) S[t][j][e] = -INFINITY;
      }
      float mn[2][2];
#pragma unroll
      for (int t = 0; t < 2; ++t) {
        float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          mx0 = fmaxf(mx0, fmaxf(S[t][j][0], S[t][j][1]));
          mx1 = fmaxf(mx1, fmaxf(S[t][j][2], S[t][j][3]));
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        // finite: every block holds at least one valid key (kb < L)
        mn[t][0] = fmaxf(m[t][0], mx0 * scale_log2e);
        mn[t][1] = fmaxf(m[t][1], mx1 * scale_log2e);
        const float c0 = ex2_approx(m[t][0] - mn[t][0]), c1 = ex2_approx(m[t][1] - mn[t][1]);
        l[t][0] *= c0; l[t][1] *= c1;
#pragma unroll
        for (int i = 0; i < 4; ++i) { O[t][i][0] *= c0; O[t][i][1] *= c0; O[t][i][2] *= c1; O[t][i][3] *= c1; }
        m[t][0] = mn[t][0]; m[t][1] = mn[t][1];
      }
#pragma unroll
      for (int t = 0; t < 2; ++t)
#pragma unroll
        for (int j = 0; j < NJ; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float pexp = ex2_approx(fmaf(S[t][j][e], scale_log2e, e < 2 ? -mn[t][0] : -mn[t][1]));   // -inf -> 0
            S[t][j][e] = pexp;
            if (e < 2) l[t][0] += pexp; else l[t][1] += pexp;
          }
#pragma unroll
      for (int kk = 0; kk < NKK; ++kk) {
        uint32_t pa[2][4];
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          pa[t][0] = pack_half2(S[t][2 * kk][0], S[t][2 * kk][1]);
          pa[t][1] = pack_half2(S[t][2 * kk][2], S[t][2 * kk][3]);
          pa[t][2] = pack_half2(S[t][2 * kk + 1][0], S[t][2 * kk + 1][1]);
          pa[t][3] = pack_half2(S[t][2 * kk + 1][2], S[t][2 * kk + 1][3]);
        }
#pragma unroll
        for (int dn2 = 0; dn2 < 2; ++dn2) {
          uint32_t vb[4];
          ldsm_x4_trans(vb, Vs + (size_t)(kb + kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * kAttPitch +
                                (dn2 * 2 + (lane >> 4)) * 8);
#pragma unroll
          for (int t = 0; t < 2; ++t) {
            mma16816(O[t][dn2 * 2], pa[t], vb[0], vb[1]);
            mma16816(O[t][dn2 * 2 + 1], pa[t], vb[2], vb[3]);
          }
        }
      }
    };
    // 64-key blocks while more than 32 keys are left (the last of them may hold padding keys), then at most one
    // 32-key block: a 200-token sequence computes 224 keys instead of 256 (L is warp-uniform).
    int kb = 0;
    for (; L - kb > 32; kb += 64) block(std::integral_constant<int, 4>{}, kb);
    if (L - kb > 0) block(std::integral_constant<int, 2>{}, kb);
    if ((pb + 4) * 32 < L) {   // the next pair's Q fragments travel while this pair's output is normalised and stored
      load_q(2 * (pb + 4), a[0]);
      load_q(2 * (pb + 4) + 1, a[1]);
    }
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      float l0 = l[t][0], l1 = l[t][1];
      l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
      l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
      const float inv0 = 1.f / l0, inv1 = 1.f / l1;
      const int q0 = (2 * pb + t) * 16 + r, q1 = q0 + 8;
#pragma unroll
      for (int dn = 0; dn < 4; ++dn) {
        if (q0 < L) *reinterpret_cast<uint32_t*>(ctx + (size_t)(t0 + q0) * H + head * 32 + dn * 8 + cp) = pack_half2(O[t][dn][0] * inv0, O[t][dn][1] * inv0);
        if (q1 < L) *reinterpret_cast<uint32_t*>(ctx + (size_t)(t0 + q1) * H + head * 32 + dn * 8 + cp) = pack_half2(O[t][dn][2] * inv1, O[t][dn][3] * inv1);
      }
    }
  }
}

// ---- attention at head_dim 64 (the encoder of rl_xenc_encode) ----------------------------------------------
// One CTA per (sequence, head, 64-query block); each of its four warps owns 16 queries.  K / V of the head stream through
// shared memory in 64-key blocks, double-buffered with cp.async (zero-filled past the sequence), so a CTA holds 36 KB
// whatever the length and several CTAs share an SM; the whole head of a 512-token sequence resident (the design of
// attention2_kernel) would take about 147 KB at this width.  S = Q K^T and O += P V on m16n8k16 (fp16 in, fp32
// accumulate), online softmax in the exp2 domain as in attention2_kernel.  CTAs walk the sequences longest first
// (seq_order_kernel), heads and then query blocks fastest.
constexpr int kAtt64Dim = 64;
constexpr int kAtt64Keys = 64;                 // keys per streamed block
constexpr int kAtt64Queries = 64;              // queries per CTA
constexpr int kAtt64Pitch = kAtt64Dim + 8;     // halves per staged row: 144 bytes, conflict-free ldmatrix
constexpr int kAtt64Threads = 128;

__global__ void __launch_bounds__(kAtt64Threads, 3) attention64_kernel(const __half* __restrict__ qkv, const int32_t* __restrict__ cu,
                                                                       const int32_t* __restrict__ order, int H, int n_heads,
                                                                       int n_qb, float scale_log2e, __half* __restrict__ ctx) {
  __shared__ __align__(16) __half Ks[2][kAtt64Keys * kAtt64Pitch];
  __shared__ __align__(16) __half Vs[2][kAtt64Keys * kAtt64Pitch];
  const int qb = (int)(blockIdx.x % (unsigned)n_qb);
  const int sh = (int)(blockIdx.x / (unsigned)n_qb);
  const int head = sh % n_heads, seq = order[sh / n_heads];
  const int t0 = cu[seq], L = cu[seq + 1] - t0;
  if (qb * kAtt64Queries >= L) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t ld = (size_t)3 * H;
  const __half* kg = qkv + (size_t)t0 * ld + H + head * kAtt64Dim;   // key j of the head: kg + j * ld; its value: + H
  auto load_kv = [&](int kb, int st) {   // keys [kb, kb + 64): 64 rows x 8 pieces of 16 bytes, for K and V
#pragma unroll
    for (int idx = threadIdx.x; idx < kAtt64Keys * 8; idx += kAtt64Threads) {
      const int j = idx >> 3, c = idx & 7;
      const bool ok = kb + j < L;
      const __half* src = kg + (size_t)(ok ? kb + j : L - 1) * ld + c * 8;   // (clamped: a zero-fill copy reads nothing)
      cp_async_16(smem_u32(&Ks[st][j * kAtt64Pitch + c * 8]), src, ok ? 16u : 0u);
      cp_async_16(smem_u32(&Vs[st][j * kAtt64Pitch + c * 8]), src + H, ok ? 16u : 0u);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  load_kv(0, 0);
  const int r = lane >> 2, cp = (lane & 3) * 2;
  const int q0 = qb * kAtt64Queries + warp * 16 + r, q1 = q0 + 8;
  const bool active = qb * kAtt64Queries + warp * 16 < L;   // warp-uniform: this warp has at least one query
  // A fragments of S = Q K^T, four 16-wide k-steps over the head's 64 columns (rows >= L read as zero)
  uint32_t a[4][4];
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    const __half* p0 = qkv + (size_t)(t0 + q0) * ld + head * kAtt64Dim + ks * 16 + cp;
    const __half* p1 = qkv + (size_t)(t0 + q1) * ld + head * kAtt64Dim + ks * 16 + cp;
    a[ks][0] = q0 < L ? __ldg(reinterpret_cast<const uint32_t*>(p0)) : 0u;
    a[ks][1] = q1 < L ? __ldg(reinterpret_cast<const uint32_t*>(p1)) : 0u;
    a[ks][2] = q0 < L ? __ldg(reinterpret_cast<const uint32_t*>(p0 + 8)) : 0u;
    a[ks][3] = q1 < L ? __ldg(reinterpret_cast<const uint32_t*>(p1 + 8)) : 0u;
  }
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  float O[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) O[i][e] = 0.f;
  const int n_kb = (L + kAtt64Keys - 1) / kAtt64Keys;
  for (int b = 0; b < n_kb; ++b) {
    const int kb = b * kAtt64Keys, st = b & 1;
    if (b + 1 < n_kb) {   // the next block travels while this one is computed
      load_kv(kb + kAtt64Keys, st ^ 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    if (active) {
      const __half* Kb = Ks[st];
      const __half* Vb = Vs[st];
      float S[8][4];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) S[j][e] = 0.f;
#pragma unroll
        for (int kp = 0; kp < 2; ++kp) {   // columns [32 kp, 32 kp + 32): k-steps 2 kp and 2 kp + 1
          uint32_t bf[4];
          ldsm_x4(bf, Kb + (j * 8 + (lane & 7)) * kAtt64Pitch + kp * 32 + (lane >> 3) * 8);
          mma16816(S[j], a[2 * kp], bf[0], bf[1]);
          mma16816(S[j], a[2 * kp + 1], bf[2], bf[3]);
        }
      }
      if (kb + kAtt64Keys > L) {   // only the last key block holds padding keys
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (kb + j * 8 + cp + (e & 1) >= L) S[j][e] = -INFINITY;
      }
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        mx0 = fmaxf(mx0, fmaxf(S[j][0], S[j][1]));
        mx1 = fmaxf(mx1, fmaxf(S[j][2], S[j][3]));
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      // finite: every key block holds a valid key (scale > 0, so max commutes with the scaling)
      const float mn0 = fmaxf(m0, mx0 * scale_log2e), mn1 = fmaxf(m1, mx1 * scale_log2e);
      const float c0 = ex2_approx(m0 - mn0), c1 = ex2_approx(m1 - mn1);
      l0 *= c0; l1 *= c1;
#pragma unroll
      for (int i = 0; i < 8; ++i) { O[i][0] *= c0; O[i][1] *= c0; O[i][2] *= c1; O[i][3] *= c1; }
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float pexp = ex2_approx(fmaf(S[j][e], scale_log2e, e < 2 ? -mn0 : -mn1));   // -inf -> 0
          S[j][e] = pexp;
          if (e < 2) l0 += pexp; else l1 += pexp;
        }
      m0 = mn0; m1 = mn1;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        uint32_t pa[4];
        pa[0] = pack_half2(S[2 * kk][0], S[2 * kk][1]);
        pa[1] = pack_half2(S[2 * kk][2], S[2 * kk][3]);
        pa[2] = pack_half2(S[2 * kk + 1][0], S[2 * kk + 1][1]);
        pa[3] = pack_half2(S[2 * kk + 1][2], S[2 * kk + 1][3]);
#pragma unroll
        for (int dn2 = 0; dn2 < 4; ++dn2) {
          uint32_t vb[4];
          ldsm_x4_trans(vb, Vb + (kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * kAtt64Pitch + (dn2 * 2 + (lane >> 4)) * 8);
          mma16816(O[dn2 * 2], pa, vb[0], vb[1]);
          mma16816(O[dn2 * 2 + 1], pa, vb[2], vb[3]);
        }
      }
    }
    __syncthreads();   // stage st is refilled by the next iteration's load
  }
  if (!active) return;
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv0 = 1.f / l0, inv1 = 1.f / l1;
#pragma unroll
  for (int dn = 0; dn < 8; ++dn) {
    if (q0 < L) *reinterpret_cast<uint32_t*>(ctx + (size_t)(t0 + q0) * H + head * kAtt64Dim + dn * 8 + cp) = pack_half2(O[dn][0] * inv0, O[dn][1] * inv0);
    if (q1 < L) *reinterpret_cast<uint32_t*>(ctx + (size_t)(t0 + q1) * H + head * kAtt64Dim + dn * 8 + cp) = pack_half2(O[dn][2] * inv1, O[dn][3] * inv1);
  }
}

// ---- pooler + classifier ----------------------------------------------------------------------------------
// logit[s][j] = Wc[j] . tanh(Wp h_s + bp) + bc[j] with h_s the [CLS] row of sequence s and NL (1 or 2) labels j.
// A CTA owns kClsSeqs sequences (their [CLS] rows sit in shared memory as fp32) and its min(H/32, 16) warps share the
// H pooler outputs; for one output the lanes stride over the H inputs, so every Wp read is a coalesced 128-byte line
// shared by the CTA's sequences, followed by one warp-shuffle reduction per sequence; the warps' NL partial logits
// per sequence meet in shared memory and are summed in a fixed order.  (Wp read row-per-lane touches 32 lines per
// load instruction; one warp per four sequences walking all H outputs one after the other is coalesced but leaves a
// few CTAs with long serial work.)  logit is [P, NL] row-major; score is sigmoid(l) at one label and softmax(l)[1]
// = 1 / (1 + exp(l0 - l1)) at two, a form that cannot overflow where exp(l1) / (exp(l0) + exp(l1)) can.
constexpr int kClsSeqs = 2;
constexpr int kClsMaxWarps = 16;
template <int NL>
__global__ void __launch_bounds__(kClsMaxWarps * 32) cls_head_kernel(const __half* __restrict__ hidden, const int32_t* __restrict__ cu,
                                                                     const float* __restrict__ Wp, const float* __restrict__ bp,
                                                                     const float* __restrict__ Wc, const float* __restrict__ bc,
                                                                     int P, int H, float* __restrict__ logit,
                                                                     float* __restrict__ score) {
  extern __shared__ float cls_smem[];  // [kClsSeqs][H] [CLS] rows as fp32, then [warps][kClsSeqs][NL] partial logits
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int seq0 = blockIdx.x * kClsSeqs;
  float* h = cls_smem;
  float* part = cls_smem + (size_t)kClsSeqs * H;
#pragma unroll
  for (int s = 0; s < kClsSeqs; ++s) {
    const bool ok = seq0 + s < P;
    const __half* src = hidden + (size_t)cu[ok ? seq0 + s : seq0] * H;  // [CLS] token
    for (int c = threadIdx.x; c < H; c += blockDim.x) h[s * H + c] = ok ? __half2float(src[c]) : 0.f;
  }
  __syncthreads();
  float out[kClsSeqs][NL];
#pragma unroll
  for (int s = 0; s < kClsSeqs; ++s)
#pragma unroll
    for (int j = 0; j < NL; ++j) out[s][j] = 0.f;
#pragma unroll 2
  for (int o = warp; o < H; o += nw) {   // this warp's pooler outputs
    const float* w = Wp + (size_t)o * H;
    float a[kClsSeqs];
#pragma unroll
    for (int s = 0; s < kClsSeqs; ++s) a[s] = 0.f;
#pragma unroll 4
    for (int c = lane; c < H; c += 32) {
      const float wv = __ldg(w + c);
#pragma unroll
      for (int s = 0; s < kClsSeqs; ++s) a[s] = fmaf(wv, h[s * H + c], a[s]);
    }
    const float b = __ldg(bp + o);
    float wc[NL];
#pragma unroll
    for (int j = 0; j < NL; ++j) wc[j] = __ldg(Wc + (size_t)j * H + o);
#pragma unroll
    for (int s = 0; s < kClsSeqs; ++s) {
      const float t = tanhf(warp_sum_f(a[s]) + b);   // identical on every lane
#pragma unroll
      for (int j = 0; j < NL; ++j) out[s][j] += t * wc[j];
    }
  }
  if (lane == 0) {
#pragma unroll
    for (int s = 0; s < kClsSeqs; ++s)
#pragma unroll
      for (int j = 0; j < NL; ++j) part[(warp * kClsSeqs + s) * NL + j] = out[s][j];
  }
  __syncthreads();
  if (threadIdx.x < kClsSeqs && seq0 + threadIdx.x < P) {   // fixed summation order: deterministic logits
    const int seq = seq0 + threadIdx.x;
    float v[NL];
#pragma unroll
    for (int j = 0; j < NL; ++j) {
      v[j] = bc[j];
      for (int wi = 0; wi < nw; ++wi) v[j] += part[(wi * kClsSeqs + threadIdx.x) * NL + j];
      logit[(size_t)seq * NL + j] = v[j];
    }
    // FlashRank: sigmoid of a single logit, softmax(logits)[1] of two
    score[seq] = NL == 1 ? 1.f / (1.f + __expf(-v[0])) : 1.f / (1.f + __expf(v[0] - v[NL - 1]));
  }
}

}  // namespace
}  // namespace rl

using namespace rl;

extern "C" size_t rl_xenc_linear_image_bytes(int N, int K) {
  const int n_ks = (K + kSliceK - 1) / kSliceK;
  const int n_pad = (N + 15) / 16 * 16;
  return (size_t)((n_pad + kPassN - 1) / kPassN) * kPassN * n_ks * kSliceK * sizeof(__half);
}

extern "C" int rl_xenc_pack_linear(const float* W, int N, int K, void* image, void* stream) {
  RL_REQUIRE(W && image && N > 0 && K > 0, RL_EINVAL, "rl_xenc_pack_linear: bad arguments");
  RL_REQUIRE(N % 16 == 0 && K % 8 == 0, RL_EUNSUPPORTED, "rl_xenc_pack_linear: N %% 16 and K %% 8 must be 0");
  RL_CUDA_CHECK(cudaMemsetAsync(image, 0, rl_xenc_linear_image_bytes(N, K), (cudaStream_t)stream));
  pack_linear_kernel<<<1024, 256, 0, (cudaStream_t)stream>>>(W, N, K, reinterpret_cast<__half*>(image));
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

// cuTensorMapEncodeTiled through the runtime's driver entry point (no -lcuda link dependency).
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = []() -> EncodeTiledFn {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
      return nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

static int launch_linear(const __half* X, const void* img, const float* bias, __half* Y, int T, int N, int K, int act,
                         int sm_count, cudaStream_t stream) {
  EncodeTiledFn enc = encode_tiled_fn();
  RL_REQUIRE(enc != nullptr, RL_ECUDA, "cuTensorMapEncodeTiled is not available from this driver");
  RL_REQUIRE((reinterpret_cast<uintptr_t>(X) & 15) == 0 && (K * 2) % 16 == 0, RL_EINVAL, "linear: X must be 16-byte aligned");
  CUtensorMap tm;
  const cuuint64_t gdim[2] = {(cuuint64_t)K, (cuuint64_t)T};          // innermost first
  const cuuint64_t gstr[1] = {(cuuint64_t)K * sizeof(__half)};        // bytes between token rows
  const cuuint32_t box[2] = {(cuuint32_t)kSliceK, (cuuint32_t)kTileM};   // 64 halves (128 B, one swizzle row) x 128 tokens
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = enc(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(X), gdim, gstr, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  RL_REQUIRE(r == CUDA_SUCCESS, RL_ECUDA, "cuTensorMapEncodeTiled failed (%d) for X[%d, %d]", (int)r, T, K);
  LinArgs t;
  t.img = reinterpret_cast<const __half*>(img); t.bias = bias; t.Y = Y; t.ldy = N; t.T = T; t.N = N; t.K = K; t.act = act;
  t.n_pass = (N + kPassN - 1) / kPassN;
  t.n_ks = (K + kSliceK - 1) / kSliceK;
  const uint32_t tail = 2 * kMaxStages * 8 + kEpiBytes;   // barriers + epilogue staging
  int stages = (int)((kSmemBudget - 1024 - tail) / kLinStageBytes);
  if (stages > kMaxStages) stages = kMaxStages;
  t.stages = stages;
  const size_t smem = (size_t)stages * kLinStageBytes + tail + 1024;
  RL_CUDA_CHECK(cudaFuncSetAttribute(linear_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t items = (int64_t)((T + kTileM - 1) / kTileM) * t.n_pass;
  const int grid = (int)(items < sm_count ? items : sm_count);
  linear_wgmma_kernel<<<grid, kLinThreads, smem, stream>>>(tm, t);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

// ---- quantized images: sizes, packing, concatenation, launch ------------------------------------------------------
static bool qlinear_shape_ok(int type, int N, int K) {
  return q_type_ok(type) && N > 0 && N % 32 == 0 && (size_t)(N + kPassN - 1) / kPassN <= kQImgMaxPasses && K > 0 &&
         K % kQSliceK == 0 && K % q_block_elems(type) == 0;
}

extern "C" size_t rl_xenc_qlinear_image_bytes(int type, int N, int K) {
  if (!qlinear_shape_ok(type, N, K)) return 0;
  size_t bytes = kQImgData;
  for (int p = 0; p < (N + kPassN - 1) / kPassN; ++p) bytes += q_pass_bytes(type, N, K, p);
  return bytes;
}

// The header of an image: written from the host (a pageable copy: the stream is synchronised before it starts).
static int write_qimg_head(void* image, int N, int K, const int* types, cudaStream_t stream) {
  unsigned char head[kQImgData];
  memset(head, 0, sizeof(head));
  const int n_pass = (N + kPassN - 1) / kPassN;
  QImgHead h{n_pass, N, K, kQImgMagic};
  memcpy(head, &h, sizeof(h));
  int64_t off = (int64_t)kQImgData;
  for (int p = 0; p < n_pass; ++p) {
    QImgPass pp{types[p], (int32_t)q_row_bytes(types[p]), off};
    memcpy(head + sizeof(QImgHead) + p * sizeof(QImgPass), &pp, sizeof(pp));
    off += (int64_t)q_pass_bytes(types[p], N, K, p);
  }
  RL_CUDA_CHECK(cudaMemcpyAsync(image, head, kQImgData, cudaMemcpyHostToDevice, stream));
  return RL_OK;
}

extern "C" int rl_xenc_pack_qlinear(int type, const void* blocks, int N, int K, void* image, void* stream_) {
  RL_REQUIRE(blocks && image, RL_EINVAL, "rl_xenc_pack_qlinear: null pointer");
  RL_REQUIRE(qlinear_shape_ok(type, N, K), RL_EUNSUPPORTED,
             "rl_xenc_pack_qlinear: type=%d N=%d K=%d unsupported (GGML Q8_0 = 8, Q4_K = 12 or Q6_K = 14; N %% 32 == 0, "
             "N <= %d, K %% 128 == 0 and a whole number of blocks)", type, N, K, (int)(kQImgMaxPasses * kPassN));
  cudaStream_t stream = (cudaStream_t)stream_;
  int types[kQImgMaxPasses];
  for (auto& ty : types) ty = type;
  const int rc = write_qimg_head(image, N, K, types, stream);
  if (rc != RL_OK) return rc;
  pack_qlinear_kernel<<<1024, 128, 0, stream>>>(type, reinterpret_cast<const unsigned char*>(blocks), N, K,
                                                reinterpret_cast<unsigned char*>(image));
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" int rl_xenc_concat_qlinear(const void* const* parts, int n_parts, void* image, void* stream_) {
  RL_REQUIRE(parts && image && n_parts > 0, RL_EINVAL, "rl_xenc_concat_qlinear: bad arguments");
  cudaStream_t stream = (cudaStream_t)stream_;
  RL_REQUIRE((size_t)n_parts <= kQImgMaxPasses, RL_EUNSUPPORTED, "rl_xenc_concat_qlinear: too many parts");
  unsigned char head[kQImgData];
  int types[kQImgMaxPasses];
  size_t payload[kQImgMaxPasses];
  int N = 0, K = 0, n_pass = 0;
  for (int i = 0; i < n_parts; ++i) {
    RL_REQUIRE(parts[i], RL_EINVAL, "rl_xenc_concat_qlinear: null part");
    RL_CUDA_CHECK(cudaMemcpyAsync(head, parts[i], kQImgData, cudaMemcpyDeviceToHost, stream));
    RL_CUDA_CHECK(cudaStreamSynchronize(stream));
    QImgHead h;
    memcpy(&h, head, sizeof(h));
    RL_REQUIRE(h.magic == kQImgMagic && h.n_pass > 0 && (size_t)h.n_pass <= kQImgMaxPasses, RL_EINVAL,
               "rl_xenc_concat_qlinear: part %d is not a quantized image", i);
    RL_REQUIRE(i == 0 || h.K == K, RL_EINVAL, "rl_xenc_concat_qlinear: parts differ in K");
    RL_REQUIRE(i == n_parts - 1 || h.N % kPassN == 0, RL_EUNSUPPORTED,
               "rl_xenc_concat_qlinear: every part but the last needs N %% %d == 0", kPassN);
    RL_REQUIRE((size_t)(n_pass + h.n_pass) <= kQImgMaxPasses, RL_EUNSUPPORTED, "rl_xenc_concat_qlinear: N too large");
    K = h.K;
    payload[i] = 0;
    for (int p = 0; p < h.n_pass; ++p) {
      QImgPass pp;
      memcpy(&pp, head + sizeof(QImgHead) + p * sizeof(QImgPass), sizeof(pp));
      types[n_pass + p] = pp.type;
      payload[i] += q_pass_bytes(pp.type, h.N, K, p);
    }
    n_pass += h.n_pass;
    N += h.N;
  }
  const int rc = write_qimg_head(image, N, K, types, stream);
  if (rc != RL_OK) return rc;
  size_t off = kQImgData;
  for (int i = 0; i < n_parts; ++i) {   // each part's passes, header excluded, one after the other
    RL_CUDA_CHECK(cudaMemcpyAsync(reinterpret_cast<unsigned char*>(image) + off,
                                  reinterpret_cast<const unsigned char*>(parts[i]) + kQImgData, payload[i],
                                  cudaMemcpyDeviceToDevice, stream));
    off += payload[i];
  }
  return RL_OK;
}

static int launch_qlinear_act(const __half* X, const void* img, const float* bias, __half* Y, int ldy, int T, int N, int K,
                              int act, int sm_count, cudaStream_t stream) {
  EncodeTiledFn enc = encode_tiled_fn();
  RL_REQUIRE(enc != nullptr, RL_ECUDA, "cuTensorMapEncodeTiled is not available from this driver");
  RL_REQUIRE((reinterpret_cast<uintptr_t>(X) & 15) == 0 && (reinterpret_cast<uintptr_t>(img) & 15) == 0, RL_EINVAL,
             "linear: X and the image must be 16-byte aligned");
  RL_REQUIRE(K % kQSliceK == 0 && (N + kPassN - 1) / kPassN <= (int)kQImgMaxPasses, RL_EUNSUPPORTED,
             "quantized linear: K %% %d == 0 and N <= %d required", kQSliceK, (int)(kQImgMaxPasses * kPassN));
  CUtensorMap tm;
  const cuuint64_t gdim[2] = {(cuuint64_t)K, (cuuint64_t)T};
  const cuuint64_t gstr[1] = {(cuuint64_t)K * sizeof(__half)};
  const cuuint32_t box[2] = {(cuuint32_t)kSliceK, (cuuint32_t)kTileM};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = enc(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(X), gdim, gstr, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  RL_REQUIRE(r == CUDA_SUCCESS, RL_ECUDA, "cuTensorMapEncodeTiled failed (%d) for X[%d, %d]", (int)r, T, K);
  QLinArgs t;
  t.img = reinterpret_cast<const unsigned char*>(img); t.bias = bias; t.Y = Y; t.ldy = ldy; t.T = T; t.N = N; t.K = K; t.act = act;
  t.n_pass = (N + kPassN - 1) / kPassN;
  t.n_qs = K / kQSliceK;
  const uint32_t tail = 3 * kQMaxStages * 8 + kEpiBytes;   // barriers + epilogue staging
  int stages = (int)((kSmemBudget - 1024 - tail) / kQStageBytes);
  if (stages > kQMaxStages) stages = kQMaxStages;
  t.stages = stages;
  const size_t smem = (size_t)stages * kQStageBytes + tail + 1024;
  RL_CUDA_CHECK(cudaFuncSetAttribute(linear_q_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t items = (int64_t)((T + kTileM - 1) / kTileM) * t.n_pass;
  const int grid = (int)(items < sm_count ? items : sm_count);
  linear_q_wgmma_kernel<<<grid, kQLinThreads, smem, stream>>>(tm, t);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

static int launch_qlinear(const __half* X, const void* img, const float* bias, __half* Y, int T, int N, int K, int act,
                          int sm_count, cudaStream_t stream) {
  return launch_qlinear_act(X, img, bias, Y, N, T, N, K, act, sm_count, stream);
}

int rl::launch_qlinear_ld(const __half* X, const void* img, const float* bias, __half* Y, int ldy, int T, int N, int K,
                          int sm_count, cudaStream_t stream) {
  RL_REQUIRE(ldy >= N && ldy % 8 == 0 && (reinterpret_cast<uintptr_t>(Y) & 15) == 0, RL_EINVAL,
             "quantized linear: ldy=%d must be >= N=%d and a multiple of 8, Y 16-byte aligned", ldy, N);
  return launch_qlinear_act(X, img, bias, Y, ldy, T, N, K, 0, sm_count, stream);
}

// The linear of an encoder layer by its image type: RL_XENC_IMAGE_F16 (rl_xenc_pack_linear) or RL_XENC_IMAGE_QUANT.
static int launch_linear_typed(int image_type, const __half* X, const void* img, const float* bias, __half* Y, int T, int N,
                               int K, int act, int sm_count, cudaStream_t stream) {
  if (image_type == RL_XENC_IMAGE_QUANT) return launch_qlinear(X, img, bias, Y, T, N, K, act, sm_count, stream);
  return launch_linear(X, img, bias, Y, T, N, K, act, sm_count, stream);
}

extern "C" int rl_xenc_linear_q(const void* X, const void* image, const float* bias, void* Y, int T, int N, int K, int act,
                                void* stream) {
  RL_REQUIRE(X && image && bias && Y && T >= 0, RL_EINVAL, "rl_xenc_linear_q: bad arguments");
  RL_REQUIRE(N > 0 && N % 32 == 0 && (size_t)(N + kPassN - 1) / kPassN <= kQImgMaxPasses && K > 0 && K % kQSliceK == 0,
             RL_EUNSUPPORTED, "rl_xenc_linear_q: N=%d K=%d unsupported (N %% 32 == 0, 0 < N <= %d, K %% 128 == 0, K > 0)", N, K,
             (int)(kQImgMaxPasses * kPassN));
  RL_REQUIRE((reinterpret_cast<uintptr_t>(bias) & 15) == 0, RL_EINVAL, "rl_xenc_linear_q: bias must be 16-byte aligned");
  if (T == 0) return RL_OK;
  int dev = 0, sms = 132;
  RL_CUDA_CHECK(cudaGetDevice(&dev));
  RL_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  return launch_qlinear(reinterpret_cast<const __half*>(X), image, bias, reinterpret_cast<__half*>(Y), T, N, K, act, sms,
                        (cudaStream_t)stream);
}

extern "C" int rl_dequant_rows_f16(int type, const void* blocks, int64_t rows, int K, void* out, void* stream) {
  RL_REQUIRE(blocks && out && rows >= 0, RL_EINVAL, "rl_dequant_rows_f16: bad arguments");
  RL_REQUIRE(q_type_ok(type) && K > 0 && K % q_block_elems(type) == 0, RL_EUNSUPPORTED,
             "rl_dequant_rows_f16: type=%d K=%d unsupported (Q8_0 = 8, Q4_K = 12 or Q6_K = 14, whole blocks per row)", type, K);
  if (rows == 0) return RL_OK;
  dequant_rows_kernel<<<2048, 256, 0, (cudaStream_t)stream>>>(type, reinterpret_cast<const unsigned char*>(blocks), rows, K,
                                                              reinterpret_cast<__half*>(out));
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" int rl_xenc_linear(const void* X, const void* image, const float* bias, void* Y, int T, int N, int K, int act,
                              void* stream) {
  RL_REQUIRE(X && image && bias && Y && T >= 0, RL_EINVAL, "rl_xenc_linear: bad arguments");
  RL_REQUIRE(N % 32 == 0 && K % 8 == 0, RL_EUNSUPPORTED, "rl_xenc_linear: N %% 32 and K %% 8 must be 0");
  RL_REQUIRE((reinterpret_cast<uintptr_t>(bias) & 15) == 0, RL_EINVAL, "rl_xenc_linear: bias must be 16-byte aligned");
  if (T == 0) return RL_OK;
  int dev = 0, sms = 132;
  RL_CUDA_CHECK(cudaGetDevice(&dev));
  RL_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  return launch_linear(reinterpret_cast<const __half*>(X), image, bias, reinterpret_cast<__half*>(Y), T, N, K, act, sms,
                       (cudaStream_t)stream);
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// ---- attention step: setup and launches, shared by rl_xenc_score, rl_xenc_encode and their attention test hooks ----
static size_t att_smem_bytes(int max_len) { return (size_t)((max_len + 63) / 64 * 64) * kAttPitch * 2 * sizeof(__half); }

// Once per forward: the length-sorted sequence order (seq_order [P]) that both attention kernels walk and, at head_dim
// 32, attention2_kernel's shared-memory limit (K and V of the longest sequence).  Refuses a too long max_len before any
// CUDA call.
static int attention_setup(int head_dim, const int32_t* cu_seqlens, int P, int max_len, int32_t* seq_order,
                           cudaStream_t stream) {
  if (head_dim == 32) {
    const size_t att_smem = att_smem_bytes(max_len);
    RL_REQUIRE(att_smem <= 200 * 1024, RL_EUNSUPPORTED, "max_len=%d too long for the attention kernel", max_len);
    RL_CUDA_CHECK(cudaFuncSetAttribute(attention2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)att_smem));
  }
  seq_order_kernel<<<1, 1024, 0, stream>>>(cu_seqlens, P, seq_order);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

// Once per layer at head_dim 32: ctx = softmax(Q K^T / sqrt(32)) V per sequence and head, from qkv [T, 3H] (Q | K | V).
static int attention_launch(const __half* qkv, const int32_t* cu_seqlens, const int32_t* seq_order, int P, int max_len,
                            int H, int nh, __half* ctx, cudaStream_t stream) {
  const float scale = 1.4426950408889634f / sqrtf(32.f);  // softmax in the exp2 domain
  attention2_kernel<<<dim3((unsigned)P * (unsigned)nh), 128, att_smem_bytes(max_len), stream>>>(qkv, cu_seqlens, seq_order,
                                                                                                  H, nh, scale, ctx);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" int rl_xenc_attention(const void* qkv, const int32_t* cu_seqlens, int P, int T, int max_len, int hidden, int n_heads,
                                 void* ctx, void* workspace, size_t workspace_bytes, void* stream_) {
  RL_REQUIRE(qkv && cu_seqlens && ctx, RL_EINVAL, "rl_xenc_attention: null pointer");
  if (P == 0 || T == 0) return RL_OK;
  RL_REQUIRE(hidden % 32 == 0 && hidden <= 512 && n_heads > 0 && hidden / n_heads == 32, RL_EUNSUPPORTED,
             "rl_xenc_attention: hidden=%d heads=%d unsupported (head_dim must be 32, hidden <= 512)", hidden, n_heads);
  RL_REQUIRE(P > 0 && P <= T && max_len > 0, RL_EINVAL, "rl_xenc_attention: bad P=%d / T=%d / max_len=%d", P, T, max_len);
  RL_REQUIRE(workspace && (reinterpret_cast<uintptr_t>(workspace) & 15) == 0 && workspace_bytes >= (size_t)P * sizeof(int32_t),
             RL_ENOSPACE, "rl_xenc_attention: workspace must be 16-byte aligned and hold %d int32", P);
  cudaStream_t stream = (cudaStream_t)stream_;
  int32_t* seq_order = reinterpret_cast<int32_t*>(workspace);
  const int rc = attention_setup(32, cu_seqlens, P, max_len, seq_order, stream);
  if (rc != RL_OK) return rc;
  return attention_launch(reinterpret_cast<const __half*>(qkv), cu_seqlens, seq_order, P, max_len, hidden, n_heads,
                          reinterpret_cast<__half*>(ctx), stream);
}

extern "C" size_t rl_xenc_workspace_bytes(const rl_xenc_weights* w, int T) {
  if (w == nullptr || T < 0) return 0;
  const size_t H = (size_t)w->hidden, F = (size_t)w->ffn;
  // hidden, qkv (3H), ctx, tmp (H), ffn (F) -- fp16 rows
  // + the length-sorted sequence order of the call (at most T sequences), 16-byte aligned behind the rows
  return ((size_t)T * (H + 3 * H + H + H + F) * sizeof(__half) + (size_t)T * sizeof(int32_t) + 4096);
}

// ---- attention at head_dim 64: launches, shared by rl_xenc_encode and the rl_xenc_encode_attention hook ----------
static int attention64_launch(const __half* qkv, const int32_t* cu_seqlens, const int32_t* seq_order, int P, int max_len,
                              int H, int nh, __half* ctx, cudaStream_t stream) {
  const int n_qb = (max_len + kAtt64Queries - 1) / kAtt64Queries;
  const float scale = 1.4426950408889634f / sqrtf((float)kAtt64Dim);  // softmax in the exp2 domain
  attention64_kernel<<<dim3((unsigned)P * (unsigned)nh * (unsigned)n_qb), kAtt64Threads, 0, stream>>>(
      qkv, cu_seqlens, seq_order, H, nh, n_qb, scale, ctx);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

// The attention launch of an encoder forward by head_dim: 32 attention2_kernel, 64 attention64_kernel.
static int encoder_attention_launch(int head_dim, const __half* qkv, const int32_t* cu_seqlens, const int32_t* seq_order, int P,
                                    int max_len, int H, int nh, __half* ctx, cudaStream_t stream) {
  return head_dim == 64 ? attention64_launch(qkv, cu_seqlens, seq_order, P, max_len, H, nh, ctx, stream)
                        : attention_launch(qkv, cu_seqlens, seq_order, P, max_len, H, nh, ctx, stream);
}

// LayerNorm launches by width: 16 columns per lane up to H = 512 (the cross-encoder's instantiations), 32 up to 1024.
static void launch_embed_ln(const rl_xenc_weights* w, const int32_t* ids, const int32_t* type_ids, const int32_t* pos_ids, int T,
                            __half* out, cudaStream_t stream) {
  const int H = w->hidden, blocks = (T + 7) / 8;
  const __half* word = reinterpret_cast<const __half*>(w->word_emb);
  const __half* pos = reinterpret_cast<const __half*>(w->pos_emb);
  const __half* type = reinterpret_cast<const __half*>(w->type_emb);
  if (H <= 512)
    embed_ln_kernel<16><<<blocks, 256, 0, stream>>>(ids, type_ids, pos_ids, word, pos, type, w->emb_ln_g, w->emb_ln_b, w->ln_eps,
                                                    T, H, w->vocab, w->max_pos, w->type_vocab, out);
  else
    embed_ln_kernel<32><<<blocks, 256, 0, stream>>>(ids, type_ids, pos_ids, word, pos, type, w->emb_ln_g, w->emb_ln_b, w->ln_eps,
                                                    T, H, w->vocab, w->max_pos, w->type_vocab, out);
}
template <typename OutT>
static void launch_add_ln(const __half* x, const __half* res, const float* g, const float* b, float eps, int T, int H, OutT* out,
                          cudaStream_t stream) {
  const int blocks = (T + 7) / 8;
  const bool vec = H % 128 == 0;   // (LayerNorm gamma / beta come from torch allocations: 16-byte aligned)
  if (H <= 512) {
    if (vec) add_ln_kernel<true, 16, OutT><<<blocks, 256, 0, stream>>>(x, res, g, b, eps, T, H, out);
    else add_ln_kernel<false, 16, OutT><<<blocks, 256, 0, stream>>>(x, res, g, b, eps, T, H, out);
  } else {
    if (vec) add_ln_kernel<true, 32, OutT><<<blocks, 256, 0, stream>>>(x, res, g, b, eps, T, H, out);
    else add_ln_kernel<false, 32, OutT><<<blocks, 256, 0, stream>>>(x, res, g, b, eps, T, H, out);
  }
}

// Pooler + classifier + score of P sequences from the fp16 rows `hidden` [T, H] (their [CLS] rows at cu_seqlens[s]).
static void launch_cls_head(const rl_xenc_weights* w, int n_labels, const __half* hidden, const int32_t* cu_seqlens, int P,
                            float* out_logit, float* out_score, cudaStream_t stream) {
  const int H = w->hidden;
  const int cls_warps = H / 32 < kClsMaxWarps ? H / 32 : kClsMaxWarps;
  const dim3 cls_grid((P + kClsSeqs - 1) / kClsSeqs);
  const size_t cls_smem = ((size_t)kClsSeqs * H + (size_t)kClsMaxWarps * kClsSeqs * n_labels) * sizeof(float);
  if (n_labels == 1)
    cls_head_kernel<1><<<cls_grid, cls_warps * 32, cls_smem, stream>>>(hidden, cu_seqlens, w->pooler_w, w->pooler_b, w->cls_w,
                                                                       w->cls_b, P, H, out_logit, out_score);
  else
    cls_head_kernel<2><<<cls_grid, cls_warps * 32, cls_smem, stream>>>(hidden, cu_seqlens, w->pooler_w, w->pooler_b, w->cls_w,
                                                                       w->cls_b, P, H, out_logit, out_score);
}

// Embeddings and every encoder layer of a packed batch, shared by rl_xenc_score and rl_xenc_encode (arguments checked by
// the caller).  The last layer's output LayerNorm writes fp16 rows into the workspace's hidden buffer or, when out_f32 is
// set, fp32 rows to out_f32 [T, H].
static int encoder_forward(const rl_xenc_weights* w, const int32_t* input_ids, const int32_t* type_ids, const int32_t* pos_ids,
                           const int32_t* cu_seqlens, int P, int T, int max_len, void* workspace, float* out_f32, int sms,
                           cudaStream_t stream) {
  const int H = w->hidden, F = w->ffn, nh = w->n_heads, head_dim = H / nh;
  __half* hidden = reinterpret_cast<__half*>(workspace);
  __half* qkv = hidden + (size_t)T * H;
  __half* ctx = qkv + (size_t)T * 3 * H;
  __half* tmp = ctx + (size_t)T * H;
  __half* ffn = tmp + (size_t)T * H;
  int32_t* seq_order = reinterpret_cast<int32_t*>(
      (reinterpret_cast<uintptr_t>(ffn + (size_t)T * F) + 15) & ~uintptr_t(15));   // [P] (P <= T)
  int rc = attention_setup(head_dim, cu_seqlens, P, max_len, seq_order, stream);
  if (rc != RL_OK) return rc;
  launch_embed_ln(w, input_ids, type_ids, pos_ids, T, hidden, stream);
  RL_CUDA_CHECK(cudaGetLastError());
  for (int l = 0; l < w->n_layers; ++l) {
    const rl_xenc_layer& L = w->layers[l];
    rc = launch_linear_typed(L.qkv_type, hidden, L.qkv_img, L.qkv_bias, qkv, T, 3 * H, H, 0, sms, stream);
    if (rc != RL_OK) return rc;
    rc = encoder_attention_launch(head_dim, qkv, cu_seqlens, seq_order, P, max_len, H, nh, ctx, stream);
    if (rc != RL_OK) return rc;
    rc = launch_linear_typed(L.o_type, ctx, L.o_img, L.o_bias, tmp, T, H, H, 0, sms, stream);
    if (rc != RL_OK) return rc;
    launch_add_ln(tmp, hidden, L.ln1_g, L.ln1_b, w->ln_eps, T, H, hidden, stream);
    RL_CUDA_CHECK(cudaGetLastError());
    rc = launch_linear_typed(L.up_type, hidden, L.up_img, L.up_bias, ffn, T, F, H, 1, sms, stream);
    if (rc != RL_OK) return rc;
    rc = launch_linear_typed(L.down_type, ffn, L.down_img, L.down_bias, tmp, T, H, F, 0, sms, stream);
    if (rc != RL_OK) return rc;
    if (out_f32 != nullptr && l == w->n_layers - 1) launch_add_ln(tmp, hidden, L.ln2_g, L.ln2_b, w->ln_eps, T, H, out_f32, stream);
    else launch_add_ln(tmp, hidden, L.ln2_g, L.ln2_b, w->ln_eps, T, H, hidden, stream);
    RL_CUDA_CHECK(cudaGetLastError());
  }
  return RL_OK;
}

// Shapes the encoder path takes: head_dim 32 or 64, H <= 1024 (LayerNorm at 32 columns per lane), up to 512 tokens.
constexpr int kEncodeMaxHidden = 1024;
constexpr int kEncodeMaxLen = 512;

// Every layer's image types, checked before the forward's first launch: RL_XENC_IMAGE_F16 or RL_XENC_IMAGE_QUANT, and a
// quantized linear's shape within launch_qlinear's (K % 128 == 0, N <= 8192).  qkv [3H, H], o [H, H], up [F, H], down [H, F].
static int check_layer_images(const rl_xenc_weights* w, const char* fn) {
  const int H = w->hidden, F = w->ffn;
  for (int l = 0; l < w->n_layers; ++l) {
    const rl_xenc_layer& L = w->layers[l];
    const int types[4] = {L.qkv_type, L.o_type, L.up_type, L.down_type};
    const int Ns[4] = {3 * H, H, F, H}, Ks[4] = {H, H, H, F};
    static const char* names[4] = {"qkv", "o", "up", "down"};
    for (int i = 0; i < 4; ++i) {
      RL_REQUIRE(types[i] == RL_XENC_IMAGE_F16 || types[i] == RL_XENC_IMAGE_QUANT, RL_EINVAL,
                 "%s: layer %d %s image type %d unsupported (RL_XENC_IMAGE_F16 = 0 or RL_XENC_IMAGE_QUANT = 1)", fn, l,
                 names[i], types[i]);
      RL_REQUIRE(types[i] != RL_XENC_IMAGE_QUANT ||
                     (Ks[i] % kQSliceK == 0 && (size_t)(Ns[i] + kPassN - 1) / kPassN <= kQImgMaxPasses),
                 RL_EUNSUPPORTED, "%s: layer %d quantized %s linear [%d, %d] unsupported (K %% %d == 0 and N <= %d required)",
                 fn, l, names[i], Ns[i], Ks[i], kQSliceK, (int)(kQImgMaxPasses * kPassN));
    }
  }
  return RL_OK;
}

// rl_xenc_score takes the union of two envelopes.  The cross-encoder's own (head_dim 32, H <= 512, max_len up to the
// position table, bounded by attention2_kernel's shared memory) and the token encoder's (head_dim 32 or 64, H <= 1024,
// max_len <= 512, at least one layer, as rl_xenc_encode).  Both run encoder_forward; the envelopes differ in checks only.
extern "C" int rl_xenc_score(const rl_xenc_weights* w, const int32_t* input_ids, const int32_t* type_ids,
                             const int32_t* pos_ids, const int32_t* cu_seqlens, int P, int T, int max_len,
                             float* out_logit, float* out_score, void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  RL_REQUIRE(w && w->layers && input_ids && type_ids && pos_ids && cu_seqlens && out_logit && out_score, RL_EINVAL,
             "rl_xenc_score: null pointer");
  const int n_labels = w->n_labels == 0 ? 1 : w->n_labels;   // 0: a zero-initialised struct of a one-label caller
  RL_REQUIRE(n_labels == 1 || n_labels == 2, RL_EUNSUPPORTED, "rl_xenc_score: n_labels=%d unsupported (1 or 2)", w->n_labels);
  if (P == 0 || T == 0) return RL_OK;
  const int H = w->hidden, F = w->ffn, nh = w->n_heads;
  const bool narrow = H % 32 == 0 && H <= 512 && nh > 0 && H / nh == 32;
  const bool wide = H % 32 == 0 && H <= kEncodeMaxHidden && nh > 0 && H % nh == 0 && (H / nh == 32 || H / nh == 64);
  RL_REQUIRE(narrow || wide, RL_EUNSUPPORTED,
             "rl_xenc_score: hidden=%d heads=%d unsupported (head_dim 32 with hidden <= 512, or head_dim 32 / 64 with "
             "hidden %% 32 == 0 and hidden <= %d)", H, nh, kEncodeMaxHidden);
  RL_REQUIRE(F % 32 == 0 && max_len > 0 && max_len <= w->max_pos, RL_EUNSUPPORTED, "rl_xenc_score: bad ffn / max_len");
  if (narrow) {
    RL_REQUIRE(att_smem_bytes(max_len) <= 200 * 1024, RL_EUNSUPPORTED, "max_len=%d too long for the attention kernel", max_len);
  } else {
    RL_REQUIRE(w->n_layers > 0, RL_EUNSUPPORTED, "rl_xenc_score: n_layers > 0 required at hidden=%d heads=%d", H, nh);
    RL_REQUIRE(max_len <= kEncodeMaxLen, RL_EUNSUPPORTED,
               "rl_xenc_score: max_len=%d unsupported at hidden=%d heads=%d (at most min(%d, max_pos=%d))", max_len, H, nh,
               kEncodeMaxLen, w->max_pos);
  }
  RL_REQUIRE(workspace && workspace_bytes >= rl_xenc_workspace_bytes(w, T), RL_ENOSPACE, "rl_xenc_score: workspace too small");
  RL_REQUIRE(P <= T, RL_EINVAL, "rl_xenc_score: more sequences than tokens");
  const int lc = check_layer_images(w, "rl_xenc_score");
  if (lc != RL_OK) return lc;
  int dev = 0, sms = 132;
  RL_CUDA_CHECK(cudaGetDevice(&dev));
  RL_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int rc = encoder_forward(w, input_ids, type_ids, pos_ids, cu_seqlens, P, T, max_len, workspace, nullptr, sms, stream);
  if (rc != RL_OK) return rc;
  launch_cls_head(w, n_labels, reinterpret_cast<const __half*>(workspace), cu_seqlens, P, out_logit, out_score, stream);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" int rl_xenc_encode(const rl_xenc_weights* w, const int32_t* input_ids, const int32_t* type_ids,
                              const int32_t* pos_ids, const int32_t* cu_seqlens, int P, int T, int max_len, float* out_hidden,
                              void* workspace, size_t workspace_bytes, void* stream_) {
  RL_REQUIRE(w && w->layers && input_ids && type_ids && pos_ids && cu_seqlens && out_hidden, RL_EINVAL,
             "rl_xenc_encode: null pointer");
  if (P == 0 || T == 0) return RL_OK;
  const int H = w->hidden, F = w->ffn, nh = w->n_heads;
  RL_REQUIRE(H % 32 == 0 && H <= kEncodeMaxHidden && nh > 0 && H % nh == 0 && (H / nh == 32 || H / nh == 64), RL_EUNSUPPORTED,
             "rl_xenc_encode: hidden=%d heads=%d unsupported (head_dim 32 or 64, hidden %% 32 == 0, hidden <= %d)", H, nh,
             kEncodeMaxHidden);
  RL_REQUIRE(F % 32 == 0 && w->n_layers > 0, RL_EUNSUPPORTED, "rl_xenc_encode: ffn %% 32 and n_layers > 0 required");
  RL_REQUIRE(max_len > 0 && max_len <= kEncodeMaxLen && max_len <= w->max_pos, RL_EUNSUPPORTED,
             "rl_xenc_encode: max_len=%d unsupported (at most min(%d, max_pos=%d))", max_len, kEncodeMaxLen, w->max_pos);
  RL_REQUIRE(P <= T, RL_EINVAL, "rl_xenc_encode: more sequences (%d) than tokens (%d)", P, T);
  RL_REQUIRE(workspace && (reinterpret_cast<uintptr_t>(workspace) & 15) == 0 && workspace_bytes >= rl_xenc_workspace_bytes(w, T),
             RL_ENOSPACE, "rl_xenc_encode: workspace must be 16-byte aligned and hold rl_xenc_workspace_bytes(w, T) bytes");
  const int lc = check_layer_images(w, "rl_xenc_encode");
  if (lc != RL_OK) return lc;
  int dev = 0, sms = 132;
  RL_CUDA_CHECK(cudaGetDevice(&dev));
  RL_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  return encoder_forward(w, input_ids, type_ids, pos_ids, cu_seqlens, P, T, max_len, workspace, out_hidden, sms,
                         (cudaStream_t)stream_);
}

extern "C" int rl_xenc_encode_attention(const void* qkv, const int32_t* cu_seqlens, int P, int T, int max_len, int hidden,
                                        int n_heads, void* ctx, void* workspace, size_t workspace_bytes, void* stream_) {
  RL_REQUIRE(qkv && cu_seqlens && ctx, RL_EINVAL, "rl_xenc_encode_attention: null pointer");
  if (P == 0 || T == 0) return RL_OK;
  RL_REQUIRE(hidden % 32 == 0 && hidden <= kEncodeMaxHidden && n_heads > 0 && hidden % n_heads == 0 &&
                 (hidden / n_heads == 32 || hidden / n_heads == 64),
             RL_EUNSUPPORTED, "rl_xenc_encode_attention: hidden=%d heads=%d unsupported (head_dim 32 or 64, hidden <= %d)",
             hidden, n_heads, kEncodeMaxHidden);
  RL_REQUIRE(P > 0 && P <= T && max_len > 0, RL_EINVAL, "rl_xenc_encode_attention: bad P=%d / T=%d / max_len=%d", P, T, max_len);
  RL_REQUIRE(max_len <= kEncodeMaxLen, RL_EUNSUPPORTED, "rl_xenc_encode_attention: max_len=%d > %d", max_len, kEncodeMaxLen);
  RL_REQUIRE(workspace && (reinterpret_cast<uintptr_t>(workspace) & 15) == 0 && workspace_bytes >= (size_t)P * sizeof(int32_t),
             RL_ENOSPACE, "rl_xenc_encode_attention: workspace must be 16-byte aligned and hold %d int32", P);
  cudaStream_t stream = (cudaStream_t)stream_;
  const int head_dim = hidden / n_heads;
  int32_t* seq_order = reinterpret_cast<int32_t*>(workspace);
  const int rc = attention_setup(head_dim, cu_seqlens, P, max_len, seq_order, stream);
  if (rc != RL_OK) return rc;
  return encoder_attention_launch(head_dim, reinterpret_cast<const __half*>(qkv), cu_seqlens, seq_order, P, max_len, hidden,
                                  n_heads, reinterpret_cast<__half*>(ctx), stream);
}

// ---- test hooks of the other forward steps: each runs the launch function that the forward itself runs ------------------
extern "C" int rl_xenc_embed_ln(const rl_xenc_weights* w, const int32_t* ids, const int32_t* type_ids, const int32_t* pos_ids,
                                int T, void* out_f16, void* stream) {
  RL_REQUIRE(w && ids && type_ids && pos_ids && out_f16 && T >= 0, RL_EINVAL, "rl_xenc_embed_ln: bad arguments");
  RL_REQUIRE(w->word_emb && w->pos_emb && w->type_emb && w->emb_ln_g && w->emb_ln_b, RL_EINVAL,
             "rl_xenc_embed_ln: null embedding table or LayerNorm");
  RL_REQUIRE(w->hidden > 0 && w->hidden % 32 == 0 && w->hidden <= kEncodeMaxHidden, RL_EUNSUPPORTED,
             "rl_xenc_embed_ln: hidden=%d unsupported (hidden %% 32 == 0, hidden <= %d)", w->hidden, kEncodeMaxHidden);
  RL_REQUIRE(w->vocab > 0 && w->max_pos > 0 && w->type_vocab > 0, RL_EINVAL, "rl_xenc_embed_ln: empty embedding table");
  if (T == 0) return RL_OK;
  launch_embed_ln(w, ids, type_ids, pos_ids, T, reinterpret_cast<__half*>(out_f16), (cudaStream_t)stream);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" int rl_xenc_add_ln(const void* x, const void* res, const float* gamma, const float* beta, float eps, int T, int H,
                              int out_f32, void* out, void* stream) {
  RL_REQUIRE(x && res && gamma && beta && out && T >= 0, RL_EINVAL, "rl_xenc_add_ln: bad arguments");
  RL_REQUIRE(H > 0 && H % 32 == 0 && H <= kEncodeMaxHidden, RL_EUNSUPPORTED,
             "rl_xenc_add_ln: H=%d unsupported (H %% 32 == 0, H <= %d)", H, kEncodeMaxHidden);
  // the vectorised path reads x / res in 8-byte and gamma / beta in 16-byte pieces and stores 8 / 16 bytes per piece
  RL_REQUIRE(aligned16(x) && aligned16(res) && aligned16(gamma) && aligned16(beta) && aligned16(out), RL_EINVAL,
             "rl_xenc_add_ln: every pointer must be 16-byte aligned");
  if (T == 0) return RL_OK;
  const __half* xh = reinterpret_cast<const __half*>(x);
  const __half* rh = reinterpret_cast<const __half*>(res);
  if (out_f32)
    launch_add_ln(xh, rh, gamma, beta, eps, T, H, reinterpret_cast<float*>(out), (cudaStream_t)stream);
  else
    launch_add_ln(xh, rh, gamma, beta, eps, T, H, reinterpret_cast<__half*>(out), (cudaStream_t)stream);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" int rl_xenc_cls_head(const rl_xenc_weights* w, const void* hidden_f16, const int32_t* cu_seqlens, int P,
                                float* out_logit, float* out_score, void* stream) {
  RL_REQUIRE(w && hidden_f16 && cu_seqlens && out_logit && out_score && P >= 0, RL_EINVAL, "rl_xenc_cls_head: bad arguments");
  RL_REQUIRE(w->pooler_w && w->pooler_b && w->cls_w && w->cls_b, RL_EINVAL, "rl_xenc_cls_head: null head weights");
  const int n_labels = w->n_labels == 0 ? 1 : w->n_labels;
  RL_REQUIRE(n_labels == 1 || n_labels == 2, RL_EUNSUPPORTED, "rl_xenc_cls_head: n_labels=%d unsupported (1 or 2)", w->n_labels);
  RL_REQUIRE(w->hidden > 0 && w->hidden % 32 == 0 && w->hidden <= kEncodeMaxHidden, RL_EUNSUPPORTED,
             "rl_xenc_cls_head: hidden=%d unsupported (hidden %% 32 == 0, hidden <= %d)", w->hidden, kEncodeMaxHidden);
  if (P == 0) return RL_OK;
  launch_cls_head(w, n_labels, reinterpret_cast<const __half*>(hidden_f16), cu_seqlens, P, out_logit, out_score,
                  (cudaStream_t)stream);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}
