// Decoder-only LLM forward for sm_90a (llama.cpp's "qwen3" architecture): the generation step of rag().
//
//   embed_rows_kernel     token rows of token_embd read from its quantized image, fp32 (the residual stream)
//   rmsnorm_kernel        x += y (the previous block's output, fp16), then RMSNorm(x) * g -> fp16
//   qgemv_kernel          y = W x over quantized images, split over (pass, K range) CTAs; the decode linears and the
//                         LM head (qgemv_combine_kernel sums the K-range partials in a fixed order)
//   qk_norm_rope_kernel   per-head RMSNorm of Q and K, NEOX RoPE, K / V into the cache
//   attention_kernel      causal GQA attention over the cache: one CTA per (KV head, 16 query vectors, key range),
//                         online softmax in fp32; attention_combine_kernel merges key ranges in a fixed order
//   swiglu_kernel         silu(gate) * up
//   sample_kernel         repeat penalty, top-k (radix select), top-p, min-p, temperature, inverse-CDF draw; its
//                         masked instance first keeps the ids a grammar state allows (grammar.cu builds the index)
// Prefill (T > 1) runs the linears on xenc.cu's wgmma quantized linear (launch_qlinear_ld).
#include <algorithm>
#include <cub/block/block_scan.cuh>
#include <cuda_fp16.h>

#include "common.cuh"
#include "qimg.cuh"

namespace rl {
namespace {

constexpr int kHd = RL_LLM_HEAD_DIM;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float ldg_half(const unsigned char* p) {
  return __half2float(__ushort_as_half(__ldg(reinterpret_cast<const unsigned short*>(p))));
}
__device__ __forceinline__ uint32_t ldg_u32(const unsigned char* p) { return __ldg(reinterpret_cast<const uint32_t*>(p)); }
// Byte i of w as a float minus `bias`: exact for bytes (2^23 + byte - 2^23 - bias).
__device__ __forceinline__ float byte_f(uint32_t w, int i, float bias) {
  return __fsub_rn(__uint_as_float(0x4B000000u | __byte_perm(w, 0u, 0x4440u + i)), 8388608.f + bias);
}

// ---- one element of a quantized image: ggml's formula in fp32, every product and difference rounded on its own ----
__device__ float image_element(const unsigned char* img, int row, int k) {
  const QImgHead h = *reinterpret_cast<const QImgHead*>(img);
  const int pass = row / kQPassRows, rr = row % kQPassRows;
  const QImgPass pp = reinterpret_cast<const QImgPass*>(img + sizeof(QImgHead))[pass];
  const int nb16 = (q_pass_rows(h.N, pass) + 15) / 16 * 16;
  const int s = k / kQSliceK, e = k % kQSliceK, g = e / 32, j = e % 32;
  const unsigned char* r = img + pp.offset + ((size_t)s * nb16 + rr) * pp.row_bytes;
  if (pp.type == kGgmlQ8_0) return __fmul_rn(ldg_half(r + 2 * g), (float)(int8_t)r[8 + e]);
  if (pp.type == kGgmlQ4_K) {
    const int q = (r[12 + 32 * (g >> 1) + j] >> (4 * (g & 1))) & 0xF;
    return __fsub_rn(__fmul_rn(__fmul_rn(ldg_half(r), (float)r[4 + g]), (float)q), __fmul_rn(ldg_half(r + 2), (float)r[8 + g]));
  }
  const int q = ((r[32 * (g & 1) + j] >> (4 * (g >> 1))) & 0xF) | (((r[64 + j] >> (2 * g)) & 3) << 4);
  return __fmul_rn(__fmul_rn(ldg_half(r + 104), (float)(int8_t)r[96 + 2 * g + j / 16]), (float)(q - 32));
}

struct Parts {   // a linear's part images, device-readable
  const unsigned char* img[RL_LLM_MAX_PARTS];
};

// out[t, k] = element (ids[t], k) of the table; one CTA per token.
__global__ void __launch_bounds__(256) embed_rows_kernel(const Parts tbl, const int32_t* __restrict__ ids, int N, int K,
                                                         float* __restrict__ out) {
  const int t = blockIdx.x;
  const int id = ids[t];
  if (id < 0 || id >= N) {   // an id outside the table: a NaN row, never a read outside the image
    for (int k = threadIdx.x; k < K; k += blockDim.x) out[(size_t)t * K + k] = __int_as_float(0x7fc00000);
    return;
  }
  const unsigned char* img = tbl.img[id / RL_LLM_PART_ROWS];
  for (int k = threadIdx.x; k < K; k += blockDim.x)
    out[(size_t)t * K + k] = image_element(img, id % RL_LLM_PART_ROWS, k);
}

// ---- RMSNorm: one CTA per row.  x (fp32 [T, H]) += add (fp16, when given); out = x / sqrt(mean(x^2) + eps) * g ----
__global__ void __launch_bounds__(256) rmsnorm_kernel(float* __restrict__ x, const __half* __restrict__ add,
                                                      const float* __restrict__ g, int H, float eps, __half* __restrict__ out) {
  __shared__ float red[8];
  float* xr = x + (size_t)blockIdx.x * H;
  float ss = 0.f;
  for (int i = threadIdx.x; i < H; i += blockDim.x) {
    float v = xr[i];
    if (add) {
      v += __half2float(add[(size_t)blockIdx.x * H + i]);
      xr[i] = v;
    }
    ss = fmaf(v, v, ss);
  }
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) tot += red[w];
  const float scale = 1.f / sqrtf(tot / (float)H + eps);
  for (int i = threadIdx.x; i < H; i += blockDim.x) out[(size_t)blockIdx.x * H + i] = __float2half_rn(xr[i] * scale * g[i]);
}

// ---- quantized GEMV ------------------------------------------------------------------------------------------------
// Work item = (pass of 128 output rows, range of K slices).  Warp w takes rows w, w + 8, ... of the pass; lane l takes
// elements 4 l .. 4 l + 3 of each 128-element slice (group g = l / 8, j = 4 (l % 8)), so one 32-bit load per lane and
// row-slice covers the row's quantized bytes.  Per lane and row the slice adds  scale * (q . x) - min * sum(x).
constexpr int kGemvThreads = 256;
constexpr int kGemvRowsPerWarp = kQPassRows / (kGemvThreads / 32);
constexpr int kGemvMaxSegs = 64;
constexpr int kGemvTargetItems = 528;   // 4 CTAs per SM of a 132-SM H100; fixed so results do not depend on the device
struct GemvSeg { const unsigned char* img; int32_t N, pass0, n0, pad_; };
struct GemvArgs {
  GemvSeg seg[kGemvMaxSegs];
  const __half* x;
  float* partial;   // [kparts][n_total] when kparts > 1
  void* y;
  int n_seg, n_pass, n_total, n_qs, kparts, spp, y_f32;
};

template <int TYPE>
__device__ __forceinline__ float row_slice_dot(const unsigned char* __restrict__ r, int lane, float4 xv, float xsum) {
  const int g = lane >> 3, j = 4 * (lane & 7);
  if (TYPE == kGgmlQ8_0) {
    const uint32_t q = ldg_u32(r + 8 + 4 * lane) ^ 0x80808080u;
    const float d = ldg_half(r + 2 * g);
    const float s = byte_f(q, 0, 128.f) * xv.x + byte_f(q, 1, 128.f) * xv.y + byte_f(q, 2, 128.f) * xv.z +
                    byte_f(q, 3, 128.f) * xv.w;
    return d * s;
  } else if (TYPE == kGgmlQ4_K) {
    const uint32_t dd = ldg_u32(r);
    const uint32_t q = (ldg_u32(r + 12 + 32 * (g >> 1) + j) >> (4 * (g & 1))) & 0x0F0F0F0Fu;
    const float d = __half2float(__ushort_as_half((unsigned short)(dd & 0xFFFF)));
    const float dmin = __half2float(__ushort_as_half((unsigned short)(dd >> 16)));
    const float d1 = d * (float)__ldg(r + 4 + g), m1 = dmin * (float)__ldg(r + 8 + g);
    const float s = byte_f(q, 0, 0.f) * xv.x + byte_f(q, 1, 0.f) * xv.y + byte_f(q, 2, 0.f) * xv.z + byte_f(q, 3, 0.f) * xv.w;
    return d1 * s - m1 * xsum;
  } else {
    const uint32_t ql = (ldg_u32(r + 32 * (g & 1) + j) >> (4 * (g >> 1))) & 0x0F0F0F0Fu;
    const uint32_t qh = (ldg_u32(r + 64 + j) >> (2 * g)) & 0x03030303u;
    const uint32_t q = ql | (qh << 4);
    const float ds = ldg_half(r + 104) * (float)(int8_t)__ldg(r + 96 + 2 * g + (j >> 4));
    const float s = byte_f(q, 0, 32.f) * xv.x + byte_f(q, 1, 32.f) * xv.y + byte_f(q, 2, 32.f) * xv.z + byte_f(q, 3, 32.f) * xv.w;
    return ds * s;
  }
}

template <int TYPE>
__device__ __forceinline__ void gemv_rows(const unsigned char* base, int nb, int nb16, int rb, int s0, int s1,
                                          const float4* xs, const float* xsum, float (&acc)[kGemvRowsPerWarp]) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int s = s0; s < s1; ++s) {
    const unsigned char* run = base + (size_t)s * nb16 * rb;
    const float4 xv = xs[(s - s0) * 32 + lane];
    const float xsm = xsum[(s - s0) * 32 + lane];
#pragma unroll
    for (int i = 0; i < kGemvRowsPerWarp; ++i) {
      const int r = warp + 8 * i;
      if (r < nb) acc[i] += row_slice_dot<TYPE>(run + (size_t)r * rb, lane, xv, xsm);
    }
  }
}

__global__ void __launch_bounds__(kGemvThreads, 3) qgemv_kernel(const __grid_constant__ GemvArgs a) {
  extern __shared__ float4 xs[];   // [spp * 32] x values of the item's K range, then [spp * 32] lane sums
  const int item = blockIdx.x;
  const int gpass = item / a.kparts, kp = item % a.kparts;
  const int s0 = kp * a.spp, s1 = min(a.n_qs, s0 + a.spp);
  float* xsum = reinterpret_cast<float*>(xs + a.spp * 32);
  for (int i = threadIdx.x; i < (s1 - s0) * 32; i += blockDim.x) {
    const __half2* xp = reinterpret_cast<const __half2*>(a.x + (size_t)(s0 * 32 + i) * 4);
    const float2 lo = __half22float2(xp[0]), hi = __half22float2(xp[1]);
    xs[i] = make_float4(lo.x, lo.y, hi.x, hi.y);
    xsum[i] = (lo.x + lo.y) + (hi.x + hi.y);
  }
  __syncthreads();
  int si = 0;
  while (si + 1 < a.n_seg && a.seg[si + 1].pass0 <= gpass) ++si;
  const GemvSeg sg = a.seg[si];
  const int pass = gpass - sg.pass0;
  const QImgPass pp = reinterpret_cast<const QImgPass*>(sg.img + sizeof(QImgHead))[pass];
  const int nb = q_pass_rows(sg.N, pass), nb16 = (nb + 15) / 16 * 16;
  float acc[kGemvRowsPerWarp];
#pragma unroll
  for (int i = 0; i < kGemvRowsPerWarp; ++i) acc[i] = 0.f;
  const unsigned char* base = sg.img + pp.offset;
  if (pp.type == kGgmlQ8_0) gemv_rows<kGgmlQ8_0>(base, nb, nb16, pp.row_bytes, s0, s1, xs, xsum, acc);
  else if (pp.type == kGgmlQ4_K) gemv_rows<kGgmlQ4_K>(base, nb, nb16, pp.row_bytes, s0, s1, xs, xsum, acc);
  else gemv_rows<kGgmlQ6_K>(base, nb, nb16, pp.row_bytes, s0, s1, xs, xsum, acc);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int i = 0; i < kGemvRowsPerWarp; ++i) {
    const int r = warp + 8 * i;
    const float v = warp_sum(acc[i]);
    if (lane == 0 && r < nb) {
      const int n = sg.n0 + pass * kQPassRows + r;
      if (a.kparts > 1) a.partial[(size_t)kp * a.n_total + n] = v;
      else if (a.y_f32) reinterpret_cast<float*>(a.y)[n] = v;
      else reinterpret_cast<__half*>(a.y)[n] = __float2half_rn(v);
    }
  }
}

__global__ void qgemv_combine_kernel(const float* __restrict__ partial, int kparts, int n_total, void* y, int y_f32) {
  for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < n_total; n += gridDim.x * blockDim.x) {
    float v = 0.f;
    for (int k = 0; k < kparts; ++k) v += partial[(size_t)k * n_total + n];
    if (y_f32) reinterpret_cast<float*>(y)[n] = v;
    else reinterpret_cast<__half*>(y)[n] = __float2half_rn(v);
  }
}

// ---- QK-norm + NEOX RoPE + cache write: one warp per (token, head) of the n_head + 2 n_kv heads ---------------------
// Lane l holds elements l, l + 32, l + 64, l + 96: the rotation pairs (l, l + 64) and (l + 32, l + 96).  The angle of
// pair i < 64 is pos * inv_freq_i in fp32 with inv_freq_i = 1 / powf(base, 2 i / 128) (fp32, one rounding each), as
// transformers' rotary embedding forms it; cos / sin by sincosf.
__global__ void __launch_bounds__(256) qk_norm_rope_kernel(const __half* __restrict__ qkv, int T, int p0, int n_head, int n_kv,
                                                           const float* __restrict__ qn, const float* __restrict__ kn, float eps,
                                                           float base, __half* __restrict__ q_out, __half* __restrict__ kc,
                                                           __half* __restrict__ vc) {
  const int nh_all = n_head + 2 * n_kv;
  const int wid = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (wid >= T * nh_all) return;
  const int t = wid / nh_all, h = wid % nh_all, pos = p0 + t;
  const __half* src = qkv + (size_t)t * nh_all * kHd + (size_t)h * kHd;
  float v[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) v[i] = __half2float(src[lane + 32 * i]);
  if (h >= n_head + n_kv) {   // V: copied
    __half* dst = vc + ((size_t)pos * n_kv + (h - n_head - n_kv)) * kHd;
#pragma unroll
    for (int i = 0; i < 4; ++i) dst[lane + 32 * i] = src[lane + 32 * i];
    return;
  }
  const bool is_q = h < n_head;
  const float* w = is_q ? qn : kn;
  const float ss = warp_sum(v[0] * v[0] + v[1] * v[1] + v[2] * v[2] + v[3] * v[3]);
  const float scale = 1.f / sqrtf(ss / (float)kHd + eps);
#pragma unroll
  for (int i = 0; i < 4; ++i) v[i] = v[i] * scale * w[lane + 32 * i];
  float o[4];
#pragma unroll
  for (int p = 0; p < 2; ++p) {   // pair (i, i + 64), i = lane + 32 p
    const int i = lane + 32 * p;
    const float inv = 1.f / powf(base, (float)(2 * i) / (float)kHd);
    float sn, cs;
    sincosf((float)pos * inv, &sn, &cs);
    o[p] = v[p] * cs - v[p + 2] * sn;
    o[p + 2] = v[p + 2] * cs + v[p] * sn;
  }
  __half* dst = is_q ? q_out + ((size_t)t * n_head + h) * kHd : kc + ((size_t)pos * n_kv + (h - n_head)) * kHd;
#pragma unroll
  for (int i = 0; i < 4; ++i) dst[lane + 32 * i] = __float2half_rn(o[i]);
}

// ---- causal GQA attention ------------------------------------------------------------------------------------------
// Query vectors r = t G + g (G = n_head / n_kv) of one KV head, 16 per CTA, against the cache rows of one key range,
// 64 keys at a time through shared memory (fp32).  Scores Q.K / sqrt(128); online softmax in fp32.  With one key range
// the output is normalised and stored fp16; with several each range stores (m, l, unnormalised O) and
// attention_combine_kernel merges them in range order.
constexpr int kAttQ = 16, kAttKeys = 64, kAttThreads = 256, kAttKPitch = kHd + 1;
constexpr int kAttTargetCtas = 264;   // two per SM of a 132-SM H100; fixed so results do not depend on the device
constexpr int kAttMaxSplits = 64;
constexpr size_t kAttSmem = (size_t)(kAttQ * kHd + kAttKeys * kAttKPitch + kAttKeys * kHd + kAttQ * kAttKeys + 3 * kAttQ) * 4;

__global__ void __launch_bounds__(kAttThreads, 2) attention_kernel(const __half* __restrict__ q, const __half* __restrict__ kc,
                                                                  const __half* __restrict__ vc, int T, int p0, int n_head,
                                                                  int n_kv, int splits, int chunk, __half* __restrict__ out,
                                                                  float* __restrict__ part_o, float* __restrict__ part_ml) {
  extern __shared__ float sm[];
  float* Qs = sm;
  float* Ks = Qs + kAttQ * kHd;
  float* Vs = Ks + kAttKeys * kAttKPitch;
  float* Ps = Vs + kAttKeys * kHd;
  float* row_m = Ps + kAttQ * kAttKeys;
  float* row_l = row_m + kAttQ;
  float* row_a = row_l + kAttQ;
  const int G = n_head / n_kv;
  const int kvh = blockIdx.y, split = blockIdx.z, r0 = blockIdx.x * kAttQ;
  const int nq = min(kAttQ, T * G - r0);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int i = tid; i < kAttQ * kHd; i += kAttThreads) {
    const int qi = i / kHd, d = i % kHd, r = r0 + qi;
    Qs[i] = qi < nq ? __half2float(q[((size_t)(r / G) * n_head + kvh * G + r % G) * kHd + d]) : 0.f;
  }
  if (tid < kAttQ) { row_m[tid] = kNegInf; row_l[tid] = 0.f; }
  const int last_pos = p0 + (r0 + nq - 1) / G;   // the largest query position of the tile
  const int k_begin = split * chunk, k_end = min(last_pos + 1, k_begin + chunk);
  const float scale = 0.08838834764831845f;   // 1 / sqrt(128)
  float o[8];
#pragma unroll
  for (int m = 0; m < 8; ++m) o[m] = 0.f;
  const int d_pv = tid & (kHd - 1), q_pv = tid >> 7;
  __syncthreads();
  for (int k0 = k_begin; k0 < k_end; k0 += kAttKeys) {
    for (int i = tid; i < kAttKeys * (kHd / 8); i += kAttThreads) {   // 16-byte loads: 8 halves
      const int j = i / (kHd / 8), c = i % (kHd / 8);
      uint4 kw = make_uint4(0, 0, 0, 0), vw = kw;
      if (k0 + j < k_end) {
        const size_t off = ((size_t)(k0 + j) * n_kv + kvh) * kHd + c * 8;
        kw = *reinterpret_cast<const uint4*>(kc + off);
        vw = *reinterpret_cast<const uint4*>(vc + off);
      }
      const __half2* kh = reinterpret_cast<const __half2*>(&kw);
      const __half2* vh = reinterpret_cast<const __half2*>(&vw);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 kf = __half22float2(kh[e]), vf = __half22float2(vh[e]);
        Ks[j * kAttKPitch + c * 8 + 2 * e] = kf.x;
        Ks[j * kAttKPitch + c * 8 + 2 * e + 1] = kf.y;
        Vs[j * kHd + c * 8 + 2 * e] = vf.x;
        Vs[j * kHd + c * 8 + 2 * e + 1] = vf.y;
      }
    }
    __syncthreads();
    {   // scores: key j = tid % 64, query vectors tid / 64 + 4 m
      const int j = tid & (kAttKeys - 1), qb = tid >> 6;
      float s[4] = {0.f, 0.f, 0.f, 0.f};
      for (int d = 0; d < kHd; ++d) {
        const float kv = Ks[j * kAttKPitch + d];
#pragma unroll
        for (int m = 0; m < 4; ++m) s[m] = fmaf(Qs[(qb + 4 * m) * kHd + d], kv, s[m]);
      }
#pragma unroll
      for (int m = 0; m < 4; ++m) {
        const int qi = qb + 4 * m;
        const int pos = p0 + (r0 + qi) / G;
        const bool ok = qi < nq && k0 + j < k_end && k0 + j <= pos;
        Ps[qi * kAttKeys + j] = ok ? s[m] * scale : kNegInf;
      }
    }
    __syncthreads();
#pragma unroll
    for (int rr = 0; rr < kAttQ / 8; ++rr) {   // online softmax: warp w, rows 2 w and 2 w + 1
      const int qi = 2 * warp + rr;
      const float a = Ps[qi * kAttKeys + lane], b = Ps[qi * kAttKeys + lane + 32];
      const float m_old = row_m[qi];
      const float m_new = fmaxf(m_old, warp_max(fmaxf(a, b)));
      const float pa = m_new == kNegInf ? 0.f : expf(a - m_new), pb = m_new == kNegInf ? 0.f : expf(b - m_new);
      const float sum = warp_sum(pa + pb);
      Ps[qi * kAttKeys + lane] = pa;
      Ps[qi * kAttKeys + lane + 32] = pb;
      __syncwarp();
      if (lane == 0) {
        const float alpha = m_old == kNegInf ? 0.f : expf(m_old - m_new);
        row_a[qi] = alpha;
        row_l[qi] = row_l[qi] * alpha + sum;
        row_m[qi] = m_new;
      }
    }
    __syncthreads();
#pragma unroll
    for (int m = 0; m < 8; ++m) {   // O[qi, d] = alpha O + P V: dim d_pv, query vectors q_pv + 2 m
      const int qi = q_pv + 2 * m;
      float acc = o[m] * row_a[qi];
      for (int j = 0; j < kAttKeys; ++j) acc = fmaf(Ps[qi * kAttKeys + j], Vs[j * kHd + d_pv], acc);
      o[m] = acc;
    }
    __syncthreads();
  }
#pragma unroll
  for (int m = 0; m < 8; ++m) {
    const int qi = q_pv + 2 * m;
    if (qi >= nq) continue;
    const int r = r0 + qi;
    const size_t row = (size_t)(r / G) * n_head + kvh * G + r % G;   // [T, n_head] order
    if (splits == 1) {
      out[row * kHd + d_pv] = __float2half_rn(o[m] / row_l[qi]);
    } else {
      const size_t rows = (size_t)T * n_head;
      part_o[((size_t)split * rows + row) * kHd + d_pv] = o[m];
      if (d_pv == 0) {
        part_ml[((size_t)split * rows + row) * 2] = row_m[qi];
        part_ml[((size_t)split * rows + row) * 2 + 1] = row_l[qi];
      }
    }
  }
}

__global__ void __launch_bounds__(kHd) attention_combine_kernel(const float* __restrict__ part_o, const float* __restrict__ part_ml,
                                                                int splits, int rows, __half* __restrict__ out) {
  const int row = blockIdx.x, d = threadIdx.x;
  float M = kNegInf;
  for (int s = 0; s < splits; ++s) M = fmaxf(M, part_ml[((size_t)s * rows + row) * 2]);
  float L = 0.f, O = 0.f;
  for (int s = 0; s < splits; ++s) {
    const float m = part_ml[((size_t)s * rows + row) * 2];
    if (m == kNegInf) continue;
    const float w = expf(m - M);
    L += part_ml[((size_t)s * rows + row) * 2 + 1] * w;
    O += part_o[((size_t)s * rows + row) * kHd + d] * w;
  }
  out[(size_t)row * kHd + d] = __float2half_rn(O / L);
}

// ---- SwiGLU: a[t, i] = silu(gate) * up, gu = [T, 2 F] (gate in columns 0 .. F, up in F .. 2 F) ----------------------
__global__ void swiglu_kernel(const __half* __restrict__ gu, int T, int F, __half* __restrict__ a) {
  const int64_t total = (int64_t)T * F;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = i / F, c = i % F;
    const float g = __half2float(gu[t * 2 * F + c]), u = __half2float(gu[t * 2 * F + F + c]);
    a[i] = __float2half_rn(g / (1.f + expf(-g)) * u);
  }
}

// ---- sampler: one CTA --------------------------------------------------------------------------------------------------
constexpr int kSampleThreads = 1024;
// The grammar of a masked draw: the token index (int16 [n_states, V], the state after the token's bytes or -1), the
// accepting states and the end-of-generation ids, allowed exactly in accepting states whatever their bytes.
struct SampleMask {
  const int16_t* index;
  const uint8_t* accept;
  int32_t* state;   // device: read, then the state after the drawn token (unchanged after an end-of-generation id)
  int n_states;
  int eog[RL_LLM_MAX_EOG];   // -1 past the given ids
};
// top-p, min-p, temperature and the inverse CDF at u over the k candidates (descending logit): the slot drawn.
__device__ int draw(const float* c_logit, int k, float temperature, float top_p, float min_p, float u) {
  int n = k;
  if (top_p < 1.f) {   // softmax at temperature 1, smallest prefix whose mass reaches top_p (the crossing one kept)
    const float mx = c_logit[0];
    float sum = 0.f;
    for (int i = 0; i < n; ++i) sum += expf(c_logit[i] - mx);
    float cum = 0.f;
    for (int i = 0; i < n; ++i) {
      cum += expf(c_logit[i] - mx) / sum;
      if (cum >= top_p) { n = i + 1; break; }
    }
  }
  if (min_p > 0.f) {   // logits >= max + log(min_p), at least one
    const float cut = c_logit[0] + logf(min_p);
    int m = 1;
    while (m < n && c_logit[m] >= cut) ++m;
    n = m;
  }
  const float mx = c_logit[0] / temperature;
  float sum = 0.f;
  for (int i = 0; i < n; ++i) sum += expf(c_logit[i] / temperature - mx);
  const float target = u * sum;
  float cum = 0.f;
  int pick = n - 1;
  for (int i = 0; i < n; ++i) {
    cum += expf(c_logit[i] / temperature - mx);
    if (target < cum) { pick = i; break; }
  }
  return pick;
}

template <bool kMasked>
__global__ void __launch_bounds__(kSampleThreads) sample_kernel(const float* __restrict__ logits, int V, const int32_t* __restrict__ hist,
                                                               int n_hist, float temperature, int top_k, float top_p, float min_p,
                                                               float penalty, float u, float* __restrict__ w,
                                                               int32_t* __restrict__ out_id, const SampleMask mask) {
  using Scan = cub::BlockScan<int, kSampleThreads>;
  __shared__ typename Scan::TempStorage scan_tmp;
  __shared__ int hist_bins[256];
  __shared__ uint32_t s_prefix, s_mask;
  __shared__ int s_need;
  __shared__ float c_logit[RL_LLM_MAX_TOP_K];
  __shared__ int c_id[RL_LLM_MAX_TOP_K];
  __shared__ int s_allowed;
  const int tid = threadIdx.x;
  int state = 0;
  if constexpr (kMasked) {
    // masked logits are -inf before the penalty (-inf * penalty stays -inf); a state outside the table allows nothing
    state = *mask.state;
    const bool valid = state >= 0 && state < mask.n_states;
    const bool eog_ok = valid && mask.accept[state];
    const int16_t* row = mask.index + (size_t)(valid ? state : 0) * V;
    if (tid == 0) s_allowed = 0;
    __syncthreads();
    int n_ok = 0;
    for (int i = tid; i < V; i += kSampleThreads) {
      bool eog = false;
#pragma unroll
      for (int e = 0; e < RL_LLM_MAX_EOG; ++e) eog |= mask.eog[e] == i;   // unused slots hold -1
      const float x = logits[i];
      // an id whose own logit is -inf or NaN counts as masked, so every candidate carries mass and the draw's
      // sums stay finite
      const bool ok = valid && (eog ? eog_ok : row[i] >= 0) && x > kNegInf;
      w[i] = ok ? x : kNegInf;
      n_ok += ok;
    }
    atomicAdd(&s_allowed, n_ok);
    __syncthreads();
    if (s_allowed == 0) {   // nothing allowed: no token, the state unchanged
      if (tid == 0) *out_id = RL_LLM_NO_TOKEN;
      return;
    }
  } else {
    for (int i = tid; i < V; i += kSampleThreads) w[i] = logits[i];
    __syncthreads();
  }
  if (tid < n_hist) {   // each distinct id once: its first occurrence applies the penalty
    const int tok = hist[tid];
    bool first = tok >= 0 && tok < V;
    for (int j = 0; j < tid && first; ++j) first = hist[j] != tok;
    if (first) {
      const float x = w[tok];
      w[tok] = x <= 0.f ? x * penalty : x / penalty;
    }
  }
  __syncthreads();
  int k = temperature == 0.f ? 1 : min(top_k, V);
  if constexpr (kMasked) k = min(k, s_allowed);   // the candidates are allowed ids only, so no fallback picks a masked one
  // radix select of the k-th largest order key, 8 bits at a time
  if (tid == 0) { s_prefix = 0; s_mask = 0; s_need = k; }
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += kSampleThreads) hist_bins[i] = 0;
    __syncthreads();
    const uint32_t prefix = s_prefix, mask = s_mask;
    for (int i = tid; i < V; i += kSampleThreads) {
      const uint32_t key = f2ord(w[i]);
      if ((key & mask) == prefix) atomicAdd(&hist_bins[(key >> shift) & 255], 1);
    }
    __syncthreads();
    if (tid == 0) {
      int need = s_need, b = 255;
      for (; b > 0; --b) {
        if (hist_bins[b] >= need) break;
        need -= hist_bins[b];
      }
      s_need = need;
      s_prefix = prefix | ((uint32_t)b << shift);
      s_mask = mask | (255u << shift);
    }
    __syncthreads();
  }
  const uint32_t thr = s_prefix;
  const int need = s_need;   // ids with key == thr taken, lowest first; k - need ids have a larger key
  // collect in id order: thread t scans ids [t c, (t + 1) c)
  const int per = (V + kSampleThreads - 1) / kSampleThreads;
  const int lo = min(V, tid * per), hi = min(V, lo + per);
  int n_gt = 0, n_eq = 0;
  for (int i = lo; i < hi; ++i) {
    const uint32_t key = f2ord(w[i]);
    n_gt += key > thr;
    n_eq += key == thr;
  }
  int o_gt, o_eq;
  Scan(scan_tmp).ExclusiveSum(n_gt, o_gt);
  __syncthreads();
  Scan(scan_tmp).ExclusiveSum(n_eq, o_eq);
  for (int i = tid; i < RL_LLM_MAX_TOP_K; i += kSampleThreads) { c_logit[i] = kNegInf; c_id[i] = 0x7fffffff; }
  __syncthreads();
  for (int i = lo; i < hi; ++i) {
    const uint32_t key = f2ord(w[i]);
    if (key > thr) { c_logit[o_gt] = w[i]; c_id[o_gt] = i; ++o_gt; }
    else if (key == thr) {
      if (o_eq < need) { c_logit[k - need + o_eq] = w[i]; c_id[k - need + o_eq] = i; }
      ++o_eq;
    }
  }
  __syncthreads();
  // bitonic sort of the 256 slots: logit descending, id ascending (empty slots last)
  for (int size = 2; size <= RL_LLM_MAX_TOP_K; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      if (tid < RL_LLM_MAX_TOP_K) {
        const int j = tid ^ stride;
        if (j > tid) {
          const bool up = (tid & size) == 0;
          const float la = c_logit[tid], lb = c_logit[j];
          const int ia = c_id[tid], ib = c_id[j];
          const bool a_first = la > lb || (la == lb && ia < ib);
          if (a_first != up) { c_logit[tid] = lb; c_logit[j] = la; c_id[tid] = ib; c_id[j] = ia; }
        }
      }
      __syncthreads();
    }
  }
  if (tid != 0) return;
  int pick = 0;
  if (temperature != 0.f) pick = draw(c_logit, k, temperature, top_p, min_p, u);
  const int tok = c_id[pick];
  *out_id = tok;
  if constexpr (kMasked) {
    bool eog = false;
#pragma unroll
    for (int e = 0; e < RL_LLM_MAX_EOG; ++e) eog |= mask.eog[e] == tok;
    if (!eog) *mask.state = mask.index[(size_t)state * V + tok];
  }
}

}  // namespace
}  // namespace rl

using namespace rl;

// ---- host side -------------------------------------------------------------------------------------------------------
static size_t align256(size_t x) { return (x + 255) / 256 * 256; }

static int sm_count_of_device(int* sms) {
  int dev = 0;
  RL_CUDA_CHECK(cudaGetDevice(&dev));
  RL_CUDA_CHECK(cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev));
  return RL_OK;
}

static bool linear_ok(const rl_llm_linear* w) {
  if (!w || w->N <= 0 || w->K <= 0 || w->K % kQSliceK || w->N % 32) return false;
  if (w->n_parts != (w->N + RL_LLM_PART_ROWS - 1) / RL_LLM_PART_ROWS || w->n_parts > RL_LLM_MAX_PARTS) return false;
  for (int i = 0; i < w->n_parts; ++i)
    if (!w->parts[i] || (reinterpret_cast<uintptr_t>(w->parts[i]) & 15)) return false;
  return true;
}
static int part_rows(const rl_llm_linear* w, int i) { return std::min(RL_LLM_PART_ROWS, w->N - RL_LLM_PART_ROWS * i); }

// The GEMV plan of segments with one K: items (pass, K range), kparts K ranges of spp slices each.
struct GemvPlan { int n_pass, kparts, spp, n_qs, n_total; };
static GemvPlan gemv_plan(int n_total, int n_pass, int K) {
  GemvPlan p;
  p.n_qs = K / kQSliceK;
  p.n_total = n_total;
  p.n_pass = n_pass;
  int kp = (kGemvTargetItems + n_pass - 1) / n_pass;
  kp = std::max(1, std::min(kp, p.n_qs));
  p.spp = (p.n_qs + kp - 1) / kp;
  p.kparts = (p.n_qs + p.spp - 1) / p.spp;
  return p;
}
static size_t gemv_partial_bytes(int N, int K) {
  const GemvPlan p = gemv_plan(N, (N + kQPassRows - 1) / kQPassRows, K);   // parts hold whole passes but the last
  return p.kparts > 1 ? (size_t)p.kparts * N * sizeof(float) : 0;
}

// y = [W_0; W_1; ...] x for linears of one K, outputs concatenated.
static int launch_gemv(const rl_llm_linear* const* ws, int n_lin, const __half* x, void* y, int y_f32, float* partial,
                       cudaStream_t stream) {
  GemvArgs a;
  memset(&a, 0, sizeof(a));
  int n0 = 0, pass0 = 0, ns = 0;
  for (int l = 0; l < n_lin; ++l)
    for (int i = 0; i < ws[l]->n_parts; ++i) {
      RL_REQUIRE(ns < kGemvMaxSegs, RL_EUNSUPPORTED, "qgemv: more than %d parts in one launch", kGemvMaxSegs);
      const int N = part_rows(ws[l], i);
      a.seg[ns++] = GemvSeg{reinterpret_cast<const unsigned char*>(ws[l]->parts[i]), N, pass0, n0, 0};
      n0 += N;
      pass0 += (N + kQPassRows - 1) / kQPassRows;
    }
  const GemvPlan p = gemv_plan(n0, pass0, ws[0]->K);
  a.x = x; a.partial = partial; a.y = y; a.y_f32 = y_f32;
  a.n_seg = ns; a.n_pass = pass0; a.n_total = n0; a.n_qs = p.n_qs; a.kparts = p.kparts; a.spp = p.spp;
  const size_t smem = (size_t)p.spp * 32 * (sizeof(float4) + sizeof(float));
  if (smem > 48 * 1024)
    RL_CUDA_CHECK(cudaFuncSetAttribute(qgemv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  qgemv_kernel<<<p.n_pass * p.kparts, kGemvThreads, smem, stream>>>(a);
  RL_CUDA_CHECK(cudaGetLastError());
  if (p.kparts > 1) {
    qgemv_combine_kernel<<<(n0 + 255) / 256, 256, 0, stream>>>(partial, p.kparts, n0, y, y_f32);
    RL_CUDA_CHECK(cudaGetLastError());
  }
  return RL_OK;
}

// The split count of an attention call: enough key ranges of whole 64-key tiles to reach kAttTargetCtas CTAs.
static int att_splits(int T, int n_head, int n_kv, int n_keys) {
  const int tiles = (T * (n_head / n_kv) + kAttQ - 1) / kAttQ;
  const int ctas = tiles * n_kv;
  int s = (kAttTargetCtas + ctas - 1) / ctas;
  const int key_tiles = (n_keys + kAttKeys - 1) / kAttKeys;
  return std::max(1, std::min({s, key_tiles, kAttMaxSplits}));
}
static size_t att_ws_bytes(int T, int n_head, int splits) {
  return splits > 1 ? align256((size_t)splits * T * n_head * kHd * 4) + align256((size_t)splits * T * n_head * 2 * 4) : 0;
}

static int launch_attention(const __half* q, const __half* kc, const __half* vc, int T, int p0, int n_head, int n_kv,
                            int splits, __half* out, void* ws, cudaStream_t stream) {
  const int n_keys = p0 + T;
  const int key_tiles = (n_keys + kAttKeys - 1) / kAttKeys;
  const int chunk = (key_tiles + splits - 1) / splits * kAttKeys;
  splits = (n_keys + chunk - 1) / chunk;   // no empty trailing range
  float* part_o = reinterpret_cast<float*>(ws);
  float* part_ml = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(ws) +
                                            align256((size_t)splits * T * n_head * kHd * 4));
  RL_CUDA_CHECK(cudaFuncSetAttribute(attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAttSmem));
  const dim3 grid((T * (n_head / n_kv) + kAttQ - 1) / kAttQ, n_kv, splits);
  attention_kernel<<<grid, kAttThreads, kAttSmem, stream>>>(q, kc, vc, T, p0, n_head, n_kv, splits, chunk, out, part_o, part_ml);
  RL_CUDA_CHECK(cudaGetLastError());
  if (splits > 1) {
    attention_combine_kernel<<<T * n_head, kHd, 0, stream>>>(part_o, part_ml, splits, T * n_head, out);
    RL_CUDA_CHECK(cudaGetLastError());
  }
  return RL_OK;
}

static bool heads_ok(int n_head, int n_kv) {
  return n_head > 0 && n_kv > 0 && n_head % n_kv == 0 && n_head / n_kv <= RL_LLM_MAX_GROUP;
}

extern "C" size_t rl_llm_qgemv_workspace_bytes(int N, int K) {
  if (N <= 0 || K <= 0 || K % kQSliceK) return 0;
  return gemv_partial_bytes(N, K);
}

extern "C" int rl_llm_qgemv(const rl_llm_linear* w, const void* x, void* y, int y_f32, void* workspace,
                            size_t workspace_bytes, void* stream) {
  RL_REQUIRE(w && x && y, RL_EINVAL, "rl_llm_qgemv: null pointer");
  RL_REQUIRE(linear_ok(w), RL_EUNSUPPORTED, "rl_llm_qgemv: N=%d K=%d n_parts=%d unsupported (N %% 32 == 0, K %% 128 == 0, "
             "ceil(N / %d) <= %d 16-byte aligned parts)", w->N, w->K, w->n_parts, RL_LLM_PART_ROWS, RL_LLM_MAX_PARTS);
  RL_REQUIRE((reinterpret_cast<uintptr_t>(x) & 7) == 0, RL_EINVAL, "rl_llm_qgemv: x must be 8-byte aligned");
  RL_REQUIRE(workspace_bytes >= gemv_partial_bytes(w->N, w->K) && (workspace || !gemv_partial_bytes(w->N, w->K)),
             RL_ENOSPACE, "rl_llm_qgemv: workspace too small");
  const rl_llm_linear* ws[1] = {w};
  return launch_gemv(ws, 1, reinterpret_cast<const __half*>(x), y, y_f32, reinterpret_cast<float*>(workspace),
                     (cudaStream_t)stream);
}

extern "C" int rl_llm_embed(const rl_llm_linear* table, const int32_t* ids, int T, float* out, void* stream) {
  RL_REQUIRE(table && ids && out && T >= 0, RL_EINVAL, "rl_llm_embed: bad arguments");
  RL_REQUIRE(linear_ok(table), RL_EUNSUPPORTED, "rl_llm_embed: the table is not a valid linear");
  if (T == 0) return RL_OK;
  Parts p;
  for (int i = 0; i < RL_LLM_MAX_PARTS; ++i) p.img[i] = reinterpret_cast<const unsigned char*>(table->parts[i]);
  embed_rows_kernel<<<T, 256, 0, (cudaStream_t)stream>>>(p, ids, table->N, table->K, out);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" int rl_llm_qk_norm_rope(const void* qkv, int T, int p0, int n_head, int n_kv, const float* q_norm,
                                   const float* k_norm, float eps, float rope_base, int n_ctx, void* q_out, void* k_cache,
                                   void* v_cache, void* stream) {
  RL_REQUIRE(qkv && q_norm && k_norm && q_out && k_cache && v_cache && T >= 0 && p0 >= 0, RL_EINVAL,
             "rl_llm_qk_norm_rope: bad arguments");
  RL_REQUIRE(heads_ok(n_head, n_kv), RL_EUNSUPPORTED, "rl_llm_qk_norm_rope: n_head=%d n_kv=%d unsupported", n_head, n_kv);
  RL_REQUIRE(p0 + T <= n_ctx, RL_EINVAL, "rl_llm_qk_norm_rope: positions %d + %d exceed n_ctx=%d", p0, T, n_ctx);
  RL_REQUIRE(rope_base > 0.f && eps >= 0.f, RL_EINVAL, "rl_llm_qk_norm_rope: rope_base=%g eps=%g", rope_base, eps);
  if (T == 0) return RL_OK;
  const int warps = T * (n_head + 2 * n_kv);
  qk_norm_rope_kernel<<<(warps + 7) / 8, 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const __half*>(qkv), T, p0, n_head, n_kv, q_norm, k_norm, eps, rope_base,
      reinterpret_cast<__half*>(q_out), reinterpret_cast<__half*>(k_cache), reinterpret_cast<__half*>(v_cache));
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" size_t rl_llm_attention_workspace_bytes(int T, int n_head, int n_kv, int n_keys, int splits) {
  if (T <= 0 || !heads_ok(n_head, n_kv) || n_keys <= 0 || splits < 0 || splits > kAttMaxSplits) return 0;
  return att_ws_bytes(T, n_head, splits ? splits : att_splits(T, n_head, n_kv, n_keys));
}

extern "C" int rl_llm_attention(const void* q, const void* k_cache, const void* v_cache, int T, int p0, int n_head, int n_kv,
                                int splits, void* out, void* workspace, size_t workspace_bytes, void* stream) {
  RL_REQUIRE(q && k_cache && v_cache && out && T >= 1 && p0 >= 0, RL_EINVAL, "rl_llm_attention: bad arguments");
  RL_REQUIRE(heads_ok(n_head, n_kv), RL_EUNSUPPORTED, "rl_llm_attention: n_head=%d n_kv=%d unsupported (n_head %% n_kv == 0, "
             "group <= %d)", n_head, n_kv, RL_LLM_MAX_GROUP);
  RL_REQUIRE(splits >= 0 && splits <= kAttMaxSplits, RL_EINVAL, "rl_llm_attention: splits=%d (0 .. %d)", splits, kAttMaxSplits);
  RL_REQUIRE((reinterpret_cast<uintptr_t>(k_cache) & 15) == 0 && (reinterpret_cast<uintptr_t>(v_cache) & 15) == 0, RL_EINVAL,
             "rl_llm_attention: caches must be 16-byte aligned");
  const int s = splits ? splits : att_splits(T, n_head, n_kv, p0 + T);
  RL_REQUIRE(workspace_bytes >= att_ws_bytes(T, n_head, s) && (workspace || s == 1), RL_ENOSPACE,
             "rl_llm_attention: workspace too small");
  return launch_attention(reinterpret_cast<const __half*>(q), reinterpret_cast<const __half*>(k_cache),
                          reinterpret_cast<const __half*>(v_cache), T, p0, n_head, n_kv, s, reinterpret_cast<__half*>(out),
                          workspace, (cudaStream_t)stream);
}

extern "C" size_t rl_llm_sample_workspace_bytes(int V) { return V > 0 ? (size_t)V * sizeof(float) : 0; }

extern "C" int rl_llm_sample(const float* logits, int V, const int32_t* hist, int n_hist, float temperature, int top_k,
                             float top_p, float min_p, float repeat_penalty, float u, int32_t* out_id, void* workspace,
                             size_t workspace_bytes, void* stream) {
  RL_REQUIRE(logits && out_id && workspace && V > 0 && n_hist >= 0 && (hist || n_hist == 0), RL_EINVAL,
             "rl_llm_sample: bad arguments");
  RL_REQUIRE(n_hist <= kSampleThreads, RL_EINVAL, "rl_llm_sample: n_hist=%d > %d", n_hist, kSampleThreads);
  RL_REQUIRE(top_k >= 1 && top_k <= RL_LLM_MAX_TOP_K, RL_EINVAL, "rl_llm_sample: top_k=%d unsupported (1 .. %d)", top_k,
             RL_LLM_MAX_TOP_K);
  RL_REQUIRE(temperature >= 0.f && top_p > 0.f && top_p <= 1.f && min_p >= 0.f && min_p <= 1.f && repeat_penalty > 0.f &&
             u >= 0.f && u < 1.f, RL_EINVAL, "rl_llm_sample: temperature=%g top_p=%g min_p=%g repeat_penalty=%g u=%g out of "
             "range", temperature, top_p, min_p, repeat_penalty, u);
  RL_REQUIRE(workspace_bytes >= rl_llm_sample_workspace_bytes(V), RL_ENOSPACE, "rl_llm_sample: workspace too small");
  sample_kernel<false><<<1, kSampleThreads, 0, (cudaStream_t)stream>>>(logits, V, hist, n_hist, temperature, top_k, top_p,
                                                                       min_p, repeat_penalty, u,
                                                                       reinterpret_cast<float*>(workspace), out_id, SampleMask{});
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" int rl_llm_sample_masked(const float* logits, int V, const int32_t* hist, int n_hist, float temperature, int top_k,
                                    float top_p, float min_p, float repeat_penalty, float u, const int16_t* index,
                                    int n_states, const uint8_t* accept, const int32_t* eog_ids, int n_eog, int32_t* state,
                                    int32_t* out_id, void* workspace, size_t workspace_bytes, void* stream) {
  RL_REQUIRE(logits && out_id && workspace && V > 0 && n_hist >= 0 && (hist || n_hist == 0), RL_EINVAL,
             "rl_llm_sample_masked: bad arguments");
  RL_REQUIRE(index && accept && state && n_states > 0 && n_states <= RL_GRAMMAR_MAX_STATES, RL_EINVAL,
             "rl_llm_sample_masked: bad grammar (n_states=%d, 1 .. %d)", n_states, RL_GRAMMAR_MAX_STATES);
  RL_REQUIRE(n_eog >= 0 && n_eog <= RL_LLM_MAX_EOG && (eog_ids || n_eog == 0), RL_EINVAL,
             "rl_llm_sample_masked: n_eog=%d (0 .. %d)", n_eog, RL_LLM_MAX_EOG);
  RL_REQUIRE(n_hist <= kSampleThreads, RL_EINVAL, "rl_llm_sample_masked: n_hist=%d > %d", n_hist, kSampleThreads);
  RL_REQUIRE(top_k >= 1 && top_k <= RL_LLM_MAX_TOP_K, RL_EINVAL, "rl_llm_sample_masked: top_k=%d unsupported (1 .. %d)",
             top_k, RL_LLM_MAX_TOP_K);
  RL_REQUIRE(temperature >= 0.f && top_p > 0.f && top_p <= 1.f && min_p >= 0.f && min_p <= 1.f && repeat_penalty > 0.f &&
             u >= 0.f && u < 1.f, RL_EINVAL, "rl_llm_sample_masked: temperature=%g top_p=%g min_p=%g repeat_penalty=%g "
             "u=%g out of range", temperature, top_p, min_p, repeat_penalty, u);
  RL_REQUIRE(workspace_bytes >= rl_llm_sample_workspace_bytes(V), RL_ENOSPACE, "rl_llm_sample_masked: workspace too small");
  SampleMask m{index, accept, state, n_states, {}};
  for (int e = 0; e < RL_LLM_MAX_EOG; ++e) m.eog[e] = e < n_eog ? eog_ids[e] : -1;
  sample_kernel<true><<<1, kSampleThreads, 0, (cudaStream_t)stream>>>(logits, V, hist, n_hist, temperature, top_k, top_p,
                                                                      min_p, repeat_penalty, u,
                                                                      reinterpret_cast<float*>(workspace), out_id, m);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

// ---- the forward step ---------------------------------------------------------------------------------------------
struct FwdLayout { size_t x, h, qkv, q, att, y, gu, a, bias, gemv, attn, total; };
static FwdLayout fwd_layout(const rl_llm_weights* w, int T) {
  const size_t H = w->hidden, F = w->ffn, nq = (size_t)w->n_head * kHd, nqkv = (size_t)(w->n_head + 2 * w->n_kv) * kHd;
  FwdLayout L;
  size_t off = 0;
  auto take = [&](size_t b) { const size_t o = off; off += align256(b); return o; };
  L.x = take((size_t)T * H * 4);
  L.h = take((size_t)T * std::max(H, nq) * 2);
  L.qkv = take((size_t)T * nqkv * 2);
  L.q = take((size_t)T * nq * 2);
  L.att = take((size_t)T * nq * 2);
  L.y = take((size_t)T * H * 2);
  L.gu = take((size_t)T * 2 * F * 2);
  L.a = take((size_t)T * F * 2);
  L.bias = take((size_t)RL_LLM_PART_ROWS * 4);
  size_t g = 0;
  for (const auto& nk : {std::make_pair((size_t)nqkv, H), std::make_pair(H, nq), std::make_pair(2 * F, H),
                         std::make_pair(H, F), std::make_pair((size_t)w->vocab, H)})
    g = std::max(g, gemv_partial_bytes((int)nk.first, (int)nk.second));
  L.gemv = take(g);
  L.attn = take(att_ws_bytes(T, w->n_head, att_splits(T, w->n_head, w->n_kv, w->n_ctx)));
  L.total = off;
  return L;
}

static const char* weights_error(const rl_llm_weights* w) {
  if (!w || !w->layers || !w->output_norm) return "null pointer";
  if (w->n_layers < 1 || w->hidden <= 0 || w->hidden % 256 || w->ffn <= 0 || w->ffn % 256 || w->vocab <= 0 || w->n_ctx <= 0)
    return "n_layers >= 1, hidden and ffn multiples of 256, vocab > 0 and n_ctx > 0 required";
  if (!heads_ok(w->n_head, w->n_kv)) return "n_head must be a multiple of n_kv with a group <= 8";
  if (!(w->eps >= 0.f) || !(w->rope_base > 0.f)) return "eps >= 0 and rope_base > 0 required";
  const int H = w->hidden, nq = w->n_head * kHd, nkv = w->n_kv * kHd;
  auto lin = [](const rl_llm_linear& l, int N, int K) { return l.N == N && l.K == K && linear_ok(&l); };
  if (!lin(w->token_embd, w->vocab, H) || !lin(w->output, w->vocab, H)) return "token_embd / output must be [vocab, hidden]";
  for (int i = 0; i < w->n_layers; ++i) {
    const rl_llm_layer& l = w->layers[i];
    if (!lin(l.q, nq, H) || !lin(l.k, nkv, H) || !lin(l.v, nkv, H) || !lin(l.o, H, nq) || !lin(l.gate, w->ffn, H) ||
        !lin(l.up, w->ffn, H) || !lin(l.down, H, w->ffn))
      return "a layer's linear has the wrong shape or parts";
    if (!l.attn_norm || !l.q_norm || !l.k_norm || !l.ffn_norm) return "a layer's norm is null";
  }
  return nullptr;
}

extern "C" size_t rl_llm_workspace_bytes(const rl_llm_weights* w, int T_max) {
  if (weights_error(w) || T_max < 1) return 0;
  size_t b = 0;   // the attention's key-range partials shrink as T grows: the largest layout of any T <= T_max
  for (int T = 1; T <= T_max; ++T) b = std::max(b, fwd_layout(w, T).total);
  return b;
}

// A linear over T rows: GEMV when T == 1, else the wgmma linear part by part into columns n0 .. of a [T, ldy] output.
static int run_linear(const rl_llm_linear& l, const __half* X, int T, __half* Y, int ldy, int col0, const float* zero_bias,
                      float* gemv_ws, int sms, cudaStream_t stream) {
  if (T == 1) {
    const rl_llm_linear* ls[1] = {&l};
    return launch_gemv(ls, 1, X, Y + col0, 0, gemv_ws, stream);
  }
  for (int i = 0; i < l.n_parts; ++i) {
    const int rc = launch_qlinear_ld(X, l.parts[i], zero_bias, Y + col0 + RL_LLM_PART_ROWS * i, ldy, T, part_rows(&l, i), l.K,
                                     sms, stream);
    if (rc != RL_OK) return rc;
  }
  return RL_OK;
}

extern "C" int rl_llm_forward(const rl_llm_weights* w, const int32_t* ids, int T, int p0, void* k_cache, void* v_cache,
                              float* logits, void* workspace, size_t workspace_bytes, void* stream_) {
  const char* err = weights_error(w);
  RL_REQUIRE(!err, RL_EINVAL, "rl_llm_forward: %s", err ? err : "");
  RL_REQUIRE(ids && k_cache && v_cache && logits && workspace && T >= 1 && p0 >= 0, RL_EINVAL, "rl_llm_forward: bad arguments");
  RL_REQUIRE(p0 + T <= w->n_ctx, RL_EINVAL, "rl_llm_forward: positions %d + %d exceed n_ctx=%d", p0, T, w->n_ctx);
  const FwdLayout L = fwd_layout(w, T);
  RL_REQUIRE(workspace_bytes >= L.total, RL_ENOSPACE, "rl_llm_forward: workspace %zu < %zu bytes", workspace_bytes, L.total);
  cudaStream_t stream = (cudaStream_t)stream_;
  int sms = 132;
  if (T > 1) {
    const int rc = sm_count_of_device(&sms);
    if (rc != RL_OK) return rc;
  }
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  float* x = reinterpret_cast<float*>(ws + L.x);
  __half* h = reinterpret_cast<__half*>(ws + L.h);
  __half* qkv = reinterpret_cast<__half*>(ws + L.qkv);
  __half* q = reinterpret_cast<__half*>(ws + L.q);
  __half* att = reinterpret_cast<__half*>(ws + L.att);
  __half* y = reinterpret_cast<__half*>(ws + L.y);
  __half* gu = reinterpret_cast<__half*>(ws + L.gu);
  __half* a = reinterpret_cast<__half*>(ws + L.a);
  float* zero_bias = reinterpret_cast<float*>(ws + L.bias);
  float* gemv_ws = reinterpret_cast<float*>(ws + L.gemv);
  const int H = w->hidden, F = w->ffn, nq = w->n_head * kHd, nkv = w->n_kv * kHd, nqkv = nq + 2 * nkv;
  const size_t cache_layer = (size_t)w->n_ctx * nkv;
  RL_CUDA_CHECK(cudaMemsetAsync(zero_bias, 0, (size_t)RL_LLM_PART_ROWS * 4, stream));
  int rc = rl_llm_embed(&w->token_embd, ids, T, x, stream);
  if (rc != RL_OK) return rc;
  for (int li = 0; li < w->n_layers; ++li) {
    const rl_llm_layer& l = w->layers[li];
    __half* kc = reinterpret_cast<__half*>(k_cache) + li * cache_layer;
    __half* vc = reinterpret_cast<__half*>(v_cache) + li * cache_layer;
    rmsnorm_kernel<<<T, 256, 0, stream>>>(x, li ? y : nullptr, l.attn_norm, H, w->eps, h);
    RL_CUDA_CHECK(cudaGetLastError());
    if (T == 1) {
      const rl_llm_linear* qkv_l[3] = {&l.q, &l.k, &l.v};
      rc = launch_gemv(qkv_l, 3, h, qkv, 0, gemv_ws, stream);
    } else {
      rc = run_linear(l.q, h, T, qkv, nqkv, 0, zero_bias, gemv_ws, sms, stream);
      if (rc == RL_OK) rc = run_linear(l.k, h, T, qkv, nqkv, nq, zero_bias, gemv_ws, sms, stream);
      if (rc == RL_OK) rc = run_linear(l.v, h, T, qkv, nqkv, nq + nkv, zero_bias, gemv_ws, sms, stream);
    }
    if (rc != RL_OK) return rc;
    rc = rl_llm_qk_norm_rope(qkv, T, p0, w->n_head, w->n_kv, l.q_norm, l.k_norm, w->eps, w->rope_base, w->n_ctx, q, kc, vc,
                             stream);
    if (rc != RL_OK) return rc;
    rc = launch_attention(q, kc, vc, T, p0, w->n_head, w->n_kv, att_splits(T, w->n_head, w->n_kv, p0 + T), att,
                          ws + L.attn, stream);
    if (rc != RL_OK) return rc;
    rc = run_linear(l.o, att, T, y, H, 0, zero_bias, gemv_ws, sms, stream);
    if (rc != RL_OK) return rc;
    rmsnorm_kernel<<<T, 256, 0, stream>>>(x, y, l.ffn_norm, H, w->eps, h);
    RL_CUDA_CHECK(cudaGetLastError());
    if (T == 1) {
      const rl_llm_linear* gu_l[2] = {&l.gate, &l.up};
      rc = launch_gemv(gu_l, 2, h, gu, 0, gemv_ws, stream);
    } else {
      rc = run_linear(l.gate, h, T, gu, 2 * F, 0, zero_bias, gemv_ws, sms, stream);
      if (rc == RL_OK) rc = run_linear(l.up, h, T, gu, 2 * F, F, zero_bias, gemv_ws, sms, stream);
    }
    if (rc != RL_OK) return rc;
    swiglu_kernel<<<std::min(4096, (T * F + 255) / 256), 256, 0, stream>>>(gu, T, F, a);
    RL_CUDA_CHECK(cudaGetLastError());
    rc = run_linear(l.down, a, T, y, H, 0, zero_bias, gemv_ws, sms, stream);
    if (rc != RL_OK) return rc;
  }
  // the last row only: x += y, output norm, LM head
  rmsnorm_kernel<<<1, 256, 0, stream>>>(x + (size_t)(T - 1) * H, y + (size_t)(T - 1) * H, w->output_norm, H, w->eps, h);
  RL_CUDA_CHECK(cudaGetLastError());
  const rl_llm_linear* head[1] = {&w->output};
  return launch_gemv(head, 1, h, logits, 1, gemv_ws, stream);
}
