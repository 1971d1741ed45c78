// The quantized weight image (rl_xenc_pack_qlinear) as every kernel that reads it sees it: GGML block types, the
// header, and the per-pass, per-128-K-slice row runs.  xenc.cu writes and runs the wgmma linear on it; decoder.cu reads
// it element by element (GEMV, embedding rows).
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace rl {

// Types by their GGML ids.  A block of K elements of one row: Q8_0 32 elements (fp16 d, 32 int8), Q4_K 256 (fp16 d,
// fp16 dmin, 12 bytes of 6-bit scales and mins, 128 bytes of nibbles), Q6_K 256 (128 bytes of low nibbles, 64 of high
// bit pairs, 16 int8 scales, fp16 d).  Every value is ggml's formula in float32, each product and difference rounded on
// its own (no contraction):
//   Q8_0 d q      Q4_K (d sc) q - (dmin m)      Q6_K (d sc) (q - 32)
constexpr int kGgmlQ8_0 = 8, kGgmlQ4_K = 12, kGgmlQ6_K = 14;

__host__ __device__ inline int q_block_elems(int type) { return type == kGgmlQ8_0 ? 32 : 256; }
__host__ __device__ inline int q_block_bytes(int type) { return type == kGgmlQ8_0 ? 34 : type == kGgmlQ4_K ? 144 : 210; }
inline bool q_type_ok(int type) { return type == kGgmlQ8_0 || type == kGgmlQ4_K || type == kGgmlQ6_K; }

// Q4_K's 6-bit scale and min of sub-block j (ggml's get_scale_min_k4).
__host__ __device__ inline void q4k_scale_min(int j, const unsigned char* s, int& sc, int& m) {
  if (j < 4) {
    sc = s[j] & 63;
    m = s[j + 4] & 63;
  } else {
    sc = (s[j + 4] & 0xF) | ((s[j - 4] >> 6) << 4);
    m = (s[j + 4] >> 4) | ((s[j] >> 6) << 4);
  }
}

// Header (QImgHead, then n_pass QImgPass) and, from kQImgData on, per pass of kQPassRows output rows and per 128-element
// K slice one run of nb16 (the pass's rows rounded up to 16) rows of row_bytes each.  A row's slice (zero bytes for the
// padding rows, which decode to +0):
//   Q8_0  136 B: four fp16 d, then 128 int8
//   Q4_K   76 B: fp16 d, fp16 dmin, the four 6-bit scales and four mins unpacked to bytes, the 64 nibble bytes of the
//                half super-block (low nibbles: elements 0-31 and 64-95, high nibbles: 32-63 and 96-127)
//   Q6_K  108 B: the half super-block's 64 ql bytes, 32 qh bytes, 8 int8 scales, fp16 d, 2 zero bytes
// In each type, element e = 32 g + j of a slice (group g, j < 32) is:
//   Q8_0  d[g] * q[8 + e]
//   Q4_K  (d sc[g]) nib - (dmin m[g]),  nib = byte 12 + 32 (g >> 1) + j, nibble g & 1
//   Q6_K  (d sc[2 g + j / 16]) (q - 32), q = nibble g >> 1 of ql[32 (g & 1) + j] | bits 2 g of qh[64 + j] << 4
// That is 1.0, 1.056 and 1.029 times the GGUF bytes.  Each pass carries its own type, so images of tensors of different
// types concatenate pass by pass (rl_xenc_concat_qlinear).
constexpr int kQPassRows = 128;
constexpr int kQSliceK = 128;
constexpr uint32_t kQMaxRowBytes = 136;
struct QImgHead { int32_t n_pass, N, K, magic; };
struct QImgPass { int32_t type, row_bytes; int64_t offset; };   // offset from the image's start
constexpr int32_t kQImgMagic = 0x51494d47;     // "QIMG"
constexpr size_t kQImgMaxPasses = 64;          // N <= 8192
constexpr size_t kQImgData = 2048;             // where the passes' rows start (1024-aligned room for the header)
static_assert(sizeof(QImgHead) + kQImgMaxPasses * sizeof(QImgPass) <= kQImgData, "the header must fit before the data");

__host__ __device__ inline uint32_t q_row_bytes(int type) { return type == kGgmlQ8_0 ? 136u : type == kGgmlQ4_K ? 76u : 108u; }
__host__ __device__ inline int q_pass_rows(int N, int pass) {
  const int rem = N - pass * kQPassRows;
  return rem < kQPassRows ? rem : kQPassRows;
}

// The wgmma linear on a quantized image (xenc.cu) with an output row stride: Y[t * ldy + n] = X[t] . W[n] + bias[n]
// rounded to fp16.  ldy >= N, ldy % 8 == 0 and Y 16-byte aligned.
int launch_qlinear_ld(const __half* X, const void* img, const float* bias, __half* Y, int ldy, int T, int N, int K,
                      int sm_count, cudaStream_t stream);

}  // namespace rl
