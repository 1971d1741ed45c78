// Sentence splitting on the GPU: the SaT token-classification head, the hat-weighted stitching of overlapping blocks,
// the token -> character map, the override with known probabilities, the whitespace-run propagation, and the
// reference's two-stage dynamic program that partitions each document into sentences (raglite/_split_sentences.py).
//
// Which blocks exist, their hat weights and which character each token writes are decided on the host
// (raglite_b200/_sentences.py); the kernels take them as arrays.  Every kernel is a gather or a per-document serial
// loop: no atomics, so results do not depend on how documents are grouped into calls.
#include "common.cuh"

namespace rl {
namespace {

constexpr int kSatMaxLabels = 16;
constexpr int kThreads = 256;

__device__ __forceinline__ int64_t upper_doc(const int64_t* off, int n_docs, int64_t x) {
  // the document d with off[d] <= x < off[d + 1] (off ascending, off[0] == 0)
  int lo = 0, hi = n_docs;   // invariant: off[lo] <= x, off[hi] > x
  while (hi - lo > 1) {
    int mid = (lo + hi) >> 1;
    if (off[mid] <= x) lo = mid; else hi = mid;
  }
  return lo;
}

// logits[r, l] = hidden[r, :] . W[l, :] + b[l]: one warp per row, lanes stride the hidden dimension, a fixed
// butterfly reduction.
__global__ void sat_head_kernel(const float* __restrict__ hidden, int64_t rows, int H, const float* __restrict__ W,
                                const float* __restrict__ bias, int NL, float* __restrict__ logits) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < rows; r += warps) {
    const float* h = hidden + r * H;
    for (int l = 0; l < NL; ++l) {
      const float* w = W + (int64_t)l * H;
      float acc = 0.f;
      for (int k = lane; k < H; k += 32) acc = fmaf(h[k], w[k], acc);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) logits[r * NL + l] = acc + bias[l];
    }
  }
}

// Stitched logit of every document token: the hat-weighted mean over the blocks that cover it, read in ascending block
// order.  A document's blocks all hold B = doc_block[d] tokens and start at blk_start[] (ascending, document-relative);
// block b's in-block position k is logits row blk_row[b] + k.  hat[B (B - 1) / 2 + k] is the weight of position k.
__global__ void sat_stitch_kernel(const float* __restrict__ logits, int NL, const int64_t* __restrict__ doc_tok_off,
                                  const int32_t* __restrict__ doc_block, int n_docs, const int64_t* __restrict__ blk_off,
                                  const int32_t* __restrict__ blk_start, const int64_t* __restrict__ blk_row,
                                  const float* __restrict__ hat, float* __restrict__ stitched) {
  const int64_t T = doc_tok_off[n_docs];
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < T; g += (int64_t)gridDim.x * blockDim.x) {
    const int d = (int)upper_doc(doc_tok_off, n_docs, g);
    const int t = (int)(g - doc_tok_off[d]);
    const int B = doc_block[d];
    const float* w = hat + (int64_t)B * (B - 1) / 2;
    // first block with start > t - B (it covers t when its start <= t)
    int64_t lo = blk_off[d], hi = blk_off[d + 1];
    while (lo < hi) {
      int64_t mid = (lo + hi) >> 1;
      if (blk_start[mid] > t - B) hi = mid; else lo = mid + 1;
    }
    float num[kSatMaxLabels], den = 0.f;
#pragma unroll
    for (int l = 0; l < kSatMaxLabels; ++l) num[l] = 0.f;
    for (int64_t b = lo; b < blk_off[d + 1] && blk_start[b] <= t; ++b) {
      const int k = t - blk_start[b];
      const float wk = w[k];
      const float* lg = logits + (blk_row[b] + k) * NL;
#pragma unroll
      for (int l = 0; l < kSatMaxLabels; ++l)
        if (l < NL) num[l] = __fadd_rn(num[l], __fmul_rn(wk, lg[l]));
      den = __fadd_rn(den, wk);
    }
#pragma unroll
    for (int l = 0; l < kSatMaxLabels; ++l)
      if (l < NL) stitched[g * NL + l] = __fdiv_rn(num[l], den);
  }
}

// dmin[d] = the minimum stitched logit of document d over all tokens and labels (-inf for a document without tokens,
// whose probabilities then come out 0).
__global__ void sat_doc_min_kernel(const float* __restrict__ stitched, int NL, const int64_t* __restrict__ doc_tok_off,
                                   float* __restrict__ dmin) {
  __shared__ float red[kThreads / 32];
  const int d = blockIdx.x;
  const int64_t a = doc_tok_off[d] * NL, e = doc_tok_off[d + 1] * NL;
  float m = __builtin_huge_valf();
  for (int64_t i = a + threadIdx.x; i < e; i += blockDim.x) m = fminf(m, stitched[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) m = fminf(m, red[w]);
    dmin[d] = a == e ? kNegInf : m;
  }
}

__global__ void sat_fill_kernel(const float* __restrict__ dmin, const int64_t* __restrict__ doc_char_off, int n_docs,
                                float* __restrict__ out) {
  const int64_t N = doc_char_off[n_docs];
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < N; c += (int64_t)gridDim.x * blockDim.x)
    out[c] = dmin[upper_doc(doc_char_off, n_docs, c)];
}

// Each token with a target writes its label-0 logit there.  The host leaves at most one writer per character.
__global__ void sat_scatter_kernel(const float* __restrict__ stitched, int NL, const int64_t* __restrict__ tok_char,
                                   int64_t T, float* __restrict__ out) {
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < T; g += (int64_t)gridDim.x * blockDim.x) {
    const int64_t c = tok_char[g];
    if (c >= 0) out[c] = stitched[g * NL];
  }
}

__global__ void sat_sigmoid_kernel(const float* __restrict__ known, int64_t N, float* __restrict__ out) {
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < N; c += (int64_t)gridDim.x * blockDim.x) {
    float p = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-out[c])));
    if (known != nullptr && !isnan(known[c])) p = known[c];
    out[c] = p;
  }
}

// Whitespace runs inside a document: for a non-space character i followed by a space, and j the first non-space after
// that run (in the same document), p[i .. j-2] = min(p[i .. j-1]) and p[j-1] = max(p[i .. j-1]).  Runs at the start or
// the end of a document are left alone.  One thread owns each run, so the reads see the values before propagation.
__global__ void sat_space_kernel(const uint8_t* __restrict__ is_space, const int64_t* __restrict__ doc_char_off,
                                 int n_docs, float* __restrict__ out) {
  const int64_t N = doc_char_off[n_docs];
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i + 1 < N; i += (int64_t)gridDim.x * blockDim.x) {
    if (is_space[i] || !is_space[i + 1]) continue;
    const int64_t end = doc_char_off[upper_doc(doc_char_off, n_docs, i) + 1];
    int64_t j = i + 1;
    while (j < end && is_space[j]) ++j;
    if (j >= end) continue;
    float mn = out[i], mx = out[i];
    for (int64_t c = i + 1; c < j; ++c) {
      const float v = out[c];
      if (isnan(v) || v < mn) mn = v;   // NaN propagates, as in np.min / np.max
      if (isnan(v) || v > mx) mx = v;
    }
    for (int64_t c = i; c < j - 1; ++c) out[c] = mn;
    out[j - 1] = mx;
  }
}

// ---- the partition ---------------------------------------------------------------------------------------------------
// One call of the reference's _split_sentences on p[0, n) (max_len <= 0 means none).  dp, back and ring are scratch of n
// entries; the boundaries come out ascending as partition indices (boundary + 1) in out.  Returns their number, 0 when the
// text stays one sentence, -1 when no split satisfies the constraints.  Every float64 step is the reference's: the
// float32 score widened, one rounded addition, strict comparisons.
__device__ int solve_partition(const float* __restrict__ p, int n, int min_len, int max_len, double* __restrict__ dp,
                               int* __restrict__ back, int* __restrict__ ring, int* __restrict__ out) {
  const double ninf = -__builtin_huge_val();
  const int first_valid = min_len - 1, last_valid = n - min_len - 1;
  if (last_valid < first_valid) return 0;
  for (int i = 0; i < n; ++i) {
    dp[i] = ninf;
    back[i] = -1;
  }
  if (max_len <= 0) {
    double best_prev = ninf;
    int best_idx = -1;
    for (int i = first_valid; i <= last_valid; ++i) {
      const int j = i - min_len;
      if (j >= first_valid && dp[j] > best_prev) {
        best_prev = dp[j];
        best_idx = j;
      }
      const double s = (double)__fsub_rn(p[i], 0.25f);
      dp[i] = s;
      if (best_prev > ninf && __dadd_rn(best_prev, s) > dp[i]) {
        dp[i] = __dadd_rn(best_prev, s);
        back[i] = best_idx;
      }
    }
  } else {
    int head = 0, tail = 0;   // the deque: ring[head, tail), each index pushed once
    for (int i = first_valid; i <= last_valid; ++i) {
      const int j = i - min_len;
      if (j >= first_valid && isfinite(dp[j])) {
        while (tail > head && dp[ring[tail - 1]] <= dp[j]) --tail;
        ring[tail++] = j;
      }
      while (tail > head && ring[head] < i - max_len) ++head;
      const double s = (double)__fsub_rn(p[i], 0.25f);
      if (i + 1 <= max_len) dp[i] = s;
      if (tail > head && __dadd_rn(dp[ring[head]], s) > dp[i]) {
        dp[i] = __dadd_rn(dp[ring[head]], s);
        back[i] = ring[head];
      }
    }
  }
  int answer_min = first_valid;
  if (max_len > 0 && n - max_len - 1 > answer_min) answer_min = n - max_len - 1;
  const bool no_boundary_valid = max_len <= 0 || max_len >= n;
  double best = no_boundary_valid ? 0.0 : ninf;
  int best_last = -1;
  for (int i = answer_min; i <= last_valid; ++i)
    if (dp[i] > best) {
      best = dp[i];
      best_last = i;
    }
  if (best_last == -1) return no_boundary_valid ? 0 : -1;
  int k = 0;
  for (int pos = best_last; pos >= 0; pos = back[pos]) ring[k++] = pos;   // the DP is done with the ring
  for (int m = 0; m < k; ++m) out[m] = ring[k - 1 - m] + 1;
  return k;
}

// One thread per document: stage 1 over the whole document with no maximum, then stage 2 (with max_len) over every
// stage-1 sentence longer than max_len, each on its own slice of the scratch.
__global__ void sentence_partition_kernel(const float* __restrict__ probas, const int64_t* __restrict__ doc_off,
                                          const int32_t* __restrict__ doc_len, const int32_t* __restrict__ min_len,
                                          const int32_t* __restrict__ max_len, int n_docs, double* __restrict__ dp,
                                          int* __restrict__ back, int* __restrict__ ring, int* __restrict__ bnd,
                                          int* __restrict__ cuts, int* __restrict__ counts, int* __restrict__ status) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= n_docs) return;
  const int64_t o = doc_off[d];
  const int n = doc_len[d], lo = min_len[d], hi = max_len[d];
  const float* p = probas + o;
  int* out = cuts + o;
  int k1 = solve_partition(p, n, lo, 0, dp + o, back + o, ring + o, bnd + o);
  if (hi <= 0) {
    for (int m = 0; m < k1; ++m) out[m] = bnd[o + m];
    counts[d] = k1;
    status[d] = 0;
    return;
  }
  int nc = 0;
  for (int s = 0; s <= k1; ++s) {
    const int a = s == 0 ? 0 : bnd[o + s - 1], e = s == k1 ? n : bnd[o + s];
    if (e - a > hi) {
      const int k2 = solve_partition(p + a, e - a, lo, hi, dp + o + a, back + o + a, ring + o + a, out + nc);
      if (k2 < 0) {
        counts[d] = 0;
        status[d] = 1;
        return;
      }
      for (int m = 0; m < k2; ++m) out[nc + m] += a;
      nc += k2;
    }
    if (s < k1) out[nc++] = e;
  }
  counts[d] = nc;
  status[d] = 0;
}

int grid_for(int64_t n) {
  int64_t g = (n + kThreads - 1) / kThreads;
  return (int)(g < 1 ? 1 : (g > 65536 ? 65536 : g));
}

}  // namespace
}  // namespace rl

using namespace rl;

extern "C" int rl_sat_token_logits(const float* hidden, int64_t rows, int hidden_size, const float* W, const float* bias,
                                   int n_labels, float* logits, void* stream) {
  RL_REQUIRE(rows >= 0 && hidden_size > 0 && n_labels >= 1 && n_labels <= kSatMaxLabels, RL_EINVAL,
             "rl_sat_token_logits: rows >= 0, hidden > 0 and 1 <= n_labels <= %d", kSatMaxLabels);
  if (rows == 0) return RL_OK;
  RL_REQUIRE(hidden && W && bias && logits, RL_EINVAL, "rl_sat_token_logits: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t blocks = (rows + (kThreads / 32) - 1) / (kThreads / 32);
  sat_head_kernel<<<(int)(blocks > 65536 ? 65536 : blocks), kThreads, 0, st>>>(hidden, rows, hidden_size, W, bias,
                                                                               n_labels, logits);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" size_t rl_sat_workspace_bytes(int64_t n_tokens, int n_docs, int n_labels) {
  if (n_tokens < 0 || n_docs < 0 || n_labels < 1) return 0;
  return (size_t)((n_tokens * n_labels * 4 + 255) / 256 * 256) + (size_t)((int64_t)n_docs * 4 + 255) / 256 * 256;
}

extern "C" int rl_sat_char_probas(const float* logits, int n_labels, const int64_t* doc_tok_off,
                                  const int64_t* doc_char_off, const int32_t* doc_block, int n_docs, int64_t n_tokens,
                                  int64_t n_chars, const int64_t* blk_off, const int32_t* blk_start,
                                  const int64_t* blk_row, const float* hat, const int64_t* tok_char, const float* known,
                                  const uint8_t* is_space, float* probas, void* workspace, size_t workspace_bytes,
                                  void* stream) {
  RL_REQUIRE(n_labels >= 1 && n_labels <= kSatMaxLabels && n_docs >= 0 && n_tokens >= 0 && n_chars >= 0, RL_EINVAL,
             "rl_sat_char_probas: 1 <= n_labels <= %d, n_docs, n_tokens, n_chars >= 0", kSatMaxLabels);
  if (n_docs == 0 || n_chars == 0) return RL_OK;
  RL_REQUIRE(doc_tok_off && doc_char_off && doc_block && blk_off && probas && workspace, RL_EINVAL,
             "rl_sat_char_probas: null pointer");
  RL_REQUIRE(n_tokens == 0 || (logits && blk_start && blk_row && hat && tok_char), RL_EINVAL,
             "rl_sat_char_probas: null pointer");
  RL_REQUIRE(workspace_bytes >= rl_sat_workspace_bytes(n_tokens, n_docs, n_labels), RL_ENOSPACE,
             "rl_sat_char_probas: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  float* stitched = (float*)workspace;
  float* dmin = (float*)((char*)workspace + (n_tokens * n_labels * 4 + 255) / 256 * 256);
  if (n_tokens) {
    sat_stitch_kernel<<<grid_for(n_tokens), kThreads, 0, st>>>(logits, n_labels, doc_tok_off, doc_block, n_docs, blk_off,
                                                               blk_start, blk_row, hat, stitched);
    RL_CUDA_CHECK(cudaGetLastError());
  }
  sat_doc_min_kernel<<<n_docs, kThreads, 0, st>>>(stitched, n_labels, doc_tok_off, dmin);
  RL_CUDA_CHECK(cudaGetLastError());
  sat_fill_kernel<<<grid_for(n_chars), kThreads, 0, st>>>(dmin, doc_char_off, n_docs, probas);
  RL_CUDA_CHECK(cudaGetLastError());
  if (n_tokens) {
    sat_scatter_kernel<<<grid_for(n_tokens), kThreads, 0, st>>>(stitched, n_labels, tok_char, n_tokens, probas);
    RL_CUDA_CHECK(cudaGetLastError());
  }
  sat_sigmoid_kernel<<<grid_for(n_chars), kThreads, 0, st>>>(known, n_chars, probas);
  RL_CUDA_CHECK(cudaGetLastError());
  if (is_space) {
    sat_space_kernel<<<grid_for(n_chars), kThreads, 0, st>>>(is_space, doc_char_off, n_docs, probas);
    RL_CUDA_CHECK(cudaGetLastError());
  }
  return RL_OK;
}

extern "C" size_t rl_sentence_partition_workspace_bytes(int64_t n_chars) {
  if (n_chars < 0) return 0;
  return (size_t)((n_chars * 8 + 255) / 256 * 256) + 3 * (size_t)((n_chars * 4 + 255) / 256 * 256);
}

extern "C" int rl_sentence_partition(const float* probas, const int64_t* doc_off, const int32_t* doc_len,
                                     const int32_t* min_len, const int32_t* max_len, int n_docs, int64_t n_chars,
                                     int32_t* cuts, int32_t* counts, int32_t* status, void* workspace,
                                     size_t workspace_bytes, void* stream) {
  RL_REQUIRE(n_docs >= 0 && n_chars >= 0, RL_EINVAL, "rl_sentence_partition: n_docs, n_chars >= 0");
  if (n_docs == 0) return RL_OK;
  RL_REQUIRE(probas && doc_off && doc_len && min_len && max_len && cuts && counts && status && workspace, RL_EINVAL,
             "rl_sentence_partition: null pointer");
  RL_REQUIRE(workspace_bytes >= rl_sentence_partition_workspace_bytes(n_chars), RL_ENOSPACE,
             "rl_sentence_partition: workspace too small");
  char* ws = (char*)workspace;
  const size_t s8 = (size_t)((n_chars * 8 + 255) / 256 * 256), s4 = (size_t)((n_chars * 4 + 255) / 256 * 256);
  double* dp = (double*)ws;
  int* back = (int*)(ws + s8);
  int* ring = (int*)(ws + s8 + s4);
  int* bnd = (int*)(ws + s8 + 2 * s4);
  constexpr int kPartThreads = 64;
  sentence_partition_kernel<<<(n_docs + kPartThreads - 1) / kPartThreads, kPartThreads, 0, (cudaStream_t)stream>>>(
      probas, doc_off, doc_len, min_len, max_len, n_docs, dp, back, ring, bnd, cuts, counts, status);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}
