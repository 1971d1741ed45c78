// Grammar-constrained sampling, the token index: for every (DFA state s, token v), the state after walking v's bytes
// from s, or -1.  decoder.cu's masked sampler reads one row of it per step (the allowed ids and the next state).
//
// One thread per (s, v), grid-stride, v fastest so that a warp reads neighbouring offsets and writes neighbouring
// entries.  The transition table goes to shared memory when it fits (n_states <= kSmemStates); each walk is then a
// chain of shared-memory loads, one per byte.
#include <algorithm>

#include "common.cuh"

namespace rl {
namespace {

constexpr int kIndexThreads = 256;
constexpr int kSmemStates = 384;   // 384 x 256 x 2 bytes = 192 KB of the H100's 227 KB per CTA

__global__ void __launch_bounds__(kIndexThreads) token_index_kernel(const int16_t* __restrict__ trans, int n_states,
                                                                   const uint8_t* __restrict__ bytes,
                                                                   const int64_t* __restrict__ offsets, int V,
                                                                   int16_t* __restrict__ index, int use_smem) {
  extern __shared__ int16_t s_trans[];
  const int16_t* tbl = trans;
  if (use_smem) {
    for (int i = threadIdx.x; i < n_states * 256; i += kIndexThreads) s_trans[i] = trans[i];
    __syncthreads();
    tbl = s_trans;
  }
  const int64_t total = (int64_t)n_states * V;
  for (int64_t p = (int64_t)blockIdx.x * kIndexThreads + threadIdx.x; p < total; p += (int64_t)gridDim.x * kIndexThreads) {
    const int s = (int)(p / V), v = (int)(p - (int64_t)s * V);
    const int64_t a = offsets[v], b = offsets[v + 1];
    int st = a < b ? s : -1;
    for (int64_t i = a; i < b && st >= 0; ++i) {
      const int nxt = tbl[st * 256 + __ldg(bytes + i)];
      st = (unsigned)nxt < (unsigned)n_states ? nxt : -1;   // anything outside the table is no transition
    }
    index[p] = (int16_t)st;
  }
}

}  // namespace
}  // namespace rl

using namespace rl;

extern "C" int rl_grammar_token_index(const int16_t* trans, int n_states, const uint8_t* token_bytes,
                                      const int64_t* offsets, int V, int16_t* index, void* stream) {
  RL_REQUIRE(trans && offsets && index && V > 0 && (token_bytes || V == 0), RL_EINVAL,
             "rl_grammar_token_index: bad arguments");
  RL_REQUIRE(n_states > 0 && n_states <= RL_GRAMMAR_MAX_STATES, RL_EUNSUPPORTED,
             "rl_grammar_token_index: n_states=%d unsupported (1 .. %d)", n_states, RL_GRAMMAR_MAX_STATES);
  int dev = 0, sms = 0;
  RL_CUDA_CHECK(cudaGetDevice(&dev));
  RL_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int use_smem = n_states <= kSmemStates;
  const size_t smem = use_smem ? (size_t)n_states * 256 * sizeof(int16_t) : 0;
  RL_CUDA_CHECK(cudaFuncSetAttribute(token_index_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;   // as many CTAs per SM as the table's shared memory lets in
  RL_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, token_index_kernel, kIndexThreads, smem));
  const int64_t total = (int64_t)n_states * V;
  const int64_t want = (total + kIndexThreads - 1) / kIndexThreads;
  const int grid = (int)std::min<int64_t>(want, (int64_t)sms * std::max(per_sm, 1));
  token_index_kernel<<<grid, kIndexThreads, smem, (cudaStream_t)stream>>>(trans, n_states, token_bytes, offsets, V, index,
                                                                          use_smem);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}
