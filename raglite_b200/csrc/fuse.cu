// The steps right after the scan, batched on device chunk indices (SURVEY.md section 8f-3, sm_90a):
//
//   rl_rrf_fuse      Reciprocal Rank Fusion of R rankings per query (reference _search.py:233-254, as used by
//                    hybrid_search :257-280): score(c) = sum_r w_r / (k + position of c in ranking r), ordered
//                    by descending score, ties in first-appearance order (Python's stable sort over a dict
//                    filled ranking by ranking).
//   rl_span_collate  The ranking half of retrieve_chunk_spans (_search.py:323-360): add the neighbours of every
//                    retrieved chunk inside its document, deduplicate, order by (document, position), cut into
//                    runs of consecutive positions, score a run with sum 1 / (rank + 1) over its retrieved members,
//                    order the runs by descending score (stable).
//
// One CTA per query; everything lives in shared memory (a few thousand entries).  Scores are float64, summed in
// the reference's order and the way its Python code sums them (`+=` for RRF, compensated `sum()` for spans), so
// they are the reference's Python floats bit for bit.
#include "common.cuh"

namespace rl {
namespace {

constexpr int kFuseThreads = 256;
constexpr int kFuseMax = 4096;   // entries per query (R * L, or retrieved chunks x (1 + neighbours))

// Ascending bitonic sort of (key, payload) pairs, lexicographic; n is a power of two.
__device__ void bitonic_pairs(uint64_t* key, uint32_t* pay, int n) {
  for (int k = 2; k <= n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const uint64_t a = key[i], b = key[ixj];
          const uint32_t pa = pay[i], pb = pay[ixj];
          const bool gt = a > b || (a == b && pa > pb);
          const bool up = (i & k) == 0;
          if (gt == up) { key[i] = b; key[ixj] = a; pay[i] = pb; pay[ixj] = pa; }
        }
      }
      __syncthreads();
    }
  }
}

// Order-preserving map double -> uint64 (ascending).
__device__ __forceinline__ uint64_t d2ord(double d) {
  const uint64_t u = (uint64_t)__double_as_longlong(d);
  return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
}

__global__ void __launch_bounds__(kFuseThreads) rrf_fuse_kernel(const int64_t* __restrict__ ids, const double* __restrict__ weights,
                                                              int R, int L, double k, int K, int64_t* __restrict__ out_ids,
                                                              double* __restrict__ out_score, int32_t* __restrict__ out_count) {
  extern __shared__ __align__(16) unsigned char fuse_smem[];
  const int n = R * L;
  int npow2 = 1;
  while (npow2 < n) npow2 <<= 1;
  uint64_t* key = reinterpret_cast<uint64_t*>(fuse_smem);           // [npow2]
  double* score = reinterpret_cast<double*>(key + npow2);            // [npow2]
  uint32_t* pay = reinterpret_cast<uint32_t*>(score + npow2);        // [npow2]
  __shared__ int n_unique;
  const int b = blockIdx.x;
  const int64_t* my = ids + (size_t)b * n;
  // 1) (id, position) pairs, padding last; sorted by id, then position: equal ids become contiguous, in ranking order
  for (int p = threadIdx.x; p < npow2; p += blockDim.x) {
    const int64_t id = p < n ? my[p] : -1;
    key[p] = id < 0 ? ~0ull : (uint64_t)id;
    pay[p] = (uint32_t)p;
  }
  if (threadIdx.x == 0) n_unique = 0;
  __syncthreads();
  bitonic_pairs(key, pay, npow2);
  // 2) the head of every group sums its members' contributions in ranking order (what the reference's dict does)
  for (int p = threadIdx.x; p < npow2; p += blockDim.x) {
    score[p] = 0.0;
    const uint64_t id = key[p];
    if (id == ~0ull || (p > 0 && key[p - 1] == id)) continue;
    double s = 0.0;
    for (int e = p; e < npow2 && key[e] == id; ++e) {
      const int r = (int)(pay[e] / (uint32_t)L), i = (int)(pay[e] % (uint32_t)L);
      s += weights[r] / (k + (double)i);
    }
    score[p] = s;
  }
  __syncthreads();
  // 3) compact the heads: (descending score, first appearance) -> ascending sort of (~ord(score), first position)
  // reuse: heads write (skey, first position | slot of the id) to the tail-free arrays after a barrier
  __shared__ int cursor;
  if (threadIdx.x == 0) cursor = 0;
  __syncthreads();
  uint64_t my_key[(kFuseMax + kFuseThreads - 1) / kFuseThreads];
  uint32_t my_pay[(kFuseMax + kFuseThreads - 1) / kFuseThreads];
  uint64_t my_id[(kFuseMax + kFuseThreads - 1) / kFuseThreads];
  int mine = 0;
  for (int p = threadIdx.x; p < npow2; p += blockDim.x) {
    const uint64_t id = key[p];
    if (id != ~0ull && (p == 0 || key[p - 1] != id)) {
      my_key[mine] = ~d2ord(score[p]);
      my_pay[mine] = pay[p];       // first appearance (smallest position of the group)
      my_id[mine] = id;
      ++mine;
    }
  }
  __syncthreads();
  // second arrays: ids ride in `score`'s storage (as raw 64-bit patterns) indexed by first position
  uint64_t* id_of_pos = reinterpret_cast<uint64_t*>(score);
  for (int m = 0; m < mine; ++m) {
    const int slot = atomicAdd(&cursor, 1);
    key[slot] = my_key[m];
    pay[slot] = my_pay[m];
    id_of_pos[my_pay[m]] = my_id[m];   // positions are unique, < n <= npow2
  }
  __syncthreads();
  const int nu = cursor;
  int upow2 = 1;
  while (upow2 < nu) upow2 <<= 1;
  for (int p = nu + threadIdx.x; p < upow2; p += blockDim.x) { key[p] = ~0ull; pay[p] = 0xFFFFFFFFu; }
  __syncthreads();
  bitonic_pairs(key, pay, upow2);
  const int n_out = nu < K ? nu : K;
  for (int i = threadIdx.x; i < K; i += blockDim.x) {
    if (i < n_out) {
      const uint64_t o = ~key[i];
      const uint64_t u = (o & 0x8000000000000000ull) ? (o & 0x7fffffffffffffffull) : ~o;
      out_score[(size_t)b * K + i] = __longlong_as_double((long long)u);
      out_ids[(size_t)b * K + i] = (int64_t)id_of_pos[pay[i]];
    } else {
      out_score[(size_t)b * K + i] = 0.0;
      out_ids[(size_t)b * K + i] = -1;
    }
  }
  if (threadIdx.x == 0) out_count[b] = n_out;
}

// ---- span collation -------------------------------------------------------------------------------------------
// chunk_doc[c] / chunk_pos[c]: document ordinal and Chunk.index of chunk c; sorted_key / sorted_chunk: the table
// (doc << 32 | pos) -> chunk, ascending by key (neighbour lookup by binary search); alive[c] != 0: not deleted.
__device__ __forceinline__ int64_t find_chunk(const uint64_t* __restrict__ sorted_key, const int64_t* __restrict__ sorted_chunk,
                                              int64_t n, uint64_t want) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (sorted_key[mid] < want) lo = mid + 1; else hi = mid;
  }
  return (lo < n && sorted_key[lo] == want) ? sorted_chunk[lo] : -1;
}

__global__ void __launch_bounds__(kFuseThreads) span_collate_kernel(
    const int64_t* __restrict__ ranked, int M, const int32_t* __restrict__ chunk_doc, const int32_t* __restrict__ chunk_pos,
    const uint8_t* __restrict__ chunk_alive, const uint64_t* __restrict__ sorted_key, const int64_t* __restrict__ sorted_chunk,
    int64_t n_chunks, const int32_t* __restrict__ neighbors, int n_nb, int64_t* __restrict__ out_member,
    int32_t* __restrict__ out_span_start, int32_t* __restrict__ out_span_len, double* __restrict__ out_span_score,
    int32_t* __restrict__ out_n_span, int32_t* __restrict__ out_n_member) {
  extern __shared__ __align__(16) unsigned char fuse_smem[];
  const int cap = M * (1 + n_nb);
  int npow2 = 1;
  while (npow2 < cap) npow2 <<= 1;
  // Shared memory, npow2 entries per array: key | score | chunk_of | rel | tmpk (8 bytes each) | pay (4 bytes).  The
  // 4-byte array comes last so that every 8-byte array starts on an 8-byte boundary for any npow2, 1 included.
  uint64_t* key = reinterpret_cast<uint64_t*>(fuse_smem);         // (doc << 32 | pos), later span sort keys
  double* score = reinterpret_cast<double*>(key + npow2);          // 1 / (rank + 1) of retrieved members, 0 for neighbours
  int64_t* chunk_of = reinterpret_cast<int64_t*>(score + npow2);   // [npow2] chunk per entry (by original slot)
  double* rel = reinterpret_cast<double*>(chunk_of + npow2);       // [npow2] relevance by unique index
  uint64_t* tmpk = reinterpret_cast<uint64_t*>(rel + npow2);       // [npow2] scratch
  uint32_t* pay = reinterpret_cast<uint32_t*>(tmpk + npow2);       // slot in `ranked x (1 + n_nb)` -> chunk, later span index
  __shared__ int n_span;
  const int b = blockIdx.x;
  // 1) entries: slot = i * (1 + n_nb) + o (o = 0: the retrieved chunk, o >= 1: its o-th neighbour offset)
  for (int e = threadIdx.x; e < npow2; e += blockDim.x) {
    uint64_t kk = ~0ull;
    int64_t c = -1;
    if (e < cap) {
      const int i = e / (1 + n_nb), o = e % (1 + n_nb);
      const int64_t base = ranked[(size_t)b * M + i];
      if (base >= 0 && base < n_chunks) {
        if (o == 0) {
          c = base;
        } else {
          const int64_t pos = (int64_t)chunk_pos[base] + neighbors[o - 1];
          if (pos >= 0) c = find_chunk(sorted_key, sorted_chunk, n_chunks, ((uint64_t)(uint32_t)chunk_doc[base] << 32) | (uint64_t)pos);
          if (c >= 0 && chunk_alive != nullptr && chunk_alive[c] == 0) c = -1;
        }
      }
      if (c >= 0) kk = ((uint64_t)(uint32_t)chunk_doc[c] << 32) | (uint64_t)(uint32_t)chunk_pos[c];
    }
    key[e] = kk;
    pay[e] = (uint32_t)e;
    chunk_of[e] = c;
  }
  if (threadIdx.x == 0) n_span = 0;
  __syncthreads();
  // sorted by (doc, pos), then by slot: of several entries for one chunk the retrieved one with the best rank comes first
  bitonic_pairs(key, pay, npow2);
  // 2) unique chunks in (doc, pos) order; a unique entry's relevance = 1 / (rank + 1) of the LAST retrieved duplicate in
  //    list order (the reference's dict comprehension keeps the last assignment) -- duplicates in `ranked` are unusual
  int* head = reinterpret_cast<int*>(score);   // scratch until scores are written: flag per sorted entry
  for (int e = threadIdx.x; e < npow2; e += blockDim.x)
    head[e] = (key[e] != ~0ull && (e == 0 || key[e - 1] != key[e])) ? 1 : 0;
  __syncthreads();
  // exclusive scan of the flags by one warp-sized sequential pass per thread block (cap is a few thousand)
  __shared__ int total_unique;
  if (threadIdx.x == 0) {
    int run = 0;
    for (int e = 0; e < npow2; ++e) { const int f = head[e]; head[e] = f ? run : -1; run += f; }
    total_unique = run;
  }
  __syncthreads();
  const int nu = total_unique;
  // member list (unique chunks in document order) + per-member relevance, written to global / kept in registers via smem
  int64_t* member = out_member + (size_t)b * cap;
  for (int e = threadIdx.x; e < npow2; e += blockDim.x) {
    const int u = head[e];
    if (u < 0) continue;
    double r = 0.0;
    for (int x = e; x < npow2 && key[x] == key[e]; ++x) {
      const int slot = (int)pay[x];
      if (slot % (1 + n_nb) == 0) r = 1.0 / (double)(slot / (1 + n_nb) + 1);   // ascending slots: the last one wins
    }
    rel[u] = r;
    member[u] = chunk_of[pay[e]];
  }
  __syncthreads();
  // 3) runs of consecutive positions inside one document; run score = sum of member relevances in document order
  uint64_t* ukey = key;   // reuse: first compact the unique keys
  __shared__ int dummy;
  (void)dummy;
  // (unique keys, in order) -- gather through a second pass (tmpk) to avoid aliasing while reading `key`
  for (int e = threadIdx.x; e < npow2; e += blockDim.x)
    if (head[e] >= 0) tmpk[head[e]] = key[e];
  __syncthreads();
  for (int u = threadIdx.x; u < nu; u += blockDim.x) ukey[u] = tmpk[u];
  __syncthreads();
  int32_t* s_start = out_span_start + (size_t)b * cap;
  int32_t* s_len = out_span_len + (size_t)b * cap;
  double* s_score = out_span_score + (size_t)b * cap;
  if (threadIdx.x == 0) {   // sequential: the reference's groupby loop (a few thousand members at most)
    // A run's score is the reference's sum() over its members, which Python (3.12 on) computes with Neumaier's
    // compensated summation: a running sum plus a compensation term that is added once at the end.
    auto py_sum = [](double acc, double comp) { return comp != 0.0 && isfinite(comp) ? acc + comp : acc; };
    int ns = 0, start = 0;
    double acc = 0.0, comp = 0.0;
    for (int u = 0; u < nu; ++u) {
      const bool cont = u > 0 && (ukey[u] >> 32) == (ukey[u - 1] >> 32) && (uint32_t)ukey[u] == (uint32_t)ukey[u - 1] + 1u;
      if (u > 0 && !cont) {
        s_start[ns] = start; s_len[ns] = u - start; s_score[ns] = py_sum(acc, comp); ++ns;
        start = u; acc = 0.0; comp = 0.0;
      }
      const double x = rel[u], t = acc + x;
      comp += fabs(acc) >= fabs(x) ? (acc - t) + x : (x - t) + acc;
      acc = t;
    }
    if (nu > 0) { s_start[ns] = start; s_len[ns] = nu - start; s_score[ns] = py_sum(acc, comp); ++ns; }
    n_span = ns;
  }
  __syncthreads();
  // 4) order the runs by descending score, stable in document order
  const int ns = n_span;
  int spow2 = 1;
  while (spow2 < ns) spow2 <<= 1;
  for (int i = threadIdx.x; i < spow2; i += blockDim.x) {
    key[i] = i < ns ? ~d2ord(s_score[i]) : ~0ull;
    pay[i] = i < ns ? (uint32_t)i : 0xFFFFFFFFu;
  }
  __syncthreads();
  bitonic_pairs(key, pay, spow2);
  // permute (start, len, score) through shared scratch
  int* p_start = reinterpret_cast<int*>(tmpk);
  int* p_len = p_start + npow2;
  for (int i = threadIdx.x; i < ns; i += blockDim.x) { p_start[i] = s_start[pay[i]]; p_len[i] = s_len[pay[i]]; rel[i] = s_score[pay[i]]; }
  __syncthreads();
  for (int i = threadIdx.x; i < cap; i += blockDim.x) {
    if (i < ns) { s_start[i] = p_start[i]; s_len[i] = p_len[i]; s_score[i] = rel[i]; }
    else { s_start[i] = 0; s_len[i] = 0; s_score[i] = 0.0; }
    if (i >= nu) member[i] = -1;
  }
  if (threadIdx.x == 0) { out_n_span[b] = ns; out_n_member[b] = nu; }
}

}  // namespace
}  // namespace rl

using namespace rl;

extern "C" int rl_rrf_fuse(const int64_t* ids, const double* weights, int B, int R, int L, double k, int K, int64_t* out_ids,
                           double* out_score, int32_t* out_count, void* stream) {
  RL_REQUIRE(B >= 0 && R >= 1 && L >= 1 && K >= 1 && k > 0.0, RL_EINVAL, "rl_rrf_fuse: bad sizes");
  if (B == 0) return RL_OK;
  RL_REQUIRE(ids && weights && out_ids && out_score && out_count, RL_EINVAL, "rl_rrf_fuse: null pointer");
  RL_REQUIRE((int64_t)R * L <= kFuseMax, RL_EUNSUPPORTED, "rl_rrf_fuse: R*L=%lld exceeds %d", (long long)R * L, kFuseMax);
  int npow2 = 1;
  while (npow2 < R * L) npow2 <<= 1;
  const size_t smem = (size_t)npow2 * (8 + 8 + 4);
  RL_CUDA_CHECK(cudaFuncSetAttribute(rrf_fuse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  rrf_fuse_kernel<<<B, kFuseThreads, smem, (cudaStream_t)stream>>>(ids, weights, R, L, k, K, out_ids, out_score, out_count);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" int rl_span_collate(const int64_t* ranked, int B, int M, const int32_t* chunk_doc, const int32_t* chunk_pos,
                               const uint8_t* chunk_alive, const uint64_t* sorted_key, const int64_t* sorted_chunk,
                               int64_t n_chunks, const int32_t* neighbors, int n_neighbors, int64_t* out_member,
                               int32_t* out_span_start, int32_t* out_span_len, double* out_span_score, int32_t* out_n_span,
                               int32_t* out_n_member, void* stream) {
  RL_REQUIRE(B >= 0 && M >= 1 && n_neighbors >= 0 && n_chunks >= 0, RL_EINVAL, "rl_span_collate: bad sizes");
  if (B == 0) return RL_OK;
  RL_REQUIRE(ranked && chunk_doc && chunk_pos && sorted_key && sorted_chunk && out_member && out_span_start && out_span_len &&
                 out_span_score && out_n_span && out_n_member && (n_neighbors == 0 || neighbors),
             RL_EINVAL, "rl_span_collate: null pointer");
  const int64_t cap = (int64_t)M * (1 + n_neighbors);
  RL_REQUIRE(cap <= kFuseMax, RL_EUNSUPPORTED, "rl_span_collate: M*(1+neighbors)=%lld exceeds %d", (long long)cap, kFuseMax);
  int npow2 = 1;
  while (npow2 < cap) npow2 <<= 1;
  const size_t smem = (size_t)npow2 * (8 + 8 + 8 + 8 + 8 + 4);   // key | score | chunk_of | rel | tmpk | pay
  RL_REQUIRE(smem <= 220 * 1024, RL_EUNSUPPORTED, "rl_span_collate: %zu bytes of shared memory", smem);
  RL_CUDA_CHECK(cudaFuncSetAttribute(span_collate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  span_collate_kernel<<<B, kFuseThreads, smem, (cudaStream_t)stream>>>(ranked, M, chunk_doc, chunk_pos, chunk_alive, sorted_key,
                                                                        sorted_chunk, n_chunks, neighbors, n_neighbors, out_member,
                                                                        out_span_start, out_span_len, out_span_score, out_n_span,
                                                                        out_n_member);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}
