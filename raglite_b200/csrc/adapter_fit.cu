// Query-adapter FIT on the device (SURVEY.md section 8f-4; reference _query_adapter.py:21-38, 172-183), sm_90a.
//
//   rl_best_vectors     For every (eval, retrieved chunk): the chunk's vector with the largest inner product with
//                       the eval's query -- argmax(chunk.embedding_matrix @ q), _query_adapter.py:172-183 -- copied
//                       out as the positive / negative example.  One CTA per (chunk slot, eval).
//   rl_adapter_targets  The bounded least squares of _optimize_query_target (:21-38) for every eval at once:
//                         min_mu 1/2 |q + D^T mu|^2,  mu >= 0,  D = {p_i - (1 + alpha) n_j},   t = q + D^T mu*.
//                       The m = |P| |N| rows of D live in the span of the r = |P| + |N| <= 64 example vectors, so the
//                       kernel never forms D: with W = [P; N], G = W W^T (r x r) and W q it has every entry of the
//                       Gram matrix H = D D^T and of g = D q in closed form, runs Lawson-Hanson active-set NNLS on
//                       (H, g) in float64 (the passive set never exceeds r columns, one Cholesky of <= 64 x 64 per
//                       step, all in shared memory) and recovers t = q + P^T a - (1 + alpha) N^T b from the row /
//                       column sums a, b of mu*.  t is the unique projection, so it equals SciPy's lsq_linear answer
//                       to rounding.  One CTA per eval.
#include <cuda_fp16.h>

#include "common.cuh"

namespace rl {
namespace {

constexpr int kFitThreads = 128;
constexpr int kFitMaxR = 64;      // retrieved chunks per eval (optimize_top_k <= 64)
constexpr int kFitMaxM = 1024;    // |P| * |N| <= 32 * 32

__device__ __forceinline__ double warp_sum_dd(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(kFitThreads) best_vectors_kernel(const float* __restrict__ E, const void* __restrict__ E16, int64_t ld, int d,
                                                                 const int64_t* __restrict__ chunk_off, const int64_t* __restrict__ chunks,
                                                                 int n_slots, const float* __restrict__ Q, float* __restrict__ best,
                                                                 int64_t* __restrict__ best_row) {
  __shared__ double s_val[kFitThreads / 32];
  __shared__ int64_t s_row[kFitThreads / 32];
  const int slot = blockIdx.x, e = blockIdx.y;
  const int64_t c = chunks[(size_t)e * n_slots + slot];
  float* out = best + ((size_t)e * n_slots + slot) * d;
  if (c < 0) {
    for (int i = threadIdx.x; i < d; i += blockDim.x) out[i] = 0.f;
    if (threadIdx.x == 0) best_row[(size_t)e * n_slots + slot] = -1;
    return;
  }
  const float* q = Q + (size_t)e * d;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const int64_t r0 = chunk_off[c], r1 = chunk_off[c + 1];
  double best_v = -__builtin_huge_val();
  int64_t best_r = -1;
  for (int64_t r = r0 + warp; r < r1; r += nw) {
    double acc = 0.0;
    if (E16 != nullptr) {
      const __half* row = reinterpret_cast<const __half*>(E16) + r * ld;
      for (int i = lane; i < d; i += 32) acc += (double)__half2float(row[i]) * (double)q[i];
    } else {
      const float* row = E + r * ld;
      for (int i = lane; i < d; i += 32) acc += (double)row[i] * (double)q[i];
    }
    acc = warp_sum_dd(acc);
    if (acc > best_v) { best_v = acc; best_r = r; }   // rows ascend within a warp: the first maximum wins
  }
  if (lane == 0) { s_val[warp] = best_v; s_row[warp] = best_r; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < nw; ++w)
      if (s_val[w] > s_val[0] || (s_val[w] == s_val[0] && s_row[w] >= 0 && (s_row[0] < 0 || s_row[w] < s_row[0]))) {
        s_val[0] = s_val[w]; s_row[0] = s_row[w];
      }
    best_row[(size_t)e * n_slots + slot] = s_row[0];
  }
  __syncthreads();
  const int64_t br = s_row[0];
  for (int i = threadIdx.x; i < d; i += blockDim.x) {
    float v = 0.f;
    if (br >= 0) v = E16 != nullptr ? __half2float(reinterpret_cast<const __half*>(E16)[br * ld + i]) : E[br * ld + i];
    out[i] = v;
  }
}

// kind[e, slot]: 1 = relevant (positive), 0 = irrelevant (negative), anything else = unused slot.
__global__ void __launch_bounds__(kFitThreads) adapter_targets_kernel(const float* __restrict__ best, const uint8_t* __restrict__ kind,
                                                                    int n_slots, int d, const float* __restrict__ Q, double alpha,
                                                                    double* __restrict__ T, int32_t* __restrict__ ok,
                                                                    int32_t* __restrict__ iters) {
  extern __shared__ __align__(16) unsigned char fit_smem[];
  double* G = reinterpret_cast<double*>(fit_smem);          // [kFitMaxR][kFitMaxR]  W W^T
  double* Hs = G + kFitMaxR * kFitMaxR;                      // [kFitMaxR][kFitMaxR]  H on the passive set, then its Cholesky factor
  double* wq = Hs + kFitMaxR * kFitMaxR;                     // [kFitMaxR]            W q
  double* mu = wq + kFitMaxR;                                // [kFitMaxM]
  double* wgrad = mu + kFitMaxM;                             // [kFitMaxM]            -(H mu + g)
  double* z = wgrad + kFitMaxM;                              // [kFitMaxR]
  double* rhs = z + kFitMaxR;                                // [kFitMaxR]
  int* widx = reinterpret_cast<int*>(rhs + kFitMaxR);        // [kFitMaxR] slot of the i-th example (positives first)
  int* S = widx + kFitMaxR;                                  // [kFitMaxR] passive set (generator indices)
  uint8_t* inS = reinterpret_cast<uint8_t*>(S + kFitMaxR);   // [kFitMaxM] 1: passive, 2: rejected until the next successful step
  __shared__ int nP, nN, s_sz, s_pick, s_flag, s_iter, s_fresh;
  __shared__ double s_best, s_step;
  const int e = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  const uint8_t* kd = kind + (size_t)e * n_slots;
  const float* q = Q + (size_t)e * d;
  double* t_out = T + (size_t)e * d;
  if (tid == 0) {
    int p = 0, n = 0;
    for (int sl = 0; sl < n_slots; ++sl) if (kd[sl] == 1) widx[p++] = sl;
    nP = p;
    for (int sl = 0; sl < n_slots; ++sl) if (kd[sl] == 0) widx[p + n++] = sl;
    nN = n;
    s_sz = 0; s_iter = 0;
  }
  __syncthreads();
  const int P = nP, N = nN, r = P + N, m = P * N;
  if (P == 0 || N == 0 || r > kFitMaxR || m > kFitMaxM) {   // nothing to optimise (reference: the eval is skipped)
    for (int i = tid; i < d; i += blockDim.x) t_out[i] = (double)q[i];
    if (tid == 0) { ok[e] = 0; iters[e] = 0; }
    return;
  }
  const float* base = best + (size_t)e * n_slots * d;
  // G = W W^T and W q in float64: one warp per (a, b) pair
  for (int pr = warp; pr < r * (r + 1) / 2 + r; pr += nw) {
    int a, b;
    if (pr < r) { a = pr; b = -1; }
    else { int k = pr - r; a = 0; while (k >= r - a) { k -= r - a; ++a; } b = a + k; }
    const float* va = base + (size_t)widx[a] * d;
    const float* vb = b < 0 ? q : base + (size_t)widx[b] * d;
    double acc = 0.0;
    for (int i = lane; i < d; i += 32) acc += (double)va[i] * (double)vb[i];
    acc = warp_sum_dd(acc);
    if (lane == 0) { if (b < 0) wq[a] = acc; else { G[a * kFitMaxR + b] = acc; G[b * kFitMaxR + a] = acc; } }
  }
  for (int j = tid; j < m; j += blockDim.x) { mu[j] = 0.0; inS[j] = 0; }
  __syncthreads();
  const double c = 1.0 + alpha;
  auto Hent = [&](int j, int k) -> double {   // <d_j, d_k>, generator j = (i, jj): p_i - c n_jj
    const int i1 = j / N, j1 = P + j % N, i2 = k / N, j2 = P + k % N;
    return G[i1 * kFitMaxR + i2] - c * G[i1 * kFitMaxR + j2] - c * G[j1 * kFitMaxR + i2] + c * c * G[j1 * kFitMaxR + j2];
  };
  auto gent = [&](int j) -> double { return wq[j / N] - c * wq[P + j % N]; };   // <d_j, q>
  double gmax = 0.0;
  for (int j = 0; j < m; ++j) gmax = fmax(gmax, fabs(gent(j)));
  // Relative to the instance, like the pivot and fresh-column tests: scaling q by 2^a and the examples by 2^b scales
  // every gradient by 2^(a+b) and t by 2^a exactly.  gmax = 0 makes every gradient 0, and nothing is picked.
  const double tol = 1e-13 * gmax;
  const int max_iter = 6 * m + 64;
  while (true) {
    // w = -(g + H mu) over the generators outside the passive set; pick the largest
    for (int j = tid; j < m; j += blockDim.x) {
      double w = -gent(j);
      for (int a = 0; a < s_sz; ++a) w -= Hent(j, S[a]) * mu[S[a]];
      wgrad[j] = inS[j] ? -1.0 : w;
    }
    if (tid == 0) { s_best = tol; s_pick = -1; }
    __syncthreads();
    if (tid == 0) {
      for (int j = 0; j < m; ++j) if (wgrad[j] > s_best) { s_best = wgrad[j]; s_pick = j; }
      ++s_iter;
    }
    __syncthreads();
    if (s_pick < 0 || s_sz >= r || s_iter > max_iter) break;
    if (tid == 0) { S[s_sz] = s_pick; inS[s_pick] = 1; ++s_sz; s_fresh = 1; }
    __syncthreads();
    // inner loop: least squares on the passive set, step back to feasibility if a coefficient went non-positive
    while (true) {
      const int s = s_sz;
      for (int ab = tid; ab < s * s; ab += blockDim.x) Hs[(ab / s) * kFitMaxR + ab % s] = Hent(S[ab / s], S[ab % s]);
      for (int a = tid; a < s; a += blockDim.x) rhs[a] = -gent(S[a]);
      if (tid == 0) s_flag = 0;
      __syncthreads();
      // Cholesky H_SS = L L^T (in place, lower), then two triangular solves
      for (int col = 0; col < s; ++col) {
        if (tid == 0) {
          double dg = Hs[col * kFitMaxR + col];
          for (int k = 0; k < col; ++k) dg -= Hs[col * kFitMaxR + k] * Hs[col * kFitMaxR + k];
          if (dg <= 1e-14 * fabs(Hs[col * kFitMaxR + col]) || dg <= 0.0) s_flag = 1;   // dependent column
          Hs[col * kFitMaxR + col] = dg > 0.0 ? sqrt(dg) : 1.0;
        }
        __syncthreads();
        if (s_flag) break;
        const double piv = Hs[col * kFitMaxR + col];
        for (int row = col + 1 + tid; row < s; row += blockDim.x) {
          double v = Hs[row * kFitMaxR + col];
          for (int k = 0; k < col; ++k) v -= Hs[row * kFitMaxR + k] * Hs[col * kFitMaxR + k];
          Hs[row * kFitMaxR + col] = v / piv;
        }
        __syncthreads();
      }
      if (s_flag) {   // the newest generator is (numerically) in the span of the others: drop it for this round
        if (tid == 0) { --s_sz; inS[S[s_sz]] = 2; }
        __syncthreads();
        break;
      }
      if (tid == 0) {
        for (int a = 0; a < s; ++a) { double v = rhs[a]; for (int k = 0; k < a; ++k) v -= Hs[a * kFitMaxR + k] * z[k]; z[a] = v / Hs[a * kFitMaxR + a]; }
        for (int a = s - 1; a >= 0; --a) { double v = z[a]; for (int k = a + 1; k < s; ++k) v -= Hs[k * kFitMaxR + a] * z[k]; z[a] = v / Hs[a * kFitMaxR + a]; }
        // Lawson-Hanson safeguard: the column just added must come out positive in the first solve (it does in exact
        // arithmetic, its gradient was positive); if rounding says otherwise, adding it would cycle -- treat it as
        // dependent instead.
        if (s_fresh && z[s - 1] <= 0.0) s_flag = 2;
        s_fresh = 0;
        double step = 1.0;
        bool feasible = true;
        for (int a = 0; a < s; ++a)
          if (z[a] <= 0.0) { feasible = false; const double cur = mu[S[a]]; step = fmin(step, cur / (cur - z[a])); }
        s_step = feasible ? -1.0 : step;
      }
      __syncthreads();
      if (s_flag == 2) {
        if (tid == 0) { --s_sz; inS[S[s_sz]] = 2; }
        __syncthreads();
        break;
      }
      if (s_step < 0.0) {
        for (int a = tid; a < s; a += blockDim.x) mu[S[a]] = z[a];
        for (int j = tid; j < m; j += blockDim.x) if (inS[j] == 2) inS[j] = 0;   // a real step: rejected columns may come back
        __syncthreads();
        break;
      }
      if (tid == 0) {   // move towards z until the first coefficient hits zero, drop the zeros from the passive set
        int keep = 0;
        for (int a = 0; a < s; ++a) {
          const int j = S[a];
          double v = mu[j] + s_step * (z[a] - mu[j]);
          if (v <= 1e-300 || z[a] <= 0.0 && mu[j] / (mu[j] - z[a]) <= s_step) v = 0.0;
          mu[j] = v;
          if (v > 0.0) S[keep++] = j; else inS[j] = 0;
        }
        s_sz = keep;
      }
      __syncthreads();
      if (s_sz == 0) break;
    }
  }
  __syncthreads();
  // t = q + sum_i a_i p_i - c sum_j b_j n_j with a_i = sum_j mu_ij, b_j = sum_i mu_ij  (z reused as [a | b])
  for (int a = tid; a < r; a += blockDim.x) {
    double v = 0.0;
    if (a < P) for (int jj = 0; jj < N; ++jj) v += mu[a * N + jj];
    else for (int i = 0; i < P; ++i) v += mu[i * N + (a - P)];
    z[a] = v;
  }
  __syncthreads();
  for (int i = tid; i < d; i += blockDim.x) {
    double v = (double)q[i];
    for (int a = 0; a < P; ++a) v += z[a] * (double)base[(size_t)widx[a] * d + i];
    for (int a = P; a < r; ++a) v -= c * z[a] * (double)base[(size_t)widx[a] * d + i];
    t_out[i] = v;
  }
  if (tid == 0) { ok[e] = 1; iters[e] = s_iter; }
}

}  // namespace
}  // namespace rl

using namespace rl;

extern "C" int rl_best_vectors(const void* E, int e_dtype, int64_t ld, int d, const int64_t* chunk_off, const int64_t* chunks,
                               int n_evals, int n_slots, const float* Q, float* best, int64_t* best_row, void* stream) {
  RL_REQUIRE(n_evals >= 0 && n_slots >= 1 && d >= 1 && ld >= d && (e_dtype == 0 || e_dtype == 1), RL_EINVAL, "rl_best_vectors: bad arguments");
  if (n_evals == 0) return RL_OK;
  RL_REQUIRE(E && chunk_off && chunks && Q && best && best_row, RL_EINVAL, "rl_best_vectors: null pointer");
  best_vectors_kernel<<<dim3(n_slots, n_evals), kFitThreads, 0, (cudaStream_t)stream>>>(
      e_dtype == 0 ? static_cast<const float*>(E) : nullptr, e_dtype == 1 ? E : nullptr, ld, d, chunk_off, chunks, n_slots, Q, best, best_row);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}

extern "C" int rl_adapter_targets(const float* best, const uint8_t* kind, int n_evals, int n_slots, int d, const float* Q, double alpha,
                                  double* T, int32_t* ok, int32_t* iters, void* stream) {
  RL_REQUIRE(n_evals >= 0 && n_slots >= 1 && n_slots <= kFitMaxR && d >= 1 && alpha >= 0.0, RL_EINVAL,
             "rl_adapter_targets: bad arguments (at most %d retrieved chunks per eval)", kFitMaxR);
  if (n_evals == 0) return RL_OK;
  RL_REQUIRE(best && kind && Q && T && ok && iters, RL_EINVAL, "rl_adapter_targets: null pointer");
  const size_t smem = (size_t)(2 * kFitMaxR * kFitMaxR + kFitMaxR + 2 * kFitMaxM + 2 * kFitMaxR) * sizeof(double) +
                      (size_t)2 * kFitMaxR * sizeof(int) + kFitMaxM + 64;
  RL_CUDA_CHECK(cudaFuncSetAttribute(adapter_targets_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  adapter_targets_kernel<<<n_evals, kFitThreads, smem, (cudaStream_t)stream>>>(best, kind, n_slots, d, Q, alpha, T, ok, iters);
  RL_CUDA_CHECK(cudaGetLastError());
  return RL_OK;
}
