// Arguments shared by the three scan kernels (fp32 CUDA-core, tensor-core wgmma and L1) and their epilogues.
#pragma once
#include "common.cuh"

namespace rl {

struct ScanArgs {
  const float* E;            // [n_rows, ld]
  const float* inv_norm;     // [n_rows]
  const float* sq_norm;      // [n_rows]
  const uint8_t* row_allowed;  // [n_rows] or null
  const uint8_t* row_alive;    // [n_rows] or null: tombstones only (read when cnt_all is set)
  int32_t* cnt_all;            // [B] or null: rows passing the threshold that row_allowed masks out
  const float* Q;            // [B, d] float32 (fp32 scan)
  const float* q_inv_norm;   // [B]
  const float* thr;          // [B] emission thresholds (EMIT mode)
  float* dump;               // [B, n_sample_rows] (DUMP mode)
  Cand* cand;                // [B, cap]
  int32_t* cand_cnt;         // [B]
  int32_t* ghist;            // [B, kHistBins] emitted-candidate histogram (online threshold refinement)
  const float* eps;          // [B] error bound of the approximate key
  const float* hist_inv_w;   // [B] 1 / histogram bin width (from the select kernel)
  int32_t sel_count;         // #vectors at/above an edge that make it a valid threshold
  int64_t n_rows, ld, n_sample_rows;
  int64_t n_mode_blocks;     // number of blocks this launch covers
  int32_t d, B, metric, S, cap;
  int32_t dump_mode;         // 1: sample blocks -> dump, 0: remaining blocks -> emit
};

__device__ __forceinline__ int64_t mode_block_index(const ScanArgs& a, int64_t ord) {
  return a.dump_mode ? ord * a.S : main_block_index(ord, a.S);
}

__device__ __forceinline__ void emit_candidate(const ScanArgs& a, int col, float key, int32_t row) {
  const int slot = atomicAdd(a.cand_cnt + col, 1);
  if (slot < a.cap) a.cand[(size_t)col * a.cap + slot] = Cand{key, row};
}

int launch_scan_fp32(const ScanArgs& a, cudaStream_t stream);
// RL_METRIC_L1 (scan_l1.cu): float32 or float16 rows (e_f16), key = -sum |e - q|.
int launch_scan_l1(const ScanArgs& a, bool e_f16, cudaStream_t stream);

}  // namespace rl
