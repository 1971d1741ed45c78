// Interface of the tensor-core (wgmma) scan (RL_ALGO_TCGEN05), see scan_wgmma.cu.
#pragma once
#include "scan_common.cuh"

namespace rl {

bool wgmma_scan_supported(const rl_scan_params* p);
size_t wgmma_qimg_bytes(const rl_scan_params* p);
// Builds the fp16, pre-swizzled shared-memory image of the (scaled) query batch.
int wgmma_prepare_queries(const rl_scan_params* p, const float* q_inv_norm, float* q_scale, void* qimg,
                          cudaStream_t stream);
int launch_scan_wgmma(const ScanArgs& a, const rl_scan_params* p, const float* q_scale, const void* qimg,
                      int sm_count, cudaStream_t stream);

}  // namespace rl
