// Probe: read bandwidth of an HBM-resident buffer vs an L2-resident buffer with LDG.128 streaming
// loads (persistent grid).  Guides the choice between stationary and streamed query tiles.
#include <cstdio>
#include <cuda_runtime.h>
__global__ void __launch_bounds__(512) rd(const float4* __restrict__ p, size_t n, int reps, float* out) {
  float acc = 0.f;
  for (int r = 0; r < reps; ++r)
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
      float4 v = __ldg(p + i);
      acc += v.x + v.y + v.z + v.w;
    }
  if (acc == 1.2345f) *out = acc;
}
int main() {
  float* out; cudaMalloc(&out, 4);
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  // 8 .. 32 MiB stay resident in an H100's 50 MB L2; 4 GiB streams from HBM
  for (size_t mb : {8, 16, 32, 4096}) {
    size_t bytes = mb << 20; float4* p; cudaMalloc(&p, bytes); cudaMemset(p, 0, bytes);
    int reps = mb <= 32 ? 200 : 4;
    for (int grid : {sms, 2 * sms, 4 * sms}) {
      cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
      rd<<<grid, 512>>>(p, bytes / 16, 2, out);
      cudaEventRecord(a); rd<<<grid, 512>>>(p, bytes / 16, reps, out); cudaEventRecord(b); cudaEventSynchronize(b);
      float ms; cudaEventElapsedTime(&ms, a, b);
      printf("buffer %5zu MiB grid %4d: %.1f GB/s\n", mb, grid, (double)bytes * reps / ms / 1e6);
    }
    cudaFree(p);
  }
  return 0;
}
