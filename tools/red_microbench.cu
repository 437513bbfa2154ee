// How fast can the L2 absorb red.global.add.v4.f32 row updates (256 B rows, random rows of a 17.8 MB
// table)?  Decides whether the row-sparse backward product should push (scatter) instead of pull.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o red_mb red_microbench.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
__global__ void __launch_bounds__(256) push_rows(float* Y, int n_rows, int updates_per_group, uint32_t seed) {
  const int lane = threadIdx.x & 31, gl = lane & 7;
  const uint32_t gid = (blockIdx.x * blockDim.x + threadIdx.x) >> 3;
  uint32_t s = gid * 2654435761u + seed;
  const float4 v = make_float4(1e-3f, 2e-3f, 3e-3f, 4e-3f);
  for (int k = 0; k < updates_per_group; ++k) {
    s = s * 1664525u + 1013904223u;
    const uint32_t row = (uint32_t)(((uint64_t)s * (uint64_t)n_rows) >> 32);
    float* p = Y + (size_t)row * 64 + gl * 4;
    atomicAdd(reinterpret_cast<float4*>(p), v);
    atomicAdd(reinterpret_cast<float4*>(p + 32), v);
  }
}
__global__ void __launch_bounds__(256) store_rows(float* Y, int n_rows, int updates_per_group, uint32_t seed) {
  const int lane = threadIdx.x & 31, gl = lane & 7;
  const uint32_t gid = (blockIdx.x * blockDim.x + threadIdx.x) >> 3;
  uint32_t s = gid * 2654435761u + seed;
  const float4 v = make_float4(1e-3f, 2e-3f, 3e-3f, 4e-3f);
  for (int k = 0; k < updates_per_group; ++k) {
    s = s * 1664525u + 1013904223u;
    const uint32_t row = (uint32_t)(((uint64_t)s * (uint64_t)n_rows) >> 32);
    float* p = Y + (size_t)row * 64 + gl * 4;
    *reinterpret_cast<float4*>(p) = v;
    *reinterpret_cast<float4*>(p + 32) = v;
  }
}
int main() {
  const int n_rows = 69716;
  float* Y;
  cudaMalloc(&Y, (size_t)n_rows * 64 * 4);
  cudaMemset(Y, 0, (size_t)n_rows * 64 * 4);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  for (int upd : {8, 32, 128}) {
    for (int blocks : {sms * 2, sms * 8}) {
      const long long groups = (long long)blocks * 256 / 8;
      for (int kind = 0; kind < 2; ++kind) {
        for (int w = 0; w < 2; ++w) (kind ? store_rows : push_rows)<<<blocks, 256>>>(Y, n_rows, upd, 7u);
        cudaEventRecord(e0);
        const int reps = 10;
        for (int r = 0; r < reps; ++r) (kind ? store_rows : push_rows)<<<blocks, 256>>>(Y, n_rows, upd, 11u + r);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms;
        cudaEventElapsedTime(&ms, e0, e1);
        const double rows = (double)groups * upd;
        printf("%s blocks=%4d upd/group=%3d: %8.0f row updates in %7.2f us -> %6.2f TB/s (%.1f G rows/s)\n", kind ? "st.v4 " : "red.v4", blocks, upd,
               rows, ms * 1000 / reps, rows * 256 / (ms / reps * 1e-3) / 1e12, rows / (ms / reps * 1e-3) / 1e9);
      }
    }
  }
  printf("last error: %s\n", cudaGetErrorString(cudaDeviceSynchronize()));
  return 0;
}
