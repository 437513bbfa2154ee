// L2 / HBM gather-bandwidth microbenchmark (evidence for DESIGN.md: the SpMM's X-row gathers
// are bound by L2->SM throughput).  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o l2mb l2_microbench.cu
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>

__global__ void stream_read(const float4* __restrict__ p, size_t n4, int reps, float* sink) {
  float acc = 0.f;
  for (int r = 0; r < reps; ++r)
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
      float4 v = __ldg(p + i);
      acc += v.x + v.y + v.z + v.w;
    }
  if (acc == 123.456f) *sink = acc;
}

// each group of LPR lanes gathers one row of ROWB bytes per index; U independent rows in flight
template <int ROWB, int U>
__global__ void gather_rows(const float* __restrict__ tab, const int* __restrict__ idx, size_t n_idx, float* sink) {
  constexpr int LPR = ROWB / 16;
  constexpr int GPW = 32 / LPR;
  const int lane = threadIdx.x & 31, sub = lane / LPR, cl = lane % LPR;
  const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  float acc = 0.f;
  for (size_t base = warp * GPW * U; base + GPW * U <= n_idx; base += nwarps * GPW * U) {
    float4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int r = __ldg(idx + base + u * GPW + sub);
      v[u] = __ldg(reinterpret_cast<const float4*>(tab + (size_t)r * (ROWB / 4)) + cl);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) acc += v[u].x + v[u].y + v[u].z + v[u].w;
  }
  if (acc == 123.456f) *sink = acc;
}


// the same gather through the TMA unit: every lane issues one cp.async.bulk of a whole row into the warp's
// shared-memory ring (ST stages of 32 rows); completion by mbarrier transaction count; the rows are then read
// back from shared memory (ld.shared.v4) like an SpMM would.
template <int ROWB, int ST>
__global__ void __launch_bounds__(256) gather_rows_bulk(const float* __restrict__ tab, const int* __restrict__ idx, size_t n_idx, float* sink) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  constexpr int WARPS = 8;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned char* ring = smem_raw + (size_t)w * ST * 32 * ROWB;
  __shared__ unsigned long long bars[WARPS][ST];
  if (lane == 0)
    for (int s = 0; s < ST; ++s) {
      unsigned a = (unsigned)__cvta_generic_to_shared(&bars[w][s]);
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(a));
    }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncwarp();
  const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  float acc = 0.f;
  size_t n_it = 0;
  for (size_t base = warp * 32; base + 32 <= n_idx; base += nwarps * 32) ++n_it;
  auto issue = [&](size_t it) {
    const int s = (int)(it % ST);
    const size_t base = (warp + it * nwarps) * 32;
    const unsigned bar = (unsigned)__cvta_generic_to_shared(&bars[w][s]);
    if (lane == 0) asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(32 * ROWB) : "memory");
    __syncwarp();
    const int r = __ldg(idx + base + lane);
    const unsigned dst = (unsigned)__cvta_generic_to_shared(ring + ((size_t)s * 32 + lane) * ROWB);
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(tab + (size_t)r * (ROWB / 4)), "r"(ROWB), "r"(bar)
                 : "memory");
  };
  for (size_t it = 0; it < (size_t)(ST - 1) && it < n_it; ++it) issue(it);
  for (size_t it = 0; it < n_it; ++it) {
    if (it + ST - 1 < n_it) issue(it + ST - 1);
    const int s = (int)(it % ST);
    const unsigned bar = (unsigned)__cvta_generic_to_shared(&bars[w][s]);
    const unsigned parity = (unsigned)((it / ST) & 1);
    asm volatile(
        "{\n\t.reg .pred P1;\n\tWAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
        "@P1 bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}" ::"r"(bar),
        "r"(parity)
        : "memory");
    // read the stage back: lane l reads 16 bytes of every row (the SpMM's lane-group mapping reads as much)
    const float4* st = reinterpret_cast<const float4*>(ring + (size_t)s * 32 * ROWB);
#pragma unroll 8
    for (int k = lane; k < 32 * ROWB / 16; k += 32) {
      const float4 v = st[k];
      acc += v.x + v.y + v.z + v.w;
    }
    __syncwarp();
  }
  if (acc == 123.456f) *sink = acc;
}

template <typename F>
float time_ms(F f, int iters) {
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  f();
  cudaDeviceSynchronize();
  cudaEventRecord(a);
  for (int i = 0; i < iters; ++i) f();
  cudaEventRecord(b);
  cudaEventSynchronize(b);
  float ms;
  cudaEventElapsedTime(&ms, a, b);
  return ms / iters;
}

int main() {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  float* sink;
  cudaMalloc(&sink, 4);
  printf("SMs %d\n", sms);
  for (size_t mb : {8, 16, 32, 64, 96, 256, 1024}) {
    size_t bytes = mb << 20;
    float4* p;
    cudaMalloc(&p, bytes);
    cudaMemset(p, 0, bytes);
    int reps = mb <= 96 ? 8 : 1;
    float ms = time_ms([&] { stream_read<<<sms * 8, 256>>>(p, bytes / 16, reps, sink); }, 10);
    printf("stream_read %5zu MB x%d: %8.1f GB/s\n", mb, reps, bytes * (double)reps / ms / 1e6);
    cudaFree(p);
  }
  const size_t n_idx = 1 << 22;
  for (size_t rows : {38048, 69716, 262144, 1048576, 8388608}) {
    std::vector<int> h(n_idx);
    unsigned s = 12345;
    for (size_t i = 0; i < n_idx; ++i) {
      s = s * 1664525u + 1013904223u;
      h[i] = (int)((s >> 8) % rows);
    }
    int* idx;
    cudaMalloc(&idx, n_idx * 4);
    cudaMemcpy(idx, h.data(), n_idx * 4, cudaMemcpyHostToDevice);
    float* tab;
    cudaMalloc(&tab, rows * 512);
    cudaMemset(tab, 0, rows * 512);
#define RUN(ROWB, U, BLK)                                                                                   \
  {                                                                                                         \
    float ms = time_ms([&] { gather_rows<ROWB, U><<<sms * BLK, 256>>>(tab, idx, n_idx, sink); }, 10);       \
    printf("gather rows=%8zu rowB=%3d U=%d blk/SM=%d table=%7.1f MB: %8.1f GB/s\n", rows, ROWB, U, BLK,     \
           rows * (double)ROWB / 1e6, n_idx * (double)ROWB / ms / 1e6);                                     \
  }
    RUN(256, 4, 8)
    RUN(256, 8, 8)
    RUN(256, 8, 4)
    RUN(128, 8, 8)
    RUN(512, 4, 8)
    RUN(512, 8, 8)
#define RUNB(ROWB, ST, BLK)                                                                                         \
  {                                                                                                                 \
    const size_t smem = (size_t)8 * ST * 32 * ROWB;                                                                 \
    cudaFuncSetAttribute(gather_rows_bulk<ROWB, ST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);       \
    float ms = time_ms([&] { gather_rows_bulk<ROWB, ST><<<sms * BLK, 256, smem>>>(tab, idx, n_idx, sink); }, 10);   \
    printf("bulk   rows=%8zu rowB=%3d stages=%d blk/SM=%d smem/blk=%3zu KB: %8.1f GB/s  (%s)\n", rows, ROWB, ST, BLK, smem >> 10, \
           n_idx * (double)ROWB / ms / 1e6, cudaGetErrorString(cudaGetLastError()));                                \
  }
    if (rows <= 262144) {
      RUNB(256, 2, 3)
      RUNB(256, 3, 2)
      RUNB(256, 2, 1)
      RUNB(256, 3, 1)
    }
    cudaFree(idx);
    cudaFree(tab);
  }
  return 0;
}
