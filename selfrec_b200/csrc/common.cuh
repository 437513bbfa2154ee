// Shared helpers for the selfrec_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include <functional>
#include <utility>
#include "selfrec_b200.h"

#define SRB_FULL_MASK 0xffffffffu

namespace srb {

void set_error(const char* fmt, ...);
extern std::atomic<long long> g_launches;

inline int check_cuda(cudaError_t e, const char* what) {
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return SRB_ERR_CUDA;
  }
  return SRB_OK;
}

// Call after every kernel launch: counts it and surfaces launch-configuration errors.
inline int post_launch(const char* what) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return check_cuda(cudaPeekAtLastError(), what);
}

// Programmatic dependent launch (PDL).  srb_train_step launches its kernels with programmatic stream serialisation
// (unless SRB_PDL=0): a kernel may then be scheduled while its predecessor on the stream still drains, so its launch
// latency and CTA ramp-up overlap that tail.  Every kernel launched through launch_kernel() therefore calls pdl_wait()
// before its first global access (read or write) of anything an earlier kernel touches, and pdl_trigger() once it runs
// (the dependent is released only when every CTA of the grid has triggered or exited, i.e. after the last wave is
// resident).  Outside PDL launches both instructions are no-ops.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

bool pdl_active();  // true while srb_train_step enqueues its kernels with PDL on this thread (engine.cu)

template <typename... KArgs, typename... Args>
inline int launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, const char* what,
                         Args&&... args) {
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_active() ? 1 : 0;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return check_cuda(e, what);
}

#define SRB_REQUIRE(cond, ...)            \
  do {                                    \
    if (!(cond)) {                        \
      srb::set_error(__VA_ARGS__);        \
      return SRB_ERR_ARG;                 \
    }                                     \
  } while (0)

#define SRB_TRY(expr)                     \
  do {                                    \
    int _rc = (expr);                     \
    if (_rc != SRB_OK) return _rc;        \
  } while (0)

int sm_count();
long long l2_bytes();  // L2 size of the current device

// sparse-row scatter with several (src, rows) segments in one launch (bpr.cu)
struct ScatterSeg {
  const float* src;     // [n, d] compact rows
  const int32_t* rows;  // [n] destination row ids
  const int32_t* n_dev; // optional device count
  int32_t n;            // capacity / host count
  int32_t row_off;
  float scale;
  int32_t mod, rem;        // optional filter (mod > 0; cyclic row ownership): only rows with row % mod == rem, stored at row / mod
  int32_t item_min;        // optional (> 0): rows[r] >= item_min are items, stored at rows[r] - item_min + item_off, unfiltered
  int32_t item_off;
};
struct ScatterSegs {
  int count;
  ScatterSeg s[16];
};
int scatter_segments(float* dst, int d, const ScatterSegs& segs, cudaStream_t st);

// The backward seed tables of a graph model's step (engine.cu, both training steps).  LightGCN, XSimGCL: F and G;
// SimGCL: F; SGL: F of the encoders on adj_view[0], adj_view[1], adj.  SeedRows places them in a step's layout.
struct SeedRows {
  int32_t user_off[3], item_off[3];  // row of user / item 0 in table t (ScatterSeg.row_off)
  int32_t user_mod, user_rem;        // cyclic user ownership (ScatterSeg.mod / rem), or 0
  int32_t item_min;                  // > 0: SGL's cat rows from item_min on are items (ScatterSeg.item_min), placed at
                                     // item_off[t]; 0: cat rows are table rows of one [N, d] table per t
};
struct SeedGrads {  // a batch's compact loss gradients, [cap, d] per batch list
  const int32_t* batch;              // SRB_BATCH_HEADER counts, then the lists u | i | j | unique u | unique i
  int cap, d;
  const float *emb, *l2;             // BPR and LightGCN's L2 term on E0: [3][cap, d] at u, i, j
  const float *nce_u[2], *nce_i[2];  // InfoNCE views 1, 2 at the unique users / items (SGL: nce_u at cat)
  const int32_t *cat, *n_cat;        // SGL: table rows of the unique users, then of the unique items
};
// Which gradient enters which table, with what scale (one scatter); returns the level where G enters, or -1 (run_chain)
int seed_segments(int model, int n_layers, int layer_cl, const SeedGrads& g, const SeedRows& r, ScatterSegs& segs);
// First kernel of a graph model's step (engine.cu): Adam's bias corrections, words[0, n_words) cleared, and the batch rows
// of the first n_seed seed tables cleared on layout r
int step_begin(int32_t* step, float* scalars, double lr, double b1, double b2, int32_t* words, int n_words, const int32_t* batch, int cap,
               int d, float* seed, int n_seed, const SeedRows& r, cudaStream_t st);

// The loss stage of both training steps (engine.cu), on [rows, d] tables: the step's output, the raw E0 (LightGCN's L2
// term), view 1 (XSimGCL: the CL view) and view 2.
struct LossRows {
  const int32_t* batch;              // SRB_BATCH_HEADER counts: b, unique users, unique items (then seed_segments' lists)
  const int32_t *u, *i, *j;          // BPR: table rows u, item_off + i, item_off + j
  int32_t item_off;
  const int32_t *uq_u, *uq_i;        // InfoNCE: table rows uq_off[0] + unique user, uq_off[1] + unique item
  int32_t uq_off[2];
  const int32_t *cat, *n_cat;        // SGL's one InfoNCE problem: table rows of the unique users, then of the unique items
  const int32_t* cat_id;             // the same entries as ids u | U + i (SeedGrads.cat)
};
struct LossBufs {
  float *g_emb, *g_l2;               // [3][cap, d]
  float* g_nce;                      // InfoNCE gradients: view v of problem p at g_nce + (2p + v) * nce_plane; SGL's one
  size_t nce_plane;                  // problem of 2 cap rows: view v at g_nce + 2v * cap * d
  float *bpr_scratch, *bpr_losses, *nce_losses;
  void* nce_ws;
  int64_t nce_ws_bytes;
  float* losses;                     // [4]
};
struct ForkRes;  // engine.cu: with one, BPR + L2 run on its side stream beside the InfoNCE
// BPR + L2, the model's InfoNCE (before_nce, if set, is enqueued on st just before it) and the step's four losses (BPR,
// L2, cl_rate x the InfoNCE losses, total) into o.losses; g gets the gradients where they were written (seed_segments)
int step_losses(int model, float reg, float l2_div, float tau, float cl_rate, int d, int cap, const float* out, const float* e0,
                const float* v1, const float* v2, const LossRows& r, const LossBufs& o, ForkRes* fork,
                const std::function<int()>& before_nce, SeedGrads& g, cudaStream_t st);

// Adam step counter + bias corrections in double, like torch's Python floats (one thread)
__device__ __forceinline__ void adam_prepare(int32_t* step, float* scalars, double lr, double b1, double b2) {
  const int t = *step + 1;
  *step = t;
  const double bc1 = 1.0 - pow(b1, (double)t);
  const double bc2 = 1.0 - pow(b2, (double)t);
  scalars[0] = (float)(lr / bc1);
  scalars[1] = (float)sqrt(bc2);
}

// One Adam element, rounded as torch.optim.Adam's CUDA kernels round it (w1 = 1 - beta1, w2 = 1 - beta2):
//   m.lerp_(g, w1)                      m = fma(w1, g - m, m)
//   v.mul_(b2).addcmul_(g, g, w2)       v = fma(w2, g * g, v * b2), both products rounded first
//   p.addcdiv_(m, denom, -step_size)    p = fma(-step_size, m / denom, p), denom = sqrt(v) / bc2_sqrt + eps
// Round-to-nearest intrinsics pin every rounding: left to contraction, the compiler folded v * b2 into an fma (v off
// torch's in a quarter of the elements) and fused the last multiply-subtract in some lanes of a kernel but not others.
__device__ __forceinline__ void adam_elem(float& p, float& m, float& v, float g, float step_size, float bc2_sqrt, float w1,
                                          float b2, float w2, float eps) {
  m = __fmaf_rn(w1, __fsub_rn(g, m), m);
  v = __fmaf_rn(w2, __fmul_rn(g, g), __fmul_rn(v, b2));
  const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bc2_sqrt), eps);
  p = __fmaf_rn(-step_size, __fdiv_rn(m, denom), p);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(SRB_FULL_MASK, v, o);
  return v;
}

__device__ __forceinline__ float4 ldg4(const float* p) {
  return __ldg(reinterpret_cast<const float4*>(p));
}

__device__ __forceinline__ void st4(float* p, const float4& v) {
  *reinterpret_cast<float4*>(p) = v;
}

__device__ __forceinline__ float4 f4_zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }

__device__ __forceinline__ float4 f4_fma(float a, const float4& x, const float4& acc) {
  return make_float4(fmaf(a, x.x, acc.x), fmaf(a, x.y, acc.y), fmaf(a, x.z, acc.z),
                     fmaf(a, x.w, acc.w));
}

__device__ __forceinline__ float4 f4_add(const float4& a, const float4& b) {
  return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
}

__device__ __forceinline__ float4 f4_scale(float s, const float4& a) {
  return make_float4(s * a.x, s * a.y, s * a.z, s * a.w);
}

__device__ __forceinline__ float f4_dot(const float4& a, const float4& b) {
  return fmaf(a.w, b.w, fmaf(a.z, b.z, fmaf(a.y, b.y, a.x * b.x)));
}

__device__ __forceinline__ float sgnf(float x) {
  return (x > 0.f) ? 1.f : ((x < 0.f) ? -1.f : 0.f);
}

// Philox4x32-10 (Salmon et al. 2011): counter-based generator for the perf-mode noise.
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
    uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0;
    key.y += W1;
  }
  return ctr;
}

__device__ __forceinline__ float u32_to_unit(uint32_t x) {
  return (float)(x >> 8) * (1.0f / 16777216.0f);  // [0, 1) with 24 random bits
}

}  // namespace srb
