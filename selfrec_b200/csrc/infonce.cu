// (iii) Fused InfoNCE forward/backward (CUDA-core fp32 tile version).
//
// Replaces InfoNCE(view1[idx], view2[idx], temperature) util/loss_torch.py:35-50
//   view = F.normalize(view, dim=1); S = view1 @ view2.T / tau;
//   loss = -mean(diag(log_softmax(S, dim=1)))
// as called by XSimGCL.py:45-50, SimGCL.py:43-50, SGL.py:115-125, plus its autograd
// backward.  The n x n logit matrix is produced tile by tile (64 x 64) in registers /
// shared memory and never written to HBM; the backward pass recomputes it (flash-style).
//
//   prep    gather rows, L2-normalise, store row-major and k-major copies, S_ii
//   lse     per (row block, column split): partial row max / sum-exp        (2 n^2 d flop)
//   grad    per (row block, column split): G = (softmax(S) - I) * w/(n tau);
//           dV1 += G V2 (registers, one atomic pass), dV2 += G^T V1 (red.v4 per tile)
//                                                                            (6 n^2 d flop)
//           (d = 256: nce_grad_wide_kernel, the column tile streamed in 128-wide halves)
//   finish  back through F.normalize, loss = mean(lse - S_ii)
//
// The same kernels, with BSM = true (infonce_tc.cuh), replace batch_softmax_loss(user_emb, item_emb, temperature)
// util/loss_torch.py:25-32 (SSL4Rec.py:33; CL4SRec imports it): only the per-row loss and a per-row gradient factor
// differ.
#include "common.cuh"
#include "infonce_tc.cuh"

namespace srb {

constexpr int NCE_T = 64;       // tile edge
constexpr int NCE_MAX_SPLITS = 8;

struct NceProblem {
  const float* table1;
  const float* table2;
  int32_t row_off1, row_off2;
  float scale1, scale2;
  const int32_t* idx;
  const int32_t* n_dev;
  int32_t n;
  float weight;
  float* g1;
  float* g2;
  float* loss;
  // workspace slices
  float* V1;   // [NP][D] normalised rows
  float* V2;
  float* V1T;  // [D][NP]
  float* V2T;
  float* inv1;  // [NP] 1/max(||v||, 1e-12)
  float* inv2;
  float* diag;  // [NP] S_ii
  float* part_m;  // [SPLITS][NP]
  float* part_l;
  float* dV1;  // [NP][D]
  float* dV2;
  float* loss_acc;  // [1]
  float* lse;       // [NP] (tensor-core path)
};

struct NceArgs {
  int32_t n_problems;
  int32_t np;  // padded capacity (multiple of 64)
  int32_t splits;
  int32_t b_cos;
  float inv_tau;
  NceProblem p[4];
};

__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

__device__ __forceinline__ int nce_n(const NceProblem& p) { return p.n_dev ? min(*p.n_dev, p.n) : p.n; }

template <int D>
__global__ void __launch_bounds__(256) nce_prep_kernel(const NceArgs a) {
  pdl_wait();
  pdl_trigger();
  const NceProblem& p = a.p[blockIdx.y];
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= a.np) return;
  const int n = nce_n(p);
  if (blockIdx.x == 0 && threadIdx.x == 0) *p.loss_acc = 0.f;
  constexpr int Q = (D + 127) / 128;
  float4 v1[Q], v2[Q];
  float s1 = 0.f, s2 = 0.f, s12 = 0.f;
  if (i < n) {
    const int r = p.idx[i];
#pragma unroll
    for (int q = 0; q < Q; ++q) {
      const int c = lane * 4 + q * 128;
      v1[q] = (c < D) ? f4_scale(p.scale1, ldg4(p.table1 + (size_t)(r + p.row_off1) * D + c)) : f4_zero();
      v2[q] = (c < D) ? f4_scale(p.scale2, ldg4(p.table2 + (size_t)(r + p.row_off2) * D + c)) : f4_zero();
      s1 += f4_dot(v1[q], v1[q]);
      s2 += f4_dot(v2[q], v2[q]);
    }
  } else {
#pragma unroll
    for (int q = 0; q < Q; ++q) v1[q] = f4_zero(), v2[q] = f4_zero();
  }
  s1 = warp_sum(s1);
  s2 = warp_sum(s2);
  float i1 = 1.f, i2 = 1.f;
  if (a.b_cos) {
    i1 = 1.f / fmaxf(sqrtf(s1), 1e-12f);
    i2 = 1.f / fmaxf(sqrtf(s2), 1e-12f);
  }
#pragma unroll
  for (int q = 0; q < Q; ++q) {
    const int c = lane * 4 + q * 128;
    if (a.b_cos) {
      // F.normalize divides (x / max(norm, eps)); keep the division for rounding parity
      const float n1 = fmaxf(sqrtf(s1), 1e-12f), n2 = fmaxf(sqrtf(s2), 1e-12f);
      v1[q] = make_float4(v1[q].x / n1, v1[q].y / n1, v1[q].z / n1, v1[q].w / n1);
      v2[q] = make_float4(v2[q].x / n2, v2[q].y / n2, v2[q].z / n2, v2[q].w / n2);
    }
    s12 += f4_dot(v1[q], v2[q]);
    if (c < D) {
      st4(p.V1 + (size_t)i * D + c, v1[q]);
      st4(p.V2 + (size_t)i * D + c, v2[q]);
      st4(p.dV1 + (size_t)i * D + c, f4_zero());
      st4(p.dV2 + (size_t)i * D + c, f4_zero());
      p.V1T[(size_t)(c + 0) * a.np + i] = v1[q].x;
      p.V1T[(size_t)(c + 1) * a.np + i] = v1[q].y;
      p.V1T[(size_t)(c + 2) * a.np + i] = v1[q].z;
      p.V1T[(size_t)(c + 3) * a.np + i] = v1[q].w;
      p.V2T[(size_t)(c + 0) * a.np + i] = v2[q].x;
      p.V2T[(size_t)(c + 1) * a.np + i] = v2[q].y;
      p.V2T[(size_t)(c + 2) * a.np + i] = v2[q].z;
      p.V2T[(size_t)(c + 3) * a.np + i] = v2[q].w;
    }
  }
  s12 = warp_sum(s12);
  if (lane == 0) {
    p.inv1[i] = i1;
    p.inv2[i] = i2;
    p.diag[i] = s12 * a.inv_tau;
  }
}

// Tensor-core pipeline (d = 64): gather + normalise 32 rows per CTA; besides the exact rows it writes the
// TF32 hi / lo parts (x = hi + lo, hi = rna_tf32(x); the tensor core truncates lo) of both views, row-major
// and transposed (through shared memory, so the transposed stores are 128-byte coalesced; columns in the
// nce_tperm order the tensor-core kernel expects), behind dV2:
//   hi: [V1 | V2 | V1^T | V2^T]   then lo: the same four
__global__ void __launch_bounds__(256) nce_prep_tc_kernel(const NceArgs a) {
  pdl_wait();
  pdl_trigger();
  constexpr int D = 64;
  __shared__ float t1[32][D + 1], t2[32][D + 1];
  const NceProblem& p = a.p[blockIdx.y];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int i0 = blockIdx.x * 32;
  const int n = nce_n(p);
  if (blockIdx.x == 0 && threadIdx.x == 0) *p.loss_acc = 0.f;
  const size_t nd = (size_t)a.np * D;
  float* hi = p.dV2 + nd;
  float* lo = hi + 4 * nd;
#pragma unroll 1
  for (int rr = 0; rr < 4; ++rr) {
    const int il = warp * 4 + rr, i = i0 + il;
    const int c = lane * 2;
    float2 v1 = make_float2(0.f, 0.f), v2 = make_float2(0.f, 0.f);
    if (i < n) {
      const int r = p.idx[i];
      v1 = *reinterpret_cast<const float2*>(p.table1 + (size_t)(r + p.row_off1) * D + c);
      v2 = *reinterpret_cast<const float2*>(p.table2 + (size_t)(r + p.row_off2) * D + c);
      v1.x *= p.scale1, v1.y *= p.scale1, v2.x *= p.scale2, v2.y *= p.scale2;
    }
    const float s1 = warp_sum(v1.x * v1.x + v1.y * v1.y);
    const float s2 = warp_sum(v2.x * v2.x + v2.y * v2.y);
    float i1 = 1.f, i2 = 1.f;
    if (a.b_cos) {  // F.normalize divides (x / max(norm, eps)); keep the division for rounding parity
      const float n1 = fmaxf(sqrtf(s1), 1e-12f), n2 = fmaxf(sqrtf(s2), 1e-12f);
      i1 = 1.f / n1, i2 = 1.f / n2;
      v1.x /= n1, v1.y /= n1, v2.x /= n2, v2.y /= n2;
    }
    const float s12 = warp_sum(v1.x * v2.x + v1.y * v2.y);
    const size_t o = (size_t)i * D + c;
    *reinterpret_cast<float2*>(p.V1 + o) = v1;
    *reinterpret_cast<float2*>(p.V2 + o) = v2;
    *reinterpret_cast<float2*>(p.dV1 + o) = make_float2(0.f, 0.f);
    *reinterpret_cast<float2*>(p.dV2 + o) = make_float2(0.f, 0.f);
    const float2 h1 = make_float2(tf32_rna(v1.x), tf32_rna(v1.y)), h2 = make_float2(tf32_rna(v2.x), tf32_rna(v2.y));
    *reinterpret_cast<float2*>(hi + o) = h1;
    *reinterpret_cast<float2*>(hi + nd + o) = h2;
    *reinterpret_cast<float2*>(lo + o) = make_float2(v1.x - h1.x, v1.y - h1.y);
    *reinterpret_cast<float2*>(lo + nd + o) = make_float2(v2.x - h2.x, v2.y - h2.y);
    t1[il][c] = v1.x, t1[il][c + 1] = v1.y;
    t2[il][c] = v2.x, t2[il][c + 1] = v2.y;
    if (lane == 0) {
      p.inv1[i] = i1;
      p.inv2[i] = i2;
      const float dg = s12 * a.inv_tau;
      p.diag[i] = dg;
      // softmax denominator l_i: its diagonal term from the exact S_ii here (the tensor-core S_ii is low by the
      // accumulator's truncation, ~2^-21 of a unit cosine, and at small tau this term is nearly all of l_i); pass A
      // adds the off-diagonal terms
      p.part_l[i] = expf(dg - a.inv_tau);
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < D * 32; e += 256) {
    const int dc = e >> 5, il = e & 31;
    const size_t o = (size_t)dc * a.np + i0 + nce_tperm(il);  // columns permuted within groups of 8 (infonce_tc.cuh)
    const float x1 = t1[il][dc], x2 = t2[il][dc];
    const float g1 = tf32_rna(x1), g2 = tf32_rna(x2);
    hi[2 * nd + o] = g1;
    hi[3 * nd + o] = g2;
    lo[2 * nd + o] = x1 - g1;
    lo[3 * nd + o] = x2 - g2;
  }
}

// cooperative copy of a [rows x 64] k-major slab (rows = D) from T[k][col0 .. col0+63]
template <int D>
__device__ __forceinline__ void load_kmajor(float (*dst)[NCE_T], const float* T, int np, int col0) {
  for (int e = threadIdx.x; e < D * (NCE_T / 4); e += blockDim.x) {
    const int k = e / (NCE_T / 4), c4 = e % (NCE_T / 4);
    *reinterpret_cast<float4*>(&dst[k][c4 * 4]) = *reinterpret_cast<const float4*>(T + (size_t)k * np + col0 + c4 * 4);
  }
}

// cooperative copy of 64 row-major rows [64][D]
template <int D>
__device__ __forceinline__ void load_rowmajor(float (*dst)[D], const float* V, int row0) {
  for (int e = threadIdx.x; e < NCE_T * (D / 4); e += blockDim.x) {
    const int r = e / (D / 4), c4 = e % (D / 4);
    *reinterpret_cast<float4*>(&dst[r][c4 * 4]) = *reinterpret_cast<const float4*>(V + (size_t)(row0 + r) * D + c4 * 4);
  }
}

// S micro-tile: rows ty*4+r, cols tx*4+c of (A^T B) over k = 0..D-1, k-major operands.
template <int D>
__device__ __forceinline__ void s_tile(const float (*AsT)[NCE_T], const float (*BsT)[NCE_T], int ty, int tx, float (&s)[4][4]) {
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) s[r][c] = 0.f;
#pragma unroll 8
  for (int k = 0; k < D; ++k) {
    const float4 av = *reinterpret_cast<const float4*>(&AsT[k][ty * 4]);
    const float4 bv = *reinterpret_cast<const float4*>(&BsT[k][tx * 4]);
    const float ar[4] = {av.x, av.y, av.z, av.w};
    const float bc[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) s[r][c] = fmaf(ar[r], bc[c], s[r][c]);
  }
}

template <int D>
struct NceLseSmem {
  float AsT[D][NCE_T];
  float BsT[D][NCE_T];
};

template <int D>
__global__ void __launch_bounds__(256) nce_lse_kernel(const NceArgs a) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ __align__(16) unsigned char smem_raw[];
  NceLseSmem<D>& sm = *reinterpret_cast<NceLseSmem<D>*>(smem_raw);
  const NceProblem& p = a.p[blockIdx.z];
  const int n = nce_n(p);
  const int i0 = blockIdx.x * NCE_T;
  if (i0 >= n) return;
  const int split = blockIdx.y;
  const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
  load_kmajor<D>(sm.AsT, p.V1T, a.np, i0);
  float m[4], l[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) m[r] = -INFINITY, l[r] = 0.f;
  const int ntiles = (n + NCE_T - 1) / NCE_T;
  const float L2E = 1.4426950408889634f;
  for (int jt = split; jt < ntiles; jt += a.splits) {
    const int j0 = jt * NCE_T;
    __syncthreads();
    load_kmajor<D>(sm.BsT, p.V2T, a.np, j0);
    __syncthreads();
    float s[4][4];
    s_tile<D>(sm.AsT, sm.BsT, ty, tx, s);
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      float tm = -INFINITY;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        s[r][c] = (j0 + tx * 4 + c < n) ? s[r][c] * a.inv_tau : -INFINITY;
        tm = fmaxf(tm, s[r][c]);
      }
      const float mn = fmaxf(m[r], tm);
      if (mn > -INFINITY) {
        float acc = 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c) acc += exp2f((s[r][c] - mn) * L2E);
        l[r] = l[r] * exp2f((m[r] - mn) * L2E) + acc;
        m[r] = mn;
      }
    }
  }
  // combine the 16 tx lanes that share a row (half-warp xor shuffles)
#pragma unroll
  for (int r = 0; r < 4; ++r) {
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {
      const float mo = __shfl_xor_sync(SRB_FULL_MASK, m[r], o);
      const float lo = __shfl_xor_sync(SRB_FULL_MASK, l[r], o);
      const float mn = fmaxf(m[r], mo);
      if (mn > -INFINITY) {
        l[r] = l[r] * exp2f((m[r] - mn) * L2E) + lo * exp2f((mo - mn) * L2E);
        m[r] = mn;
      }
    }
    if (tx == 0) {
      const int i = i0 + ty * 4 + r;
      p.part_m[(size_t)split * a.np + i] = m[r];
      p.part_l[(size_t)split * a.np + i] = l[r];
    }
  }
}

template <int D>
struct NceGradSmem {
  float AsT[D][NCE_T];
  float BsT[D][NCE_T];
  float Ar[NCE_T][D];
  float Br[NCE_T][D];
  float Gs[NCE_T][NCE_T];   // G[i][j]
  float GsT[NCE_T][NCE_T];  // G^T[j][i], float4 column index xor-swizzled with (j >> 2)
  float lse[NCE_T];
  float red[8];
};

// batch_softmax_loss: gscale times the row factor c_r of this thread's rows ty*4 + r (after sm.lse is written)
__device__ __forceinline__ void bsm_row_scales(const NceProblem& p, const float* lse, int i0, int ty, int n, float gscale,
                                               float (&gs)[4]) {
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int i = i0 + ty * 4 + r;
    gs[r] = (i < n) ? gscale * bsm_row_coef(lse[ty * 4 + r], p.diag[i]) : 0.f;
  }
}

template <int D, bool BSM>
__global__ void __launch_bounds__(256) nce_grad_kernel(const NceArgs a) {
  pdl_wait();
  pdl_trigger();
  constexpr int CW = D / 16;  // output columns per thread in the G V products
  extern __shared__ __align__(16) unsigned char smem_raw[];
  NceGradSmem<D>& sm = *reinterpret_cast<NceGradSmem<D>*>(smem_raw);
  const NceProblem& p = a.p[blockIdx.z];
  const int n = nce_n(p);
  const int i0 = blockIdx.x * NCE_T;
  if (i0 >= n) return;
  const int split = blockIdx.y;
  const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
  const float L2E = 1.4426950408889634f;
  load_kmajor<D>(sm.AsT, p.V1T, a.np, i0);
  load_rowmajor<D>(sm.Ar, p.V1, i0);
  if (threadIdx.x < NCE_T) {
    const int i = i0 + threadIdx.x;
    float M = -INFINITY;
    for (int s = 0; s < a.splits; ++s) M = fmaxf(M, p.part_m[(size_t)s * a.np + i]);
    float Lsum = 0.f;
    for (int s = 0; s < a.splits; ++s) {
      const float ms = p.part_m[(size_t)s * a.np + i];
      if (ms > -INFINITY) Lsum += p.part_l[(size_t)s * a.np + i] * exp2f((ms - M) * L2E);
    }
    const float lse = (i < n) ? M + logf(Lsum) : 0.f;
    sm.lse[threadIdx.x] = lse;
    // loss contribution (split 0 only): sum_i loss_i
    float contrib = (split == 0 && i < n) ? (BSM ? bsm_row_loss(lse, p.diag[i]) : lse - p.diag[i]) : 0.f;
    contrib = warp_sum(contrib);
    if ((threadIdx.x & 31) == 0) sm.red[threadIdx.x >> 5] = contrib;
  }
  __syncthreads();
  if (threadIdx.x == 0 && split == 0) atomicAdd(p.loss_acc, sm.red[0] + sm.red[1]);
  const float gscale = p.weight * a.inv_tau / (float)n;  // d loss / d S_ij = (P_ij - delta_ij) / n
  float gs[4];  // BSM: gscale * c_r
  if constexpr (BSM) bsm_row_scales(p, sm.lse, i0, ty, n, gscale, gs);
  float o1[4][CW];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int q = 0; q < CW; ++q) o1[r][q] = 0.f;
  const int ntiles = (n + NCE_T - 1) / NCE_T;
  for (int jt = split; jt < ntiles; jt += a.splits) {
    const int j0 = jt * NCE_T;
    __syncthreads();  // previous tile's readers of BsT/Br/Gs are done
    load_kmajor<D>(sm.BsT, p.V2T, a.np, j0);
    load_rowmajor<D>(sm.Br, p.V2, j0);
    __syncthreads();
    float s[4][4];
    s_tile<D>(sm.AsT, sm.BsT, ty, tx, s);
    // G = (exp(S - lse_i) - delta_ij) * gscale, zero outside the valid n x n block
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int i = i0 + ty * 4 + r;
      const float lse = sm.lse[ty * 4 + r];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int j = j0 + tx * 4 + c;
        float g = 0.f;
        if (i < n && j < n) {
          g = exp2f((s[r][c] * a.inv_tau - lse) * L2E);
          if (i == j) g -= 1.f;
          if constexpr (BSM) g *= gs[r];
          else g *= gscale;
        }
        s[r][c] = g;
      }
      *reinterpret_cast<float4*>(&sm.Gs[ty * 4 + r][tx * 4]) = make_float4(s[r][0], s[r][1], s[r][2], s[r][3]);
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int jl = tx * 4 + c;
      *reinterpret_cast<float4*>(&sm.GsT[jl][((ty ^ (jl >> 2)) & 15) * 4]) = make_float4(s[0][c], s[1][c], s[2][c], s[3][c]);
    }
    __syncthreads();
    // O1[i][c] += sum_j G[i][j] V2[j][c]   (A operand = G^T k-major, B operand = Br row-major)
#pragma unroll 4
    for (int j = 0; j < NCE_T; ++j) {
      const float4 av = *reinterpret_cast<const float4*>(&sm.GsT[j][((ty ^ (j >> 2)) & 15) * 4]);
      const float ar[4] = {av.x, av.y, av.z, av.w};
      float bq[CW];
#pragma unroll
      for (int q = 0; q < CW; ++q) bq[q] = sm.Br[j][tx * CW + q];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int q = 0; q < CW; ++q) o1[r][q] = fmaf(ar[r], bq[q], o1[r][q]);
    }
    // Q[j][c] = sum_i G[i][j] V1[i][c]  (A operand = Gs k-major over i, B operand = Ar)
    float qv[4][CW];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int q = 0; q < CW; ++q) qv[r][q] = 0.f;
#pragma unroll 4
    for (int i = 0; i < NCE_T; ++i) {
      const float4 av = *reinterpret_cast<const float4*>(&sm.Gs[i][ty * 4]);
      const float ar[4] = {av.x, av.y, av.z, av.w};
      float bq[CW];
#pragma unroll
      for (int q = 0; q < CW; ++q) bq[q] = sm.Ar[i][tx * CW + q];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int q = 0; q < CW; ++q) qv[r][q] = fmaf(ar[r], bq[q], qv[r][q]);
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int j = j0 + ty * 4 + r;
      if (j < n) {
#pragma unroll
        for (int q = 0; q < CW; ++q) atomicAdd(p.dV2 + (size_t)j * D + tx * CW + q, qv[r][q]);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int i = i0 + ty * 4 + r;
    if (i < n) {
#pragma unroll
      for (int q = 0; q < CW; ++q) atomicAdd(p.dV1 + (size_t)i * D + tx * CW + q, o1[r][q]);
    }
  }
}

// D = 256: NceGradSmem<256> would take 288 KB, over the 227 KB a CTA may opt into.  The CTA's own 64 rows stay
// resident (k-major and row-major, 128 KB) and every column tile is streamed in 128-wide halves: S accumulates over the
// two k-halves of V2^T in the k order of s_tile (so S matches nce_lse_kernel<256> bit for bit), then G V2 and G^T V1
// run over the two column halves of V2 and V1.  Per thread: o1 over both halves (2 x 4 x 8 registers), qv over one.
constexpr int NCE_WIDE_D = 256;
constexpr int NCE_WIDE_H = NCE_WIDE_D / 2;

struct NceGradWideSmem {
  float AsT[NCE_WIDE_D][NCE_T];  // own rows, k-major
  float Ar[NCE_T][NCE_WIDE_D];   // own rows, row-major
  float BsT[NCE_WIDE_H][NCE_T];  // one k-half of the column tile
  float Br[NCE_T][NCE_WIDE_H];   // one column half of the column tile
  float Gs[NCE_T][NCE_T];
  float GsT[NCE_T][NCE_T];  // float4 column index xor-swizzled with (j >> 2), as in nce_grad_kernel
  float lse[NCE_T];
  float red[8];
};

template <bool BSM>
__global__ void __launch_bounds__(256) nce_grad_wide_kernel(const NceArgs a) {
  pdl_wait();
  pdl_trigger();
  constexpr int D = NCE_WIDE_D, H = NCE_WIDE_H;
  constexpr int CW = H / 16;  // output columns per thread and half in the G V products
  extern __shared__ __align__(16) unsigned char smem_raw[];
  NceGradWideSmem& sm = *reinterpret_cast<NceGradWideSmem*>(smem_raw);
  const NceProblem& p = a.p[blockIdx.z];
  const int n = nce_n(p);
  const int i0 = blockIdx.x * NCE_T;
  if (i0 >= n) return;
  const int split = blockIdx.y;
  const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
  const float L2E = 1.4426950408889634f;
  load_kmajor<D>(sm.AsT, p.V1T, a.np, i0);
  load_rowmajor<D>(sm.Ar, p.V1, i0);
  if (threadIdx.x < NCE_T) {
    const int i = i0 + threadIdx.x;
    float M = -INFINITY;
    for (int s = 0; s < a.splits; ++s) M = fmaxf(M, p.part_m[(size_t)s * a.np + i]);
    float Lsum = 0.f;
    for (int s = 0; s < a.splits; ++s) {
      const float ms = p.part_m[(size_t)s * a.np + i];
      if (ms > -INFINITY) Lsum += p.part_l[(size_t)s * a.np + i] * exp2f((ms - M) * L2E);
    }
    const float lse = (i < n) ? M + logf(Lsum) : 0.f;
    sm.lse[threadIdx.x] = lse;
    float contrib = (split == 0 && i < n) ? (BSM ? bsm_row_loss(lse, p.diag[i]) : lse - p.diag[i]) : 0.f;
    contrib = warp_sum(contrib);
    if ((threadIdx.x & 31) == 0) sm.red[threadIdx.x >> 5] = contrib;
  }
  __syncthreads();
  if (threadIdx.x == 0 && split == 0) atomicAdd(p.loss_acc, sm.red[0] + sm.red[1]);
  const float gscale = p.weight * a.inv_tau / (float)n;
  float gs[4];  // BSM: gscale * c_r
  if constexpr (BSM) bsm_row_scales(p, sm.lse, i0, ty, n, gscale, gs);
  float o1[2][4][CW];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int q = 0; q < CW; ++q) o1[h][r][q] = 0.f;
  // one column half [h*H, h*H + H) of 64 row-major rows of V (row stride D)
  auto load_half = [&](float (*dst)[H], const float* V, int row0, int h) {
    for (int e = threadIdx.x; e < NCE_T * (H / 4); e += blockDim.x) {
      const int r = e / (H / 4), c4 = e % (H / 4);
      *reinterpret_cast<float4*>(&dst[r][c4 * 4]) = *reinterpret_cast<const float4*>(V + (size_t)(row0 + r) * D + h * H + c4 * 4);
    }
  };
  const int ntiles = (n + NCE_T - 1) / NCE_T;
  for (int jt = split; jt < ntiles; jt += a.splits) {
    const int j0 = jt * NCE_T;
    float s[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) s[r][c] = 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      __syncthreads();  // h = 0: the previous tile's readers of BsT / Br / Gs are done; h = 1: the readers of k-half 0
      load_kmajor<H>(sm.BsT, p.V2T + (size_t)h * H * a.np, a.np, j0);
      if (h == 1) load_half(sm.Br, p.V2, j0, 0);
      __syncthreads();
#pragma unroll 8
      for (int k = 0; k < H; ++k) {
        const float4 av = *reinterpret_cast<const float4*>(&sm.AsT[h * H + k][ty * 4]);
        const float4 bv = *reinterpret_cast<const float4*>(&sm.BsT[k][tx * 4]);
        const float ar[4] = {av.x, av.y, av.z, av.w};
        const float bc[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c) s[r][c] = fmaf(ar[r], bc[c], s[r][c]);
      }
    }
    // G = (exp(S - lse_i) - delta_ij) * gscale, zero outside the valid n x n block
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int i = i0 + ty * 4 + r;
      const float lse = sm.lse[ty * 4 + r];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int j = j0 + tx * 4 + c;
        float g = 0.f;
        if (i < n && j < n) {
          g = exp2f((s[r][c] * a.inv_tau - lse) * L2E);
          if (i == j) g -= 1.f;
          if constexpr (BSM) g *= gs[r];
          else g *= gscale;
        }
        s[r][c] = g;
      }
      *reinterpret_cast<float4*>(&sm.Gs[ty * 4 + r][tx * 4]) = make_float4(s[r][0], s[r][1], s[r][2], s[r][3]);
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int jl = tx * 4 + c;
      *reinterpret_cast<float4*>(&sm.GsT[jl][((ty ^ (jl >> 2)) & 15) * 4]) = make_float4(s[0][c], s[1][c], s[2][c], s[3][c]);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (h == 1) {
        __syncthreads();  // the readers of column half 0 are done
        load_half(sm.Br, p.V2, j0, 1);
      }
      __syncthreads();
      // O1[i][h*H + c] += sum_j G[i][j] V2[j][h*H + c]
#pragma unroll 4
      for (int j = 0; j < NCE_T; ++j) {
        const float4 av = *reinterpret_cast<const float4*>(&sm.GsT[j][((ty ^ (j >> 2)) & 15) * 4]);
        const float ar[4] = {av.x, av.y, av.z, av.w};
        float bq[CW];
#pragma unroll
        for (int q = 0; q < CW; ++q) bq[q] = sm.Br[j][tx * CW + q];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int q = 0; q < CW; ++q) o1[h][r][q] = fmaf(ar[r], bq[q], o1[h][r][q]);
      }
      // Q[j][h*H + c] = sum_i G[i][j] V1[i][h*H + c]
      float qv[4][CW];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int q = 0; q < CW; ++q) qv[r][q] = 0.f;
#pragma unroll 4
      for (int i = 0; i < NCE_T; ++i) {
        const float4 av = *reinterpret_cast<const float4*>(&sm.Gs[i][ty * 4]);
        const float ar[4] = {av.x, av.y, av.z, av.w};
        float bq[CW];
#pragma unroll
        for (int q = 0; q < CW; ++q) bq[q] = sm.Ar[i][h * H + tx * CW + q];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int q = 0; q < CW; ++q) qv[r][q] = fmaf(ar[r], bq[q], qv[r][q]);
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int j = j0 + ty * 4 + r;
        if (j < n) {
#pragma unroll
          for (int q = 0; q < CW; ++q) atomicAdd(p.dV2 + (size_t)j * D + h * H + tx * CW + q, qv[r][q]);
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int i = i0 + ty * 4 + r;
    if (i < n) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int q = 0; q < CW; ++q) atomicAdd(p.dV1 + (size_t)i * D + h * H + tx * CW + q, o1[h][r][q]);
    }
  }
}

template <int D>
__global__ void __launch_bounds__(256) nce_finish_kernel(const NceArgs a) {
  pdl_wait();
  pdl_trigger();
  const NceProblem& p = a.p[blockIdx.y];
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int n = nce_n(p);
  if (blockIdx.x == 0 && threadIdx.x == 0) *p.loss = (n > 0) ? *p.loss_acc / (float)n : 0.f;
  if (i >= n) return;
  constexpr int Q = (D + 127) / 128;
#pragma unroll 1
  for (int side = 0; side < 2; ++side) {
    const float* V = side ? p.V2 : p.V1;
    const float* dV = side ? p.dV2 : p.dV1;
    float* g = side ? p.g2 : p.g1;
    const float inv = side ? p.inv2[i] : p.inv1[i];
    float4 vh[Q], dv[Q];
    float dot = 0.f;
#pragma unroll
    for (int q = 0; q < Q; ++q) {
      const int c = lane * 4 + q * 128;
      vh[q] = (c < D) ? *reinterpret_cast<const float4*>(V + (size_t)i * D + c) : f4_zero();
      dv[q] = (c < D) ? *reinterpret_cast<const float4*>(dV + (size_t)i * D + c) : f4_zero();
      dot += f4_dot(vh[q], dv[q]);
    }
    dot = warp_sum(dot);
#pragma unroll
    for (int q = 0; q < Q; ++q) {
      const int c = lane * 4 + q * 128;
      if (c >= D) continue;
      float4 o = dv[q];
      if (a.b_cos) {
        // d/dv of v/||v||:  (dvh - vh * <vh, dvh>) / ||v||
        o = make_float4((dv[q].x - vh[q].x * dot) * inv, (dv[q].y - vh[q].y * dot) * inv, (dv[q].z - vh[q].z * dot) * inv,
                        (dv[q].w - vh[q].w * dot) * inv);
      }
      st4(g + (size_t)i * D + c, o);
    }
  }
}

static inline int64_t align_up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }
static inline int nce_np(int n) { return (int)align_up(n > 0 ? n : 1, 128); }  // 128: tile edge of the tensor-core path

static int64_t nce_problem_floats(int np, int d) {
  // V1 V2 V1T V2T dV1 dV2 + TF32 hi and lo parts of V1 V2 V1T V2T: 14 * np * d ; inv1 inv2 diag: 3 * np ;
  // part_m part_l: 2 * splits * np ; loss_acc (padded)
  return 14ll * np * d + 4ll * np + 2ll * NCE_MAX_SPLITS * np + 64;  // + lse[np]
}

// finish for the tensor-core path: pass A left dV1 unnormalised (sum_j exp(S_ij - 1/tau) v2_j) and the
// denominators l_i in part_l; dV1hat = w/(n tau l_i) dV1, both sides get the diagonal term
// (P_ii - 1) * w/(n tau) * vhat_other in exact fp32, then the same normalisation backward as nce_finish_kernel
// (BSM: w/(n tau) times c_i)
template <bool BSM>
__global__ void __launch_bounds__(256) nce_tc_finish_kernel(const NceArgs a) {
  pdl_wait();
  pdl_trigger();
  constexpr int D = 64;
  const NceProblem& p = a.p[blockIdx.y];
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int n = nce_n(p);
  if (blockIdx.x == 0 && threadIdx.x == 0) *p.loss = (n > 0) ? *p.loss_acc / (float)n : 0.f;
  if (i >= n) return;
  const float li = p.part_l[i];
  const float pii = expf(p.diag[i] - a.inv_tau) / li;
  float gs = p.weight * a.inv_tau / (float)n;
  if constexpr (BSM) gs *= pii / (pii + BSM_EPS);
  const float cd = (pii - 1.f) * gs;
  const float2 v1 = *reinterpret_cast<const float2*>(p.V1 + (size_t)i * D + lane * 2);
  const float2 v2 = *reinterpret_cast<const float2*>(p.V2 + (size_t)i * D + lane * 2);
#pragma unroll 1
  for (int side = 0; side < 2; ++side) {
    const float2 vh = side ? v2 : v1;
    const float2 vo = side ? v1 : v2;
    float2 dv = *reinterpret_cast<const float2*>((side ? p.dV2 : p.dV1) + (size_t)i * D + lane * 2);
    if (side == 0) dv.x *= gs / li, dv.y *= gs / li;
    dv.x = fmaf(cd, vo.x, dv.x);
    dv.y = fmaf(cd, vo.y, dv.y);
    const float dot = warp_sum(vh.x * dv.x + vh.y * dv.y);
    const float inv = side ? p.inv2[i] : p.inv1[i];
    float2 o = dv;
    if (a.b_cos) o = make_float2((dv.x - vh.x * dot) * inv, (dv.y - vh.y * dot) * inv);
    *reinterpret_cast<float2*>((side ? p.g2 : p.g1) + (size_t)i * D + lane * 2) = o;
  }
}

// tensor-core pipeline: prep (exact rows + TF32 hi/lo parts) -> pass A (LSE + view-1 gradient) -> pass B -> finish
template <bool BSM>
static int nce_launch_tc(const NceArgs& a, int n_problems, cudaStream_t st) {
  const int np = a.np;
  const int d = NT_D;
  {
    dim3 grid(np / 32, n_problems);
    SRB_TRY(launch_kernel(nce_prep_tc_kernel, grid, 256, 0, st, "nce_prep_tc_kernel", a));
  }
  NtMaps maps;
  NtArgs t;
  t.np = np;
  t.inv_tau = a.inv_tau;
  const int row_blocks = np / NT_T;
  // one CTA per SM (193 KB of shared memory each): as many column splits as fit in a single wave
  int splits = sm_count() / (row_blocks * n_problems);
  if (splits < 1) splits = 1;
  if (splits > NT_MAX_SPLITS) splits = NT_MAX_SPLITS;
  if (splits > row_blocks) splits = row_blocks;
  t.splits = splits;
  const long long nd = (long long)np * d;
  for (int q = 0; q < n_problems; ++q) {
    const NceProblem& p = a.p[q];
    // hi / lo parts live behind dV2 (written by prep): hi of (V1 V2 V1T V2T) then lo of the same four
    float* hi = p.dV2 + nd;
    float* lo = hi + 4 * nd;
    for (int h = 0; h < 2; ++h) {
      float* r = h ? lo : hi;
      SRB_REQUIRE(make_tmap_f32_rows(&maps.v1r[q][h], r, (uint64_t)np, d, NT_T) == 0 &&
                      make_tmap_f32_rows(&maps.v2r[q][h], r + nd, (uint64_t)np, d, NT_T) == 0 &&
                      make_tmap_f32_rows(&maps.v1c[q][h], r, (uint64_t)np, d, NT_C) == 0 &&
                      make_tmap_f32_rows(&maps.v2c[q][h], r + nd, (uint64_t)np, d, NT_C) == 0 &&
                      make_tmap_f32_rows(&maps.v1t[q][h], r + 2 * nd, (uint64_t)d, (uint64_t)np, NT_D) == 0 &&
                      make_tmap_f32_rows(&maps.v2t[q][h], r + 3 * nd, (uint64_t)d, (uint64_t)np, NT_D) == 0,
                  "infonce: cuTensorMapEncodeTiled failed");
    }
    NtProblem& o = t.p[q];
    o.n = p.n;
    o.n_dev = p.n_dev;
    o.weight = p.weight;
    o.diag = p.diag;
    o.lsum = p.part_l;  // [np] softmax denominators (first split slice of the partials area)
    o.dV1 = p.dV1;
    o.dV2 = p.dV2;
    o.loss_acc = p.loss_acc;
  }
  for (int q = n_problems; q < 2; ++q) {
    for (int h = 0; h < 2; ++h) {
      maps.v1r[q][h] = maps.v1r[0][h];
      maps.v2r[q][h] = maps.v2r[0][h];
      maps.v1c[q][h] = maps.v1c[0][h];
      maps.v2c[q][h] = maps.v2c[0][h];
      maps.v1t[q][h] = maps.v1t[0][h];
      maps.v2t[q][h] = maps.v2t[0][h];
    }
    t.p[q] = t.p[0];
  }
  const size_t smem = NtSmem::total + 1024;
  static bool attr_done = false;
  if (!attr_done) {
    SRB_TRY(check_cuda(cudaFuncSetAttribute(nce_tc_kernel<1, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "nce tc attr"));
    SRB_TRY(check_cuda(cudaFuncSetAttribute(nce_tc_kernel<2, BSM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "nce tc attr"));
    attr_done = true;
  }
  dim3 grid(row_blocks, splits, n_problems);
  SRB_TRY(launch_kernel(nce_tc_kernel<1, false>, grid, NT_THREADS, smem, st, "nce_tc_kernel<pass_a>", maps, t));
  SRB_TRY(launch_kernel(nce_tc_kernel<2, BSM>, grid, NT_THREADS, smem, st, "nce_tc_kernel<pass_b>", maps, t));
  return launch_kernel(nce_tc_finish_kernel<BSM>, dim3((np + 7) / 8, n_problems), 256, 0, st, "nce_tc_finish_kernel", a);
}

template <int D, bool BSM>
static int nce_launch(const NceArgs& a, int n_problems, cudaStream_t st) {
  const int np = a.np;
  {
    dim3 grid((np + 7) / 8, n_problems);
    SRB_TRY(launch_kernel(nce_prep_kernel<D>, grid, 256, 0, st, "nce_prep_kernel", a));
  }
  {
    void (*grad)(const NceArgs);
    size_t grad_smem;
    if constexpr (D == NCE_WIDE_D) {
      grad = nce_grad_wide_kernel<BSM>;
      grad_smem = sizeof(NceGradWideSmem);
    } else {
      grad = nce_grad_kernel<D, BSM>;
      grad_smem = sizeof(NceGradSmem<D>);
    }
    static bool attr_done = false;
    if (!attr_done) {
      SRB_TRY(check_cuda(cudaFuncSetAttribute(nce_lse_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(NceLseSmem<D>)), "nce lse smem attr"));
      SRB_TRY(check_cuda(cudaFuncSetAttribute(grad, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)grad_smem), "nce grad smem attr"));
      attr_done = true;
    }
    dim3 grid(np / NCE_T, a.splits, n_problems);
    SRB_TRY(launch_kernel(nce_lse_kernel<D>, grid, 256, sizeof(NceLseSmem<D>), st, "nce_lse_kernel", a));
    SRB_TRY(launch_kernel(grad, grid, 256, grad_smem, st, D == NCE_WIDE_D ? "nce_grad_wide_kernel" : "nce_grad_kernel", a));
  }
  {
    dim3 grid((np + 7) / 8, n_problems);
    SRB_TRY(launch_kernel(nce_finish_kernel<D>, grid, 256, 0, st, "nce_finish_kernel", a));
  }
  return SRB_OK;
}

// srb_infonce_fwd_bwd (BSM = false) and srb_batch_softmax_fwd_bwd (BSM = true): the same checks, workspace and routes
template <bool BSM>
static int nce_fwd_bwd(const srb_infonce_desc* d, void* stream) {
  const char* what = BSM ? "batch_softmax" : "infonce";
  SRB_REQUIRE(d != nullptr, "%s: null desc", what);
  SRB_REQUIRE(d->n_problems >= 1 && d->n_problems <= 4, "%s: n_problems must be 1..4", what);
  SRB_REQUIRE(d->temperature > 0.f, "%s: temperature must be positive", what);
  SRB_REQUIRE(!BSM || d->b_cos, "%s: b_cos must be 1 (the loss normalises both inputs)", what);
  SRB_REQUIRE(d->d == 16 || d->d == 32 || d->d == 64 || d->d == 128 || d->d == 256, "%s: unsupported d=%d (16, 32, 64, 128, 256)", what, d->d);
  int max_n = 0;
  for (int q = 0; q < d->n_problems; ++q) {
    const srb_infonce_problem& s = d->prob[q];
    SRB_REQUIRE(s.table1 && s.table2 && s.idx && s.g1 && s.g2 && s.loss, "%s: null pointer in problem %d", what, q);
    SRB_REQUIRE(s.n >= 0, "%s: negative n", what);
    if (s.n > max_n) max_n = s.n;
  }
  SRB_REQUIRE(d->workspace && d->workspace_bytes >= srb_infonce_workspace_bytes(max_n, d->d, d->n_problems),
              "%s: workspace too small (%lld < %lld)", what, (long long)d->workspace_bytes,
              (long long)srb_infonce_workspace_bytes(max_n, d->d, d->n_problems));
  if (max_n == 0) {
    for (int q = 0; q < d->n_problems; ++q)
      SRB_TRY(check_cuda(cudaMemsetAsync(d->prob[q].loss, 0, 4, (cudaStream_t)stream), what));
    return SRB_OK;
  }
  NceArgs a;
  a.n_problems = d->n_problems;
  a.np = nce_np(max_n);
  a.b_cos = d->b_cos;
  a.inv_tau = 1.0f / d->temperature;
  // enough CTAs for ~2 waves: row blocks x splits x problems
  const int row_blocks = a.np / NCE_T;
  int splits = (2 * sm_count() + row_blocks * d->n_problems - 1) / (row_blocks * d->n_problems);
  if (splits < 1) splits = 1;
  if (splits > NCE_MAX_SPLITS) splits = NCE_MAX_SPLITS;
  if (splits > row_blocks) splits = row_blocks;
  a.splits = splits;
  float* w = reinterpret_cast<float*>(d->workspace);
  const int64_t per = nce_problem_floats(a.np, d->d);
  for (int q = 0; q < d->n_problems; ++q) {
    const srb_infonce_problem& s = d->prob[q];
    NceProblem& p = a.p[q];
    p.table1 = s.table1;
    p.table2 = s.table2;
    p.row_off1 = s.row_off1;
    p.row_off2 = s.row_off2;
    p.scale1 = s.scale1;
    p.scale2 = s.scale2;
    p.idx = s.idx;
    p.n_dev = s.n_dev;
    p.n = s.n;
    p.weight = s.weight;
    p.g1 = s.g1;
    p.g2 = s.g2;
    p.loss = s.loss;
    float* base = w + per * q;
    const int64_t nd = (int64_t)a.np * d->d;
    p.V1 = base;
    p.V2 = base + nd;
    p.V1T = base + 2 * nd;
    p.V2T = base + 3 * nd;
    p.dV1 = base + 4 * nd;
    p.dV2 = base + 5 * nd;
    float* t = base + 14 * nd;  // [6 nd, 14 nd): TF32 hi / lo parts (tensor-core path)
    p.inv1 = t;
    p.inv2 = t + a.np;
    p.diag = t + 2 * a.np;
    p.part_m = t + 3 * a.np;
    p.part_l = t + 3 * a.np + (int64_t)NCE_MAX_SPLITS * a.np;
    p.lse = t + 3 * a.np + 2ll * NCE_MAX_SPLITS * a.np;
    p.loss_acc = p.lse + a.np;
  }
  cudaStream_t st = (cudaStream_t)stream;
  // the tensor-core LSE pass shifts by the bound 1/tau of a cosine logit: needs exp(-2/tau) representable
  if (d->d == 64 && d->b_cos && d->n_problems <= 2 && a.inv_tau <= 40.f) return nce_launch_tc<BSM>(a, d->n_problems, st);
  switch (d->d) {
    case 16: return nce_launch<16, BSM>(a, d->n_problems, st);
    case 32: return nce_launch<32, BSM>(a, d->n_problems, st);
    case 64: return nce_launch<64, BSM>(a, d->n_problems, st);
    case 128: return nce_launch<128, BSM>(a, d->n_problems, st);
    default: return nce_launch<256, BSM>(a, d->n_problems, st);
  }
}

}  // namespace srb

extern "C" int64_t srb_infonce_workspace_bytes(int32_t max_n, int32_t d, int32_t n_problems) {
  if (max_n < 0 || d <= 0 || n_problems <= 0) return 0;
  return srb::nce_problem_floats(srb::nce_np(max_n), d) * 4 * n_problems;
}

extern "C" int srb_infonce_fwd_bwd(const srb_infonce_desc* d, void* stream) { return srb::nce_fwd_bwd<false>(d, stream); }

extern "C" int srb_batch_softmax_fwd_bwd(const srb_infonce_desc* d, void* stream) { return srb::nce_fwd_bwd<true>(d, stream); }
