// (iii) InfoNCE forward/backward on the Hopper tensor cores (wgmma, TF32), d = 64.
//
// Same contract as infonce.cu (util/loss_torch.py:35-50 + autograd backward); the n x n logit matrix
// lives only in registers.  Per problem, with V1, V2 the L2-normalised gathered views:
//   pass A  rows = view-1 rows i:  E = exp(S - 1/tau)  (|S| <= 1/tau: cosines, so the shift needs no running max);
//           l_i += sum_{j != i} E_ij (the softmax denominator; prep seeds it with exp(S_ii - 1/tau) from the exact
//           S_ii) and, unnormalised, dV1_i += sum_{j != i} E_ij V2_j
//           -- forward (LSE) and the view-1 gradient in ONE sweep: the 1/l_i factor is applied afterwards
//   pass B  rows = view-2 rows j:  G' = exp(S^T - lse_i) * w/(n tau), i != j;  dV2 += G' V1   (needs every l_i)
//   finish  scales dV1 by w/(n tau l_i), adds the diagonal term (P_ii - 1) w/(n tau) v_i in exact fp32, then the
//           normalisation backward
// batch_softmax_loss (BSM below) runs the same passes: its row factor c_i multiplies w/(n tau) in pass B and finish.
// Each CTA owns a block of 128 rows and a strided subset of the 64-column tiles:
//   warp 8        TMA producer: per tile, the column operand [64 x 64] (K-major over d, for S) and the same tile
//                 from the transposed copy [64 d x 64 cols] (K-major over the column index, for G V), hi and lo
//                 parts, 128-byte swizzle, 2-stage ring
//   warpgroups 0, 1 (64 rows each):
//                 S[64 x 64]  = A B^T         wgmma m64n64k8, 8 k-steps x 3 products, operands in smem
//                 G = exp(...) in registers, split into TF32 hi / lo
//                 D[64 x 64] += G Vt^T        same shape, the G operand taken straight from the registers that
//                                             held S; finally D -> global (red.v2 over splits)
// The accumulator fragment of S holds columns 2t, 2t+1 of every 8-column k-step where the register A fragment
// of the next product wants columns t, t+4.  Instead of shuffling, the transposed copy is written with the columns
// of every group of 8 permuted (column o stored at position (o >> 1) + 4 (o & 1), nce_tperm), so that the k-step's
// B rows match the A fragment as it stands.
// fp32 accuracy on a TF32 pipe: every operand is split x = hi + lo (hi = rna_tf32(x), lo = x - hi, which
// the tensor core truncates to TF32) and each product is evaluated as hi*hi + hi*lo + lo*hi ("3xTF32",
// error ~2^-21 instead of 2^-11).  S_ii and the normalisation backward use the exact fp32 rows.
#pragma once
#include "common.cuh"
#include "tc_common.cuh"

namespace srb {

using namespace tc;

constexpr int NT_D = 64;
constexpr int NT_T = 128;        // rows per CTA (two warpgroups of wgmma M = 64)
constexpr int NT_C = 64;         // columns per tile (wgmma N of the S product, K of the G V product)
constexpr int NT_STAGES = 2;
constexpr int NT_THREADS = 256 + 32;  // warpgroups 0-1 MMA + exponentials, warp 8 TMA
constexpr int NT_MAX_SPLITS = 8;
constexpr uint32_t NT_ATILE = NT_T * NT_D * 4;   // 32 KB: 2 k-chunks x [128][32]      (x2: hi, lo)
constexpr uint32_t NT_BTILE = NT_C * NT_D * 4;   // 16 KB: 2 k-chunks x [64][32]       (x2: hi, lo)
constexpr uint32_t NT_TTILE = NT_D * NT_C * 4;   // 16 KB: 2 column chunks x [64][32]  (x2: hi, lo)
constexpr uint32_t NT_STAGE = 2 * NT_BTILE + 2 * NT_TTILE;  // one ring stage: B hi | B lo | Bt hi | Bt lo

// position of column i of a 64-column tile in the transposed copies (see above)
__host__ __device__ __forceinline__ int nce_tperm(int i) { return (i & ~7) | (((i & 7) >> 1) + 4 * (i & 1)); }

struct NtSmem {
  static constexpr uint32_t a_off = 0;                                  // row-operand tile hi|lo (fixed per CTA)  64 KB
  static constexpr uint32_t b_off = a_off + 2 * NT_ATILE;               // 2 stages x (B hi|lo, Bt hi|lo)        128 KB
  static constexpr uint32_t bar_off = b_off + NT_STAGES * NT_STAGE;
  static constexpr uint32_t total = bar_off + 1024;                     // barriers + column constants (pass B)
};

struct NtProblem {
  int32_t n;
  const int32_t* n_dev;
  float weight;
  const float* diag;     // [NP] exact S_ii
  float* lsum;           // [NP] softmax denominators l_i = sum_j exp(S_ij - 1/tau) (diagonal term by prep, the rest by pass A)
  float* dV1;            // [NP][64] accumulators (zeroed by prep)
  float* dV2;
  float* loss_acc;
};

struct NtArgs {
  int32_t np;      // padded capacity, multiple of 128
  int32_t splits;
  float inv_tau;
  NtProblem p[2];
};

struct NtMaps {
  // per problem (<= 2), hi and lo parts [2]: row-major views as row operand (box [128][32]) and as column
  // operand (box [64][32]), and the transposed views ([64 rows][NP], box [64][32])
  CUtensorMap v1r[2][2], v2r[2][2], v1c[2][2], v2c[2][2], v1t[2][2], v2t[2][2];
};

// The two losses over the in-batch softmax of S (row r: lse_r, p_r = exp(S_rr - lse_r)) differ only per row; BSM
// selects batch_softmax_loss at compile time in the kernels of both paths:
//   InfoNCE             loss_r = lse_r - S_rr          dL/dS_rj = (P_rj - delta_rj) / n
//   batch_softmax_loss  loss_r = -log(p_r + 1e-5)      dL/dS_rj = c_r (P_rj - delta_rj) / n,  c_r = p_r / (p_r + 1e-5)
// The reference (util/loss_torch.py:25-32) sums exp(S) without a shift and overflows once 1/tau > 88.7; here p_r comes
// from the log-sum-exp and stays finite.
constexpr float BSM_EPS = 1e-5f;  // the reference's 10e-6

__device__ __forceinline__ float bsm_row_loss(float lse, float s_rr) { return -logf(expf(s_rr - lse) + BSM_EPS); }

__device__ __forceinline__ float bsm_row_coef(float lse, float s_rr) {
  const float p = expf(s_rr - lse);
  return p / (p + BSM_EPS);
}

__device__ __forceinline__ int nt_n(const NtProblem& p) { return p.n_dev ? min(*p.n_dev, p.n) : p.n; }

__device__ __forceinline__ float to_tf32_rna(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

__device__ __forceinline__ float ex2_approx(float x) {  // 2^x, flush-to-zero, 2 ulp (the MUFU unit)
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// mode 1: pass A (rows = view 1)   mode 2: pass B (rows = view 2).  Pass A is the same for both losses: BSM (the
// batch_softmax_loss row factor c_i, folded into pass B's column constants) applies to pass B only.
template <int MODE, bool BSM>
__global__ void __launch_bounds__(NT_THREADS, 1) nce_tc_kernel(const __grid_constant__ NtMaps maps, const NtArgs a) {
  static_assert(MODE == 2 || !BSM, "pass A does not depend on the loss");
  pdl_wait();
  pdl_trigger();
  extern __shared__ __align__(1024) uint8_t nt_smem_raw[];
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(nt_smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sm + NtSmem::bar_off);
  uint64_t* bar_full = bars;                // [2] TMA -> MMA (column tiles, both layouts)
  uint64_t* bar_empty = bars + NT_STAGES;   // [2] both warpgroups' G V products done -> TMA
  uint64_t* bar_a = bars + 2 * NT_STAGES;   // [1] row tile loaded
  float* colc = reinterpret_cast<float*>(bars + 8);  // [2][64] pass B: per-column exponent offsets, double-buffered

  const int prob = blockIdx.z;
  const NtProblem& P = a.p[prob];
  const int n = nt_n(P);
  const int r0 = blockIdx.x * NT_T;
  if (r0 >= n) return;
  const int split = blockIdx.y;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int n_tiles = (n + NT_C - 1) / NT_C;
  const int my_tiles = (n_tiles - split + a.splits - 1) / a.splits;  // tiles split, split+S, ...
  if (my_tiles <= 0) return;
  const CUtensorMap* map_row = (MODE == 2) ? maps.v2r[prob] : maps.v1r[prob];    // [2]: hi, lo
  const CUtensorMap* map_col = (MODE == 2) ? maps.v1c[prob] : maps.v2c[prob];
  const CUtensorMap* map_colt = (MODE == 2) ? maps.v1t[prob] : maps.v2t[prob];

  if (threadIdx.x == 0) {
    for (int s = 0; s < NT_STAGES; ++s) {
      mbar_init(bar_full + s, 1);
      mbar_init(bar_empty + s, 2);  // one arrive per consumer warpgroup
    }
    mbar_init(bar_a, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (elect_one()) {
      mbar_arrive_expect_tx(bar_a, 2 * NT_ATILE);
      for (int h = 0; h < 2; ++h)
        for (int c = 0; c < 2; ++c) tma_load_2d(sm + NtSmem::a_off + h * NT_ATILE + c * 16384, &map_row[h], bar_a, c * 32, r0);
      for (int k = 0; k < my_tiles; ++k) {
        const int t = split + k * a.splits;
        const int s = k % NT_STAGES;
        uint8_t* st = sm + NtSmem::b_off + s * NT_STAGE;
        mbar_wait(bar_empty + s, ((k / NT_STAGES) & 1) ^ 1);
        mbar_arrive_expect_tx(bar_full + s, NT_STAGE);
        for (int h = 0; h < 2; ++h)
          for (int c = 0; c < 2; ++c) {
            tma_load_2d(st + h * NT_BTILE + c * 8192, &map_col[h], bar_full + s, c * 32, t * NT_C);
            tma_load_2d(st + 2 * NT_BTILE + h * NT_TTILE + c * 8192, &map_colt[h], bar_full + s, t * NT_C + c * 32, 0);
          }
      }
    }
    return;
  }
  // ===== consumer warpgroup wg: rows r0 + 64 wg .. +63 =====
  const int wg = warp >> 2;
  const int w4 = warp & 3, g = lane >> 2, tq = lane & 3;
  const int et = threadIdx.x;            // 0..255
  const int row_a = r0 + wg * 64 + w4 * 16 + g;  // accumulator rows of this thread: row_a, row_a + 8
  const float L2E = 1.4426950408889634f;
  const float sc = a.inv_tau * L2E;      // exponent scale: 2^(s*sc + off) = e^(s/tau + off/log2(e))
  const float gscale = P.weight * a.inv_tau / (float)n;
  const float lg = log2f(gscale);
  float l_run[2] = {0.f, 0.f};  // pass A: sum of exp(S - 1/tau) over my columns, rows row_a and row_a + 8
  // pass B: exponent offset of column c = log2(w/(n tau)) - lse_c log2(e), lse_c = 1/tau + ln l_c; the CTAs of the
  // first row block see every column exactly once and also accumulate the loss = mean(lse_i - S_ii), S_ii exact
  auto col_const = [&](int col) -> float {
    float off = -INFINITY, contrib = 0.f;
    if (col < n) {
      const float lse = a.inv_tau + logf(P.lsum[col]);
      off = lg - lse * L2E;
      contrib = BSM ? bsm_row_loss(lse, P.diag[col]) : lse - P.diag[col];
      if constexpr (BSM) off += log2f(bsm_row_coef(lse, P.diag[col]));  // c_col = 0 gives -inf: a zero column of G'
    }
    if (blockIdx.x == 0) {
      contrib = warp_sum(contrib);
      if (lane == 0) atomicAdd(P.loss_acc, contrib);
    }
    return off;
  };
  float next_colc = 0.f;
  if (MODE == 2) {  // column constants of tile 0
    if (et < NT_C) colc[et] = col_const(split * NT_C + et);
    named_bar_sync(1, 256);
  }
  const uint32_t a_base = smem_u32(sm + NtSmem::a_off + wg * 8192);
  float d[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) d[j] = 0.f;
  mbar_wait(bar_a, 0);
  for (int k = 0; k < my_tiles; ++k) {
    const int t = split + k * a.splits;
    const int s = k % NT_STAGES;
    const int cb = t * NT_C;  // first column of the tile
    if (MODE == 2 && et < NT_C && k + 1 < my_tiles) next_colc = col_const((t + a.splits) * NT_C + et);  // prefetch
    mbar_wait(bar_full + s, (k / NT_STAGES) & 1);
    const uint32_t b_base = smem_u32(sm + NtSmem::b_off + s * NT_STAGE);
    // S = Ahi Bhi + Ahi Blo + Alo Bhi
    float sv[32];
    wgmma_fence();
#pragma unroll
    for (int pr = 0; pr < 3; ++pr) {
      const uint32_t ab = a_base + (pr == 2 ? NT_ATILE : 0);
      const uint32_t bb = b_base + (pr == 1 ? NT_BTILE : 0);
#pragma unroll
      for (int c = 0; c < 2; ++c)
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
          wgmma_m64n64k8_tf32_ss(sv, make_smem_desc_k_sw128(ab + c * 16384 + kk * 32), make_smem_desc_k_sw128(bb + c * 8192 + kk * 32),
                                 (pr | c | kk) ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    // G: pass A x = exp(s/tau - 1/tau), pass B x = exp(s/tau - lse_col) * w/(n tau).  The diagonal term
    // (P_ii - 1) v_i is added in exact fp32 by the finish kernel: through the tensor core its TF32 rounding
    // (|G_ii| ~ 1) would dominate the row.  Rows >= n only reach rows >= n of D, which are never written.
    uint32_t hi[32], lo[32];
    const float* cc = colc + (k & 1) * NT_C;
    // (selects, not branches: a divergent path between the wgmma groups would serialise them)
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int cl = 8 * (j >> 2) + 2 * tq + (j & 1);  // column within the tile
      const int rh = (j >> 1) & 1;                     // row_a or row_a + 8
      const float off = (MODE == 1) ? -sc : cc[cl];    // pass B: -inf for columns >= n
      float x = ex2_approx(fmaf(sv[j], sc, off));
      x = (cb + cl == row_a + 8 * rh) ? 0.f : x;
      if (MODE == 1) {
        x = (cb + cl < n) ? x : 0.f;
        l_run[rh] += x;  // off-diagonal terms only: prep seeded l_i with the exact diagonal term
      }
      const float h = to_tf32_rna(x);
      hi[j] = __float_as_uint(h);
      lo[j] = __float_as_uint(x - h);
    }
    // D += Ghi Vhi + Glo Vhi + Ghi Vlo      (K = the 64 columns of this tile, 8 per MMA; G from registers)
    const uint32_t bt_base = b_base + 2 * NT_BTILE;
    wgmma_fence();
#pragma unroll
    for (int pr = 0; pr < 3; ++pr) {
      const uint32_t (&ga)[32] = (pr == 1) ? lo : hi;
      const uint32_t vb = bt_base + (pr == 2 ? NT_TTILE : 0);
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)
        wgmma_m64n64k8_tf32_rs(d, ga[4 * kk], ga[4 * kk + 2], ga[4 * kk + 1], ga[4 * kk + 3],
                               make_smem_desc_k_sw128(vb + (kk >> 2) * 8192 + (kk & 3) * 32), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    if ((threadIdx.x & 127) == 0) mbar_arrive(bar_empty + s);  // this warpgroup is done with the stage
    if (MODE == 2) {
      if (et < NT_C && k + 1 < my_tiles) colc[((k + 1) & 1) * NT_C + et] = next_colc;
      named_bar_sync(1, 256);
    }
  }
#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    const int row = row_a + 8 * rh;
    if (MODE == 1) {
      float l = l_run[rh];
      l += __shfl_xor_sync(SRB_FULL_MASK, l, 1);
      l += __shfl_xor_sync(SRB_FULL_MASK, l, 2);
      if (tq == 0 && row < n) atomicAdd(P.lsum + row, l);
    }
    if (row < n) {
      float* out = ((MODE == 1) ? P.dV1 : P.dV2) + (size_t)row * NT_D;
#pragma unroll
      for (int cg = 0; cg < 8; ++cg)  // red.global.add.v2.f32
        atomicAdd(reinterpret_cast<float2*>(out + 8 * cg + 2 * tq), make_float2(d[4 * cg + 2 * rh], d[4 * cg + 2 * rh + 1]));
    }
  }
}

}  // namespace srb
