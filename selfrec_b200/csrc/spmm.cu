// (i) CSR SpMM  Y = A * X  with fused epilogue (noise, layer sum, Adam, peer all-gather).
//
// Replaces torch.sparse.mm(self.sparse_norm_adj, ego_embeddings) -- LightGCN.py:72,
// SimGCL.py:85, XSimGCL.py:88, SGL.py:104-108 -- plus the elementwise tail of the encoders
// (XSimGCL.py:90-96) and, for the last backward product, torch.optim.Adam.step.
//
// HBM/L2-bound integer + fp32 work: no tensor cores here by design (see the kernel comment
// for the lane mapping).
#include "spmm_args.cuh"

namespace srb {

__device__ __forceinline__ void st4_cs(float* p, const float4& v, int stream) {
  if (stream) __stcs(reinterpret_cast<float4*>(p), v);
  else st4(p, v);
}

// store to another rank's copy: a plain P2P store, or one multimem.st that the NVSwitch replicates into every
// rank's copy of a multicast-mapped buffer
__device__ __forceinline__ void st4_peer(float* p, const float4& v, int mc) {
  if (mc) asm volatile("multimem.st.weak.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
  else st4(p, v);
}

// 16-byte ld.global.nc when `pred`, else zeros: one predicated load, no branch, so a sub-batch's gathers stay in flight
// together (a `pred ? ldg4(p) : f4_zero()` compiles to a branch around every load: the yelp2018 XSimGCL step went
// from 0.539 to 0.550 ms, H100 80GB HBM3 at 400 W)
__device__ __forceinline__ float4 ldg4_if(const float* p, bool pred) {
  float4 r = f4_zero();
  asm("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %5, 0;\n\t@q ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4];\n\t}"
      : "+f"(r.x), "+f"(r.y), "+f"(r.z), "+f"(r.w)
      : "l"(p), "r"((int)pred));
  return r;
}

// Epilogue of one output row held by a lane group (gl = lane within the group): dense addend, noise,
// store / peer pushes, running layer sum, Adam.  All lanes of the warp must call it (shuffles);
// `valid` gates the memory traffic.
template <int D>
__device__ __forceinline__ void spmm_epilogue(const SpmmArgs& a, int row, int gl, float4 acc0, float4 acc1, bool valid) {
  constexpr int LPR = D / 8;
  constexpr int HALF = D / 2;
  {
    // ---- epilogue (per lane group = per row) ----
    if (a.stage_peer[0]) {  // partial product of a sharded item row: hand it to the row's owner, nothing else
      if (!valid) return;
      int o = 0;
#pragma unroll 1
      while (row >= a.stage_bounds[o + 1]) ++o;
      float* dst = a.stage_peer[o] + ((size_t)a.stage_rank * a.stage_cap + (row - a.stage_bounds[o])) * D + gl * 4;
      st4(dst, acc0);
      st4(dst + HALF, acc1);
      return;
    }
    const size_t off = (size_t)row * D + gl * 4;
    float4 y0 = acc0, y1 = acc1;
    if (a.extra && valid) {
      y0 = f4_fma(a.extra_scale, *reinterpret_cast<const float4*>(a.extra + off), y0);
      y1 = f4_fma(a.extra_scale, *reinterpret_cast<const float4*>(a.extra + off + HALF), y1);
    }
    if (a.seed && valid) {
      if ((__ldg(a.seed_mask + (row >> 5)) >> (row & 31)) & 1u) {
        y0 = f4_add(y0, *reinterpret_cast<const float4*>(a.seed + off));
        y1 = f4_add(y1, *reinterpret_cast<const float4*>(a.seed + off + HALF));
      }
    }
    if (a.noise_mode) {
      float4 n0 = f4_zero(), n1 = f4_zero();
      if (a.noise_mode == 1) {
        if (valid) {
          n0 = ldg4(a.noise + off);
          n1 = ldg4(a.noise + off + HALF);
        }
      } else {
        const uint32_t stp = a.pstep ? (uint32_t)*a.pstep : 0u;
        const uint32_t grow = (uint32_t)(a.noise_row_base + row * a.noise_row_stride);
        // counter = (row, column block | view << 16, layer tag, step): (view, step) pairs never share a stream; the
        // column block (c / 4: gl and gl + LPR) stays below 64, clear of the view bits, up to D = 256
        const uint32_t vw = a.poff.y << 16;
        const uint32_t cb0 = (uint32_t)gl | vw;
        // (at LPR = 32, cb0 + 32: one add in place of a second loop-invariant word, which spilled at 64 registers)
        const uint32_t cb1 = LPR == 32 ? cb0 + LPR : (uint32_t)(gl + LPR) | vw;
        const uint4 r0 = philox4x32_10(make_uint4(grow, cb0, a.poff.x, stp), a.pkey);
        const uint4 r1 = philox4x32_10(make_uint4(grow, cb1, a.poff.x, stp), a.pkey);
        n0 = make_float4(u32_to_unit(r0.x), u32_to_unit(r0.y), u32_to_unit(r0.z), u32_to_unit(r0.w));
        n1 = make_float4(u32_to_unit(r1.x), u32_to_unit(r1.y), u32_to_unit(r1.z), u32_to_unit(r1.w));
      }
      float ss = f4_dot(n0, n0) + f4_dot(n1, n1);
#pragma unroll
      for (int o = LPR / 2; o > 0; o >>= 1) ss += __shfl_xor_sync(SRB_FULL_MASK, ss, o);
      const float nrm = fmaxf(sqrtf(ss), 1e-12f);  // F.normalize eps
#define SRB_PERT(Y, N, F) Y.F += sgnf(Y.F) * (N.F / nrm) * a.eps;
      SRB_PERT(y0, n0, x) SRB_PERT(y0, n0, y) SRB_PERT(y0, n0, z) SRB_PERT(y0, n0, w)
      SRB_PERT(y1, n1, x) SRB_PERT(y1, n1, y) SRB_PERT(y1, n1, z) SRB_PERT(y1, n1, w)
#undef SRB_PERT
    }
    if (!valid) return;
    if (a.Y) {  // written once, read (randomly) by the NEXT product
      st4_cs(a.Y + off, y0, a.stream);
      st4_cs(a.Y + off + HALF, y1, a.stream);
    }
    if (a.world > 0 && a.peer[0]) {  // fused all-gather: NVLink P2P stores into every rank's layer buffer
#pragma unroll 1
      for (int g = 0; g < a.world; ++g) {
        st4_peer(a.peer[g] + off, y0, a.peer_mc);
        st4_peer(a.peer[g] + off + HALF, y1, a.peer_mc);
      }
    }
    if (a.sum_out) {
      float4 s0 = y0, s1 = y1;
      if (a.sum_in) {
        float4 t0 = *reinterpret_cast<const float4*>(a.sum_in + off);
        float4 t1 = *reinterpret_cast<const float4*>(a.sum_in + off + HALF);
#pragma unroll
        for (int j = 0; j < 3; ++j) {
          if (!a.sum_add[j]) break;
          t0 = f4_add(*reinterpret_cast<const float4*>(a.sum_add[j] + off), t0);
          t1 = f4_add(*reinterpret_cast<const float4*>(a.sum_add[j] + off + HALF), t1);
        }
        s0 = f4_add(s0, t0);
        s1 = f4_add(s1, t1);
      }
      s0 = f4_scale(a.sum_scale, s0);
      s1 = f4_scale(a.sum_scale, s1);
      st4_cs(a.sum_out + off, s0, a.stream);
      st4_cs(a.sum_out + off + HALF, s1, a.stream);
      if (a.world > 0 && a.peer_sum[0]) {
#pragma unroll 1
        for (int g = 0; g < a.world; ++g) {
          st4_peer(a.peer_sum[g] + off, s0, a.peer_mc);
          st4_peer(a.peer_sum[g] + off + HALF, s1, a.peer_mc);
        }
      }
    }
    if (a.ap) {
      const float step_size = a.ascal[0];
      const float bc2_sqrt = a.ascal[1];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const size_t o2 = off + h * HALF;
        const float4 g = h ? y1 : y0;
        float4 p4 = *reinterpret_cast<const float4*>(a.ap + o2);
        float4 m = *reinterpret_cast<const float4*>(a.am + o2);
        float4 v4 = *reinterpret_cast<const float4*>(a.av + o2);
#define SRB_ADAM1(F) adam_elem(p4.F, m.F, v4.F, g.F, step_size, bc2_sqrt, a.w1, a.b2, a.w2, a.aeps);
        SRB_ADAM1(x) SRB_ADAM1(y) SRB_ADAM1(z) SRB_ADAM1(w)
#undef SRB_ADAM1
        st4(a.ap + o2, p4);
        st4_cs(a.am + o2, m, a.stream);
        st4_cs(a.av + o2, v4, a.stream);
        if (a.world > 0 && a.peer_p[0]) {
#pragma unroll 1
          for (int g = 0; g < a.world; ++g) st4_peer(a.peer_p[g] + o2, p4, a.peer_mc);
        }
      }
    }
  }
}

// Mapping: a row vector of D floats lives on LPR = D/8 lanes (two float4 per lane: columns
// [4*gl, 4*gl+4) and [D/2 + 4*gl, ...)), so a warp holds 32/LPR lane groups: 16 at D = 16, 8 at D = 32, one (the whole
// warp) at D = 256.  Rows are taken in `row_order` (degree-descending), in three
// classes so that no row is a long chain of dependent L2 round trips (a row of thousands of non-zeros handled by
// one warp alone would take as long as the rest of the matrix):
//   * the first n_vlong rows get a whole CTA: 8 warps x 32/LPR lane groups stride through the row, partial
//     sums meet in shared memory;
//   * the next n_long rows get a warp each (the 32/LPR lane groups stride 32 non-zeros per iteration
//     and are xor-shuffled together; at D = 256 the warp is one group and there is nothing to combine);
//   * the remaining rows are processed RPW = 32/LPR at a time, one per lane group (neighbours in the
//     sorted order are equally long; at D = 256 a warp per row).
// Each lane loads one (col, val) pair per iteration (coalesced, prefetched one iteration ahead) and
// the pairs are walked with group-wide shuffles; every X-row gather is two 128-bit ld.global.nc per
// lane (LPR lanes x 16 B = one contiguous half row), issued 2*SB at a time before the FMAs.
template <int D, bool MASKED>
__device__ __forceinline__ void spmm_gather(const SpmmArgs& a, int p, int end, int stride, int gl, float4& acc0, float4& acc1) {
  constexpr int LPR = D / 8;
  constexpr int HALF = D / 2;
  constexpr int SB = LPR < 4 ? LPR : 4;  // sub-batch: 2*SB independent 128-bit gathers per lane in flight
  constexpr bool masked = MASKED;  // compile-time: the plain product must not pay for the mask logic
  const int lane = threadIdx.x & 31;
  const int gbase = lane - gl;  // first lane of my group
  // (col, val) of the current iteration; padding slots gather row 0 with weight 0 (an L1 hit)
  int c = 0;
  float v = 0.f;
  bool hit = false;
  if (p + gl < end) {
    // tables beyond L2 (config-5 size: the product is bound by re-reads of gathered X rows): the CSR arrays are read
    // once per product, so they go evict-first and do not push X rows out; small graphs keep everything L2-resident
    c = a.stream ? __ldcs(a.colidx + p + gl) : __ldg(a.colidx + p + gl);
    v = a.stream ? __ldcs(a.vals + p + gl) : __ldg(a.vals + p + gl);
    if (masked) hit = (__ldg(a.col_mask + (c >> 5)) >> (c & 31)) & 1u;
  }
  while (__any_sync(SRB_FULL_MASK, p < end)) {
    int cn = 0;
    float vn = 0.f;
    bool hitn = false;
    if (p + stride + gl < end) {  // prefetch the next iteration's pair
      cn = a.stream ? __ldcs(a.colidx + p + stride + gl) : __ldg(a.colidx + p + stride + gl);
      vn = a.stream ? __ldcs(a.vals + p + stride + gl) : __ldg(a.vals + p + stride + gl);
      if (masked) hitn = (__ldg(a.col_mask + (cn >> 5)) >> (cn & 31)) & 1u;
    }
    if (!masked) {
#pragma unroll
      for (int j0 = 0; j0 < LPR; j0 += SB) {
        if (j0 > 0 && !__any_sync(SRB_FULL_MASK, p + j0 < end)) break;
        float vv[SB];
        float4 x0[SB], x1[SB];
#pragma unroll
        for (int j = 0; j < SB; ++j) {
          const int cc = __shfl_sync(SRB_FULL_MASK, c, j0 + j, LPR);
          vv[j] = __shfl_sync(SRB_FULL_MASK, v, j0 + j, LPR);
          const float* xr = a.X + (size_t)cc * D + gl * 4;
          x0[j] = ldg4(xr);
          x1[j] = ldg4(xr + HALF);
        }
#pragma unroll
        for (int j = 0; j < SB; ++j) {
          acc0 = f4_fma(vv[j], x0[j], acc0);
          acc1 = f4_fma(vv[j], x1[j], acc1);
        }
      }
    } else {
      // row-sparse X: only the non-zeros whose column bit is set are gathered.  Each lane group compacts its
      // hits (ballot + find-first-set) so a sub-batch holds SB real gathers; the warp stops when every
      // group has run out -- fewer dependent L2 round trips, which is what bounds this product.  A slot past the
      // group's last hit loads nothing and adds an exact zero: X is a seed table whose rows outside the batch hold
      // whatever an earlier step left there (a NaN there would survive a multiplication by weight 0)
      // (the group's LPR ballot bits; a whole-warp group at LPR = 32 keeps all of them -- 1u << 32 is undefined)
      constexpr uint32_t GROUP_BITS = LPR >= 32 ? 0xffffffffu : (1u << (LPR & 31)) - 1u;
      uint32_t gm = (__ballot_sync(SRB_FULL_MASK, hit) >> gbase) & GROUP_BITS;
      while (__any_sync(SRB_FULL_MASK, gm != 0)) {
        float vv[SB];
        float4 x0[SB], x1[SB];
#pragma unroll
        for (int j = 0; j < SB; ++j) {
          const int src = gm ? (__ffs(gm) - 1) : 0;
          const bool live = gm != 0;
          gm &= gm - 1;
          const int cc = __shfl_sync(SRB_FULL_MASK, c, gbase + src);
          const float vs = __shfl_sync(SRB_FULL_MASK, v, gbase + src);
          vv[j] = live ? vs : 0.f;
          const float* xr = a.X + (size_t)cc * D + gl * 4;
          x0[j] = ldg4_if(xr, live);
          x1[j] = ldg4_if(xr + HALF, live);
        }
#pragma unroll
        for (int j = 0; j < SB; ++j) {
          acc0 = f4_fma(vv[j], x0[j], acc0);
          acc1 = f4_fma(vv[j], x1[j], acc1);
        }
      }
    }
    c = cn;
    v = vn;
    hit = hitn;
    p += stride;
  }
}

// sums the 32/lpr lane groups of a warp into every group (no shuffle at all when one group fills the warp)
__device__ __forceinline__ void xor_reduce_groups(float4& acc0, float4& acc1, int lpr) {
  for (int o = lpr; o < 32; o <<= 1) {
    acc0.x += __shfl_xor_sync(SRB_FULL_MASK, acc0.x, o);
    acc0.y += __shfl_xor_sync(SRB_FULL_MASK, acc0.y, o);
    acc0.z += __shfl_xor_sync(SRB_FULL_MASK, acc0.z, o);
    acc0.w += __shfl_xor_sync(SRB_FULL_MASK, acc0.w, o);
    acc1.x += __shfl_xor_sync(SRB_FULL_MASK, acc1.x, o);
    acc1.y += __shfl_xor_sync(SRB_FULL_MASK, acc1.y, o);
    acc1.z += __shfl_xor_sync(SRB_FULL_MASK, acc1.z, o);
    acc1.w += __shfl_xor_sync(SRB_FULL_MASK, acc1.w, o);
  }
}

// Partial sums of the chunks of split ("huge") rows: one CTA per (row, chunk) work item, SRB_HUB_CHUNK non-zeros each.
// A power-law graph at config-5 scale has rows with millions of non-zeros; one CTA walking such a row alone would
// take longer than the rest of the product, so those rows are cut into chunks here and summed (in chunk order:
// deterministic) by the main kernel.
template <int D, bool MASKED>
__global__ void __launch_bounds__(256) spmm_hub_kernel(const SpmmArgs a) {
  constexpr int LPR = D / 8;
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int grp = lane / LPR;
  const int gl = lane % LPR;
  pdl_wait();
  pdl_trigger();
  const int n_work = a.seg ? a.n_cta : (a.n_vlong_dev ? min(a.n_vlong_dev[4], a.n_work) : a.n_work);
  __shared__ float4 part[8][2][LPR];
  for (int k = blockIdx.x; k < n_work; k += gridDim.x) {
    int w = k, beg, end;
    if (a.seg) {  // column-blocked segments, in (column block, row) order
      w = __ldg(a.order_cta + k);
      beg = __ldg(a.seg + 2 * w);
      end = __ldg(a.seg + 2 * w + 1);
    } else {
      const int row = __ldg(a.hub_work + 2 * w);
      const int ci = __ldg(a.hub_work + 2 * w + 1);
      const int rbeg = __ldg(a.rowptr + row), rend = __ldg(a.rowptr + row + 1);
      beg = min(rend, rbeg + ci * SRB_HUB_CHUNK);
      end = min(rend, beg + SRB_HUB_CHUNK);
    }
    // non-zeros per warp: a multiple of 32, the segment spread over all 8 warps (column-blocked segments and the last
    // chunk of a row are shorter than a full chunk; with a fixed 256 per warp most warps of such a CTA sat idle)
    const int per = ((end - beg + 255) / 256) * 32;
    const int wbeg = beg + wib * per;
    const int wend = min(end, wbeg + per);
    float4 acc0 = f4_zero(), acc1 = f4_zero();
    spmm_gather<D, MASKED>(a, wbeg + grp * LPR, wend, 32, gl, acc0, acc1);
    xor_reduce_groups(acc0, acc1, LPR);
    if (grp == 0) {
      part[wib][0][gl] = acc0;
      part[wib][1][gl] = acc1;
    }
    __syncthreads();
    if (wib == 0 && grp == 0) {
      acc0 = f4_zero();
      acc1 = f4_zero();
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        acc0 = f4_add(acc0, part[q][0][gl]);
        acc1 = f4_add(acc1, part[q][1][gl]);
      }
      float* dst = a.hub_part + (size_t)w * D + gl * 4;
      st4(dst, acc0);
      st4(dst + D / 2, acc1);
    }
    __syncthreads();
  }
}

// Short segments of the column-blocked lists: a warp each (lane groups stride the segment, like a "long" row).
template <int D, bool MASKED>
__global__ void __launch_bounds__(256) spmm_seg_warp_kernel(const SpmmArgs a) {
  constexpr int LPR = D / 8;
  const int lane = threadIdx.x & 31;
  const int grp = lane / LPR;
  const int gl = lane % LPR;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  pdl_wait();
  pdl_trigger();
  for (int k = warp0; k < a.n_warp; k += nwarps) {
    const int w = __ldg(a.order_warp + k);
    const int beg = __ldg(a.seg + 2 * w), end = __ldg(a.seg + 2 * w + 1);
    float4 acc0 = f4_zero(), acc1 = f4_zero();
    spmm_gather<D, MASKED>(a, beg + grp * LPR, end, 32, gl, acc0, acc1);
    xor_reduce_groups(acc0, acc1, LPR);
    if (grp == 0) {
      float* dst = a.hub_part + (size_t)w * D + gl * 4;
      st4(dst, acc0);
      st4(dst + D / 2, acc1);
    }
  }
}

// Split rows, second half: add up the chunk sums of spmm_hub_kernel (chunk order), then the common epilogue.
// One warp per row; its own launch so that the main kernel's register budget stays what it was.
template <int D>
__global__ void __launch_bounds__(256) spmm_hub_finish_kernel(const SpmmArgs a) {
  constexpr int LPR = D / 8;
  constexpr int RPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int grp = lane / LPR;
  const int gl = lane % LPR;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  pdl_wait();
  pdl_trigger();
  const int n_huge = a.n_vlong_dev ? min(a.n_vlong_dev[0], a.n_rows) : a.n_huge;
  peer_wait(a.ps);  // (its epilogue may store to peers; the signal is the main kernel's, launched after this one)
  for (int vr = warp0; vr < n_huge; vr += nwarps) {
    const int row = __ldg(a.row_order + vr);
    const int first = __ldg(a.hub_first + vr);
    const int deg = __ldg(a.rowptr + row + 1) - __ldg(a.rowptr + row);
    const int nch = a.seg ? __ldg(a.seg_cnt + vr) : (deg + SRB_HUB_CHUNK - 1) / SRB_HUB_CHUNK;
    float4 acc0 = f4_zero(), acc1 = f4_zero();
    for (int c = grp; c < nch; c += RPW) {
      const float* src = a.hub_part + (size_t)(first + c) * D + gl * 4;
      acc0 = f4_add(acc0, *reinterpret_cast<const float4*>(src));
      acc1 = f4_add(acc1, *reinterpret_cast<const float4*>(src + D / 2));
    }
    xor_reduce_groups(acc0, acc1, LPR);
    spmm_epilogue<D>(a, row, gl, acc0, acc1, grp == 0);
  }
}

template <int D, bool MASKED>
__global__ void __launch_bounds__(256) spmm_csr_kernel(const SpmmArgs a) {
  constexpr int LPR = D / 8;     // lanes per row
  constexpr int RPW = 32 / LPR;  // rows per warp (short rows)
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int grp = lane / LPR;
  const int gl = lane % LPR;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;

  pdl_wait();
  pdl_trigger();
  peer_wait(a.ps);
  // (the split rows -- the first n_huge entries of the list -- belong to spmm_hub_kernel / spmm_hub_finish_kernel)
  int n_vlong = a.n_vlong, n_long = a.n_long, n_short = a.n_rows - a.n_huge - a.n_vlong - a.n_long;
  const int32_t* ro_v = a.row_order ? a.row_order + a.n_huge : nullptr;  // the three classes' row lists (null: identity order)
  const int32_t* ro_l = a.row_order ? ro_v + n_vlong : nullptr;
  const int32_t* ro_s = a.row_order ? ro_l + n_long : nullptr;
  int id_l = n_vlong, id_s = n_vlong + n_long;
  if (a.n_vlong_dev) {  // row list classified on the device: four segments of capacity n_rows (split, very long, long, short)
    n_vlong = min(a.n_vlong_dev[1], a.n_rows);
    n_long = min(a.n_vlong_dev[2], a.n_rows);
    n_short = min(a.n_vlong_dev[3], a.n_rows);
    ro_v = a.row_order + a.n_rows;
    ro_l = a.row_order + 2 * a.n_rows;
    ro_s = a.row_order + 3 * a.n_rows;
  }
  // ---- class 1: one CTA per very long row ----
  __shared__ float4 part[8][2][LPR];
  for (int vr = blockIdx.x; vr < n_vlong; vr += gridDim.x) {
    const int row = ro_v ? __ldg(ro_v + vr) : vr;
    const int beg = __ldg(a.rowptr + row);
    const int end = __ldg(a.rowptr + row + 1);
    const int per = ((end - beg + 255) / 256) * 32;  // non-zeros per warp, a multiple of 32
    const int wbeg = beg + wib * per;
    const int wend = min(end, wbeg + per);
    float4 acc0 = f4_zero(), acc1 = f4_zero();
    spmm_gather<D, MASKED>(a, wbeg + grp * LPR, wend, 32, gl, acc0, acc1);
    xor_reduce_groups(acc0, acc1, LPR);
    if (grp == 0) {
      part[wib][0][gl] = acc0;
      part[wib][1][gl] = acc1;
    }
    __syncthreads();
    if (wib == 0) {
      acc0 = f4_zero();
      acc1 = f4_zero();
#pragma unroll
      for (int w = 0; w < 8; ++w) {
        acc0 = f4_add(acc0, part[w][0][gl]);
        acc1 = f4_add(acc1, part[w][1][gl]);
      }
      spmm_epilogue<D>(a, row, gl, acc0, acc1, grp == 0);
    }
    __syncthreads();
  }

  // ---- classes 2 and 3: one warp per long row, one lane group per short row ----
  const int n_items = n_long + (n_short + RPW - 1) / RPW;
  for (int item = warp0; item < n_items; item += nwarps) {
    const bool is_long = item < n_long;  // warp-uniform
    const int k = is_long ? item : (item - n_long) * RPW + grp;  // index within the class
    bool valid = is_long || k < n_short;
    int row = 0, p = 0, end = 0;
    if (valid) {
      if (is_long) row = ro_l ? __ldg(ro_l + k) : id_l + k;
      else row = ro_s ? __ldg(ro_s + k) : id_s + k;
      p = __ldg(a.rowptr + row);
      end = __ldg(a.rowptr + row + 1);
    }
    if (is_long) p += grp * LPR;
    float4 acc0 = f4_zero(), acc1 = f4_zero();
    spmm_gather<D, MASKED>(a, p, end, is_long ? 32 : LPR, gl, acc0, acc1);
    if (is_long) {  // combine the lane groups; group 0 owns the row
      xor_reduce_groups(acc0, acc1, LPR);
      valid = valid && grp == 0;
    }
    spmm_epilogue<D>(a, row, gl, acc0, acc1, valid);
  }
  peer_signal(a.ps);  // (sharded item-side product: this rank's partial rows are in the owners' staging areas)
}

// sum over the ranks' copies of a multicast-mapped buffer, added by the NVSwitch (NVLS): 16 bytes per request
__device__ __forceinline__ float4 multimem_ld_reduce_add4(const float* mc) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}

// Owner-side reduction of an item slice (bipartite sharding): every rank's item-side product left its partial rows
// in this rank's staging area; one lane group per slice row adds them in rank order (deterministic, and the only
// writer of the row) and runs the common epilogue -- noise, layer sum, Adam, and the pushes that hand the finished
// row to every rank (the all-gather half of the exchange).
template <int D>
__global__ void __launch_bounds__(256) reduce_rows_kernel(const SpmmArgs a, const ReduceArgs r) {
  constexpr int LPR = D / 8;
  constexpr int RPW = 32 / LPR;
  constexpr int HALF = D / 2;
  const int lane = threadIdx.x & 31;
  const int grp = lane / LPR;
  const int gl = lane % LPR;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int n_items = (r.n_slice + RPW - 1) / RPW;
  peer_wait(a.ps);  // every rank's partial rows have landed in the staging area
  if (r.mc_part) {
    // NVLS route: four rows per lane group in flight (8 x 16 B per lane): the kernel is bound by NVLink latency x
    // bytes in flight and runs on one CTA per SM beside the user-side SpMM
    constexpr int UN = 4;
    for (int item = warp0 * UN; item < n_items; item += nwarps * UN) {
      float4 p0[UN], p1[UN];
      bool ok[UN];
#pragma unroll
      for (int u = 0; u < UN; ++u) {
        const int k = (item + u) * RPW + grp;
        ok[u] = (item + u) < n_items && k < r.n_slice;
        if (ok[u] && r.mask) {
          const int row = r.slice_begin + k;
          ok[u] = (__ldg(r.mask + (row >> 5)) >> (row & 31)) & 1u;
        }
        p0[u] = p1[u] = f4_zero();
        if (ok[u]) {
          const float* src = r.mc_part + (size_t)(r.slice_begin + k) * D + gl * 4;
          p0[u] = multimem_ld_reduce_add4(src);
          p1[u] = multimem_ld_reduce_add4(src + HALF);
        }
      }
#pragma unroll
      for (int u = 0; u < UN; ++u) {
        if (!__any_sync(SRB_FULL_MASK, ok[u])) continue;
        spmm_epilogue<D>(a, r.slice_begin + (item + u) * RPW + grp, gl, p0[u], p1[u], ok[u]);
      }
    }
    peer_signal(a.ps);
    return;
  }
  for (int item = warp0; item < n_items; item += nwarps) {
    const int k = item * RPW + grp;
    bool valid = k < r.n_slice;
    if (r.mask) {  // last forward layer: only the batch's items carry a fresh partial sum (warp-uniform skip)
      const int row = r.slice_begin + k;
      valid = valid && ((__ldg(r.mask + (row >> 5)) >> (row & 31)) & 1u);
      if (!__any_sync(SRB_FULL_MASK, valid)) continue;
    }
    float4 acc0 = f4_zero(), acc1 = f4_zero();
    if (valid) {
      const float* src = r.stage + (size_t)k * D + gl * 4;
      const size_t plane = (size_t)r.stage_cap * D;
#pragma unroll 1
      for (int q = 0; q < r.world; q += 2) {  // two ranks' partials in flight
        const bool two = q + 1 < r.world;
        const float4 p0 = ldg4(src + (size_t)q * plane), p1 = ldg4(src + (size_t)q * plane + HALF);
        float4 p2 = f4_zero(), p3 = f4_zero();
        if (two) {
          p2 = ldg4(src + (size_t)(q + 1) * plane);
          p3 = ldg4(src + (size_t)(q + 1) * plane + HALF);
        }
        acc0 = f4_add(acc0, p0);
        acc1 = f4_add(acc1, p1);
        if (two) {
          acc0 = f4_add(acc0, p2);
          acc1 = f4_add(acc1, p3);
        }
      }
    }
    spmm_epilogue<D>(a, r.slice_begin + k, gl, acc0, acc1, valid);
  }
  peer_signal(a.ps);  // the finished rows are in every rank's copy
}

// The epilogue alone (identity product): one lane group per row reads X[row] and runs the common epilogue on it.
template <int D>
__global__ void __launch_bounds__(256) rows_epilogue_kernel(const SpmmArgs a) {
  constexpr int LPR = D / 8;
  constexpr int RPW = 32 / LPR;
  constexpr int HALF = D / 2;
  const int lane = threadIdx.x & 31;
  const int grp = lane / LPR;
  const int gl = lane % LPR;
  const int warp0 = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int n_items = (a.n_rows + RPW - 1) / RPW;
  pdl_wait();
  pdl_trigger();
  for (int item = warp0; item < n_items; item += nwarps) {
    const int row = item * RPW + grp;
    const bool valid = row < a.n_rows;
    float4 acc0 = f4_zero(), acc1 = f4_zero();
    if (valid) {
      const float* src = a.X + (size_t)row * D + gl * 4;
      acc0 = a.stream ? __ldcs(reinterpret_cast<const float4*>(src)) : ldg4(src);
      acc1 = a.stream ? __ldcs(reinterpret_cast<const float4*>(src + HALF)) : ldg4(src + HALF);
    }
    spmm_epilogue<D>(a, row, gl, acc0, acc1, valid);
  }
}

int launch_rows_epilogue(const SpmmArgs& a, int d, cudaStream_t st) {
  if (a.n_rows <= 0) return SRB_OK;
  const int rpw = 32 / (d / 8);
  long long blocks = ((long long)(a.n_rows + rpw - 1) / rpw + 7) / 8;
  const long long cap = (long long)sm_count() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  switch (d) {
    case 16: return launch_kernel(rows_epilogue_kernel<16>, (int)blocks, 256, 0, st, "rows_epilogue_kernel", a);
    case 32: return launch_kernel(rows_epilogue_kernel<32>, (int)blocks, 256, 0, st, "rows_epilogue_kernel", a);
    case 64: return launch_kernel(rows_epilogue_kernel<64>, (int)blocks, 256, 0, st, "rows_epilogue_kernel", a);
    case 128: return launch_kernel(rows_epilogue_kernel<128>, (int)blocks, 256, 0, st, "rows_epilogue_kernel", a);
    case 256: return launch_kernel(rows_epilogue_kernel<256>, (int)blocks, 256, 0, st, "rows_epilogue_kernel", a);
    default: set_error("rows_epilogue: unsupported d=%d (16, 32, 64, 128, 256)", d); return SRB_ERR_ARG;
  }
}

int launch_reduce_rows(const SpmmArgs& a, const ReduceArgs& r, int d, cudaStream_t st) {
  if (r.n_slice <= 0) return SRB_OK;
  const int rpw = 32 / (d / 8);
  long long blocks = ((long long)(r.n_slice + rpw - 1) / rpw + 7) / 8;
  const long long cap = (long long)sm_count() * (r.small_grid ? 1 : 8);
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  switch (d) {
    case 16: reduce_rows_kernel<16><<<(int)blocks, 256, 0, st>>>(a, r); break;
    case 32: reduce_rows_kernel<32><<<(int)blocks, 256, 0, st>>>(a, r); break;
    case 64: reduce_rows_kernel<64><<<(int)blocks, 256, 0, st>>>(a, r); break;
    case 128: reduce_rows_kernel<128><<<(int)blocks, 256, 0, st>>>(a, r); break;
    case 256: reduce_rows_kernel<256><<<(int)blocks, 256, 0, st>>>(a, r); break;
    default: set_error("reduce_rows: unsupported d=%d (16, 32, 64, 128, 256)", d); return SRB_ERR_ARG;
  }
  return post_launch("reduce_rows_kernel");
}

template <int D, bool M>
static int launch_spmm_dma(const SpmmArgs& a, int hub_blocks, int blocks, cudaStream_t st) {
  if (hub_blocks > 0) {
    if (a.seg && a.n_warp > 0) {
      const int wb = max(1, min((a.n_warp + 7) / 8, blocks));
      SRB_TRY(launch_kernel(spmm_seg_warp_kernel<D, M>, wb, 256, 0, st, "spmm_seg_warp_kernel", a));
    }
    SRB_TRY(launch_kernel(spmm_hub_kernel<D, M>, hub_blocks, 256, 0, st, "spmm_hub_kernel", a));
    const int nh = a.n_vlong_dev ? a.n_rows : a.n_huge;  // (device-counted lists: the capacity)
    SRB_TRY(launch_kernel(spmm_hub_finish_kernel<D>, max(1, min((nh + 7) / 8, hub_blocks)), 256, 0, st, "spmm_hub_finish_kernel", a));
  }
  return launch_kernel(spmm_csr_kernel<D, M>, blocks, 256, 0, st, "spmm_csr_kernel", a);
}

template <int D>
static int launch_spmm_d(const SpmmArgs& a, int hub_blocks, int blocks, cudaStream_t st) {
  if (a.col_mask != nullptr) return launch_spmm_dma<D, true>(a, hub_blocks, blocks, st);
  return launch_spmm_dma<D, false>(a, hub_blocks, blocks, st);
}

int launch_spmm(const SpmmArgs& a, int d, cudaStream_t st) {
  if (a.n_rows == 0) return SRB_OK;
  const int threads = 256;
  const int rpw = 32 / (d / 8);
  const long long items = (long long)a.n_long + ((long long)a.n_rows - a.n_huge - a.n_vlong - a.n_long + rpw - 1) / rpw;
  long long blocks = (items + threads / 32 - 1) / (threads / 32);
  if (a.n_vlong_dev) blocks = ((long long)a.n_rows + threads / 32 - 1) / (threads / 32);  // worst case: every row long, a warp each
  if (blocks < a.n_vlong) blocks = a.n_vlong;
  const long long cap = (long long)sm_count() * 8;  // 8 x 256 threads = full residency
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  long long hub_blocks = a.seg ? (a.n_cta > 0 ? a.n_cta : (a.n_work > 0 ? 1 : 0)) : a.n_work;  // (device-counted lists: the capacity)
  if (hub_blocks > cap) hub_blocks = cap;
  switch (d) {
    case 16: return launch_spmm_d<16>(a, (int)hub_blocks, (int)blocks, st);
    case 32: return launch_spmm_d<32>(a, (int)hub_blocks, (int)blocks, st);
    case 64: return launch_spmm_d<64>(a, (int)hub_blocks, (int)blocks, st);
    case 128: return launch_spmm_d<128>(a, (int)hub_blocks, (int)blocks, st);
    case 256: return launch_spmm_d<256>(a, (int)hub_blocks, (int)blocks, st);
    default: set_error("spmm: unsupported d=%d (16, 32, 64, 128, 256)", d); return SRB_ERR_ARG;
  }
}

int fill_args(const srb_spmm_desc* d, SpmmArgs& a) {
  SRB_REQUIRE(d != nullptr, "spmm: null desc");
  SRB_REQUIRE(d->rowptr && d->colidx && d->vals && d->X, "spmm: null CSR/X pointer");
  SRB_REQUIRE(d->n_rows >= 0 && d->n_cols >= 0, "spmm: negative shape");
  SRB_REQUIRE(d->noise_mode >= 0 && d->noise_mode <= 2, "spmm: bad noise_mode");
  SRB_REQUIRE(d->noise_mode != 1 || d->noise, "spmm: noise_mode 1 needs a noise tensor");
  SRB_REQUIRE(!d->adam_p || (d->adam_m && d->adam_v && d->adam_scalars), "spmm: incomplete adam pointers");
  SRB_REQUIRE(d->X != d->Y, "spmm: Y must not alias X");
  a.rowptr = d->rowptr;
  a.colidx = d->colidx;
  a.vals = d->vals;
  a.row_order = d->row_order;
  a.n_rows = d->n_rows;
  a.n_vlong_dev = d->row_order ? d->n_vlong_dev : nullptr;
  // split rows: static lists take the counts from the desc, device-classified lists from n_vlong_dev[0] / [4]
  const bool hub = d->row_order && d->hub.n_work > 0 && (a.n_vlong_dev || d->hub.n_rows > 0);
  SRB_REQUIRE(!hub || (d->hub.first && (d->hub.work || d->hub.seg) && d->hub.part), "spmm: split-row lists incomplete");
  SRB_REQUIRE(!hub || d->hub.n_rows <= d->n_rows, "spmm: more split rows than rows");
  a.n_huge = (hub && !a.n_vlong_dev) ? d->hub.n_rows : 0;
  a.hub_first = hub ? d->hub.first : nullptr;
  a.hub_work = hub ? d->hub.work : nullptr;
  a.hub_part = hub ? d->hub.part : nullptr;
  a.n_work = hub ? d->hub.n_work : 0;
  const bool segs = hub && !a.n_vlong_dev && d->hub.seg != nullptr;
  SRB_REQUIRE(!segs || (d->hub.seg_cnt && (d->hub.n_cta == 0 || d->hub.order_cta) && (d->hub.n_warp == 0 || d->hub.order_warp)),
              "spmm: column-blocked split-row lists incomplete");
  a.seg = segs ? d->hub.seg : nullptr;
  a.seg_cnt = segs ? d->hub.seg_cnt : nullptr;
  a.order_cta = segs ? d->hub.order_cta : nullptr;
  a.order_warp = segs ? d->hub.order_warp : nullptr;
  a.n_cta = segs ? d->hub.n_cta : 0;
  a.n_warp = segs ? d->hub.n_warp : 0;
  const int rest = d->n_rows - a.n_huge;
  a.n_vlong = (d->row_order && d->n_vlong_rows > 0) ? (d->n_vlong_rows < rest ? d->n_vlong_rows : rest) : 0;
  a.col_mask = d->col_mask;
  a.n_long = (d->row_order && d->n_long_rows > 0) ? (d->n_long_rows < rest - a.n_vlong ? d->n_long_rows : rest - a.n_vlong) : 0;
  a.X = d->X;
  a.Y = d->Y;
  a.extra = d->extra;
  a.extra_scale = d->extra_scale;
  a.seed_mask = nullptr;
  a.seed = nullptr;
  a.noise_mode = d->noise_mode;
  a.noise = d->noise;
  a.eps = d->eps;
  a.pkey = make_uint2((uint32_t)d->philox_seed, (uint32_t)(d->philox_seed >> 32));
  a.poff = make_uint2((uint32_t)d->philox_offset, (uint32_t)(d->philox_offset >> 32));
  a.pstep = d->philox_step_dev;
  a.sum_in = d->sum_in;
  a.sum_add[0] = a.sum_add[1] = a.sum_add[2] = nullptr;
  a.sum_out = d->sum_out;
  a.sum_scale = d->sum_scale;
  a.ap = d->adam_p;
  a.am = d->adam_m;
  a.av = d->adam_v;
  a.ascal = d->adam_scalars;
  a.b2 = (float)d->beta2;
  a.w1 = (float)(1.0 - d->beta1);
  a.w2 = (float)(1.0 - d->beta2);
  a.aeps = d->adam_eps;
  a.world = 0;
  a.noise_row_base = 0;
  a.noise_row_stride = 1;
  a.peer_mc = 0;
  a.ps = PeerSync{};
  // (rows + columns) x d x 4 bytes of dense operands beyond 3/4 of the L2 (37.5 MB on an H100): stream the one-touch data
  a.stream = ((long long)d->n_rows + d->n_cols) * d->d * 4 > l2_bytes() / 4 * 3;
  a.stage_rank = a.stage_cap = 0;
  for (int g = 0; g < 8; ++g) a.peer[g] = a.peer_sum[g] = a.peer_p[g] = a.stage_peer[g] = nullptr;
  for (int g = 0; g < 9; ++g) a.stage_bounds[g] = 0;
  return SRB_OK;
}

int graph_args(const srb_graph_csr& g, int n_rows, int n_cols, int d, const float* X, SpmmArgs& a) {
  srb_spmm_desc p = {};
  p.rowptr = g.rowptr;
  p.colidx = g.colidx;
  p.vals = g.vals;
  p.row_order = g.row_order;
  p.n_long_rows = g.n_long_rows;
  p.n_vlong_rows = g.n_vlong_rows;
  p.hub = g.hub;
  p.n_rows = n_rows;
  p.n_cols = n_cols;
  p.d = d;
  p.X = X;
  p.extra_scale = 1.f;
  p.sum_scale = 1.f;
  return fill_args(&p, a);
}

}  // namespace srb

extern "C" int srb_spmm_csr(const srb_spmm_desc* desc, void* stream) {
  srb::SpmmArgs a;
  SRB_TRY(srb::fill_args(desc, a));
  return srb::launch_spmm(a, desc->d, (cudaStream_t)stream);
}

extern "C" int srb_spmm_epilogue_rows(const srb_spmm_desc* desc, void* stream) {
  srb::SpmmArgs a;
  SRB_TRY(srb::fill_args(desc, a));
  SRB_REQUIRE(desc->Y || desc->sum_out || desc->adam_p, "spmm_epilogue_rows: nothing to write");
  return srb::launch_rows_epilogue(a, desc->d, (cudaStream_t)stream);
}

extern "C" int srb_encoder_forward(const srb_encoder_desc* e, void* stream) {
  SRB_REQUIRE(e != nullptr, "encoder: null desc");
  SRB_REQUIRE(e->E0 && e->final_out, "encoder: null E0/final_out");
  SRB_REQUIRE(e->n_layers >= 0, "encoder: negative n_layers");
  SRB_REQUIRE(e->n_layers == 0 || (e->work0 && e->work1), "encoder: work buffers required");
  SRB_REQUIRE(e->include_ego || e->n_layers > 0, "encoder: mean over zero layers");
  SRB_REQUIRE(!e->last_rows || (e->last_rows_out && e->last_rows_out != e->final_out && e->last_rows_out != e->E0),
              "encoder: last_rows needs a separate last_rows_out buffer");
  // (with no layer, or with the last layer as the CL view, the last layer is the identity or runs in full, and the
  // mean would land in final_out instead: refused rather than leave last_rows_out unwritten)
  SRB_REQUIRE(!e->last_rows || (e->n_layers > 0 && !(e->cl_out && e->layer_cl == e->n_layers)),
              "encoder: last_rows needs n_layers >= 1 and no CL view at the last layer");
  const size_t nd = (size_t)e->n * e->d;
  cudaStream_t st = (cudaStream_t)stream;
  const int L = e->n_layers;
  if (L == 0) {  // MF: the encoder is the identity
    SRB_TRY(srb::check_cuda(cudaMemcpyAsync(e->final_out, e->E0, nd * 4, cudaMemcpyDeviceToDevice, st), "encoder copy"));
    if (e->cl_out)
      SRB_TRY(srb::check_cuda(cudaMemcpyAsync(e->cl_out, e->E0, nd * 4, cudaMemcpyDeviceToDevice, st), "encoder copy"));
    return SRB_OK;
  }
  const float inv = 1.0f / (float)(e->include_ego ? L + 1 : L);
  const bool want_cl = e->cl_out != nullptr;
  const bool cl_hit = want_cl && e->layer_cl >= 1 && e->layer_cl <= L;
  if (want_cl && !cl_hit)  // XSimGCL.py:86: default CL view is the ego embedding
    SRB_TRY(srb::check_cuda(cudaMemcpyAsync(e->cl_out, e->E0, nd * 4, cudaMemcpyDeviceToDevice, st), "encoder copy"));
  const float* x = e->E0;
  int k0 = 0;
  if (e->x1) {  // layer 1 was evaluated by the caller (shared by several encoders)
    SRB_REQUIRE(L >= 2 && !e->include_ego && !(cl_hit && e->layer_cl == 1) && e->x1 != e->work0 && e->x1 != e->work1,
                "encoder: x1 needs n_layers >= 2, include_ego == 0, layer_cl != 1 and a buffer of its own");
    x = e->x1;
    k0 = 1;
  }
  const bool last_on_rows = e->last_rows && e->n_last_rows > 0 && !(cl_hit && e->layer_cl == L);
  // Layer mean on the batch rows only: when the last layer runs on the listed rows and every earlier layer output is
  // still in a buffer of its own (cl_out, work0/1, x1: L <= 3), the full-size layers keep no running sum; the last
  // layer's epilogue adds E0 (when the ego layer counts), E1, ..., E(L-1) at its rows, in the order the running sum
  // would have (((E0 + E1) + E2) + E3), so the mean is bit-identical.
  const float* src[4];
  int n_src = 0;
  bool live = true;
  if (e->include_ego) src[n_src++] = e->E0;
  const float* px = e->E0;
  for (int k = 0; k < L - 1 && live; ++k) {  // where the loop below leaves the output of layer k + 1
    const float* py = (k == 0 && e->x1) ? e->x1 : (cl_hit && k == e->layer_cl - 1) ? e->cl_out : (px == e->work0 ? e->work1 : e->work0);
    for (int j = 0; j < n_src; ++j) live = live && src[j] != py;
    live = live && n_src < 4;
    if (live) src[n_src++] = py;
    px = py;
  }
  const bool batch_mean = last_on_rows && live;
  for (int k = k0; k < L; ++k) {
    srb_spmm_desc s = {};
    s.rowptr = e->rowptr;
    s.colidx = e->colidx;
    s.vals = e->vals;
    s.row_order = e->row_order;
    s.n_long_rows = e->n_long_rows;
    s.n_vlong_rows = e->n_vlong_rows;
    s.hub = e->hub;
    s.n_rows = e->n;
    s.n_cols = e->n;
    s.d = e->d;
    s.X = x;
    const bool last = (k == L - 1);
    float* y = nullptr;
    if (cl_hit && k == e->layer_cl - 1) y = e->cl_out;  // this layer's output is the CL view
    else if (!last) y = (x == e->work0) ? e->work1 : e->work0;
    s.Y = y;
    s.noise_mode = e->noise_mode;
    if (e->noise_mode == 1) s.noise = e->noise + (size_t)k * nd;
    s.eps = e->eps;
    s.philox_seed = e->philox_seed;
    s.philox_offset = e->philox_offset + (uint64_t)k;
    s.philox_step_dev = e->philox_step_dev;
    // running sum lives in final_out; layer 1 seeds it (with E0 when the ego layer counts)
    s.sum_in = (k == 0) ? (e->include_ego ? e->E0 : nullptr) : ((k == 1 && e->x1) ? e->x1 : e->final_out);
    s.sum_out = (batch_mean && !last) ? nullptr : e->final_out;
    s.sum_scale = last ? inv : 1.0f;
    if (batch_mean && last) s.sum_in = n_src ? src[0] : nullptr;
    if (last && last_on_rows) {
      // only the listed rows of the final mean are consumed: one warp per listed row
      s.row_order = e->last_rows;
      s.n_rows = e->n_last_rows;
      if (e->last_rows_nv_dev) {  // list classified on the device: four segments of n_last_rows entries
        s.n_vlong_rows = 0;
        s.n_long_rows = 0;
        s.n_vlong_dev = e->last_rows_nv_dev;
        s.hub = e->last_rows_hub;
      } else {
        s.n_vlong_rows = e->n_last_rows;  // unsorted, degree-biased rows: a CTA per listed row
        s.n_long_rows = 0;
        s.hub = srb_hub_split{};
      }
      s.Y = nullptr;
      s.sum_out = e->last_rows_out;  // out of place: duplicates in the list stay idempotent
    }
    srb::SpmmArgs a;
    SRB_TRY(srb::fill_args(&s, a));
    if (batch_mean && last)
      for (int j = 1; j < n_src; ++j) a.sum_add[j - 1] = src[j];
    SRB_TRY(srb::launch_spmm(a, s.d, st));
    x = y;
  }
  return SRB_OK;
}
