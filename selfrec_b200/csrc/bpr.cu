// (ii) Fused (u,i,j) gather + BPR + L2 forward/backward, sparse-row scatter, Adam.
//
// Replaces, for one batch of triples:
//   rec_user_emb[user_idx], rec_item_emb[pos_idx], rec_item_emb[neg_idx]   XSimGCL.py:30 & peers
//   bpr_loss      util/loss_torch.py:6-10   mean(-log(10e-6 + sigmoid(<u,p> - <u,n>)))
//   l2_reg_loss   util/loss_torch.py:18-22  reg * sum_e ||e||_F / e.shape[0]   (NOT squared)
// and their autograd backward (gather backward = index_put_ accumulate -> srb_scatter_add_rows).
// One warp per triple; warp-shuffle reductions; two launches because the Frobenius norm
// must be complete before its gradient can be formed.
#include "common.cuh"

namespace srb {

struct BprArgs {
  const float* emb;
  const float* l2_emb;
  int32_t n_users;
  const int32_t* u_idx;
  const int32_t* i_idx;
  const int32_t* j_idx;
  const int32_t* b_dev;
  int32_t b;
  float emb_scale;
  float reg;
  int32_t l2_terms;
  float l2_div;
  float grad_scale;
  float* losses;
  float* g_emb;
  float* g_l2;
  float* scratch;  // [0]=sum bpr, [1..3]=sum of squares of l2 rows (u, p, n)
};

template <int D>
__device__ __forceinline__ void load_row(const float* base, int row, int lane, float scale, float4 (&r)[(D + 127) / 128]) {
#pragma unroll
  for (int q = 0; q < (D + 127) / 128; ++q) {
    const int c = lane * 4 + q * 128;
    r[q] = (c < D) ? f4_scale(scale, ldg4(base + (size_t)row * D + c)) : f4_zero();
  }
}

template <int D>
__global__ void __launch_bounds__(256) bpr_reduce_kernel(const BprArgs a) {
  constexpr int Q = (D + 127) / 128;
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int t = blockIdx.x * (blockDim.x >> 5) + wib;
  pdl_wait();
  pdl_trigger();
  const int b = a.b_dev ? min(*a.b_dev, a.b) : a.b;
  float bpr = 0.f, su = 0.f, sp = 0.f, sn = 0.f;
  if (t < b) {
    const int u = a.u_idx[t], p = a.n_users + a.i_idx[t], n = a.n_users + a.j_idx[t];
    float4 ru[Q], rp[Q], rn[Q];
    load_row<D>(a.emb, u, lane, a.emb_scale, ru);
    load_row<D>(a.emb, p, lane, a.emb_scale, rp);
    load_row<D>(a.emb, n, lane, a.emb_scale, rn);
    float pos = 0.f, neg = 0.f;
#pragma unroll
    for (int q = 0; q < Q; ++q) {
      pos += f4_dot(ru[q], rp[q]);
      neg += f4_dot(ru[q], rn[q]);
    }
    pos = warp_sum(pos);
    neg = warp_sum(neg);
    if (a.l2_emb != a.emb) {
      load_row<D>(a.l2_emb, u, lane, 1.f, ru);
      load_row<D>(a.l2_emb, p, lane, 1.f, rp);
      load_row<D>(a.l2_emb, n, lane, 1.f, rn);
    }
#pragma unroll
    for (int q = 0; q < Q; ++q) {
      su += f4_dot(ru[q], ru[q]);
      sp += f4_dot(rp[q], rp[q]);
      sn += f4_dot(rn[q], rn[q]);
    }
    su = warp_sum(su);
    sp = warp_sum(sp);
    sn = warp_sum(sn);
    const float x = pos - neg;
    const float sig = 1.f / (1.f + expf(-x));
    bpr = -logf(1e-5f + sig);  // 10e-6 in the reference
  }
  __shared__ float red[8][4];
  if (lane == 0) {
    red[wib][0] = bpr;
    red[wib][1] = su;
    red[wib][2] = sp;
    red[wib][3] = sn;
  }
  __syncthreads();
  if (threadIdx.x < 4) {
    float s = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w][threadIdx.x];
    atomicAdd(a.scratch + threadIdx.x, s);
  }
}

template <int D>
__global__ void __launch_bounds__(256) bpr_grad_kernel(const BprArgs a) {
  constexpr int Q = (D + 127) / 128;
  const int lane = threadIdx.x & 31;
  const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  pdl_wait();
  pdl_trigger();
  const int b = a.b_dev ? min(*a.b_dev, a.b) : a.b;
  const float fb = (float)b;
  const float nu = sqrtf(a.scratch[1]), np = sqrtf(a.scratch[2]), nn = sqrtf(a.scratch[3]);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    a.losses[0] = (b > 0) ? a.scratch[0] / fb : 0.f;
    float l2 = nu + np + (a.l2_terms >= 3 ? nn : 0.f);
    a.losses[1] = (b > 0) ? a.reg * (l2 / fb) / a.l2_div : 0.f;
  }
  if (t >= b) return;
  const int u = a.u_idx[t], p = a.n_users + a.i_idx[t], n = a.n_users + a.j_idx[t];
  float4 ru[Q], rp[Q], rn[Q];
  load_row<D>(a.emb, u, lane, a.emb_scale, ru);
  load_row<D>(a.emb, p, lane, a.emb_scale, rp);
  load_row<D>(a.emb, n, lane, a.emb_scale, rn);
  float pos = 0.f, neg = 0.f;
#pragma unroll
  for (int q = 0; q < Q; ++q) {
    pos += f4_dot(ru[q], rp[q]);
    neg += f4_dot(ru[q], rn[q]);
  }
  pos = warp_sum(pos);
  neg = warp_sum(neg);
  const float x = pos - neg;
  const float sig = 1.f / (1.f + expf(-x));
  // d/dx of -log(1e-5 + sigmoid(x)), averaged over the batch
  const float c = a.grad_scale * (-(sig * (1.f - sig)) / (1e-5f + sig)) / fb;
  // d/de of reg * ||e||_F / b / l2_div  =  reg / (b * l2_div) * e / ||e||_F   (0 at the origin)
  const float k2 = a.grad_scale * a.reg / (fb * a.l2_div);
  const float ku = nu > 0.f ? k2 / nu : 0.f;
  const float kp = np > 0.f ? k2 / np : 0.f;
  const float kn = (a.l2_terms >= 3 && nn > 0.f) ? k2 / nn : 0.f;
  const bool l2_sep = (a.g_l2 != nullptr);
  float4 lu[Q], lp[Q], ln[Q];
  if (a.l2_emb != a.emb) {
    load_row<D>(a.l2_emb, u, lane, 1.f, lu);
    load_row<D>(a.l2_emb, p, lane, 1.f, lp);
    load_row<D>(a.l2_emb, n, lane, 1.f, ln);
  } else {
#pragma unroll
    for (int q = 0; q < Q; ++q) lu[q] = ru[q], lp[q] = rp[q], ln[q] = rn[q];
  }
  const size_t plane = (size_t)a.b * D;
#pragma unroll
  for (int q = 0; q < Q; ++q) {
    const int col = lane * 4 + q * 128;
    if (col >= D) continue;
    float4 gu = make_float4(c * (rp[q].x - rn[q].x), c * (rp[q].y - rn[q].y), c * (rp[q].z - rn[q].z), c * (rp[q].w - rn[q].w));
    float4 gp = f4_scale(c, ru[q]);
    float4 gn = f4_scale(-c, ru[q]);
    const float4 l2u = f4_scale(ku, lu[q]), l2p = f4_scale(kp, lp[q]), l2n = f4_scale(kn, ln[q]);
    const size_t o = (size_t)t * D + col;
    if (l2_sep) {
      st4(a.g_l2 + o, l2u);
      st4(a.g_l2 + plane + o, l2p);
      st4(a.g_l2 + 2 * plane + o, l2n);
    } else {
      gu = f4_add(gu, l2u);
      gp = f4_add(gp, l2p);
      gn = f4_add(gn, l2n);
    }
    st4(a.g_emb + o, gu);
    st4(a.g_emb + plane + o, gp);
    st4(a.g_emb + 2 * plane + o, gn);
  }
}

// SPLIT: some segment lists users and items together (ScatterSeg.item_min); without it the kernel is the plain scatter
template <int D, bool SPLIT>
__global__ void __launch_bounds__(256) scatter_add_rows_kernel(float* dst, const ScatterSegs segs) {
  const ScatterSeg& sg = segs.s[blockIdx.y];
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  pdl_wait();
  pdl_trigger();
  const int nn = sg.n_dev ? min(*sg.n_dev, sg.n) : sg.n;
  if (r >= nn) return;
  int row = sg.rows[r];
  if (SPLIT && sg.item_min > 0 && row >= sg.item_min) {
    row += sg.item_off - sg.item_min;  // an item row of a mixed user / item list: every rank keeps the complete item table
  } else {
    row += sg.row_off;
    if (sg.mod > 0) {  // cyclic ownership (bipartite sharding: user u lives on rank u % world, local row u / world)
      if (row % sg.mod != sg.rem) return;
      row /= sg.mod;
    }
  }
  for (int c = lane * 4; c < D; c += 128) {
    const float4 v = f4_scale(sg.scale, ldg4(sg.src + (size_t)r * D + c));
    atomicAdd(reinterpret_cast<float4*>(dst + (size_t)row * D + c), v);  // red.global.add.v4.f32 (sm_90+)
  }
}

int scatter_segments(float* dst, int d, const ScatterSegs& segs, cudaStream_t st) {
  if (segs.count == 0) return SRB_OK;
  int max_n = 0;
  for (int q = 0; q < segs.count; ++q) max_n = segs.s[q].n > max_n ? segs.s[q].n : max_n;
  if (max_n == 0) return SRB_OK;
  bool split = false;
  for (int q = 0; q < segs.count; ++q) split = split || segs.s[q].item_min > 0;
  dim3 grid((max_n + 7) / 8, segs.count);
#define SRB_SCATTER(D)                                                                                                            \
  return split ? launch_kernel(scatter_add_rows_kernel<D, true>, grid, 256, 0, st, "scatter_add_rows_kernel", dst, segs)        \
               : launch_kernel(scatter_add_rows_kernel<D, false>, grid, 256, 0, st, "scatter_add_rows_kernel", dst, segs);
  switch (d) {
    case 16: SRB_SCATTER(16)
    case 32: SRB_SCATTER(32)
    case 64: SRB_SCATTER(64)
    case 128: SRB_SCATTER(128)
    case 256: SRB_SCATTER(256)
    default: set_error("scatter: unsupported d=%d (16, 32, 64, 128, 256)", d); return SRB_ERR_ARG;
  }
#undef SRB_SCATTER
}

// Standalone l2_reg_loss (util/loss_torch.py:18-22) for the op-level drop-in, where the
// embeddings arrive already gathered: sumsq[t] = ||e_t||_F^2 (atomic), then
// loss = reg * sum_t sqrt(sumsq[t]) / rows_t and grad_t = g * reg / rows_t * e_t / ||e_t||_F.
struct L2Args {
  int n_terms;
  const float* x[4];
  float* g[4];
  long long n[4];   // elements
  int rows[4];
};

__global__ void __launch_bounds__(256) l2_sumsq_kernel(const L2Args a, float* sumsq) {
  const int t = blockIdx.y;
  const long long n = a.n[t];
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = a.x[t][i];
    acc = fmaf(v, v, acc);
  }
  acc = warp_sum(acc);
  __shared__ float red[8];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
    atomicAdd(sumsq + t, s);
  }
}

__global__ void l2_loss_kernel(const L2Args a, const float* sumsq, float reg, float* loss) {
  float l = 0.f;
  for (int t = 0; t < a.n_terms; ++t) l += sqrtf(sumsq[t]) / (float)a.rows[t];
  *loss = l * reg;
}

__global__ void __launch_bounds__(256) l2_grad_kernel(const L2Args a, const float* sumsq, float reg, const float* gout) {
  const int t = blockIdx.y;
  const long long n = a.n[t];
  const float nrm = sqrtf(sumsq[t]);
  const float k = (nrm > 0.f) ? (*gout) * reg / ((float)a.rows[t] * nrm) : 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    a.g[t][i] = k * a.x[t][i];
}

__global__ void adam_prepare_kernel(int32_t* step, float* scalars, double lr, double b1, double b2) {
  adam_prepare(step, scalars, lr, b1, b2);
}

__global__ void __launch_bounds__(256) adam_step_kernel(float* __restrict__ p, float* __restrict__ m, float* __restrict__ v,
                                                        const float* __restrict__ g, long long n4, long long n,
                                                        const float* __restrict__ scal, float w1, float b2, float w2, float eps) {
  pdl_wait();
  pdl_trigger();
  const float step_size = scal[0], bc2_sqrt = scal[1];
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 pp = reinterpret_cast<float4*>(p)[i], mm = reinterpret_cast<float4*>(m)[i], vv = reinterpret_cast<float4*>(v)[i];
    const float4 gg = reinterpret_cast<const float4*>(g)[i];
#define SRB_ADAM1(F) adam_elem(pp.F, mm.F, vv.F, gg.F, step_size, bc2_sqrt, w1, b2, w2, eps);
    SRB_ADAM1(x) SRB_ADAM1(y) SRB_ADAM1(z) SRB_ADAM1(w)
#undef SRB_ADAM1
    reinterpret_cast<float4*>(p)[i] = pp;
    reinterpret_cast<float4*>(m)[i] = mm;
    reinterpret_cast<float4*>(v)[i] = vv;
  }
  // scalar tail (n not a multiple of 4)
  for (long long i = n4 * 4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    float pp = p[i], mm = m[i], vv = v[i];
    adam_elem(pp, mm, vv, g[i], step_size, bc2_sqrt, w1, b2, w2, eps);
    p[i] = pp;
    m[i] = mm;
    v[i] = vv;
  }
}

}  // namespace srb

extern "C" int srb_bpr_l2_fwd_bwd(const srb_bpr_desc* d, void* stream) {
  SRB_REQUIRE(d != nullptr, "bpr: null desc");
  SRB_REQUIRE(d->emb && d->u_idx && d->i_idx && d->j_idx && d->losses && d->g_emb && d->scratch, "bpr: null pointer");
  SRB_REQUIRE(d->l2_terms == 2 || d->l2_terms == 3, "bpr: l2_terms must be 2 or 3");
  SRB_REQUIRE(d->b >= 0, "bpr: negative batch");
  SRB_REQUIRE(d->l2_div > 0.f, "bpr: l2_div must be positive");
  srb::BprArgs a;
  a.emb = d->emb;
  a.l2_emb = d->l2_emb ? d->l2_emb : d->emb;
  SRB_REQUIRE(a.l2_emb == a.emb || d->g_l2, "bpr: a separate l2 table needs g_l2");
  a.n_users = d->n_users;
  a.u_idx = d->u_idx;
  a.i_idx = d->i_idx;
  a.j_idx = d->j_idx;
  a.b_dev = d->b_dev;
  a.b = d->b;
  a.emb_scale = d->emb_scale;
  a.reg = d->reg;
  a.l2_terms = d->l2_terms;
  a.l2_div = d->l2_div;
  a.grad_scale = d->grad_scale;
  a.losses = d->losses;
  a.g_emb = d->g_emb;
  a.g_l2 = d->g_l2;
  a.scratch = d->scratch;
  cudaStream_t st = (cudaStream_t)stream;
  SRB_TRY(srb::check_cuda(cudaMemsetAsync(d->scratch, 0, 8 * sizeof(float), st), "bpr memset"));
  const int blocks = d->b > 0 ? (d->b + 7) / 8 : 1;
  switch (d->d) {
#define SRB_CASE(DD)                                                                                 \
  case DD:                                                                                           \
    SRB_TRY(srb::launch_kernel(srb::bpr_reduce_kernel<DD>, blocks, 256, 0, st, "bpr_reduce_kernel", a)); \
    return srb::launch_kernel(srb::bpr_grad_kernel<DD>, blocks, 256, 0, st, "bpr_grad_kernel", a);
    SRB_CASE(16)
    SRB_CASE(32)
    SRB_CASE(64)
    SRB_CASE(128)
    SRB_CASE(256)
#undef SRB_CASE
    default: srb::set_error("bpr: unsupported d=%d (16, 32, 64, 128, 256)", d->d); return SRB_ERR_ARG;
  }
}

extern "C" int srb_scatter_add_rows(float* dst, int32_t d, const float* src, const int32_t* rows, int32_t n,
                                    const int32_t* n_dev, int32_t row_off, float scale, void* stream) {
  SRB_REQUIRE(dst && src && rows, "scatter: null pointer");
  SRB_REQUIRE(n >= 0, "scatter: negative n");
  srb::ScatterSegs segs;
  segs.count = 1;
  segs.s[0] = {src, rows, n_dev, n, row_off, scale};
  return srb::scatter_segments(dst, d, segs, (cudaStream_t)stream);
}

extern "C" int srb_scatter_add_segments(float* dst, int32_t d, int32_t n_segs, const srb_scatter_seg* in, void* stream) {
  SRB_REQUIRE(dst && in, "scatter: null pointer");
  SRB_REQUIRE(n_segs >= 0 && n_segs <= 8, "scatter: 0..8 segments per launch");
  srb::ScatterSegs segs;
  segs.count = n_segs;
  for (int q = 0; q < n_segs; ++q) {
    SRB_REQUIRE(in[q].src && in[q].rows && in[q].n >= 0, "scatter: bad segment %d", q);
    segs.s[q] = {in[q].src, in[q].rows, in[q].n_dev, in[q].n, in[q].row_off, in[q].scale};
  }
  return srb::scatter_segments(dst, d, segs, (cudaStream_t)stream);
}

extern "C" int srb_adam_prepare(int32_t* step_dev, float* scalars_dev, double lr, double beta1, double beta2, void* stream) {
  SRB_REQUIRE(step_dev && scalars_dev, "adam_prepare: null pointer");
  srb::adam_prepare_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(step_dev, scalars_dev, lr, beta1, beta2);
  return srb::post_launch("adam_prepare_kernel");
}

extern "C" int srb_adam_step(float* p, float* m, float* v, const float* g, int64_t n, const float* scalars_dev, double beta1,
                             double beta2, float eps, void* stream) {
  SRB_REQUIRE(p && m && v && g && scalars_dev, "adam_step: null pointer");
  SRB_REQUIRE(n >= 0, "adam_step: negative n");
  if (n == 0) return SRB_OK;
  const long long n4 = (((uintptr_t)p | (uintptr_t)m | (uintptr_t)v | (uintptr_t)g) & 15) ? 0 : n / 4;
  long long blocks = (n4 + 255) / 256;
  const long long cap = (long long)srb::sm_count() * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return srb::launch_kernel(srb::adam_step_kernel, (int)blocks, 256, 0, (cudaStream_t)stream, "adam_step_kernel", p, m, v, g, n4, n,
                            scalars_dev, (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), eps);
}

extern "C" int srb_l2_reg_fwd(int32_t n_terms, const float* const* x, const int64_t* n_elems, const int32_t* rows, float reg,
                              float* sumsq_dev, float* loss_dev, void* stream) {
  SRB_REQUIRE(n_terms >= 1 && n_terms <= 4, "l2_reg: 1..4 terms");
  SRB_REQUIRE(x && n_elems && rows && sumsq_dev && loss_dev, "l2_reg: null pointer");
  srb::L2Args a = {};
  a.n_terms = n_terms;
  long long mx = 1;
  for (int t = 0; t < n_terms; ++t) {
    SRB_REQUIRE(x[t] && rows[t] > 0 && n_elems[t] >= 0, "l2_reg: bad term %d", t);
    a.x[t] = x[t];
    a.n[t] = n_elems[t];
    a.rows[t] = rows[t];
    if (n_elems[t] > mx) mx = n_elems[t];
  }
  cudaStream_t st = (cudaStream_t)stream;
  SRB_TRY(srb::check_cuda(cudaMemsetAsync(sumsq_dev, 0, 4 * sizeof(float), st), "l2 memset"));
  long long bx = (mx + 255) / 256;
  if (bx > 1024) bx = 1024;
  srb::l2_sumsq_kernel<<<dim3((unsigned)bx, n_terms), 256, 0, st>>>(a, sumsq_dev);
  SRB_TRY(srb::post_launch("l2_sumsq_kernel"));
  srb::l2_loss_kernel<<<1, 1, 0, st>>>(a, sumsq_dev, reg, loss_dev);
  return srb::post_launch("l2_loss_kernel");
}

extern "C" int srb_l2_reg_bwd(int32_t n_terms, const float* const* x, float* const* g, const int64_t* n_elems,
                              const int32_t* rows, float reg, const float* sumsq_dev, const float* gout_dev, void* stream) {
  SRB_REQUIRE(n_terms >= 1 && n_terms <= 4, "l2_reg: 1..4 terms");
  SRB_REQUIRE(x && g && n_elems && rows && sumsq_dev && gout_dev, "l2_reg: null pointer");
  srb::L2Args a = {};
  a.n_terms = n_terms;
  long long mx = 1;
  for (int t = 0; t < n_terms; ++t) {
    SRB_REQUIRE(x[t] && g[t] && rows[t] > 0, "l2_reg: bad term %d", t);
    a.x[t] = x[t];
    a.g[t] = g[t];
    a.n[t] = n_elems[t];
    a.rows[t] = rows[t];
    if (n_elems[t] > mx) mx = n_elems[t];
  }
  long long bx = (mx + 255) / 256;
  if (bx > 1024) bx = 1024;
  srb::l2_grad_kernel<<<dim3((unsigned)bx, n_terms), 256, 0, (cudaStream_t)stream>>>(a, sumsq_dev, reg, gout_dev);
  return srb::post_launch("l2_grad_kernel");
}
