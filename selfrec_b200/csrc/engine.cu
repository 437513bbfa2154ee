// One whole training step as a single stream-ordered call (graph-capturable).
//
// Replaces the body of the batch loop of <Model>.train():
//   MF.py:17-25  LightGCN.py:21-29  SimGCL.py:25-36  XSimGCL.py:27-37  SGL.py:30-41
// i.e. encoder forward (R4) -> gather + BPR + L2 (R5-R7) -> InfoNCE (R8) -> autograd
// backward -> Adam (R10).
//
// Backward through the propagation uses the fact that every encoder is linear in E0 and the
// SimGCL/XSimGCL noise has zero gradient (sign() and the noise are constants):
//   final = c * sum_k A^k E0   =>   dE0 = c * sum_k A^k G      (A symmetric)
// evaluated by Horner's rule with L SpMMs and no saved activations; the row-sparse loss
// gradients G (<= 3B + 2B rows) are scattered once into [N, d] seed tables that hold data only
// at the batch rows, and each Horner level adds its table in the SpMM epilogue (run_chain).
// SimGCL's three encoders share A, so their three backward chains collapse into one.  The last
// SpMM applies Adam in its epilogue.
#include <stdlib.h>
#include <algorithm>
#include <mutex>
#include "spmm_args.cuh"

namespace srb {

// SRB_PDL=0 launches the step's kernels without programmatic dependent launch (measurement switch, same results)
static bool pdl_enabled() {
  static const bool on = [] {
    const char* e = getenv("SRB_PDL");
    return !(e && e[0] == '0');
  }();
  return on;
}

static thread_local bool t_pdl = false;
bool pdl_active() { return t_pdl; }

// PDL for the launches of one srb_train_step call on this thread (the sharded step and the standalone ops launch
// without it)
struct PdlScope {
  PdlScope() { t_pdl = pdl_enabled(); }
  ~PdlScope() { t_pdl = false; }
};

struct Ws {
  float* final_;  // [N,d] main encoder output
  float* cl;      // [N,d] XSimGCL CL view / SimGCL,SGL view-1 output
  float* v2;      // [N,d] SimGCL,SGL view-2 output
  float* work0;
  float* work1;
  float* acc0;
  float* acc1;
  float* gd;      // [N,d] SimGCL: view 2's first layer (L >= 2); SGL: the sum of the two view chains
  float* rsum;    // running layer sum of the encoder being evaluated (training forwards)
  float* seed;    // [n_seed][N,d] backward seed tables (see run_chain); valid at batch rows only
  int32_t n_seed; // LightGCN, XSimGCL: F | G; SimGCL: F; SGL: F of the encoders on adj_view[0] | adj_view[1] | adj
  float* g_emb;   // [3,B,d]
  float* g_l2;    // [3,B,d]
  float* g_nce;   // 4 x [2B,d]
  float* bpr_scratch;  // [8]
  float* bpr_losses;   // [2]
  float* nce_losses;   // [4]
  int32_t* idx_cat;    // [2B] SGL concatenated unique ids
  int32_t* n_cat;      // [1]
  int32_t* batch_rows; // [4][3B] distinct table rows of the batch (u, U+i, U+j) by class: split, CTA, warp, lane group
  int32_t* n_hub;      // [8] rows per class [0..3], chunks of the split rows [4]
  uint32_t* row_mask;  // [(N+31)/32] bitmap of the batch's table rows (the rows the gradient seed touches)
  int32_t* hub_first;  // [3B] first chunk slot of each split batch row
  int32_t* hub_work;   // [hub_cap][2]
  float* hub_part;     // [hub_cap, d]
  int32_t hub_cap;
  void* nce_ws;
  int64_t nce_ws_bytes;
};

static int64_t al(int64_t x) { return (x + 255) / 256 * 256; }

static int64_t carve(const srb_step_desc* s, Ws* w, char* base) {
  const int64_t N = (int64_t)s->n_users + s->n_items, d = s->d, B = s->batch_cap;
  const int64_t nd = al(N * d * 4);
  int64_t off = 0;
  auto take = [&](int64_t bytes) {
    char* p = base ? base + off : nullptr;
    off += al(bytes);
    return p;
  };
  const bool graph = s->model != SRB_MODEL_MF;
  const bool two_views = s->model == SRB_MODEL_SIMGCL || s->model == SRB_MODEL_SGL;
  const bool has_cl = s->model == SRB_MODEL_XSIMGCL || two_views;
  const int n_seed = s->model == SRB_MODEL_SGL ? 3 : (s->model == SRB_MODEL_SIMGCL ? 1 : (graph ? 2 : 0));
  // the small per-step buffers first, at offsets that do not depend on which [N, d] tables the model has: behind the
  // tables, one table less moved them and made the yelp2018 XSimGCL step 0.7 us slower (H100 80GB HBM3, 700 W)
  float* f_gemb = (float*)take(3 * B * d * 4);
  float* f_gl2 = (float*)take(3 * B * d * 4);
  float* f_gnce = (float*)take(has_cl ? 4 * 2 * B * d * 4 : 0);
  float* f_bs = (float*)take(8 * 4);
  float* f_bl = (float*)take(2 * 4);
  float* f_nl = (float*)take(4 * 4);
  int32_t* i_cat = (int32_t*)take(2 * B * 4);
  int32_t* i_ncat = (int32_t*)take(4);
  int32_t* i_brows = (int32_t*)take(4 * 3 * B * 4);
  // [class counters (8 words) | row bitmap]: one memset clears all of it
  int32_t* i_nhub = (int32_t*)take(graph ? 32 + ((N + 31) / 32) * 4 : 32);
  uint32_t* u_mask = (uint32_t*)(i_nhub + 8);
  const int64_t hub_cap = graph ? s->adj.hub.n_work : 0;  // distinct batch rows: never more chunks than the whole graph has
  int32_t* i_hfirst = (int32_t*)take(hub_cap ? 3 * B * 4 : 0);
  int32_t* i_hwork = (int32_t*)take(hub_cap * 2 * 4);
  float* f_hpart = (float*)take(hub_cap * d * 4);
  const int64_t nws = has_cl ? srb_infonce_workspace_bytes((int32_t)(2 * B), (int32_t)d, 2) : 0;
  void* v_nws = take(nws);
  float* f_final = (float*)take(graph ? nd : 0);
  float* f_cl = (float*)take(has_cl ? nd : 0);
  float* f_v2 = (float*)take(two_views ? nd : 0);
  float* f_w0 = (float*)take(graph ? nd : 0);
  float* f_w1 = (float*)take(graph ? nd : 0);
  float* f_a0 = (float*)take(nd);
  float* f_a1 = (float*)take(graph ? nd : 0);
  float* f_gd = (float*)take(two_views ? nd : 0);
  float* f_rsum = (float*)take(graph ? nd : 0);
  float* f_seed = (float*)take(n_seed * nd);
  if (w) {
    w->final_ = f_final;
    w->cl = f_cl;
    w->v2 = f_v2;
    w->work0 = f_w0;
    w->work1 = f_w1;
    w->acc0 = f_a0;
    w->acc1 = f_a1;
    w->gd = f_gd;
    w->rsum = f_rsum;
    w->seed = f_seed;
    w->n_seed = n_seed;
    w->g_emb = f_gemb;
    w->g_l2 = f_gl2;
    w->g_nce = f_gnce;
    w->bpr_scratch = f_bs;
    w->bpr_losses = f_bl;
    w->nce_losses = f_nl;
    w->idx_cat = i_cat;
    w->n_cat = i_ncat;
    w->batch_rows = i_brows;
    w->n_hub = i_nhub;
    w->row_mask = u_mask;
    w->hub_first = i_hfirst;
    w->hub_work = i_hwork;
    w->hub_part = f_hpart;
    w->hub_cap = (int32_t)hub_cap;
    w->nce_ws = v_nws;
    w->nce_ws_bytes = nws;
  }
  return off;
}

// SGL: one InfoNCE over cat(users, items) (SGL.py:120-125) needs one combined id list.
__global__ void build_cat_idx_kernel(const int32_t* batch, int cap, int n_users, int32_t* idx_cat, int32_t* n_cat) {
  pdl_wait();
  pdl_trigger();
  const int nu = min(batch[1], cap), ni = min(batch[2], cap);
  const int32_t* uu = batch + SRB_BATCH_HEADER + 3 * cap;
  const int32_t* ui = uu + cap;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < nu + ni; t += gridDim.x * blockDim.x)
    idx_cat[t] = (t < nu) ? uu[t] : n_users + ui[t - nu];
  if (blockIdx.x == 0 && threadIdx.x == 0) *n_cat = nu + ni;
}

// rows of the [N, d] tables a batch touches: u, U + i, U + j, each listed ONCE (the bitmap de-duplicates: a hub user
// sits in a batch many times) and classified by degree for the last-layer SpMM into four segments of capacity 3*cap
// (list_batch_row).  counters[0..7] and row_mask are zeroed by step_begin_kernel.
__global__ void __launch_bounds__(256) build_batch_rows_kernel(const int32_t* batch, int cap, int n_users, const int32_t* rowptr,
                                                               int32_t* rows, int32_t* counters, uint32_t* row_mask,
                                                               int32_t* hub_first, int32_t* hub_work, int hub_cap) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  pdl_wait();
  pdl_trigger();
  const int b = min(batch[0], cap);
  const int sec = t / cap, k = t % cap;
  if (sec >= 3 || k >= b) return;
  const int32_t* u = batch + SRB_BATCH_HEADER;
  const int row = (sec == 0) ? u[k] : n_users + u[sec * cap + k];
  const uint32_t bit = 1u << (row & 31);
  if (atomicOr(row_mask + (row >> 5), bit) & bit) return;  // listed already
  list_batch_row(row, rowptr[row + 1] - rowptr[row], 0, rows, 3 * cap, counters, hub_first, hub_work, hub_cap);
}

// first kernel of a graph model's step (both training steps): Adam's bias corrections, n_words words cleared (the
// batch-row counters + bitmaps), and the batch rows u, i, j of the first n_seed seed tables cleared where the seed
// scatter puts them (layout r), a float4 per thread (duplicates only repeat a store).  One node instead of a kernel and
// two memsets.  OWNED: r has cyclic user ownership (r.user_mod > 0: the sharded step).  A compile-time switch: with the
// ownership test and division behind a runtime flag, the single-GPU step's kernel took 3.26 us instead of 2.88 us
// (yelp2018 XSimGCL, H100 80GB HBM3, 700 W).
template <bool OWNED>
__global__ void __launch_bounds__(256) step_begin_kernel(int32_t* step, float* scalars, double lr, double b1, double b2, int32_t* words,
                                                         int n_words, const int32_t* batch, int cap, int d, float* seed, int n_seed,
                                                         const SeedRows r) {
  pdl_wait();
  pdl_trigger();
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t == 0) adam_prepare(step, scalars, lr, b1, b2);
  if (t < n_words) words[t] = 0;
  const int k0 = t / (d / 4), c = (t % (d / 4)) * 4;
  const int sec = k0 / cap, k = k0 % cap;
  if (sec >= 3 || k >= min(batch[0], cap)) return;
  const int id = batch[SRB_BATCH_HEADER + sec * cap + k];
  const bool owned = OWNED && sec == 0;  // local row (id + user_off) / user_mod
  if (owned && id % r.user_mod != r.user_rem) return;  // another rank's user
  for (int q = 0; q < n_seed; ++q) {
    const int row = id + (sec == 0 ? r.user_off[q] : r.item_off[q]);
    st4(seed + (size_t)(owned ? row / r.user_mod : row) * d + c, f4_zero());
  }
}

int step_begin(int32_t* step, float* scalars, double lr, double b1, double b2, int32_t* words, int n_words, const int32_t* batch, int cap,
               int d, float* seed, int n_seed, const SeedRows& r, cudaStream_t st) {
  const int threads = std::max(n_words, 3 * cap * (d / 4));
  return launch_kernel(r.user_mod > 0 ? step_begin_kernel<true> : step_begin_kernel<false>, (threads + 255) / 256, 256, 0, st,
                       "step_begin_kernel", step, scalars, lr, b1, b2, words, n_words, batch, cap, d, seed, n_seed, r);
}

__global__ void finalize_losses_kernel(const float* bpr_losses, const float* nce_losses, int n_nce, float cl_rate, float* out) {
  pdl_wait();
  pdl_trigger();
  float cl = 0.f;
  for (int q = 0; q < n_nce; ++q) cl += nce_losses[q];
  cl *= cl_rate;
  out[0] = bpr_losses[0];
  out[1] = bpr_losses[1];
  out[2] = cl;
  out[3] = bpr_losses[0] + bpr_losses[1] + cl;
}

int seed_segments(int model, int n_layers, int layer_cl, const SeedGrads& g, const SeedRows& r, ScatterSegs& segs) {
  const int B = g.cap, L = n_layers;
  const size_t plane = (size_t)B * g.d;
  const int32_t* rows = g.batch + SRB_BATCH_HEADER;  // u | i | j | unique u | unique i
  const int32_t* n_dev = g.batch;                    // b, unique users, unique items
  const float cm = 1.f / (float)((model == SRB_MODEL_LIGHTGCN || model == SRB_MODEL_SGL) ? L + 1 : L);
  segs.count = 0;
  auto add = [&](int t, bool item, const float* src, const int32_t* idx, const int32_t* n, int cap, float scale) {
    segs.s[segs.count++] = {src, idx, n, cap, item ? r.item_off[t] : r.user_off[t], scale, item ? 0 : r.user_mod, item ? 0 : r.user_rem};
  };
  auto add_bpr = [&](int t, const float* src, float scale) {  // rows u, i, j
    add(t, false, src, rows, n_dev, B, scale);
    add(t, true, src + plane, rows + B, n_dev, B, scale);
    add(t, true, src + 2 * plane, rows + 2 * B, n_dev, B, scale);
  };
  auto add_nce = [&](int t, int view, float scale) {  // unique batch users, unique items
    add(t, false, g.nce_u[view], rows + 3 * B, n_dev + 1, B, scale);
    add(t, true, g.nce_i[view], rows + 4 * B, n_dev + 2, B, scale);
  };
  int g_level = -1;
  switch (model) {
    case SRB_MODEL_LIGHTGCN:  // the L2 term regularises the raw E0: G = F + its gradient at the ego level
      add_bpr(0, g.emb, cm);
      add_bpr(1, g.emb, cm);
      add_bpr(1, g.l2, 1.f);
      g_level = 0;
      break;
    case SRB_MODEL_XSIMGCL:
      // view 1 = final (mean) rows, view 2 = layer l* output (XSimGCL.py:45-50); G = view 2's gradient, plus F unless
      // l* is the ego layer, which the mean leaves out
      g_level = (layer_cl >= 1 && layer_cl <= L) ? layer_cl : 0;
      for (int t = 0; t < (g_level ? 2 : 1); ++t) {
        add_bpr(t, g.emb, cm);
        add_nce(t, 0, cm);
      }
      add_nce(1, 1, 1.f);
      break;
    case SRB_MODEL_SIMGCL:  // all three encoders are the same linear map of E0: one merged chain
      add_bpr(0, g.emb, cm);
      add_nce(0, 0, cm);
      add_nce(0, 1, cm);
      break;
    case SRB_MODEL_SGL:  // cat holds users u and items U + i: one table row each (item_min 0), or split at item_min
      for (int t = 0; t < 2; ++t) {
        add(t, false, g.nce_u[t], g.cat, g.n_cat, 2 * B, cm);
        segs.s[segs.count - 1].item_min = r.item_min;
        segs.s[segs.count - 1].item_off = r.item_min > 0 ? r.item_off[t] : 0;
      }
      add_bpr(2, g.emb, cm);
      break;
  }
  return g_level;
}

static int spmm_simple(const srb_step_desc* s, const srb_graph_csr* g, const float* x, float* y, const float* extra,
                       bool adam, cudaStream_t st, const uint32_t* col_mask = nullptr, const float* seed = nullptr,
                       const uint32_t* seed_mask = nullptr) {
  SpmmArgs a;
  SRB_TRY(graph_args(*g, s->n_users + s->n_items, s->n_users + s->n_items, s->d, x, a));
  a.col_mask = col_mask;
  a.Y = y;
  a.extra = extra;
  a.seed_mask = seed_mask;
  a.seed = seed;
  if (adam) {
    a.ap = s->params;
    a.am = s->adam_m;
    a.av = s->adam_v;
    a.ascal = s->scalars;
    a.b2 = (float)s->beta2;
    a.w1 = (float)(1.0 - s->beta1);
    a.w2 = (float)(1.0 - s->beta2);
    a.aeps = s->adam_eps;
  }
  return launch_spmm(a, s->d, st);
}

// BPR + L2 and InfoNCE only read the encoder outputs and write disjoint buffers: the step forks BPR onto a
// side stream (event dependencies, so a stream capture records the fork and join) and joins before the
// losses are combined.
struct ForkRes {
  cudaStream_t side;
  cudaEvent_t fork, join;
  bool ok;
};
// Default resources: one side stream + two events per device, created on first use (before any capture: capture()
// warms up eagerly).  An engine that may run beside another one on the same device brings its own through
// srb_step_desc.fork_stream / fork_event / join_event, so that two engines never re-record each other's events.
static ForkRes* fork_res(const srb_step_desc* s, ForkRes* own) {
  if (s->fork_stream && s->fork_event && s->join_event) {
    own->side = (cudaStream_t)s->fork_stream;
    own->fork = (cudaEvent_t)s->fork_event;
    own->join = (cudaEvent_t)s->join_event;
    own->ok = true;
    return own;
  }
  static ForkRes res[64] = {};
  static std::mutex mu;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  std::lock_guard<std::mutex> lock(mu);
  ForkRes& r = res[dev];
  if (!r.ok) {
    if (cudaStreamCreateWithFlags(&r.side, cudaStreamNonBlocking) != cudaSuccess) return nullptr;
    if (cudaEventCreateWithFlags(&r.fork, cudaEventDisableTiming) != cudaSuccess) return nullptr;
    if (cudaEventCreateWithFlags(&r.join, cudaEventDisableTiming) != cudaSuccess) return nullptr;
    r.ok = true;
  }
  return &r;
}

int step_losses(int model, float reg, float l2_div, float tau, float cl_rate, int d, int cap, const float* out, const float* e0,
                const float* v1, const float* v2, const LossRows& r, const LossBufs& o, ForkRes* fork,
                const std::function<int()>& before_nce, SeedGrads& g, cudaStream_t st) {
  const bool lg = model == SRB_MODEL_LIGHTGCN, xs = model == SRB_MODEL_XSIMGCL, sg = model == SRB_MODEL_SIMGCL;
  if (fork) {
    SRB_TRY(check_cuda(cudaEventRecord(fork->fork, st), "fork record"));
    SRB_TRY(check_cuda(cudaStreamWaitEvent(fork->side, fork->fork, 0), "fork wait"));
  }
  srb_bpr_desc p = {};
  p.emb = out;
  p.l2_emb = lg ? e0 : out;  // LightGCN.py:25 regularises the raw parameters
  p.n_users = r.item_off;
  p.d = d;
  p.u_idx = r.u;
  p.i_idx = r.i;
  p.j_idx = r.j;
  p.b_dev = r.batch;
  p.b = cap;
  p.emb_scale = 1.f;
  p.reg = reg;
  // (u,p,n)/batch_size: MF.py:21, LightGCN.py:25 | (u,p): SimGCL.py:31, XSimGCL.py:33 | (u,p,n): SGL.py:36
  p.l2_terms = (sg || xs) ? 2 : 3;
  p.l2_div = l2_div;
  p.grad_scale = 1.f;
  p.losses = o.bpr_losses;
  p.g_emb = o.g_emb;
  p.g_l2 = lg ? o.g_l2 : nullptr;
  p.scratch = o.bpr_scratch;
  SRB_TRY(srb_bpr_l2_fwd_bwd(&p, fork ? fork->side : st));
  if (fork) SRB_TRY(check_cuda(cudaEventRecord(fork->join, fork->side), "join record"));
  if (before_nce) SRB_TRY(before_nce());

  g = SeedGrads{r.batch, cap, d, o.g_emb, p.g_l2, {}, {}, nullptr, nullptr};
  srb_infonce_desc q = {};
  q.d = d;
  q.b_cos = 1;
  q.temperature = tau;
  q.workspace = o.nce_ws;
  q.workspace_bytes = o.nce_ws_bytes;
  if (xs || sg) {  // users and items: XSimGCL contrasts the output with its CL view, SimGCL its two views
    const float* t1 = xs ? out : v1;
    const float* t2 = xs ? v1 : v2;
    float* gp[4];
    for (int k = 0; k < 4; ++k) gp[k] = o.g_nce + k * o.nce_plane;
    q.n_problems = 2;
    q.prob[0] = {t1, t2, r.uq_off[0], r.uq_off[0], 1.f, 1.f, r.uq_u, r.batch + 1, cap, cl_rate, gp[0], gp[1], o.nce_losses + 0};
    q.prob[1] = {t1, t2, r.uq_off[1], r.uq_off[1], 1.f, 1.f, r.uq_i, r.batch + 2, cap, cl_rate, gp[2], gp[3], o.nce_losses + 1};
    g.nce_u[0] = gp[0];
    g.nce_u[1] = gp[1];
    g.nce_i[0] = gp[2];
    g.nce_i[1] = gp[3];
  } else if (model == SRB_MODEL_SGL) {  // one problem over cat(users, items) (SGL.py:120-125)
    float* g2 = o.g_nce + (size_t)2 * cap * d;
    q.n_problems = 1;
    q.prob[0] = {v1, v2, 0, 0, 1.f, 1.f, r.cat, r.n_cat, 2 * cap, cl_rate, o.g_nce, g2, o.nce_losses + 0};
    g.nce_u[0] = o.g_nce;
    g.nce_u[1] = g2;
    g.cat = r.cat_id;
    g.n_cat = r.n_cat;
  }
  if (q.n_problems) SRB_TRY(srb_infonce_fwd_bwd(&q, st));
  if (fork) SRB_TRY(check_cuda(cudaStreamWaitEvent(st, fork->join, 0), "join wait"));
  return launch_kernel(finalize_losses_kernel, 1, 1, 0, st, "finalize_losses_kernel", o.bpr_losses, o.nce_losses, q.n_problems, cl_rate,
                       o.losses);
}

// The Horner backward chain of one encoder on graph g.  Its loss gradients were scattered beforehand into [N, d] seed
// tables whose batch rows step_begin_kernel cleared:
//   F = the gradient w.r.t. the encoder's mean, which enters at levels L .. 1 (and at the ego level with include_ego);
//   G (optional, else nullptr with g_level = -1) = what enters at level g_level instead of F (XSimGCL's layer l* or
//       ego-layer gradient, LightGCN's L2 gradient on E0), plus F when that level also takes F.
// The first product gathers its input (F, or G when g_level = L) through the batch-row bitmap, and every later level
// adds its table in the SpMM epilogue at the rows whose batch bit is set -- no dense memset and no scatter per level.
// The last product adds the dense `extra` (may be nullptr) and applies Adam, or with `out` stores into it instead
// (out == extra is allowed: each row reads its addend before it stores).
static int run_chain(const srb_step_desc* s, const Ws& w, const srb_graph_csr* g, const float* F, const float* G, int g_level,
                     bool include_ego, float* out, const float* extra, cudaStream_t st) {
  const int L = s->n_layers;
  const float* x = g_level == L ? G : F;
  for (int k = L - 1; k >= 1; --k) {  // acc_k = A acc_{k+1} + F (G at level g_level)
    float* y = (x == w.acc0) ? w.acc1 : w.acc0;
    SRB_TRY(spmm_simple(s, g, x, y, nullptr, false, st, k == L - 1 ? w.row_mask : nullptr, g_level == k ? G : F, w.row_mask));
    x = y;
  }
  const float* seed0 = g_level == 0 ? G : (include_ego ? F : nullptr);
  return spmm_simple(s, g, x, out, extra, out == nullptr, st, L == 1 ? w.row_mask : nullptr, seed0, w.row_mask);
}

static ScatterSeg seg(const float* src, const int32_t* rows, const int32_t* n_dev, int n, int row_off, float scale) {
  ScatterSeg g = {src, rows, n_dev, n, row_off, scale};
  return g;
}

static int encoder(const srb_step_desc* s, const Ws& w, const srb_graph_csr* g, bool include_ego, int noise_mode, int view,
                   int layer_cl, float* final_out, float* cl_out, cudaStream_t st, const float* x1 = nullptr) {
  // training forward: the final mean is only read at the batch rows, so the last layer skips the rest
  srb_encoder_desc e = {};
  e.rowptr = g->rowptr;
  e.colidx = g->colidx;
  e.vals = g->vals;
  e.row_order = g->row_order;
  e.n_long_rows = g->n_long_rows;
  e.n_vlong_rows = g->n_vlong_rows;
  e.hub = g->hub;
  e.n = s->n_users + s->n_items;
  e.d = s->d;
  e.n_layers = s->n_layers;
  e.include_ego = include_ego;
  e.layer_cl = layer_cl;
  e.noise_mode = noise_mode;
  if (noise_mode == 1) e.noise = s->noise + (size_t)view * s->n_layers * e.n * e.d;
  e.eps = s->eps;
  e.philox_seed = s->philox_seed;
  e.philox_offset = noise_offset(view, 0);  // (+ layer in srb_encoder_forward)
  e.philox_step_dev = s->step_dev;
  e.E0 = s->params;
  if (cl_out && layer_cl == s->n_layers) {
    e.final_out = final_out;  // the last layer is the CL view and is needed in full
  } else {
    e.last_rows = w.batch_rows;
    e.n_last_rows = 3 * s->batch_cap;
    e.last_rows_nv_dev = w.n_hub;
    e.last_rows_hub = srb_hub_split{0, w.hub_cap, w.hub_first, w.hub_work, w.hub_part};
    e.last_rows_out = final_out;  // batch rows of the mean land here; the running sum lives in w.rsum
    e.final_out = w.rsum;
  }
  e.cl_out = cl_out;
  e.work0 = w.work0;
  e.work1 = w.work1;
  e.x1 = x1;
  return srb_encoder_forward(&e, st);
}

// out = x + sign(x) * normalize(noise) * eps, row by row: the noise one perturbed SimGCL encoder adds to the shared
// first product (SimGCL.py:87-88), drawn exactly as the fused SpMM epilogue of layer 1 of view `view` would draw it.
static int perturb_rows(const srb_step_desc* s, const float* x, float* out, int view, cudaStream_t st) {
  const int N = s->n_users + s->n_items;
  SpmmArgs a;
  SRB_TRY(graph_args(s->adj, N, N, s->d, x, a));  // (the graph is not read by the epilogue-only kernel)
  a.Y = out;
  a.noise_mode = s->noise_mode;
  if (s->noise_mode == 1) a.noise = s->noise + (size_t)view * s->n_layers * N * s->d;
  a.eps = s->eps;
  const uint64_t poff = noise_offset(view, 0);
  a.pkey = make_uint2((uint32_t)s->philox_seed, (uint32_t)(s->philox_seed >> 32));
  a.poff = make_uint2((uint32_t)poff, (uint32_t)(poff >> 32));
  a.pstep = s->step_dev;
  return launch_rows_epilogue(a, s->d, st);
}

}  // namespace srb

extern "C" int64_t srb_step_workspace_bytes(int32_t model, int32_t n, int32_t d, int32_t batch_cap, int32_t n_hub_work) {
  srb_step_desc s = {};
  s.adj.hub.n_work = n_hub_work > 0 ? n_hub_work : 0;
  s.model = model;
  s.n_users = n;
  s.n_items = 0;
  s.d = d;
  s.batch_cap = batch_cap;
  return srb::carve(&s, nullptr, nullptr);
}

extern "C" int srb_train_step(const srb_step_desc* s, void* stream) {
  using namespace srb;
  SRB_REQUIRE(s != nullptr, "step: null desc");
  SRB_REQUIRE(s->model >= SRB_MODEL_MF && s->model <= SRB_MODEL_SGL, "step: unknown model %d", s->model);
  SRB_REQUIRE(s->d == 16 || s->d == 32 || s->d == 64 || s->d == 128 || s->d == 256, "step: unsupported d=%d (16, 32, 64, 128, 256)", s->d);
  SRB_REQUIRE(s->n_users > 0 && s->n_items > 0 && s->batch_cap > 0, "step: bad sizes");
  SRB_REQUIRE(s->params && s->adam_m && s->adam_v && s->step_dev && s->scalars && s->losses && s->batch, "step: null pointer");
  SRB_REQUIRE(s->model == SRB_MODEL_MF || s->n_layers >= 1, "step: graph models need n_layers >= 1");
  SRB_REQUIRE(s->model == SRB_MODEL_MF || (s->adj.rowptr && s->adj.colidx && s->adj.vals), "step: null adjacency");
  const int N = s->n_users + s->n_items;
  const int64_t need = srb_step_workspace_bytes(s->model, N, s->d, s->batch_cap, s->model != SRB_MODEL_MF ? s->adj.hub.n_work : 0);
  SRB_REQUIRE(s->workspace && s->workspace_bytes >= need, "step: workspace too small (%lld < %lld)",
              (long long)s->workspace_bytes, (long long)need);
  SRB_REQUIRE(((uintptr_t)s->workspace & 255) == 0, "step: workspace must be 256-byte aligned");
  Ws w;
  carve(s, &w, (char*)s->workspace);
  cudaStream_t st = (cudaStream_t)stream;
  const int B = s->batch_cap, d = s->d, U = s->n_users, L = s->n_layers;
  const int32_t* u_idx = s->batch + SRB_BATCH_HEADER;
  const int32_t* i_idx = u_idx + B;
  const int32_t* j_idx = i_idx + B;
  const int32_t* uq_u = j_idx + B;
  const int32_t* uq_i = uq_u + B;
  const int32_t* b_dev = s->batch;
  const SeedRows rows = {{0, N, 2 * N}, {U, N + U, 2 * N + U}, 0, 0};  // seed table t: rows t * N + [0, N)

  PdlScope pdl;

  // ---- forward ----
  if (s->model != SRB_MODEL_MF) {
    const int n_words = 8 + (U + s->n_items + 31) / 32;  // [class counters | row bitmap]
    SRB_TRY(step_begin(s->step_dev, s->scalars, s->lr, s->beta1, s->beta2, w.n_hub, n_words, s->batch, B, d, w.seed, w.n_seed, rows, st));
    SRB_TRY(launch_kernel(build_batch_rows_kernel, (3 * B + 255) / 256, 256, 0, st, "build_batch_rows_kernel", s->batch, B, U, s->adj.rowptr,
                          w.batch_rows, w.n_hub, w.row_mask, w.hub_cap ? w.hub_first : nullptr, w.hub_work, w.hub_cap));
  } else {
    SRB_TRY(srb_adam_prepare(s->step_dev, s->scalars, s->lr, s->beta1, s->beta2, stream));
  }
  const float* table = s->params;  // table BPR gathers from
  switch (s->model) {
    case SRB_MODEL_MF: break;
    case SRB_MODEL_LIGHTGCN:
      SRB_TRY(encoder(s, w, &s->adj, true, 0, 0, 0, w.final_, nullptr, st));
      table = w.final_;
      break;
    case SRB_MODEL_XSIMGCL:
      SRB_REQUIRE(s->noise_mode == 1 || s->noise_mode == 2, "step: XSimGCL needs noise_mode 1 or 2");
      SRB_REQUIRE(s->noise_mode != 1 || s->noise, "step: noise tensor missing");
      SRB_TRY(encoder(s, w, &s->adj, false, s->noise_mode, 0, s->layer_cl, w.final_, w.cl, st));
      table = w.final_;
      break;
    case SRB_MODEL_SIMGCL:
      SRB_REQUIRE(s->noise_mode == 1 || s->noise_mode == 2, "step: SimGCL needs noise_mode 1 or 2");
      SRB_REQUIRE(s->noise_mode != 1 || s->noise, "step: noise tensor missing");
      if (L >= 2) {
        // layer 1 of the three encoders is the same product A * E0 (SimGCL.py:85); only the noise added to it differs
        // (:87-88).  It is evaluated once; acc0 / acc1 belong to the backward pass and are free until then.
        SRB_TRY(spmm_simple(s, &s->adj, s->params, w.acc0, nullptr, false, st));
        SRB_TRY(perturb_rows(s, w.acc0, w.acc1, 0, st));
        SRB_TRY(perturb_rows(s, w.acc0, w.gd, 1, st));
        SRB_TRY(encoder(s, w, &s->adj, false, 0, 0, 0, w.final_, nullptr, st, w.acc0));
        SRB_TRY(encoder(s, w, &s->adj, false, s->noise_mode, 0, 0, w.cl, nullptr, st, w.acc1));
        SRB_TRY(encoder(s, w, &s->adj, false, s->noise_mode, 1, 0, w.v2, nullptr, st, w.gd));
      } else {
        SRB_TRY(encoder(s, w, &s->adj, false, 0, 0, 0, w.final_, nullptr, st));
        SRB_TRY(encoder(s, w, &s->adj, false, s->noise_mode, 0, 0, w.cl, nullptr, st));
        SRB_TRY(encoder(s, w, &s->adj, false, s->noise_mode, 1, 0, w.v2, nullptr, st));
      }
      table = w.final_;
      break;
    case SRB_MODEL_SGL:
      SRB_REQUIRE(s->adj_view[0].rowptr && s->adj_view[1].rowptr, "step: SGL needs two view graphs");
      SRB_TRY(encoder(s, w, &s->adj, true, 0, 0, 0, w.final_, nullptr, st));
      SRB_TRY(encoder(s, w, &s->adj_view[0], true, 0, 0, 0, w.cl, nullptr, st));
      SRB_TRY(encoder(s, w, &s->adj_view[1], true, 0, 0, 0, w.v2, nullptr, st));
      table = w.final_;
      break;
  }

  // ---- BPR + L2 (on the side stream when an InfoNCE follows), InfoNCE ----
  ForkRes fk_own = {};
  ForkRes* fk = (s->model == SRB_MODEL_XSIMGCL || s->model == SRB_MODEL_SIMGCL || s->model == SRB_MODEL_SGL) ? fork_res(s, &fk_own) : nullptr;
  std::function<int()> build_cat;  // SGL: the cat list on the main stream, after the fork (BPR does not wait for it)
  if (s->model == SRB_MODEL_SGL)
    build_cat = [&] { return launch_kernel(build_cat_idx_kernel, 8, 256, 0, st, "build_cat_idx_kernel", s->batch, B, U, w.idx_cat, w.n_cat); };
  const LossRows lr = {s->batch, u_idx, i_idx, j_idx, U, uq_u, uq_i, {0, U}, w.idx_cat, w.n_cat, w.idx_cat};
  const LossBufs lb = {w.g_emb, w.g_l2, w.g_nce, (size_t)2 * B * d, w.bpr_scratch, w.bpr_losses, w.nce_losses, w.nce_ws, w.nce_ws_bytes, s->losses};
  SeedGrads gr;
  SRB_TRY(step_losses(s->model, s->reg, s->l2_div, s->tau, s->cl_rate, d, B, table, s->params, w.cl, w.v2, lr, lb, fk, build_cat, gr, st));

  // ---- backward + Adam ----
  const size_t plane = (size_t)B * d;
  if (s->model == SRB_MODEL_MF) {
    const size_t bytes = (size_t)N * d * 4;
    SRB_TRY(check_cuda(cudaMemsetAsync(w.acc0, 0, bytes, st), "mf memset"));
    ScatterSegs sg;
    sg.count = 3;
    sg.s[0] = seg(w.g_emb, u_idx, b_dev, B, 0, 1.f);
    sg.s[1] = seg(w.g_emb + plane, i_idx, b_dev, B, U, 1.f);
    sg.s[2] = seg(w.g_emb + 2 * plane, j_idx, b_dev, B, U, 1.f);
    SRB_TRY(scatter_segments(w.acc0, d, sg, st));
    return srb_adam_step(s->params, s->adam_m, s->adam_v, w.acc0, (int64_t)N * d, s->scalars, s->beta1, s->beta2, s->adam_eps,
                         stream);
  }
  auto seed_table = [&](int t) { return w.seed + (size_t)t * N * d; };
  ScatterSegs sg = {};
  const int g_level = seed_segments(s->model, L, s->layer_cl, gr, rows, sg);
  SRB_TRY(scatter_segments(w.seed, d, sg, st));
  if (s->model != SRB_MODEL_SGL)
    return run_chain(s, w, &s->adj, seed_table(0), g_level >= 0 ? seed_table(1) : nullptr, g_level, s->model == SRB_MODEL_LIGHTGCN,
                     nullptr, nullptr, st);
  // SGL's three graphs differ: the two view chains sum into gd, then the main chain adds it and applies Adam
  SRB_TRY(run_chain(s, w, &s->adj_view[0], seed_table(0), nullptr, -1, true, w.gd, nullptr, st));
  SRB_TRY(run_chain(s, w, &s->adj_view[1], seed_table(1), nullptr, -1, true, w.gd, w.gd, st));
  return run_chain(s, w, &s->adj, seed_table(2), nullptr, -1, true, nullptr, w.gd, st);
}
