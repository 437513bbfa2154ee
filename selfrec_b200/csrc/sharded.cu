// Bipartite-sharded training step (SURVEY 8e), one process per GPU, no NCCL on the data path.
//
// The normalised adjacency is  A = [[0, R], [R^T, 0]]  (users x items block R).  Rank g owns the USERS u with
// u % world == g (local row u / world): their rows of every [U, d] table (parameters, moments, layer buffers) never
// leave the GPU.  The cyclic assignment gives every rank the same mix of heavy and light users -- ids follow first
// appearance in the training file (ui_graph.py:29-40), so on a power-law graph contiguous nnz-balanced blocks put a
// few hundred hub users on rank 0 and millions of cold ones on the last rank, whose products (cold gathers, far more
// rows to write) then take much longer.  The (5-50x smaller) ITEM tables are replicated.  One propagation layer is
//     X_u' [block g] = R_g  X_i                 local SpMM over the replicated item table, nothing to exchange
//     X_i'           = sum_g R_g^T X_u[block g]  every rank contributes a partial [I, d] product
// and only the item half crosses NVLink: the item-side SpMM stores each finished partial row straight into the
// staging area of the rank that owns that item slice (reduce-scatter fused into the SpMM epilogue, P2P stores);
// after a device-side barrier the owner adds the partials in rank order, applies the layer's epilogue (noise,
// running layer sum, Adam on the last backward level) and stores the finished row into every rank's copy
// (all-gather fused into the reduction epilogue; one NVSwitch-multicast store per row when a multicast mapping
// exists).  Per layer and rank that is ~2 x I x d x 4 bytes over NVLink instead of the (U+I) x d x 4 of a
// row-sharded all-gather -- at config 5 (10 M users, 2 M items, d = 128) 1.8 GB instead of 5.4 GB.
// The user-side SpMM of a layer is issued between the partial pushes and the barrier, so the NVLink writes drain
// while it runs.
//
// Batch losses: the <= 5B rows a batch reads are pushed by their owners into a compact [5B, d] table on every
// rank (sections u, i, j, unique u, unique i), BPR / InfoNCE run replicated on it with the single-GPU kernels,
// and the compact gradients are scattered once into engine.cu's backward seed tables (user rows on their owner, item
// rows on every rank), whose chain runs on layer().  Persistent state (parameters, Adam moments) has exactly one writer
// per row, so the replicas of the item table are bit-identical on all ranks by construction.
//
// SGL propagates over three graphs: the normalised adjacency and the epoch's two dropped views, each given as this rank's
// Ru / Rt blocks (srb_shard_desc.Ru_view / Rt_view).  Every layer() takes the block pair it runs on; the exchange is the same.
//
// Replaces the same reference code as engine.cu (the batch-loop bodies of LightGCN.py:21-29, SimGCL.py:25-36,
// XSimGCL.py:27-37, SGL.py:30-41); world == 1 runs the same sequence without staging or barriers.
#include <stdlib.h>
#include "spmm_args.cuh"

namespace srb {

// ---------------------------------------------------------------------------------------
// device-side barrier over symmetric flags (one 32-thread block; graph-capturable)
// ---------------------------------------------------------------------------------------
struct BarrierArgs {
  int* flags[8];  // every rank's flag array [8] (flags[rank] is local)
  int* epoch;     // local counter: the number of barriers passed
  int* err;       // local: set to 1 when a peer did not arrive in time
  int world, rank;
};

__global__ void shard_barrier_kernel(const BarrierArgs b) {
  __shared__ int e_s;
  if (threadIdx.x == 0) {
    e_s = *b.epoch + 1;
    *b.epoch = e_s;
  }
  __syncthreads();
  const int e = e_s;
  if ((int)threadIdx.x < b.world) {
    __threadfence_system();  // the kernels before this one are complete; order their peer stores before the flag
    st_release_sys(b.flags[threadIdx.x] + b.rank, e);
    const int* mine = b.flags[b.rank] + threadIdx.x;
    const long long t0 = clock64();
    while (ld_acquire_sys(mine) < e) {
      if (clock64() - t0 > 60000000000ll) {  // ~30 s: a peer died; do not hang the GPU
        *b.err = 1;
        break;
      }
      __nanosleep(64);
    }
  }
}

// Bits of the batch's (local) users / items (masks of the row-sparse first backward product: umask over this rank's
// local user rows, imask over all items), and -- from the thread that sets
// a bit first, so every row is listed once -- the batch's rows of this rank's two blocks, classified by degree for the
// last forward layer (nothing but the batch rows of the final mean is read): local users -> rows of Ru, items ->
// rows of Rt.  Lists follow srb_spmm_desc.n_vlong_dev: four segments (split, CTA, warp, lane group -- unused) of
// capacity cap (users) / 2 * cap (items); cnt[0..3] class sizes and cnt[4] chunks of the user list, cnt[8..] of the
// item list.  cnt and both bitmaps are zeroed by step_begin_kernel.
// SGL's three graphs share the batch rows and the bitmaps but not the degrees: the same thread lists the row for each.
struct BatchRowLists {  // one graph's lists
  const int32_t* ru_rowptr;
  const int32_t* rt_rowptr;
  int32_t* rows_u;    // [4][cap]
  int32_t* rows_i;    // [4][2 * cap]
  int32_t* cnt;       // [16]
  int32_t* hfirst_u;  // [cap] or null (no split rows in Ru)
  int32_t* hwork_u;   // [hcap_u][2]
  int hcap_u;
  int32_t* hfirst_i;  // [2 * cap] or null
  int32_t* hwork_i;
  int hcap_i;
};
struct BatchRowsArgs {
  const int32_t* batch;
  int cap;
  uint32_t* umask;
  uint32_t* imask;
  int world, rank;   // user u lives on rank u % world as local row u / world
  int n_graphs;      // 1, or SGL's 3 (the graph, view 1, view 2)
  BatchRowLists g[3];
};

__global__ void __launch_bounds__(256) shard_batch_rows_kernel(const BatchRowsArgs a) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = min(a.batch[0], a.cap);
  const int sec = t / a.cap, k = t % a.cap;
  if (sec >= 3 || k >= b) return;
  const int id = a.batch[SRB_BATCH_HEADER + sec * a.cap + k];
  const bool user = sec == 0;
  int row = id;
  if (user) {
    if (id % a.world != a.rank) return;  // another rank's user
    row = id / a.world;
  }
  const uint32_t bit = 1u << (row & 31);
  if (atomicOr((user ? a.umask : a.imask) + (row >> 5), bit) & bit) return;  // listed already
  for (int q = 0; q < a.n_graphs; ++q) {
    const BatchRowLists& l = a.g[q];
    const int32_t* rowptr = user ? l.ru_rowptr : l.rt_rowptr;
    // a warp may list users and items at once: item keys are offset by 4 so that the two lists allocate slots apart
    list_batch_row(row, rowptr[row + 1] - rowptr[row], user ? 0 : 4, user ? l.rows_u : l.rows_i, user ? a.cap : 2 * a.cap,
                   l.cnt + (user ? 0 : 8), user ? l.hfirst_u : l.hfirst_i, user ? l.hwork_u : l.hwork_i, user ? l.hcap_u : l.hcap_i);
  }
}

// compact table of the rows a batch reads: slot = section * cap + k (sections: u, i, j, unique u, unique i).
// The owner of a row (user block / item slice) stores it into every rank's compact table.
struct GatherArgs {
  const int32_t* batch;
  int cap;
  int sec_lo, sec_hi;
  const float* utab;  // [n_local_users, D] local
  const float* itab;  // [n_items, D] (owned slice valid)
  int world, rank, ib, ib_end;
  float* dst[8];
  int n_dst;
  int32_t* ar;  // [2*cap]: k and cap + k (index lists of the compact tables), written by block 0
  // SGL (written by block 0 when cat is set): the unique users, then the unique items (SGL.py:120-121) as compact
  // slots 3 cap + k / 4 cap + k (cat) and as table rows u / n_users + i (cat_id); n_cat = their count
  int32_t* cat;
  int32_t* cat_id;
  int32_t* n_cat;
  int n_users;
};

template <int D>
__global__ void __launch_bounds__(256) shard_gather_kernel(const GatherArgs a) {
  const int lane = threadIdx.x & 31;
  const int w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (a.ar && blockIdx.x == 0)
    for (int t = threadIdx.x; t < 2 * a.cap; t += blockDim.x) a.ar[t] = t;
  if (a.cat && blockIdx.x == 0) {
    const int nu = min(a.batch[1], a.cap), ni = min(a.batch[2], a.cap);
    const int32_t* uq = a.batch + SRB_BATCH_HEADER + 3 * a.cap;  // unique users, then (at + cap) unique items
    for (int t = threadIdx.x; t < nu + ni; t += blockDim.x) {
      a.cat[t] = t < nu ? 3 * a.cap + t : 4 * a.cap + t - nu;
      a.cat_id[t] = t < nu ? uq[t] : a.n_users + uq[a.cap + t - nu];
    }
    if (threadIdx.x == 0) *a.n_cat = nu + ni;
  }
  const int slot = a.sec_lo * a.cap + w;
  if (slot >= a.sec_hi * a.cap) return;
  const int sec = slot / a.cap, k = slot % a.cap;
  const int cnt = min(sec <= 2 ? a.batch[0] : a.batch[sec - 2], a.cap);  // b, b, b, n_uniq_u, n_uniq_i
  if (k >= cnt) return;
  const int id = a.batch[SRB_BATCH_HEADER + sec * a.cap + k];
  const bool user = (sec == 0 || sec == 3);
  const float* src;
  if (user) {
    if (id % a.world != a.rank) return;
    src = a.utab + (size_t)(id / a.world) * D;
  } else {
    if (id < a.ib || id >= a.ib_end) return;
    src = a.itab + (size_t)id * D;
  }
  for (int c = lane * 4; c < D; c += 128) {
    const float4 v = *reinterpret_cast<const float4*>(src + c);
#pragma unroll 1
    for (int q = 0; q < a.n_dst; ++q) st4(a.dst[q] + (size_t)slot * D + c, v);
  }
}

static int64_t al256(int64_t x) { return (x + 255) / 256 * 256; }

// ---------------------------------------------------------------------------------------
// memory plans
// ---------------------------------------------------------------------------------------
struct SymPlan {  // byte offsets inside every rank's symmetric region
  int64_t flags, pi, fin_i, xi[2], cl_i, ai[2], stage, cmain, cv1, cv2, cp, total;
  int32_t stage_cap;
};

static SymPlan sym_plan(int64_t I, int64_t d, int64_t B, int world) {
  SymPlan p;
  int64_t off = 0;
  auto take = [&](int64_t bytes) {
    const int64_t o = off;
    off += al256(bytes);
    return o;
  };
  const int64_t nd = I * d * 4;
  p.stage_cap = (int32_t)((I + world - 1) / world);
  p.flags = take(256);
  p.pi = take(nd);
  p.fin_i = take(nd);
  p.xi[0] = take(nd);
  p.xi[1] = take(nd);
  p.cl_i = take(nd);
  p.ai[0] = take(nd);
  p.ai[1] = take(nd);
  p.stage = take(world > 1 ? (int64_t)world * p.stage_cap * d * 4 : 0);
  p.cmain = take(5 * B * d * 4);
  p.cv1 = take(5 * B * d * 4);
  p.cv2 = take(5 * B * d * 4);
  p.cp = take(5 * B * d * 4);
  p.total = off;
  return p;
}

struct LocalPlan {
  int64_t ctrl;  // [0] barrier epoch, [1] error flag (zeroed once by the host, never by a step)
  int64_t xu[2], su, clu, v2u, au[2];
  int64_t seed;  // backward seed slots, [n_seed][Ug, d] (this rank's users) then [n_seed][I, d] (the complete item replica)
  int64_t v2_i;
  int64_t g_emb, g_l2, g_nce, bpr_scratch, bpr_losses, nce_losses, ar, umask, imask, cnt, nce_ws, total;
  // batch-row lists of the last forward layer, per graph (cnt: 16 words per graph)
  int64_t rows_u[3], rows_i[3], hfirst_u[3], hfirst_i[3], hwork_u[3], hwork_i[3];
  int64_t cat, cat_id, n_cat;  // SGL's InfoNCE rows (GatherArgs)
  int64_t nce_ws_bytes;
  int n_seed, n_graphs;
};

// Every model but SGL gets the layout it always had; SGL adds a third seed slot per side, the batch-row lists of its two
// views (whose split-row chunks must fit the graph's: hub_u / hub_t), and an InfoNCE workspace of one 2B problem.
static LocalPlan local_plan(int model, int64_t I, int64_t Ug, int64_t d, int64_t B, int64_t hub_u, int64_t hub_t) {
  LocalPlan p;
  int64_t off = 0;
  auto take = [&](int64_t bytes) {
    const int64_t o = off;
    off += al256(bytes);
    return o;
  };
  const bool sgl = model == SRB_MODEL_SGL;
  p.n_seed = sgl ? 3 : 2;
  p.n_graphs = sgl ? 3 : 1;
  const int64_t und = Ug * d * 4, ind = I * d * 4;
  p.ctrl = take(256);
  p.xu[0] = take(und);
  p.xu[1] = take(und);
  p.su = take(und);
  p.clu = take(und);
  p.v2u = take(und);
  p.au[0] = take(und);
  p.au[1] = take(und);
  p.seed = take(p.n_seed * (und + ind));  // contiguous: one scatter fills every slot
  p.v2_i = take(ind);
  p.g_emb = take(3 * B * d * 4);
  p.g_l2 = take(3 * B * d * 4);
  p.g_nce = take(4 * B * d * 4);
  p.bpr_scratch = take(8 * 4);
  p.bpr_losses = take(2 * 4);
  p.nce_losses = take(4 * 4);
  p.ar = take(2 * B * 4);
  // step_begin_kernel clears both bitmaps and the list counters: [umask, nce_ws)
  p.umask = take(((Ug + 31) / 32) * 4 + 4);  // bitmap over this rank's local user rows
  p.imask = take(((I + 31) / 32) * 4);
  p.cnt = take(p.n_graphs * 16 * 4);
  p.nce_ws_bytes = sgl ? srb_infonce_workspace_bytes((int32_t)(2 * B), (int32_t)d, 1) : srb_infonce_workspace_bytes((int32_t)B, (int32_t)d, 2);
  p.nce_ws = take(p.nce_ws_bytes);
  for (int q = 0; q < p.n_graphs; ++q) {
    p.rows_u[q] = take(4 * B * 4);
    p.rows_i[q] = take(4 * 2 * B * 4);
    p.hfirst_u[q] = take(B * 4);
    p.hfirst_i[q] = take(2 * B * 4);
    p.hwork_u[q] = take(hub_u * 2 * 4);
    p.hwork_i[q] = take(hub_t * 2 * 4);
  }
  p.cat = take(sgl ? 2 * B * 4 : 0);
  p.cat_id = take(sgl ? 2 * B * 4 : 0);
  p.n_cat = take(sgl ? 4 : 0);
  p.total = off;
  return p;
}

struct Ctx {
  const srb_shard_desc* s;
  SymPlan sp;
  LocalPlan lp;
  cudaStream_t st;
  int G, rank, U, I, Ug, ib, ib_end, d, L, B;
  char* sym;   // local symmetric region
  char* loc;   // local workspace
  float* symf(int64_t off, int q) const { return (float*)((char*)s->sym[q] + off); }
  float* mine(int64_t off) const { return (float*)(sym + off); }
  float* lw(int64_t off) const { return (float*)(loc + off); }
  float* seed_u(int t) const { return lw(lp.seed) + (size_t)t * Ug * d; }
  float* seed_i(int t) const { return lw(lp.seed) + ((size_t)lp.n_seed * Ug + (size_t)t * I) * d; }
};

// One graph's blocks on this rank and the index of their batch-row lists: 0 = Ru / Rt, 1 and 2 = SGL's two views
struct Blocks {
  const srb_graph_csr* ru;  // [Ug x I]
  const srb_graph_csr* rt;  // [I x Ug]
  int q;
};

static Blocks blocks(const Ctx& c, int q) {
  return q == 0 ? Blocks{&c.s->Ru, &c.s->Rt, 0} : Blocks{&c.s->Ru_view[q - 1], &c.s->Rt_view[q - 1], q};
}

// SRB_SHARD_SYNC=barrier: separate barrier launches between the kernels of a layer instead of waits / signals folded
// into them (measurement switch; both are parity-tested: the folded mode by the one-process-per-GPU checks, barrier mode
// by tests/test_gpu_shard_loopback.py, whose ranks share one GPU -- the only mode that can, since no other kernel waits)
static bool sync_in_kernels() {
  static const int mode = [] {
    const char* e = getenv("SRB_SHARD_SYNC");
    return (e && e[0] == 'b') ? 0 : 1;
  }();
  return mode != 0;
}

// NVLS route of the partial-sum exchange (needs the multicast mapping): partial products stay in the rank's own copy of
// the staging buffer and the owner reads their sum with multimem.ld_reduce.  Opt-in (srb_shard_desc.nvls; parity-tested
// like the default): it halves a rank's NVLink ingress, which only matters from 4-8 ranks, at the price of an in-switch
// reduction whose rate bounds the owner's read.
static bool nvls(const Ctx& c) { return c.s->nvls != 0 && c.G > 1 && c.s->sym_mc != nullptr; }

// wait / signal folded into the kernels of a layer (PeerSync in spmm_args.cuh)
static PeerSync peer_sync(const Ctx& c, bool wait, bool signal) {
  PeerSync p = {};
  if (c.G <= 1 || !sync_in_kernels()) return p;
  for (int q = 0; q < c.G; ++q) p.flags[q] = (int*)((char*)c.s->sym[q] + c.sp.flags);
  p.epoch = (int*)(c.loc + c.lp.ctrl);
  p.err = p.epoch + 1;
  p.counter = p.epoch + 2;
  p.world = c.G;
  p.rank = c.rank;
  p.wait = wait;
  p.signal = signal;
  return p;
}

// wait for the peers' latest signal without sending one (e.g. before adding into rows the peers' reductions store)
__global__ void shard_wait_kernel(const PeerSync s) { peer_wait(s); }

static int barrier(const Ctx& c);

static int wait_peers(const Ctx& c) {
  if (c.G <= 1) return SRB_OK;
  if (!sync_in_kernels()) return SRB_OK;  // (barrier mode: every layer already ends with a full barrier)
  shard_wait_kernel<<<1, 32, 0, c.st>>>(peer_sync(c, true, false));
  return post_launch("shard_wait_kernel");
}

static int barrier(const Ctx& c) {
  if (c.G <= 1) return SRB_OK;
  BarrierArgs b = {};
  for (int q = 0; q < c.G; ++q) b.flags[q] = (int*)((char*)c.s->sym[q] + c.sp.flags);
  b.epoch = (int*)(c.loc + c.lp.ctrl);
  b.err = b.epoch + 1;
  b.world = c.G;
  b.rank = c.rank;
  shard_barrier_kernel<<<1, 32, 0, c.st>>>(b);
  return post_launch("shard_barrier_kernel");
}

// epilogue options of one propagation layer (both halves)
struct Epi {
  int noise_mode = 0;
  uint64_t poff = 0;
  // user half (local tables) / item half (item-id indexed tables)
  float* y_u = nullptr;
  int64_t y_i = -1;            // symmetric offset of the item output (pushed to every rank) or -1
  float* y_i_loc = nullptr;    // or: local item output, not pushed (world > 1: valid on the owner's slice only)
  const float* extra_u = nullptr;    // dense addend of every row (the outputs' layouts), or null
  const float* extra_i = nullptr;
  const float* sum_in_u = nullptr;
  float* sum_out_u = nullptr;
  const float* sum_in_i = nullptr;
  float* sum_out_i = nullptr;
  int64_t sum_push_i = -1;     // symmetric offset: the item running sum also goes to every rank (clean forward for eval)
  float sum_scale = 1.f;
  const float* seed_u = nullptr;     // backward seed slot added at the batch rows (umask / imask), or null
  const float* seed_i = nullptr;
  bool adam = false;
  const uint32_t* mask_u = nullptr;  // bitmap over this rank's users (columns of Rt)
  const uint32_t* mask_i = nullptr;  // bitmap over items (columns of Ru)
  bool rows_only = false;            // last forward layer: only the batch rows (lists of shard_batch_rows_kernel)
};

// Restrict a product over block g (Ru or Rt of graph q) to the batch rows listed by shard_batch_rows_kernel
// (device-classified list, dynamic chunk lists of the split rows; the graph's own partial-sum scratch is reused).
static void use_batch_rows(const Ctx& c, const srb_graph_csr& g, int q, bool item_side, SpmmArgs& a) {
  const int hcap = g.hub.n_work;
  a.row_order = (const int32_t*)(c.loc + (item_side ? c.lp.rows_i[q] : c.lp.rows_u[q]));
  a.n_rows = item_side ? 2 * c.B : c.B;
  a.n_vlong_dev = (const int32_t*)(c.loc + c.lp.cnt) + 16 * q + (item_side ? 8 : 0);
  a.n_huge = a.n_vlong = a.n_long = 0;
  a.hub_first = hcap ? (const int32_t*)(c.loc + (item_side ? c.lp.hfirst_i[q] : c.lp.hfirst_u[q])) : nullptr;
  a.hub_work = hcap ? (const int32_t*)(c.loc + (item_side ? c.lp.hwork_i[q] : c.lp.hwork_u[q])) : nullptr;
  a.hub_part = hcap ? g.hub.part : nullptr;
  a.n_work = hcap;
  a.seg = a.seg_cnt = a.order_cta = a.order_warp = nullptr;
  a.n_cta = a.n_warp = 0;
}

static void epi_common(const Ctx& c, const Epi& e, SpmmArgs& a) {
  const srb_shard_desc* s = c.s;
  a.noise_mode = e.noise_mode;
  a.eps = s->eps;
  a.pkey = make_uint2((uint32_t)s->philox_seed, (uint32_t)(s->philox_seed >> 32));
  a.poff = make_uint2((uint32_t)e.poff, (uint32_t)(e.poff >> 32));
  a.pstep = s->step_dev;
  a.sum_scale = e.sum_scale;
  a.extra_scale = 1.f;
  a.b2 = (float)s->beta2;
  a.w1 = (float)(1.0 - s->beta1);
  a.w2 = (float)(1.0 - s->beta2);
  a.aeps = s->adam_eps;
  a.ascal = s->scalars;
}

static void item_epilogue(const Ctx& c, const Epi& e, SpmmArgs& a) {
  const srb_shard_desc* s = c.s;
  epi_common(c, e, a);
  a.noise_row_base = c.U;
  a.Y = e.y_i >= 0 ? c.mine(e.y_i) : e.y_i_loc;
  a.extra = e.extra_i;
  a.seed = e.seed_i;  // (world > 1: added by the owner's reduction only, after the rank-ordered sum)
  a.seed_mask = (const uint32_t*)(c.loc + c.lp.imask);
  a.sum_in = e.sum_in_i;
  a.sum_out = e.sum_out_i;
  if (e.adam) {
    a.ap = c.mine(c.sp.pi);
    a.am = s->mi;
    a.av = s->vi;
  }
  a.world = 0;
  if (c.G > 1) {  // finished rows go to every other rank's copy (the local store is the plain one above)
    const bool mc = s->sym_mc != nullptr;
    int n = 0;
    for (int q = 0; q < c.G && !mc; ++q) {
      if (q == c.rank) continue;
      a.peer[n] = e.y_i >= 0 ? c.symf(e.y_i, q) : nullptr;
      a.peer_sum[n] = e.sum_push_i >= 0 ? c.symf(e.sum_push_i, q) : nullptr;
      a.peer_p[n] = e.adam ? c.symf(c.sp.pi, q) : nullptr;
      ++n;
    }
    if (mc) {
      a.peer[0] = e.y_i >= 0 ? (float*)((char*)s->sym_mc + e.y_i) : nullptr;
      a.peer_sum[0] = e.sum_push_i >= 0 ? (float*)((char*)s->sym_mc + e.sum_push_i) : nullptr;
      a.peer_p[0] = e.adam ? (float*)((char*)s->sym_mc + c.sp.pi) : nullptr;
      n = 1;
      a.peer_mc = 1;
    }
    a.world = n;
  }
}

// One propagation layer over the block pair bl: (xu [Ug,d] local, xi [I,d] replicated) -> outputs per `e`.
static int layer(const Ctx& c, const Blocks& bl, const float* xu, const float* xi, const Epi& e) {
  const srb_shard_desc* s = c.s;
  // ---- item half, part 1: this rank's partial product R_g^T xu ----
  {
    SpmmArgs a;
    SRB_TRY(graph_args(*bl.rt, c.I, c.Ug, c.d, xu, a));
    a.col_mask = e.mask_u;
    if (e.rows_only) use_batch_rows(c, *bl.rt, bl.q, true, a);
    if (c.G == 1) {
      item_epilogue(c, e, a);
    } else {
      if (nvls(c)) {  // the partial product stays local: one "owner" covering every row, plain stores
        a.stage_peer[0] = c.mine(c.sp.stage);
        a.stage_bounds[0] = 0;
        for (int q = 1; q <= 8; ++q) a.stage_bounds[q] = c.I;
        a.stage_rank = 0;
        a.stage_cap = c.I;
      } else {
        for (int q = 0; q < c.G; ++q) a.stage_peer[q] = c.symf(c.sp.stage, q);
        for (int q = 0; q <= c.G; ++q) a.stage_bounds[q] = (int32_t)((int64_t)q * c.I / c.G);
        a.stage_rank = c.rank;
        a.stage_cap = c.sp.stage_cap;
      }
      // wait: the owners have finished reading the staging areas (and every rank the buffers this layer rewrites);
      // signal: this rank's partial rows are in place
      a.ps = peer_sync(c, true, true);
    }
    SRB_TRY(launch_spmm(a, c.d, c.st));
  }
  // ---- item half, part 2 (owner-side reduction + epilogue + push to every rank) beside the user half ----
  // The reduction is NVLink-bound and the user-side product is local compute: with the caller's fork stream the two
  // run concurrently (the reduction on one CTA per SM), so the exchange hides behind the product.
  const bool overlap = c.G > 1 && sync_in_kernels() && s->fork_stream && s->fork_event && s->join_event;
  cudaStream_t rs = overlap ? (cudaStream_t)s->fork_stream : c.st;
  auto reduce = [&]() -> int {
    SpmmArgs a;
    SRB_TRY(graph_args(*bl.rt, c.I, c.Ug, c.d, xu, a));
    item_epilogue(c, e, a);
    ReduceArgs r = {};
    r.stage = c.mine(c.sp.stage);
    r.world = c.G;
    r.stage_cap = c.sp.stage_cap;
    r.slice_begin = c.ib;
    r.n_slice = c.ib_end - c.ib;
    r.mask = e.rows_only ? (const uint32_t*)(c.loc + c.lp.imask) : nullptr;
    r.mc_part = nvls(c) ? (const float*)((const char*)s->sym_mc + c.sp.stage) : nullptr;
    r.small_grid = overlap ? 1 : 0;
    a.ps = peer_sync(c, true, true);  // wait: all partials are in place; signal: the finished rows are everywhere
    return launch_reduce_rows(a, r, c.d, rs);
  };
  auto user_half = [&]() -> int {
    if (c.Ug <= 0) return SRB_OK;
    SpmmArgs a;
    SRB_TRY(graph_args(*bl.ru, c.Ug, c.I, c.d, xi, a));
    a.col_mask = e.mask_i;
    if (e.rows_only) use_batch_rows(c, *bl.ru, bl.q, false, a);
    epi_common(c, e, a);
    a.noise_row_base = c.rank;  // global id of local user row r: rank + r * world
    a.noise_row_stride = c.G;
    a.Y = e.y_u;
    a.extra = e.extra_u;
    a.seed = e.seed_u;
    a.seed_mask = (const uint32_t*)(c.loc + c.lp.umask);
    a.sum_in = e.sum_in_u;
    a.sum_out = e.sum_out_u;
    if (e.adam) {
      a.ap = s->pu;
      a.am = s->mu;
      a.av = s->vu;
    }
    return launch_spmm(a, c.d, c.st);
  };
  if (c.G == 1) return user_half();
  if (overlap) {
    SRB_TRY(check_cuda(cudaEventRecord((cudaEvent_t)s->fork_event, c.st), "shard fork record"));
    SRB_TRY(check_cuda(cudaStreamWaitEvent(rs, (cudaEvent_t)s->fork_event, 0), "shard fork wait"));
    SRB_TRY(reduce());      // launched first: its one CTA per SM is resident before the product fills the rest
    SRB_TRY(user_half());
    SRB_TRY(check_cuda(cudaEventRecord((cudaEvent_t)s->join_event, rs), "shard join record"));
    return check_cuda(cudaStreamWaitEvent(c.st, (cudaEvent_t)s->join_event, 0), "shard join wait");
  }
  SRB_TRY(user_half());  // (runs while the partial rows drain over NVLink)
  if (!sync_in_kernels()) SRB_TRY(barrier(c));
  SRB_TRY(reduce());
  return sync_in_kernels() ? SRB_OK : barrier(c);
}

// Encoder forward on the sharded tables (R4).  sums: running layer sum / final mean (user local, item owner slice).
// batch_rows: training forward -- the final mean is only read at the batch rows, so the last layer skips the rest.
// x1u / x1i: output of layer 1 evaluated by the caller (SimGCL's shared first product); the loop starts at layer 2.
static int encoder(const Ctx& c, const Blocks& bl, bool include_ego, int noise_mode, int view, int layer_cl, float* sum_u, float* sum_i,
                   float* cl_u, int64_t cl_i_off, bool push_final_items, bool batch_rows, const float* x1u = nullptr,
                   const float* x1i = nullptr) {
  const srb_shard_desc* s = c.s;
  const int L = c.L;
  const float inv = 1.0f / (float)(include_ego ? L + 1 : L);
  const float* xu = x1u ? x1u : s->pu;
  const float* xi = x1u ? x1i : c.mine(c.sp.pi);
  int pp = 0;
  for (int k = x1u ? 1 : 0; k < L; ++k) {
    const bool last = k == L - 1;
    const bool is_cl = cl_u && layer_cl == k + 1;
    Epi e;
    e.noise_mode = noise_mode;
    e.poff = noise_offset(view, k);
    if (is_cl) {
      e.y_u = cl_u;
      e.y_i = cl_i_off;
    } else if (!last) {
      e.y_u = c.lw(c.lp.xu[pp]);
      e.y_i = c.sp.xi[pp];
      pp ^= 1;
    }
    e.sum_in_u = k == 0 ? (include_ego ? s->pu : nullptr) : ((k == 1 && x1u) ? x1u : sum_u);
    e.sum_in_i = k == 0 ? (include_ego ? c.mine(c.sp.pi) : nullptr) : ((k == 1 && x1u) ? x1i : sum_i);
    e.sum_out_u = sum_u;
    e.sum_out_i = sum_i;
    e.sum_scale = last ? inv : 1.f;
    e.rows_only = batch_rows && last && !is_cl;  // (a CL view at the last layer is needed in full)
    if (last && push_final_items) e.sum_push_i = (int64_t)((char*)sum_i - c.sym);
    SRB_TRY(layer(c, bl, xu, xi, e));
    if (e.y_u) {
      xu = e.y_u;
      xi = c.mine(e.y_i);
    }
  }
  return SRB_OK;
}

static int gather(const Ctx& c, const float* utab, const float* itab, int64_t ctab_off, int sec_lo, int sec_hi, bool write_ar) {
  GatherArgs g = {};
  g.batch = c.s->batch;
  g.cap = c.B;
  g.sec_lo = sec_lo;
  g.sec_hi = sec_hi;
  g.utab = utab;
  g.itab = itab;
  g.world = c.G;
  g.rank = c.rank;
  g.ib = c.ib;
  g.ib_end = c.ib_end;
  for (int q = 0; q < c.G; ++q) g.dst[q] = c.symf(ctab_off, q);
  g.n_dst = c.G;
  g.ar = write_ar ? (int32_t*)(c.loc + c.lp.ar) : nullptr;
  if (write_ar && c.s->model == SRB_MODEL_SGL) {
    g.cat = (int32_t*)(c.loc + c.lp.cat);
    g.cat_id = (int32_t*)(c.loc + c.lp.cat_id);
    g.n_cat = (int32_t*)(c.loc + c.lp.n_cat);
    g.n_users = c.U;
  }
  const int slots = (sec_hi - sec_lo) * c.B;
  const int blocks = (slots + 7) / 8;
  switch (c.d) {
    case 16: shard_gather_kernel<16><<<blocks, 256, 0, c.st>>>(g); break;
    case 32: shard_gather_kernel<32><<<blocks, 256, 0, c.st>>>(g); break;
    case 64: shard_gather_kernel<64><<<blocks, 256, 0, c.st>>>(g); break;
    case 128: shard_gather_kernel<128><<<blocks, 256, 0, c.st>>>(g); break;
    case 256: shard_gather_kernel<256><<<blocks, 256, 0, c.st>>>(g); break;
    default: set_error("shard gather: unsupported d=%d (16, 32, 64, 128, 256)", c.d); return SRB_ERR_ARG;
  }
  return post_launch("shard_gather_kernel");
}

static int make_ctx(const srb_shard_desc* s, void* stream, Ctx& c) {
  SRB_REQUIRE(s != nullptr, "shard: null desc");
  SRB_REQUIRE(s->model == SRB_MODEL_LIGHTGCN || s->model == SRB_MODEL_SIMGCL || s->model == SRB_MODEL_XSIMGCL || s->model == SRB_MODEL_SGL,
              "shard: the sharded step covers LightGCN, SimGCL, XSimGCL and SGL (model %d)", s->model);
  SRB_REQUIRE(s->world >= 1 && s->world <= 8 && s->rank >= 0 && s->rank < s->world, "shard: bad world/rank %d/%d", s->world, s->rank);
  SRB_REQUIRE(s->d == 16 || s->d == 32 || s->d == 64 || s->d == 128 || s->d == 256, "shard: unsupported d=%d (16, 32, 64, 128, 256)", s->d);
  SRB_REQUIRE(s->n_users > 0 && s->n_items > 0 && s->batch_cap > 0 && s->n_layers >= 1, "shard: bad sizes");
  SRB_REQUIRE(s->noise_mode == 0 || s->noise_mode == 2, "shard: noise comes from the in-kernel Philox stream (noise_mode 2)");
  SRB_REQUIRE(s->model != SRB_MODEL_SGL || s->noise_mode == 0, "shard: SGL adds no noise (noise_mode 0)");
  for (int g = 0; g < s->world; ++g) SRB_REQUIRE(s->sym[g] != nullptr, "shard: null symmetric region of rank %d", g);
  SRB_REQUIRE(s->Ru.rowptr && s->Ru.colidx && s->Ru.vals && s->Rt.rowptr && s->Rt.colidx && s->Rt.vals, "shard: null matrix");
  SRB_REQUIRE(s->pu && s->mu && s->vu && s->mi && s->vi && s->step_dev && s->scalars && s->losses, "shard: null pointer");
  c.s = s;
  c.st = (cudaStream_t)stream;
  c.G = s->world;
  c.rank = s->rank;
  c.U = s->n_users;
  c.I = s->n_items;
  c.Ug = (s->n_users - s->rank + s->world - 1) / s->world;  // users rank, rank + world, rank + 2 world, ...
  c.ib = (int)((int64_t)s->rank * c.I / c.G);
  c.ib_end = (int)((int64_t)(s->rank + 1) * c.I / c.G);
  SRB_REQUIRE(c.Ug > 0, "shard: rank %d owns no users", s->rank);
  c.d = s->d;
  c.L = s->n_layers;
  c.B = s->batch_cap;
  c.sp = sym_plan(c.I, c.d, c.B, c.G);
  c.lp = local_plan(s->model, c.I, c.Ug, c.d, c.B, s->Ru.hub.n_work, s->Rt.hub.n_work);
  SRB_REQUIRE(s->sym_bytes >= c.sp.total, "shard: symmetric region too small (%lld < %lld)", (long long)s->sym_bytes, (long long)c.sp.total);
  SRB_REQUIRE(s->workspace && s->workspace_bytes >= c.lp.total, "shard: workspace too small (%lld < %lld)",
              (long long)s->workspace_bytes, (long long)c.lp.total);
  SRB_REQUIRE(((uintptr_t)s->workspace & 255) == 0 && ((uintptr_t)s->sym[s->rank] & 255) == 0, "shard: regions must be 256-byte aligned");
  c.sym = (char*)s->sym[s->rank];
  c.loc = (char*)s->workspace;
  return SRB_OK;
}

// engine.cu's run_chain on layer() over the block pair bl: seed slot f (F) enters at levels L-1 .. 1 and, with include_ego,
// at the ego level; slot 1 (G) enters at level g_level instead (at the ego level: G only -- LightGCN's G holds F too).  The
// first product gathers its input through the batch bitmaps.  Every rank reads only its own complete item slots, so the
// chain needs no synchronisation beyond layer()'s: the owner's reduction adds the item seed after the rank-ordered sum.
// The last product applies Adam, or with to_gd stores into gd (this rank's users, and the items of its own slice -- the
// rows the last product of a later chain reads); with add_gd it adds gd first.
static int chain(const Ctx& c, const Blocks& bl, int f, int g_level, bool include_ego, float* gd_u, float* gd_i, bool to_gd, bool add_gd) {
  const int L = c.L;
  const uint32_t* umask = (const uint32_t*)(c.loc + c.lp.umask);
  const uint32_t* imask = (const uint32_t*)(c.loc + c.lp.imask);
  auto slot = [&](int k) { return g_level == k ? 1 : f; };
  float* au[2] = {c.lw(c.lp.au[0]), c.lw(c.lp.au[1])};
  const float *xu = c.seed_u(slot(L)), *xi = c.seed_i(slot(L));
  for (int k = L - 1, x = 0; k >= 1; --k, x ^= 1) {
    Epi e;
    e.y_u = au[x];
    e.y_i = c.sp.ai[x];
    e.seed_u = c.seed_u(slot(k));
    e.seed_i = c.seed_i(slot(k));
    if (k == L - 1) {  // the input is a seed slot: valid at the batch rows only
      e.mask_u = umask;
      e.mask_i = imask;
    }
    SRB_TRY(layer(c, bl, xu, xi, e));
    xu = au[x];
    xi = c.mine(c.sp.ai[x]);
  }
  Epi e;
  const int s0 = g_level == 0 ? 1 : (include_ego ? f : -1);
  e.seed_u = s0 >= 0 ? c.seed_u(s0) : nullptr;
  e.seed_i = s0 >= 0 ? c.seed_i(s0) : nullptr;
  if (L == 1) {
    e.mask_u = umask;
    e.mask_i = imask;
  }
  if (to_gd) {
    e.y_u = gd_u;
    e.y_i_loc = gd_i;
  } else {
    e.adam = true;
  }
  if (add_gd) {  // (out == extra: each row reads its addend before it stores)
    e.extra_u = gd_u;
    e.extra_i = gd_i;
  }
  return layer(c, bl, xu, xi, e);
}

}  // namespace srb

extern "C" int srb_shard_plan(int32_t model, int32_t n_users, int32_t n_items, int32_t n_local_users, int32_t d, int32_t batch_cap,
                              int32_t world, int32_t hub_chunks_u, int32_t hub_chunks_t, srb_shard_layout* out) {
  SRB_REQUIRE(out && world >= 1 && world <= 8 && n_items > 0 && d > 0 && batch_cap > 0 && hub_chunks_u >= 0 && hub_chunks_t >= 0,
              "shard_plan: bad arguments");
  SRB_REQUIRE(model == SRB_MODEL_LIGHTGCN || model == SRB_MODEL_SIMGCL || model == SRB_MODEL_XSIMGCL || model == SRB_MODEL_SGL,
              "shard_plan: the sharded step covers LightGCN, SimGCL, XSimGCL and SGL (model %d)", model);
  const srb::SymPlan sp = srb::sym_plan(n_items, d, batch_cap, world);
  (void)n_users;  // (the local workspace only depends on the rank's own user count)
  const srb::LocalPlan lp = srb::local_plan(model, n_items, n_local_users, d, batch_cap, hub_chunks_u, hub_chunks_t);
  out->sym_bytes = sp.total;
  out->workspace_bytes = lp.total;
  out->item_params = sp.pi;
  out->item_final = sp.fin_i;
  out->ctrl = lp.ctrl;
  return SRB_OK;
}

extern "C" int srb_shard_step(const srb_shard_desc* s, void* stream) {
  using namespace srb;
  Ctx c;
  SRB_TRY(make_ctx(s, stream, c));
  SRB_REQUIRE(s->batch != nullptr, "shard: null batch");
  cudaStream_t st = c.st;
  const int B = c.B, d = c.d, L = c.L;
  const bool xs = s->model == SRB_MODEL_XSIMGCL, sg = s->model == SRB_MODEL_SIMGCL, lg = s->model == SRB_MODEL_LIGHTGCN,
             sgl = s->model == SRB_MODEL_SGL;
  SRB_REQUIRE(lg || sgl || s->noise_mode == 2, "shard: SimGCL / XSimGCL need noise_mode 2");
  if (sgl) {
    for (int v = 0; v < 2; ++v) {
      const srb_graph_csr &ru = s->Ru_view[v], &rt = s->Rt_view[v];
      SRB_REQUIRE(ru.rowptr && ru.colidx && ru.vals && rt.rowptr && rt.colidx && rt.vals,
                  "shard: SGL needs the epoch's two view graphs as this rank's blocks (Ru_view / Rt_view of view %d are null)", v + 1);
      SRB_REQUIRE(ru.hub.n_work <= s->Ru.hub.n_work && rt.hub.n_work <= s->Rt.hub.n_work,
                  "shard: view %d has more split-row chunks (%d, %d) than the graph the plan was made for (%d, %d)", v + 1,
                  ru.hub.n_work, rt.hub.n_work, s->Ru.hub.n_work, s->Rt.hub.n_work);
    }
  }

  uint32_t* umask = (uint32_t*)(c.loc + c.lp.umask);
  uint32_t* imask = (uint32_t*)(c.loc + c.lp.imask);
  // seed slot t: user u at row u / world + t * Ug, item i at n_seed * Ug + t * I + i; SimGCL's slot 1 holds a forward
  // buffer.  SGL's cat lists users u and items U + i: the items go to every rank's item slots.
  const int ns = c.lp.n_seed;
  const SeedRows rows = {{0, c.G * c.Ug, 2 * c.G * c.Ug}, {ns * c.Ug, ns * c.Ug + c.I, ns * c.Ug + 2 * c.I}, c.G, c.rank, sgl ? c.U : 0};
  SRB_TRY(step_begin(s->step_dev, s->scalars, s->lr, s->beta1, s->beta2, (int32_t*)umask, (int)((c.lp.nce_ws - c.lp.umask) / 4), s->batch, B,
                     d, c.lw(c.lp.seed), sg ? 1 : ns, rows, st));
  {
    BatchRowsArgs br = {};
    br.batch = s->batch;
    br.cap = B;
    br.umask = umask;
    br.imask = imask;
    br.world = c.G;
    br.rank = c.rank;
    br.n_graphs = c.lp.n_graphs;
    for (int q = 0; q < c.lp.n_graphs; ++q) {
      const Blocks bl = blocks(c, q);
      BatchRowLists& l = br.g[q];
      l.ru_rowptr = bl.ru->rowptr;
      l.rt_rowptr = bl.rt->rowptr;
      l.rows_u = (int32_t*)(c.loc + c.lp.rows_u[q]);
      l.rows_i = (int32_t*)(c.loc + c.lp.rows_i[q]);
      l.cnt = (int32_t*)(c.loc + c.lp.cnt) + 16 * q;
      l.hcap_u = bl.ru->hub.n_work;
      l.hcap_i = bl.rt->hub.n_work;
      l.hfirst_u = l.hcap_u ? (int32_t*)(c.loc + c.lp.hfirst_u[q]) : nullptr;
      l.hwork_u = (int32_t*)(c.loc + c.lp.hwork_u[q]);
      l.hfirst_i = l.hcap_i ? (int32_t*)(c.loc + c.lp.hfirst_i[q]) : nullptr;
      l.hwork_i = (int32_t*)(c.loc + c.lp.hwork_i[q]);
    }
    shard_batch_rows_kernel<<<(3 * B + 255) / 256, 256, 0, st>>>(br);
    SRB_TRY(post_launch("shard_batch_rows_kernel"));
  }
  const Blocks full = blocks(c, 0);

  // ---- forward ----
  float* su = c.lw(c.lp.su);
  float* si = c.mine(c.sp.fin_i);
  float* clu = c.lw(c.lp.clu);
  float* v2u = c.lw(c.lp.v2u);
  float* v2i = c.lw(c.lp.v2_i);
  const bool cl_hit = xs && s->layer_cl >= 1 && s->layer_cl <= L;
  if (lg) {
    SRB_TRY(encoder(c, full, true, 0, 0, 0, su, si, nullptr, -1, false, true));
  } else if (xs) {
    SRB_TRY(encoder(c, full, false, 2, 0, cl_hit ? s->layer_cl : 0, su, si, cl_hit ? clu : nullptr, c.sp.cl_i, false, true));
  } else if (sgl) {  // three encoders with the ego layer in the mean (SGL.py:98-113), the views into SimGCL's view buffers
    SRB_TRY(encoder(c, full, true, 0, 0, 0, su, si, nullptr, -1, false, true));
    SRB_TRY(encoder(c, blocks(c, 1), true, 0, 0, 0, clu, c.mine(c.sp.cl_i), nullptr, -1, false, true));
    SRB_TRY(encoder(c, blocks(c, 2), true, 0, 0, 0, v2u, v2i, nullptr, -1, false, true));
  } else if (L >= 2) {
    // layer 1 of SimGCL's three encoders is the same product (SimGCL.py:85): evaluated once into the backward
    // buffers (free until the backward pass), then perturbed per view (:87-88) -- users locally, the replicated
    // item table on every rank (the Philox stream is keyed by global row id: all replicas agree)
    float* zu = c.lw(c.lp.au[0]);
    float* zi = c.mine(c.sp.ai[0]);
    float* x1u[2] = {c.lw(c.lp.au[1]), c.seed_u(1)};
    float* x1i[2] = {c.mine(c.sp.ai[1]), c.seed_i(1)};
    {
      Epi e;
      e.y_u = zu;
      e.y_i = c.sp.ai[0];
      SRB_TRY(layer(c, full, s->pu, c.mine(c.sp.pi), e));
      SRB_TRY(wait_peers(c));  // every slice of the item half has arrived
    }
    for (int v = 0; v < 2; ++v) {
      Epi e;
      e.noise_mode = 2;
      e.poff = noise_offset(v, 0);
      if (c.Ug > 0) {
        SpmmArgs a;
        SRB_TRY(graph_args(s->Ru, c.Ug, c.I, c.d, zu, a));
        epi_common(c, e, a);
        a.noise_row_base = c.rank;
        a.noise_row_stride = c.G;
        a.Y = x1u[v];
        SRB_TRY(launch_rows_epilogue(a, c.d, st));
      }
      SpmmArgs a;
      SRB_TRY(graph_args(s->Rt, c.I, c.Ug, c.d, zi, a));
      epi_common(c, e, a);
      a.noise_row_base = c.U;
      a.Y = x1i[v];
      SRB_TRY(launch_rows_epilogue(a, c.d, st));
    }
    SRB_TRY(encoder(c, full, false, 0, 0, 0, su, si, nullptr, -1, false, true, zu, zi));
    SRB_TRY(encoder(c, full, false, 2, 0, 0, clu, c.mine(c.sp.cl_i), nullptr, -1, false, true, x1u[0], x1i[0]));
    SRB_TRY(encoder(c, full, false, 2, 1, 0, v2u, v2i, nullptr, -1, false, true, x1u[1], x1i[1]));
  } else {
    SRB_TRY(encoder(c, full, false, 0, 0, 0, su, si, nullptr, -1, false, true));
    SRB_TRY(encoder(c, full, false, 2, 0, 0, clu, c.mine(c.sp.cl_i), nullptr, -1, false, true));
    SRB_TRY(encoder(c, full, false, 2, 1, 0, v2u, v2i, nullptr, -1, false, true));
  }

  // ---- the rows the batch reads -> compact tables on every rank ----
  SRB_TRY(gather(c, su, si, c.sp.cmain, 0, sgl ? 3 : 5, true));
  if (xs) SRB_TRY(gather(c, cl_hit ? clu : s->pu, cl_hit ? c.mine(c.sp.cl_i) : c.mine(c.sp.pi), c.sp.cv1, 3, 5, false));
  if (sg || sgl) {
    SRB_TRY(gather(c, clu, c.mine(c.sp.cl_i), c.sp.cv1, 3, 5, false));
    SRB_TRY(gather(c, v2u, v2i, c.sp.cv2, 3, 5, false));
  }
  if (lg) SRB_TRY(gather(c, s->pu, c.mine(c.sp.pi), c.sp.cp, 0, 3, false));
  SRB_TRY(barrier(c));

  // ---- BPR + L2, InfoNCE on the compact tables (replicated); serial: the fork stream belongs to layer() ----
  // compact rows: u at k, i at B + k, j at 2B + k, unique users at 3B + k, unique items at 4B + k
  const int32_t* ar = (const int32_t*)(c.loc + c.lp.ar);
  const LossRows lr = {s->batch, ar, ar, ar + B, B, ar, ar, {3 * B, 4 * B}, (const int32_t*)(c.loc + c.lp.cat),
                       (const int32_t*)(c.loc + c.lp.n_cat), (const int32_t*)(c.loc + c.lp.cat_id)};
  const LossBufs lb = {c.lw(c.lp.g_emb), c.lw(c.lp.g_l2), c.lw(c.lp.g_nce), (size_t)B * d, c.lw(c.lp.bpr_scratch), c.lw(c.lp.bpr_losses),
                       c.lw(c.lp.nce_losses), c.loc + c.lp.nce_ws, c.lp.nce_ws_bytes, s->losses};
  SeedGrads gr;
  SRB_TRY(step_losses(s->model, s->reg, s->l2_div, s->tau, s->cl_rate, d, B, c.mine(c.sp.cmain), c.mine(c.sp.cp), c.mine(c.sp.cv1),
                      c.mine(c.sp.cv2), lr, lb, nullptr, nullptr, gr, st));

  // ---- backward: engine.cu's Horner chains on layer() + Adam ----
  ScatterSegs segs = {};
  const int g_level = seed_segments(s->model, L, s->layer_cl, gr, rows, segs);
  SRB_TRY(scatter_segments(c.lw(c.lp.seed), d, segs, st));
  if (!sgl) return chain(c, full, 0, g_level, lg, nullptr, nullptr, false, false);
  // SGL's three graphs differ: the two view chains sum into gd, then the graph's chain adds it and applies Adam.  gd is a
  // local table (view 2's forward buffers, free once gathered) and is never pushed: its item rows are only read by this
  // rank's reduction of its own slice.
  SRB_TRY(chain(c, blocks(c, 1), 0, -1, true, v2u, v2i, true, false));
  SRB_TRY(chain(c, blocks(c, 2), 1, -1, true, v2u, v2i, true, true));
  return chain(c, full, 2, -1, true, v2u, v2i, false, true);
}

/* Clean forward for evaluation / save() (XSimGCL.py:40-41, 53-55): the final mean of this rank's users goes to
 * out_user [n_local_users, d]; the item half lands, complete, in every rank's symmetric region at
 * srb_shard_layout.item_final. */
extern "C" int srb_shard_forward(const srb_shard_desc* s, float* out_user, void* stream) {
  using namespace srb;
  Ctx c;
  SRB_TRY(make_ctx(s, stream, c));
  SRB_REQUIRE(out_user != nullptr || c.Ug == 0, "shard_forward: null output");
  const bool ego = s->model == SRB_MODEL_LIGHTGCN || s->model == SRB_MODEL_SGL;
  SRB_TRY(encoder(c, blocks(c, 0), ego, 0, 0, 0, out_user, c.mine(c.sp.fin_i), nullptr, -1, true, false));
  return wait_peers(c);  // every slice of the item output has arrived
}
