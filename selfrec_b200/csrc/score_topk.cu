// (iv) Full-catalog scoring + rated-item mask + top-k   (impl 1: CUDA-core fp32).
//
// Replaces the per-user loop of GraphRecommender.test() base/graph_recommender.py:38-58:
//   candidates = predict(user)            XSimGCL.py:57-60  (user_emb[u] @ item_emb.T)
//   candidates[rated] = -10e8             graph_recommender.py:48-50
//   find_k_largest(max_N, candidates)     util/algorithm.py:144-156
//
// One CTA scores 32 users against the whole catalogue in tiles of 128 items, each score the
// exact fp32 chain of rank_common.cuh.  The warp that computed a user's scores also owns that
// user's top-k list (list_offer32, one entry per lane) and visits the items in id order, so the
// final set equals find_k_largest's, ties included.
#include "common.cuh"
#include "rank_common.cuh"

namespace srb {

constexpr int TK_TM = 32;   // users per CTA
constexpr int TK_TN = 128;  // items per tile

struct TopkArgs {
  const float* user_emb;
  const float* item_emb;
  int32_t n_items;
  const int32_t* users;
  int32_t n_q;
  const int32_t* rated_ptr;
  const int32_t* rated_idx;
  int32_t k;
  int32_t* out_ids;
  float* out_scores;
  const int32_t* q_map;    // optional: output row of query q (fallback path of impl 2)
  const int32_t* n_q_dev;  // optional: device-side query count (<= n_q)
  int32_t q_skip;          // first q_skip queries are handled elsewhere (fast fallback)
};

template <int D>
__global__ void __launch_bounds__(256) score_topk_kernel(const TopkArgs a) {
  extern __shared__ __align__(16) float tk_smem[];
  float (*Us)[TK_TM] = reinterpret_cast<float (*)[TK_TM]>(tk_smem);                   // [D][32] k-major
  float (*Is)[D + 1] = reinterpret_cast<float (*)[D + 1]>(tk_smem + D * TK_TM);       // [128][D+1]
  const int lane = threadIdx.x & 31;
  const int ty = threadIdx.x >> 5;  // warp id: users ty*4 .. ty*4+3 of the CTA tile
  const int q0 = a.q_skip + blockIdx.x * TK_TM;
  const int n_q = a.n_q_dev ? min(*a.n_q_dev, a.n_q) : a.n_q;
  if (q0 >= n_q) return;

  // user tile (gathered by id), transposed to k-major
  for (int e = threadIdx.x; e < TK_TM * (D / 4); e += blockDim.x) {
    const int u = e % TK_TM, k4 = e / TK_TM;
    float4 v = f4_zero();
    if (q0 + u < n_q) v = ldg4(a.user_emb + (size_t)a.users[q0 + u] * D + k4 * 4);
    Us[k4 * 4 + 0][u] = v.x;
    Us[k4 * 4 + 1][u] = v.y;
    Us[k4 * 4 + 2][u] = v.z;
    Us[k4 * 4 + 3][u] = v.w;
  }

  // per-user state of this warp: sorted list entry per lane, mask cursor
  float ls[4];
  int li[4];
  int cur[4], cend[4];
  int ev[4];  // lane l holds rated_idx[cur + l] of user r (reloaded only when the cursor moves)
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    ls[r] = -INFINITY;
    li[r] = -1;
    const int q = q0 + ty * 4 + r;
    if (q < n_q && a.rated_ptr) {
      const int u = a.users[q];
      cur[r] = a.rated_ptr[u];
      cend[r] = a.rated_ptr[u + 1];
    } else {
      cur[r] = cend[r] = 0;
    }
    ev[r] = (cur[r] + lane < cend[r]) ? a.rated_idx[cur[r] + lane] : 0x7fffffff;
  }
  const int K = a.k;

  for (int n0 = 0; n0 < a.n_items; n0 += TK_TN) {
    __syncthreads();
    for (int e = threadIdx.x; e < TK_TN * (D / 4); e += blockDim.x) {
      const int row = e / (D / 4), c4 = e % (D / 4);
      float4 v = f4_zero();
      if (n0 + row < a.n_items) v = ldg4(a.item_emb + (size_t)(n0 + row) * D + c4 * 4);
      Is[row][c4 * 4 + 0] = v.x;
      Is[row][c4 * 4 + 1] = v.y;
      Is[row][c4 * 4 + 2] = v.z;
      Is[row][c4 * 4 + 3] = v.w;
    }
    __syncthreads();
    float s[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) s[r][c] = 0.f;
    // register-blocked 4 x 4 form of exact_score (rank_common.cuh): each s[r][c] is the same chain, k = 0..D-1 from +0
#pragma unroll 8
    for (int k = 0; k < D; ++k) {
      const float4 uv = *reinterpret_cast<const float4*>(&Us[k][ty * 4]);
      const float ur[4] = {uv.x, uv.y, uv.z, uv.w};
      float iv[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) iv[c] = Is[lane + 32 * c][k];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) s[r][c] = fmaf(ur[r], iv[c], s[r][c]);
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      // items past the end of the catalogue can never enter
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (n0 + lane + 32 * c >= a.n_items) s[r][c] = -INFINITY;
      // rated-item mask: walk this user's sorted rated list through the tile
      while (true) {
        const unsigned in = __ballot_sync(SRB_FULL_MASK, ev[r] < n0 + TK_TN);
        const int cnt = __popc(in);
        if (cnt == 0) break;
        for (int t = 0; t < cnt; ++t) {
          const int et = __shfl_sync(SRB_FULL_MASK, ev[r], t) - n0;
          if (et >= 0 && (et & 31) == lane) {
            const int c = et >> 5;
#pragma unroll
            for (int cc = 0; cc < 4; ++cc)
              if (cc == c) s[r][cc] = TK_MASKED;
          }
        }
        cur[r] += cnt;
        ev[r] = (cur[r] + lane < cend[r]) ? a.rated_idx[cur[r] + lane] : 0x7fffffff;
        if (cnt < 32) break;
      }
      // sequential (id-ordered) insertion, 32 candidates per round
#pragma unroll
      for (int c = 0; c < 4; ++c) list_offer32(ls[r], li[r], s[r][c], n0 + lane + 32 * c, K);
    }
  }
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int q = q0 + ty * 4 + r;
    if (q < n_q && lane < K) {
      const size_t orow = a.q_map ? (size_t)a.q_map[q] : (size_t)q;
      a.out_ids[orow * K + lane] = li[r];
      a.out_scores[orow * K + lane] = ls[r];
    }
  }
}

// top-k of score rows, one warp per row, same sequential insertion rule as above: precomputed rows of models whose
// predict() is not a single dot product (SURVEY 8b), and the exact rows of impl 2's fast fallback.  Optional: n_q_dev,
// a device-side row count (<= n_q); q_map, the output row of row q.
__global__ void __launch_bounds__(256) topk_rows_kernel(const float* scores, int n_q, const int32_t* n_q_dev, const int32_t* q_map,
                                                        int n_items, int k, int32_t* out_ids, float* out_scores) {
  const int lane = threadIdx.x & 31;
  const int q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (q >= n_q || (n_q_dev && q >= *n_q_dev)) return;
  float ls = -INFINITY;
  int li = -1;
  const float* row = scores + (size_t)q * n_items;
  for (int n0 = 0; n0 < n_items; n0 += 32) {
    const int id = n0 + lane;
    list_offer32(ls, li, (id < n_items) ? row[id] : -INFINITY, id, k);
  }
  if (lane < k) {
    const size_t orow = q_map ? (size_t)q_map[q] : (size_t)q;
    out_ids[orow * k + lane] = li;
    out_scores[orow * k + lane] = ls;
  }
}

// exact score of item i for user u, whose row `us` sits in shared memory; TK_MASKED when i is in u's sorted rated list
template <int D>
__device__ __forceinline__ float masked_score(const float* us, const float* item_emb, int i, int u, const int32_t* rated_ptr,
                                              const int32_t* rated_idx) {
  const float* it = item_emb + (size_t)i * D;
  const float acc = exact_score<D>([&](int c) { return reinterpret_cast<const float4*>(us)[c]; }, [&](int c) { return ldg4(it + c * 4); });
  return (rated_ptr && sorted_contains(rated_idx, rated_ptr[u], rated_ptr[u + 1], i)) ? TK_MASKED : acc;
}

// dense score rows out[q][i] = <user_emb[users[q]], item_emb[i]>: the reference's predict() (XSimGCL.py:57-60) for
// callers that want the raw vector, and, with the rated CSR and a device-side row count n_q_dev (<= n_q), the masked
// rows of impl 2's fast fallback.  Rows stride over gridDim.y: the fallback usually has no rows, and a small grid.y
// keeps that case cheap.
template <int D>
__global__ void __launch_bounds__(256) score_rows_kernel(const float* user_emb, const float* item_emb, const int32_t* users, int n_q,
                                                         const int32_t* n_q_dev, const int32_t* rated_ptr, const int32_t* rated_idx,
                                                         int n_items, float* out) {
  __shared__ __align__(16) float us[D];
  const int count = n_q_dev ? min(*n_q_dev, n_q) : n_q;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  for (int q = blockIdx.y; q < count; q += gridDim.y) {
    const int u = users[q];
    __syncthreads();
    for (int k = threadIdx.x; k < D; k += blockDim.x) us[k] = user_emb[(size_t)u * D + k];
    __syncthreads();
    if (i < n_items) out[(size_t)q * n_items + i] = masked_score<D>(us, item_emb, i, u, rated_ptr, rated_idx);
  }
}

int score_topk_tc(const srb_topk_desc* d, cudaStream_t st);  // score_topk_tc.cu

static TopkArgs topk_args(const srb_topk_desc* d) {
  return TopkArgs{d->user_emb, d->item_emb, d->n_items, d->users, d->n_q, d->rated_ptr, d->rated_idx, d->k, d->out_ids, d->out_scores,
                  nullptr, nullptr, 0};
}

template <int D>
static int launch_topk(const TopkArgs& a, cudaStream_t st) {
  const size_t smem = sizeof(float) * (D * TK_TM + TK_TN * (D + 1));
  static bool attr_done = false;
  if (!attr_done) {
    SRB_TRY(check_cuda(cudaFuncSetAttribute(score_topk_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "topk smem attr"));
    attr_done = true;
  }
  const int blocks = (a.n_q - a.q_skip + TK_TM - 1) / TK_TM;
  if (blocks <= 0) return SRB_OK;
  score_topk_kernel<D><<<blocks, 256, smem, st>>>(a);
  return post_launch("score_topk_kernel");
}

// ---- fallback of impl 2: exact re-run of the users it could not certify (device-side list) ----
// Long lists (k > 32): one CTA per uncertified user at a time, at most `cap` users in flight (one scratch row each).
// The CTA writes the user's exact masked row, finds the k-th largest score s* by a 4-pass 8-bit radix select, keeps
// every score above it and, of the scores equal to it, find_k_largest's choice: among those within the first k items
// (in id order) scoring >= s* -- the ones that entered the list -- the largest ids, as many as the list has room for
// (tc_rescore_long_kernel states the rule), and writes the list score-descending, ties by id descending.
template <int D>
__global__ void __launch_bounds__(256, 1) fb_long_kernel(const float* __restrict__ user_emb, const float* __restrict__ item_emb,
                                                     const int32_t* __restrict__ fb_users, const int32_t* __restrict__ fb_rows,
                                                     const int32_t* __restrict__ fb_count, const int32_t* __restrict__ rated_ptr,
                                                     const int32_t* __restrict__ rated_idx, int n_items, int k, float* scratch,
                                                     int32_t* out_ids, float* out_scores) {
  __shared__ __align__(16) float us[D];
  __shared__ int hist[256];
  __shared__ uint32_t sel_k[256];  // kept entries: okey of the score, id
  __shared__ int32_t sel_i[256];
  __shared__ int32_t tie_i[256];  // tied items that entered the list, in id order
  __shared__ int wsum[8];
  __shared__ int s_need, s_nsel, s_ent;
  __shared__ uint32_t s_pref;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int count = *fb_count;
  float* row = scratch + (size_t)blockIdx.x * n_items;
  for (int slot = blockIdx.x; slot < count; slot += gridDim.x) {
    const int u = fb_users[slot];
    __syncthreads();
    for (int kk = tid; kk < D; kk += 256) us[kk] = user_emb[(size_t)u * D + kk];
    __syncthreads();
    for (int i = tid; i < n_items; i += 256) row[i] = masked_score<D>(us, item_emb, i, u, rated_ptr, rated_idx);
    __syncthreads();
    // radix select of the k-th largest key: pref = its key, need = how many of the entries equal to it to keep
    uint32_t pref = 0, pmask = 0;
    int need = k;
    for (int shift = 24; shift >= 0; shift -= 8) {
      hist[tid] = 0;
      __syncthreads();
      for (int i = tid; i < n_items; i += 256) {
        const uint32_t key = okey(row[i]);
        if ((key & pmask) == pref) atomicAdd(&hist[(key >> shift) & 255], 1);
      }
      __syncthreads();
      if (tid == 0) {
        int cum = 0, b = 255;
        for (; b > 0 && cum + hist[b] < need; --b) cum += hist[b];
        s_need = need - cum;
        s_pref = pref | ((uint32_t)b << shift);
        s_nsel = 0;
      }
      __syncthreads();
      need = s_need;
      pref = s_pref;
      pmask |= 0xffu << shift;
    }
    // above the k-th: any slot of the first k - need; equal to it: the `need` smallest ids, visited in id order
    for (int i = tid; i < n_items; i += 256) {
      const uint32_t key = okey(row[i]);
      if (key > pref) {
        const int p = atomicAdd(&s_nsel, 1);
        sel_k[p] = key;
        sel_i[p] = i;
      }
    }
    // walk the items in id order until k of them score >= s*; the tied ones among them entered
    int seen = 0, ties = 0;
    if (tid == 0) s_ent = 0;
    __syncthreads();
    for (int base = 0; base < n_items && seen < k; base += 256) {
      const int i = base + tid;
      const uint32_t key = i < n_items ? okey(row[i]) : 0u;
      const bool ge = i < n_items && key >= pref, tie = i < n_items && key == pref;
      const unsigned bg = __ballot_sync(SRB_FULL_MASK, ge), bt = __ballot_sync(SRB_FULL_MASK, tie);
      if (lane == 0) wsum[wid] = __popc(bg) | (__popc(bt) << 16);
      __syncthreads();
      int og = 0, ot = 0, tg = 0, tt = 0;
#pragma unroll
      for (int w = 0; w < 8; ++w) {
        const int v = wsum[w];
        og += (w < wid) ? (v & 0xffff) : 0;
        ot += (w < wid) ? (v >> 16) : 0;
        tg += v & 0xffff;
        tt += v >> 16;
      }
      const unsigned lt = (1u << lane) - 1u;
      if (tie && seen + og + __popc(bg & lt) < k) {  // entered: the entered ties are a prefix of the ties
        const int t = ties + ot + __popc(bt & lt);
        tie_i[t] = i;
        atomicMax(&s_ent, t + 1);
      }
      seen += tg;
      ties += tt;
      __syncthreads();
    }
    ties = s_ent;
    for (int t = tid; t < k; t += 256) {
      if (t >= k - need) {  // the largest `need` ids of the entered ties
        sel_k[t] = pref;
        sel_i[t] = tie_i[ties - (k - t)];
      }
    }
    __syncthreads();
    const size_t orow = (size_t)fb_rows[slot];
    write_ranked(sel_k, sel_i, k, [](int) { return true; }, out_ids + orow * k, out_scores + orow * k);
  }
}

template <int D>
static int score_topk_fallback_d(const srb_topk_desc* d, const int32_t* fb_users, const int32_t* fb_rows, const int32_t* fb_count,
                                 float* scratch, int fb_cap, cudaStream_t st) {
  if (d->k > 32) {  // long lists: every uncertified user, fb_cap at a time
    fb_long_kernel<D><<<fb_cap, 256, 0, st>>>(d->user_emb, d->item_emb, fb_users, fb_rows, fb_count, d->rated_ptr, d->rated_idx,
                                              d->n_items, d->k, scratch, d->out_ids, d->out_scores);
    return post_launch("fb_long_kernel");
  }
  // fast path for the first fb_cap users: exact score rows spread over many CTAs + one warp per user for the sequential
  // top-k (a handful of users must not cost a full impl-1 pass over the catalogue)
  dim3 grid((d->n_items + 255) / 256, fb_cap < 8 ? fb_cap : 8);
  score_rows_kernel<D><<<grid, 256, 0, st>>>(d->user_emb, d->item_emb, fb_users, fb_cap, fb_count, d->rated_ptr, d->rated_idx, d->n_items,
                                             scratch);
  SRB_TRY(post_launch("score_rows_kernel"));
  topk_rows_kernel<<<(fb_cap + 7) / 8, 256, 0, st>>>(scratch, fb_cap, fb_count, fb_rows, d->n_items, d->k, d->out_ids, d->out_scores);
  SRB_TRY(post_launch("topk_rows_kernel"));
  // slow path: everyone beyond fb_cap goes through the impl-1 kernel (CTAs without work exit at once)
  if (d->n_q <= fb_cap) return SRB_OK;
  TopkArgs a = topk_args(d);
  a.users = fb_users;
  a.q_map = fb_rows;
  a.n_q_dev = fb_count;
  a.q_skip = fb_cap;
  return launch_topk<D>(a, st);
}

int score_topk_fallback(const srb_topk_desc* d, const int32_t* fb_users, const int32_t* fb_rows, const int32_t* fb_count,
                        float* scratch, int fb_cap, cudaStream_t st) {
  switch (d->d) {  // the widths score_topk_tc accepts
    case 16: return score_topk_fallback_d<16>(d, fb_users, fb_rows, fb_count, scratch, fb_cap, st);
    case 32: return score_topk_fallback_d<32>(d, fb_users, fb_rows, fb_count, scratch, fb_cap, st);
    case 128: return score_topk_fallback_d<128>(d, fb_users, fb_rows, fb_count, scratch, fb_cap, st);
    case 256: return score_topk_fallback_d<256>(d, fb_users, fb_rows, fb_count, scratch, fb_cap, st);
    default: return score_topk_fallback_d<64>(d, fb_users, fb_rows, fb_count, scratch, fb_cap, st);
  }
}

}  // namespace srb

extern "C" int srb_score_topk(const srb_topk_desc* d, void* stream) {
  SRB_REQUIRE(d != nullptr, "topk: null desc");
  SRB_REQUIRE(d->n_q >= 0, "topk: negative n_q");
  if (d->n_q == 0) return SRB_OK;  // empty query list: nothing to launch (pointers may be null)
  SRB_REQUIRE(d->user_emb && d->item_emb && d->users && d->out_ids && d->out_scores, "topk: null pointer");
  SRB_REQUIRE((d->rated_ptr == nullptr) == (d->rated_idx == nullptr), "topk: rated_ptr/rated_idx must both be set or both null");
  SRB_REQUIRE(d->n_items >= 1, "topk: bad shape");
  SRB_REQUIRE(d->impl >= 0 && d->impl <= 2, "topk: bad impl");
  // auto (impl 0): impl 2 from 1024 items on, at every width for lists of up to 32 and at d = 64 / 128 for longer ones
  const bool tc_width = d->d == 64 || d->d == 128 || (d->k <= 32 && (d->d == 16 || d->d == 32 || d->d == 256));
  const bool tc = d->impl == 2 || (d->impl == 0 && tc_width && d->workspace != nullptr && d->n_items >= 1024);
  // impl 1 keeps one list entry per lane (k <= 32); impl 2 also takes the long lists (k <= 256)
  SRB_REQUIRE(d->k >= 1 && d->k <= (tc ? 256 : 32), "topk: k=%d unsupported (1..32; impl 2: 1..256)", d->k);
  SRB_REQUIRE(d->k <= 32 || d->k <= d->n_items, "topk: k=%d exceeds n_items=%d", d->k, d->n_items);
  if (tc) return srb::score_topk_tc(d, (cudaStream_t)stream);
  const srb::TopkArgs a = srb::topk_args(d);
  switch (d->d) {
    case 16: return srb::launch_topk<16>(a, (cudaStream_t)stream);
    case 32: return srb::launch_topk<32>(a, (cudaStream_t)stream);
    case 64: return srb::launch_topk<64>(a, (cudaStream_t)stream);
    case 128: return srb::launch_topk<128>(a, (cudaStream_t)stream);
    case 256: return srb::launch_topk<256>(a, (cudaStream_t)stream);  // 164 KB of shared memory (opt-in)
    default: srb::set_error("topk: unsupported d=%d (16, 32, 64, 128, 256)", d->d); return SRB_ERR_ARG;
  }
}

extern "C" int srb_topk_rows(const float* scores, int32_t n_q, int32_t n_items, int32_t k, int32_t* out_ids,
                             float* out_scores, void* stream) {
  SRB_REQUIRE(scores && out_ids && out_scores, "topk_rows: null pointer");
  SRB_REQUIRE(k >= 1 && k <= 32, "topk_rows: k=%d unsupported (1..32)", k);
  SRB_REQUIRE(n_q >= 0 && n_items >= 1, "topk_rows: bad shape");
  if (n_q == 0) return SRB_OK;
  srb::topk_rows_kernel<<<(n_q + 7) / 8, 256, 0, (cudaStream_t)stream>>>(scores, n_q, nullptr, nullptr, n_items, k, out_ids, out_scores);
  return srb::post_launch("topk_rows_kernel");
}

extern "C" int srb_score_rows(const float* user_emb, const float* item_emb, int32_t d, const int32_t* users, int32_t n_q,
                              int32_t n_items, float* out, void* stream) {
  SRB_REQUIRE(user_emb && item_emb && users && out, "score_rows: null pointer");
  SRB_REQUIRE(n_q >= 0 && n_q <= 65535 && n_items >= 1, "score_rows: bad shape (n_q <= 65535)");
  if (n_q == 0) return SRB_OK;
  dim3 grid((n_items + 255) / 256, n_q);
  cudaStream_t st = (cudaStream_t)stream;
  switch (d) {
    case 16: srb::score_rows_kernel<16><<<grid, 256, 0, st>>>(user_emb, item_emb, users, n_q, nullptr, nullptr, nullptr, n_items, out); break;
    case 32: srb::score_rows_kernel<32><<<grid, 256, 0, st>>>(user_emb, item_emb, users, n_q, nullptr, nullptr, nullptr, n_items, out); break;
    case 64: srb::score_rows_kernel<64><<<grid, 256, 0, st>>>(user_emb, item_emb, users, n_q, nullptr, nullptr, nullptr, n_items, out); break;
    case 128: srb::score_rows_kernel<128><<<grid, 256, 0, st>>>(user_emb, item_emb, users, n_q, nullptr, nullptr, nullptr, n_items, out); break;
    case 256: srb::score_rows_kernel<256><<<grid, 256, 0, st>>>(user_emb, item_emb, users, n_q, nullptr, nullptr, nullptr, n_items, out); break;
    default: srb::set_error("score_rows: unsupported d=%d (16, 32, 64, 128, 256)", d); return SRB_ERR_ARG;
  }
  return srb::post_launch("score_rows_kernel");
}

namespace srb {
// one warp per query row: lane r (and r + 32, ...) looks its recommended id up in the user's sorted test list;
// ceil(k / 64) words per row, bit r % 64 of word r / 64 for rank r
__global__ void __launch_bounds__(256) rank_hit_masks_kernel(const int32_t* __restrict__ ids, int n_q, int k, const int32_t* __restrict__ users,
                                                             const int32_t* __restrict__ test_ptr, const int32_t* __restrict__ test_idx,
                                                             unsigned long long* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (q >= n_q) return;
  const int u = users[q];
  const int beg = test_ptr[u], end = test_ptr[u + 1];
  const int words = (k + 63) / 64;
  for (int wd = 0; wd < words; ++wd) {
  unsigned long long mask = 0;
  for (int half = 0; half < 2; ++half) {
    const int r = wd * 64 + half * 32 + lane;
    const bool hit = r < k && sorted_contains(test_idx, beg, end, ids[(size_t)q * k + r]);
    mask |= (unsigned long long)__ballot_sync(SRB_FULL_MASK, hit) << (32 * half);
  }
  if (lane == 0) out[(size_t)q * words + wd] = mask;
  }
}
}  // namespace srb

extern "C" int srb_rank_hit_masks(const int32_t* topk_ids, int32_t n_q, int32_t k, const int32_t* users, const int32_t* test_ptr,
                                  const int32_t* test_idx, uint64_t* hit_mask, void* stream) {
  SRB_REQUIRE(n_q >= 0 && k >= 1 && k <= 256, "rank_hit_masks: k must be 1..256");
  if (n_q == 0) return SRB_OK;
  SRB_REQUIRE(topk_ids && users && test_ptr && test_idx && hit_mask, "rank_hit_masks: null pointer");
  srb::rank_hit_masks_kernel<<<(n_q + 7) / 8, 256, 0, (cudaStream_t)stream>>>(topk_ids, n_q, k, users, test_ptr, test_idx,
                                                                              reinterpret_cast<unsigned long long*>(hit_mask));
  return srb::post_launch("rank_hit_masks_kernel");
}
