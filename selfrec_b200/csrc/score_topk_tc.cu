// (iv) impl 2: full-catalog scoring on the Hopper tensor cores (wgmma, TF32) with fused
// rated-item mask + candidate selection, followed by exact fp32 re-scoring.
//
// Replaces GraphRecommender.test() base/graph_recommender.py:38-58 (predict XSimGCL.py:57-60,
// mask :48-50, find_k_largest util/algorithm.py:144-156), same contract as impl 1.
//
// The kernels are templated on the embedding size D in {16, 32, 64, 128, 256}.
//
// Stage 1  tc_gather_kernel     users[q] rows -> contiguous [n_q, d] table (TMA cannot gather),
//                               ||u_q||, max_i ||item_i||
// Stage 2  tc_score_kernel      one CTA per block of UB <= 128 users, streaming the whole catalogue in
//                               tiles of 128 items:
//            warp 8     TMA producer: item tiles [128 x D] fp32 in 32-float k-chunks, 128B-swizzled, through an
//                       mbarrier ring (D = 64: a stage is a whole tile; D = 128: a stage is one k-chunk, four stages
//                       per tile, so the 64 KB user tile fits beside the ring; D = 16: a chunk is the 16 columns and
//                       TMA's zero fill; D = 256: a stage is one item k-chunk and the users' same k-chunk, three
//                       stages, since a resident 128 KB user tile would not fit -- DESIGN 4.4)
//            warpgroups 0, 1  (64 users each): wgmma m64n128k8 kind tf32, D/8 k-steps per tile, accumulators in
//                       registers -> staged to shared memory row-major -> select: thread = one user row x one
//                       64-column half of the tile, rated-item cursor, per-thread top-24 candidate list
//                       (3 buckets of 8, minima in registers) in shared memory -> 2 x 24 candidates per user
//          The raw fp32 tables are fed to the tensor core, which reads them as TF32 (low 13
//          mantissa bits ignored): scores carry <= 2^-9 ||u|| ||i|| error -- candidates only.
// Stage 3  tc_rescore_kernel    warp per user: exact fp32 fma-chain scores of the 2 x 24 candidates
//                               (bit-identical to impl 1 / the oracle), find_k_largest's sequential
//                               insertion in id order, and a safety test: every non-candidate of a column
//                               half has approx score <= that half's 24th best, so the result is exact iff
//                               thr32 := max of the two + E(D) < exact k-th score.  Users failing it (or with fewer than
//                               k unrated items) are re-run by the exact CUDA-core kernel (impl 1).
// Lists of 33..256 (tc_score_kernel<D, true>): the select keeps, per user row x column half, a candidate buffer in global
// memory behind a running threshold instead of the 24-slot list; tc_rescore_long_kernel (CTA per user) rescoring and
// certifying them, fb_long_kernel (score_topk.cu) re-running the uncertified users (DESIGN 4.4).
#include "common.cuh"
#include "rank_common.cuh"
#include "tc_common.cuh"

namespace srb {

using namespace tc;

constexpr int TC_TN = 128;        // items per tile (wgmma N)
constexpr int TC_UB = 128;        // users per CTA: two consumer warpgroups of 64 (wgmma M)
constexpr int TC_STAGES = 2;      // smem ring depth at d <= 128 (a tile's select takes microseconds: one tile of prefetch is enough)
constexpr int TC_LIST = 24;       // candidates per list; every user has two lists, one per column half of the tiles
constexpr int TC_CAND = 2 * TC_LIST;
constexpr int TC_THREADS = 256 + 32;   // warpgroups 0-1 MMA + select, warp 8 TMA
constexpr int TC_SROW = TC_TN + 4;     // staged accumulator row stride (floats): conflict-free float4 row reads
constexpr uint32_t TC_CHUNK_BYTES = 128 * 32 * 4;     // 16 KB: one k-chunk [128 rows][32] fp32 of a user or item tile

// per-width layout: a tile row is KC 32-float k-chunks (D = 16: one, half of it TMA's zero fill beyond the row, of which
// the MMA reads the first 16 columns); a ring stage holds SC item chunks and, when the users stream (US), the users'
// same chunk
template <int D>
struct TcShape {
  static_assert(D == 16 || D == 32 || D == 64 || D == 128 || D == 256, "tensor-core ranking: D in {16, 32, 64, 128, 256}");
  static constexpr int KC = D < 32 ? 1 : D / 32;          // k-chunks per tile row
  static constexpr int KS = D < 32 ? D / 8 : 4;           // wgmma k-steps per k-chunk
  static constexpr int SC = (D == 64) ? 2 : 1;            // item k-chunks per ring stage
  static constexpr int SPT = KC / SC;                     // ring stages per item tile
  static constexpr bool US = D == 256;                    // user chunks stream through the ring beside the items'
  static constexpr int STAGES = US ? 3 : TC_STAGES;
  static constexpr uint32_t STAGE_BYTES = (SC + US) * TC_CHUNK_BYTES;      // 32 KB (D = 64, 256) / 16 KB (others)
  static constexpr uint32_t USER_BYTES = US ? 0 : KC * TC_CHUNK_BYTES;     // resident user tile: 16 / 16 / 32 / 64 KB
  // |approx - exact| <= E * ||u|| * max||i||: the TF32 operand term 2^-9 (independent of D), the accumulation term
  // 2^-19 per k-step of 8 (it grows with the chain of D / 8 k-steps: 2^-18 at D = 16 ... 2^-14 at D = 256) and 2^-18
  // for the slot tags and the final roundings (DESIGN 4.4)
  static constexpr float E = 1.0f / 512.0f + (float)(D / 8) * (1.0f / 524288.0f) + 1.0f / 262144.0f;
};

template <int D>
struct TcSmem {
  // dynamic shared memory, 1024-byte aligned base:
  //   [0, U)            resident user tile: chunk c at c * 16 KB (warpgroup w's 64 rows at + w * 8 KB); U = 0 at D = 256
  //   [U, U + N S)      N ring stages of S bytes: item chunk c at + c * 16 KB, then (D = 256) the users' chunk
  //   then the staged accumulators [2 warpgroups][64][TC_SROW] f32                  (66 KB)
  //   then candidate lists: scores [24][256] f32, ids [24][256] i32               (48 KB)
  //   then barriers         total 162 KB (D = 16, 32) / 210 KB (D = 64, 128, 256) + 256 B
  static constexpr uint32_t users_off = 0;
  static constexpr uint32_t items_off = TcShape<D>::USER_BYTES;
  static constexpr uint32_t stage_off = items_off + TcShape<D>::STAGES * TcShape<D>::STAGE_BYTES;
  static constexpr uint32_t cand_s_off = stage_off + TC_UB * TC_SROW * 4;
  static constexpr uint32_t cand_i_off = cand_s_off + TC_LIST * 2 * TC_UB * 4;
  static constexpr uint32_t bar_off = cand_i_off + TC_LIST * 2 * TC_UB * 4;
  static constexpr uint32_t total = bar_off + 256;
};

// the workspace carved by tc_carve; the rescoring kernels read it and the caller's srb_topk_desc in place from the
// parameter space (__grid_constant__)
struct TcWorkspace {
  float* ug;          // gathered user rows [n_q_pad][d]
  float* unorm;       // ||u_q|| (tc_gather_kernel)
  unsigned int* bmax; // bits of max ||item||: with unorm, the scale of the error bound E
  float* cand_s;      // [n_q][2][24] approx scores
  int32_t* cand_i;    // [n_q][2][24]
  int32_t* cand_n;    // [n_q][2]
  float* cand_thr;    // [n_q][2] min approx score of a full list, else -inf (long lists: final running threshold)
  int32_t* fb_count;  // device counter of users needing the exact fallback
  int32_t* fb_rows;   // their query rows
  int32_t* fb_users;  // their user ids
  float* fb_scratch;  // [fb_cap][n_items] exact score rows of the users re-run by the fast fallback
  int32_t fb_cap;
  float* buf_s;       // long lists: [n_q][2][cap] candidate buffers (empty at k <= 32)
  int32_t* buf_i;
  int32_t cap;
  int64_t bytes;
};

// tc_score_kernel's arguments, taken from the desc and the workspace.  The kernel does not take those two whole as the
// rescoring kernels do: ptxas then allocates its registers differently (102 -> 100 at d = 64, DESIGN 4.4), and the
// hot kernel is kept as it was measured
struct TcArgs {
  const int32_t* users;
  const int32_t* rated_ptr;
  const int32_t* rated_idx;
  int32_t n_q;
  int32_t n_items;
  int32_t ub;                // users per CTA (<= TC_UB)
  float* cand_s;
  int32_t* cand_i;
  int32_t* cand_n;
  float* cand_thr;
  int32_t k;
  int32_t cap;
  float* buf_s;
  int32_t* buf_i;
  const float* unorm;
  const unsigned int* bmax_bits;
};

constexpr int TC_LONG_MAX = 256;  // longest list of the long-list route

// per-half candidate capacity of a long list of k: room for the k best, the 2E band below them and a refill
static int tc_long_cap(int k) { return (2 * k + 256 + 31) / 32 * 32; }

template <int D>
struct TcVec;  // the D/32 floats of a row that one lane gathers (D = 16: lanes 0-15 one float each)
template <>
struct TcVec<16> {
  using T = float;
  static __device__ __forceinline__ T zero() { return 0.f; }
  static __device__ __forceinline__ float ss(T v) { return v * v; }
};
template <>
struct TcVec<32> : TcVec<16> {};
template <>
struct TcVec<64> {
  using T = float2;
  static __device__ __forceinline__ T zero() { return make_float2(0.f, 0.f); }
  static __device__ __forceinline__ float ss(T v) { return v.x * v.x + v.y * v.y; }
};
template <>
struct TcVec<128> {
  using T = float4;
  static __device__ __forceinline__ T zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
  static __device__ __forceinline__ float ss(T v) { return v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w; }
};
struct alignas(16) TcF8 {
  float4 a, b;
};
template <>
struct TcVec<256> {
  using T = TcF8;
  static __device__ __forceinline__ T zero() { return TcF8{TcVec<128>::zero(), TcVec<128>::zero()}; }
  static __device__ __forceinline__ float ss(T v) { return TcVec<128>::ss(v.a) + TcVec<128>::ss(v.b); }
};

template <int D>
__global__ void __launch_bounds__(256) tc_gather_kernel(const float* __restrict__ user_emb, const int32_t* __restrict__ users, int n_q,
                                                       int n_q_pad, float* __restrict__ ug, float* __restrict__ unorm,
                                                       const float* __restrict__ item_emb, int n_items, unsigned int* bmax_bits) {
  const int lane = threadIdx.x & 31;
  const int w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  // rows [0, n_q_pad): gathered user rows; rows [n_q_pad, n_q_pad + n_items): item norms
  using V = TcVec<D>;
  constexpr int PL = D < 32 ? 1 : D / 32;  // floats per lane
  const bool ln = D >= 32 || lane < D;    // this lane holds floats of the row
  if (w < n_q_pad) {
    typename V::T v = V::zero();
    if (w < n_q && ln) v = *reinterpret_cast<const typename V::T*>(user_emb + (size_t)users[w] * D + lane * PL);
    if (ln) *reinterpret_cast<typename V::T*>(ug + (size_t)w * D + lane * PL) = v;
    const float ss = warp_sum(V::ss(v));
    if (lane == 0 && w < n_q) unorm[w] = sqrtf(ss);
  } else if (w < n_q_pad + n_items) {
    const int i = w - n_q_pad;
    typename V::T v = V::zero();
    if (ln) v = *reinterpret_cast<const typename V::T*>(item_emb + (size_t)i * D + lane * PL);
    const float ss = warp_sum(V::ss(v));
    // non-negative floats order like uints; 38 k atomics on one word serialise, so look before touching it
    const unsigned int bits = __float_as_uint(sqrtf(ss));
    if (lane == 0 && bits > *reinterpret_cast<volatile unsigned int*>(bmax_bits)) atomicMax(bmax_bits, bits);
  }
}

template <int D, bool LONG>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_score_kernel(const __grid_constant__ CUtensorMap tm_users, const __grid_constant__ CUtensorMap tm_items, const TcArgs a) {
  extern __shared__ __align__(1024) uint8_t tc_smem_raw[];
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(tc_smem_raw) + 1023) & ~(uintptr_t)1023);
  using Sh = TcShape<D>;
  using Sm = TcSmem<D>;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sm + Sm::bar_off);
  uint64_t* bar_full = bars;                    // [STAGES]  TMA -> MMA
  uint64_t* bar_empty = bars + Sh::STAGES;      // [STAGES]  both warpgroups' MMAs done -> TMA
  uint64_t* bar_users = bars + 2 * Sh::STAGES;  // [1]
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * a.ub;             // first query row of this CTA
  const int n_tiles = (a.n_items + TC_TN - 1) / TC_TN;

  if (threadIdx.x == 0) {
    for (int s = 0; s < Sh::STAGES; ++s) {
      mbar_init(bar_full + s, 1);
      mbar_init(bar_empty + s, 2);  // one arrive per consumer warpgroup
    }
    mbar_init(bar_users, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ===== TMA producer =====
    if (elect_one()) {
      tma_prefetch_desc(&tm_users);
      tma_prefetch_desc(&tm_items);
      if constexpr (!Sh::US) {
        mbar_arrive_expect_tx(bar_users, Sh::USER_BYTES);
        for (int c = 0; c < Sh::KC; ++c) tma_load_2d(sm + Sm::users_off + c * 16384, &tm_users, bar_users, c * 32, q0);
      }
      for (int n = 0; n < n_tiles * Sh::SPT; ++n) {  // ring stage n: tile n / SPT, k-chunks (n % SPT) * SC ...
        const int s = n % Sh::STAGES;
        const uint32_t ph = (n / Sh::STAGES) & 1;
        mbar_wait(bar_empty + s, ph ^ 1);  // first pass through the ring passes immediately
        mbar_arrive_expect_tx(bar_full + s, Sh::STAGE_BYTES);
        for (int c = 0; c < Sh::SC; ++c)
          tma_load_2d(sm + Sm::items_off + s * Sh::STAGE_BYTES + c * 16384, &tm_items, bar_full + s, ((n % Sh::SPT) * Sh::SC + c) * 32,
                      (n / Sh::SPT) * TC_TN);
        if constexpr (Sh::US)  // the users' k-chunk n % SPT behind the item chunk
          tma_load_2d(sm + Sm::items_off + s * Sh::STAGE_BYTES + 16384, &tm_users, bar_full + s, (n % Sh::SPT) * 32, q0);
      }
    }
    return;
  }
  // ===== consumer warpgroup wg: MMA for its 64 users, then select: thread = one user row x one 64-column half =====
  const int wg = warp >> 2;
  const int lt = threadIdx.x & 127;
  const int chalf = lt >> 6;      // column half of every tile
  const int rloc = lt & 63;       // row within the warpgroup's 64
  const int row = wg * 64 + rloc;
  const int q = q0 + row;
  const bool active = row < a.ub && q < a.n_q;
  const int tix = chalf * TC_UB + row;  // column in the candidate arrays
  float* cs = reinterpret_cast<float*>(sm + Sm::cand_s_off);
  int32_t* ci = reinterpret_cast<int32_t*>(sm + Sm::cand_i_off);
  float* stg = reinterpret_cast<float*>(sm + Sm::stage_off) + wg * 64 * TC_SROW;
  constexpr int LS = 2 * TC_UB;  // candidate slot stride
  float thr = -INFINITY;
  int cnt = 0;
  // cursor into this user's sorted rated list; the id after next is prefetched so that advancing the
  // cursor never makes the warp wait for a global load
  int cur = 0, cend = 0, next_rated = 0x7fffffff, after_next = 0x7fffffff;
  if (active && a.rated_ptr) {
    const int u = a.users[q];
    cur = a.rated_ptr[u];
    cend = a.rated_ptr[u + 1];
    if (cur < cend) next_rated = a.rated_idx[cur];
    if (cur + 1 < cend) after_next = a.rated_idx[cur + 1];
  }
  // candidate list: 24 (score, id) slots in shared memory (column `tix`), organised as 3 buckets of 8.
  // Registers keep each bucket's minimum, so replacing the global minimum re-scans only one bucket
  // (8 independent shared-memory loads) instead of the whole list.
  // Each stored score carries its slot-in-bucket in the 3 low mantissa bits (the scores only rank candidates;
  // the certificate in tc_rescore_kernel accounts for the 2^-20 relative perturbation), so a bucket's minimum
  // names its own slot and 7 FMNMX replace a compare/select scan.
  float bm0 = INFINITY, bm1 = INFINITY, bm2 = INFINITY;  // bucket minima (valid once full)
  // long lists: thr is a running threshold; every unrated item of the half with approx score > thr is appended to the
  // half's buffer.  A full buffer is compacted: thr rises to (a lower bound of the k-th best approx score in the
  // buffer) - 2E and entries <= thr are dropped.  thr only rises, so at the end every item above the final thr is in
  // the buffer.  A compaction that frees less than a quarter of it (a band of near-ties wider than the buffer) marks
  // the half uncertified: cnt = -1, thr = +inf.
  float* bs = nullptr;
  int32_t* bi = nullptr;
  float twoE = 0.f;
  if constexpr (LONG) {
    if (active) {
      bs = a.buf_s + ((size_t)q * 2 + chalf) * a.cap;
      bi = a.buf_i + ((size_t)q * 2 + chalf) * a.cap;
      twoE = 2.0f * Sh::E * a.unorm[q] * __uint_as_float(*a.bmax_bits);
    }
  }
  auto compact = [&]() {
    // largest key v with 12 low zero bits such that >= k buffered scores have key >= v: v <= the k-th best key
    uint32_t v = 0;
    for (int b = 31; b >= 12; --b) {
      const uint32_t t = v | (1u << b);
      int c = 0;
      for (int p = 0; p < a.cap; ++p) c += okey(bs[p]) >= t;
      if (c >= a.k) v = t;
    }
    if (v != 0) thr = fmaxf(thr, ofloat(v) - twoE);
    int kept = 0;
    for (int p = 0; p < a.cap; ++p) {
      const float s = bs[p];
      if (s > thr) {
        bi[kept] = bi[p];
        bs[kept++] = s;
      }
    }
    cnt = kept;
    if (kept > a.cap - a.cap / 4) {
      cnt = -1;
      thr = INFINITY;
    }
  };
  auto process_group = [&](const uint32_t (&r)[32], int g0) {
    uint32_t mask = 0;
#pragma unroll
    for (int j = 0; j < 32; ++j)  // two instructions per score: FSETP + predicated LOP3
      asm("{\n\t.reg .pred p;\n\tsetp.gt.f32 p, %1, %2;\n\t@p or.b32 %0, %0, %3;\n\t}"
          : "+r"(mask)
          : "f"(__uint_as_float(r[j])), "f"(thr), "r"(1u << j));
    if (g0 + 32 > a.n_items) mask &= (g0 < a.n_items) ? (0xffffffffu >> (g0 + 32 - a.n_items)) : 0u;  // zero-filled OOB rows
    if (!active) mask = 0;
    // rated items never become candidates: walk the sorted rated list through this group
    while (next_rated < g0 + 32) {
      if (next_rated >= g0) mask &= ~(1u << (next_rated - g0));
      ++cur;
      next_rated = after_next;
      after_next = (cur + 1 < cend) ? a.rated_idx[cur + 1] : 0x7fffffff;
    }
    while (mask) {
      const int j = __ffs(mask) - 1;
      mask &= mask - 1;
      // r[j] with a per-lane j: a 5-level select tree on the bits of j (31 selects)
      uint32_t t16[16], t8[8], t4[4];
#pragma unroll
      for (int i = 0; i < 16; ++i) t16[i] = (j & 1) ? r[2 * i + 1] : r[2 * i];
#pragma unroll
      for (int i = 0; i < 8; ++i) t8[i] = (j & 2) ? t16[2 * i + 1] : t16[2 * i];
#pragma unroll
      for (int i = 0; i < 4; ++i) t4[i] = (j & 4) ? t8[2 * i + 1] : t8[2 * i];
      const uint32_t t2a = (j & 8) ? t4[1] : t4[0], t2b = (j & 8) ? t4[3] : t4[2];
      float sc = __uint_as_float((j & 16) ? t2b : t2a);
      if (!(sc > thr)) continue;  // thr may have risen inside this group
      const int id = g0 + j;
      if constexpr (LONG) {
        bs[cnt] = sc;
        bi[cnt] = id;
        if (++cnt == a.cap) compact();
        continue;
      }
      if (cnt < TC_LIST) {
        cs[cnt * LS + tix] = sc;
        ci[cnt * LS + tix] = id;
        ++cnt;
        if (cnt == TC_LIST) {  // list full: tag every slot and establish the bucket minima
#pragma unroll
          for (int b = 0; b < 3; ++b) {
            float mn = INFINITY;
#pragma unroll
            for (int qq = 0; qq < 8; ++qq) {
              const float v = __uint_as_float((__float_as_uint(cs[(b * 8 + qq) * LS + tix]) & ~7u) | (uint32_t)qq);
              cs[(b * 8 + qq) * LS + tix] = v;
              mn = fminf(mn, v);
            }
            if (b == 0) bm0 = mn;
            if (b == 1) bm1 = mn;
            if (b == 2) bm2 = mn;
          }
          thr = fminf(fminf(bm0, bm1), bm2);
        }
      } else {
        // evict the global minimum: it sits in the bucket whose minimum equals thr, in the slot its tag names
        const int b = (bm0 == thr) ? 0 : ((bm1 == thr) ? 1 : 2);
        const int pos = b * 8 + (int)(__float_as_uint(thr) & 7u);
        cs[pos * LS + tix] = __uint_as_float((__float_as_uint(sc) & ~7u) | (__float_as_uint(thr) & 7u));
        ci[pos * LS + tix] = id;
        float mn = cs[(b * 8) * LS + tix];
#pragma unroll
        for (int qq = 1; qq < 8; ++qq) mn = fminf(mn, cs[(b * 8 + qq) * LS + tix]);
        if (b == 0) bm0 = mn;
        else if (b == 1) bm1 = mn;
        else bm2 = mn;
        thr = fminf(fminf(bm0, bm1), bm2);
      }
    }
  };
  const uint32_t ua = smem_u32(sm + Sm::users_off + wg * 8192);
  const int w4 = warp & 3, g = lane >> 2, tq = lane & 3;
  if constexpr (!Sh::US) mbar_wait(bar_users, 0);
  for (int t = 0; t < n_tiles; ++t) {
    float acc[64];
#pragma unroll
    for (int p = 0; p < Sh::SPT; ++p) {
      const int n = t * Sh::SPT + p;
      const int s = n % Sh::STAGES;
      mbar_wait(bar_full + s, (n / Sh::STAGES) & 1);
      const uint32_t ib = smem_u32(sm + Sm::items_off + s * Sh::STAGE_BYTES);
      wgmma_fence();
#pragma unroll
      for (int c = 0; c < Sh::SC; ++c)
#pragma unroll
        for (int k = 0; k < Sh::KS; ++k)
          wgmma_m64n128k8_tf32_ss(acc,
                                  make_smem_desc_k_sw128(Sh::US ? ib + 16384 + wg * 8192 + k * 32 : ua + (p * Sh::SC + c) * 16384 + k * 32),
                                  make_smem_desc_k_sw128(ib + c * 16384 + k * 32), (p | c | k) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      if (lt == 0) mbar_arrive(bar_empty + s);  // this warpgroup is done reading the stage
    }
    named_bar_sync(1 + wg, 128);             // the previous tile's staged scores have been read
#pragma unroll
    for (int j = 0; j < 64; j += 2) {
      const int rr = w4 * 16 + g + 8 * ((j >> 1) & 1);
      const int cc = 8 * (j >> 2) + 2 * tq;
      *reinterpret_cast<float2*>(stg + rr * TC_SROW + cc) = make_float2(acc[j], acc[j + 1]);
    }
    named_bar_sync(1 + wg, 128);
    const int c0 = t * TC_TN + chalf * 64;
    const float* src = stg + rloc * TC_SROW + chalf * 64;
    uint32_t r[32];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int j = 0; j < 32; j += 4) {
        const float4 v = *reinterpret_cast<const float4*>(src + h * 32 + j);
        r[j] = __float_as_uint(v.x), r[j + 1] = __float_as_uint(v.y), r[j + 2] = __float_as_uint(v.z), r[j + 3] = __float_as_uint(v.w);
      }
      process_group(r, c0 + h * 32);
    }
  }
  if constexpr (LONG) {
    if (active) {
      a.cand_n[(size_t)q * 2 + chalf] = cnt;
      a.cand_thr[(size_t)q * 2 + chalf] = thr;
    }
    return;
  }
  if (active) {
    const size_t o = ((size_t)q * 2 + chalf) * TC_LIST;
    for (int p = 0; p < TC_LIST; ++p) {
      a.cand_s[o + p] = (p < cnt) ? cs[p * LS + tix] : -INFINITY;
      a.cand_i[o + p] = (p < cnt) ? ci[p * LS + tix] : -1;
    }
    a.cand_n[(size_t)q * 2 + chalf] = cnt;
    a.cand_thr[(size_t)q * 2 + chalf] = (cnt == TC_LIST) ? thr : -INFINITY;
  }
}

template <int D>
__global__ void __launch_bounds__(256) tc_rescore_kernel(const __grid_constant__ srb_topk_desc d, const __grid_constant__ TcWorkspace w) {
  const int lane = threadIdx.x & 31;
  const int q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (q >= d.n_q) return;
  const int cnt_a = w.cand_n[(size_t)q * 2], cnt_b = w.cand_n[(size_t)q * 2 + 1];
  const int K = d.k;
  const float bmax = __uint_as_float(*w.bmax);
  const float E = TcShape<D>::E * w.unorm[q] * bmax;  // TF32 truncation + k-step accumulation + slot tags
  // ---- prune by approximate score before any exact work ----
  // Every exact score lies within E of its approximate score.  Let a_K be the K-th largest approximate score of the
  // candidates: K candidates have an exact score >= a_K - E, so one whose approximate score is below a_K - 2E is beaten
  // by at least K others and can never end in the top-K, whatever the insertion order.  Typically half of the 48 go,
  // the survivors fit one lane each, and the second exact pass and half of the sequential insertions disappear.
  __shared__ int32_t surv[8][TC_CAND];
  int32_t* sv = surv[threadIdx.x >> 5];
  int cnt;
  {
    float ap[2];
    int cid[2];
    bool have[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int c = lane + 32 * h;
      have[h] = c < TC_CAND && (c % TC_LIST) < ((c < TC_LIST) ? cnt_a : cnt_b);
      ap[h] = have[h] ? w.cand_s[(size_t)q * TC_CAND + c] : -INFINITY;
      cid[h] = have[h] ? w.cand_i[(size_t)q * TC_CAND + c] : 0x7fffffff;
    }
    float cut = -INFINITY;
    if (cnt_a + cnt_b > K) {
      // descending rank of my approximate scores (ties broken by slot), then the value of rank K-1
      int rk[2] = {0, 0};
#pragma unroll 8
      for (int l = 0; l < 32; ++l) {
        const float o0 = __shfl_sync(SRB_FULL_MASK, ap[0], l);
        const float o1 = __shfl_sync(SRB_FULL_MASK, ap[1], l);
        rk[0] += (o0 > ap[0] || (o0 == ap[0] && l < lane)) + (o1 > ap[0]);
        rk[1] += (o0 > ap[1] || o0 == ap[1]) + (o1 > ap[1] || (o1 == ap[1] && l < lane));
      }
      const unsigned b0 = __ballot_sync(SRB_FULL_MASK, have[0] && rk[0] == K - 1);
      const unsigned b1 = __ballot_sync(SRB_FULL_MASK, have[1] && rk[1] == K - 1);
      const float ak = b0 ? __shfl_sync(SRB_FULL_MASK, ap[0], __ffs(b0) - 1) : __shfl_sync(SRB_FULL_MASK, ap[1], b1 ? __ffs(b1) - 1 : 0);
      if (b0 | b1) cut = ak - 2.0f * E;
    }
    const unsigned k0 = __ballot_sync(SRB_FULL_MASK, have[0] && ap[0] >= cut);
    const unsigned k1 = __ballot_sync(SRB_FULL_MASK, have[1] && ap[1] >= cut);
    const unsigned lt = (1u << lane) - 1u;
    if ((k0 >> lane) & 1u) sv[__popc(k0 & lt)] = cid[0];
    if ((k1 >> lane) & 1u) sv[__popc(k0) + __popc(k1 & lt)] = cid[1];
    cnt = __popc(k0) + __popc(k1);
    __syncwarp();
  }
  // survivor slots on 32 lanes: lane l owns slots l and l + 32 (the second pass only runs when more than 32 survive)
  int id[2];
  float s[2];
  bool mine[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int c = lane + 32 * h;
    mine[h] = c < cnt;
    id[h] = 0x7fffffff;
    s[h] = -INFINITY;
    if (h == 1 && cnt <= 32) continue;  // warp-uniform
    if (mine[h]) id[h] = sv[c];
    if (mine[h]) {
      const float4* u = reinterpret_cast<const float4*>(w.ug + (size_t)q * D);
      const float4* it = reinterpret_cast<const float4*>(d.item_emb + (size_t)id[h] * D);
      // the whole row in flight before the first fma: this kernel is bound by the latency of these gathers.  D = 256
      // takes the row in two pieces of 128 floats, so that its loads fit the registers without spilling
      constexpr int P = D > 128 ? 128 : D;
      float acc = 0.f;
#pragma unroll
      for (int o = 0; o < D / 4; o += P / 4) {
        float4 iv[P / 4];
#pragma unroll
        for (int c = 0; c < P / 4; ++c) iv[c] = __ldg(it + o + c);
        acc = exact_score<P, P / 4>([&](int c) { return u[o + c]; }, [&](int c) { return iv[c]; }, acc);
      }
      s[h] = acc;
    }
  }
  // rank of my candidates by item id (ids are distinct; empty slots carry INT_MAX and never count)
  int rank[2] = {0, 0};
#pragma unroll 8
  for (int l = 0; l < 32; ++l) {
    const int o0 = __shfl_sync(SRB_FULL_MASK, id[0], l);
    const int o1 = __shfl_sync(SRB_FULL_MASK, id[1], l);
    rank[0] += (o0 < id[0]) + (o1 < id[0]);
    rank[1] += (o0 < id[1]) + (o1 < id[1]);
  }
  // find_k_largest's sequential process over the candidates in id order (see score_topk.cu).  The candidates
  // are first laid out in id order in shared memory, so that each step is one broadcast load and a
  // warp-uniform compare instead of a ballot / find-first-set / shuffle chain
  __shared__ float2 ord[8][TC_CAND];
  float2* mo = ord[threadIdx.x >> 5];
#pragma unroll
  for (int h = 0; h < 2; ++h)
    if (mine[h]) mo[rank[h]] = make_float2(s[h], __int_as_float(id[h]));
  __syncwarp();
  float ls = -INFINITY;
  int li = -1;
  float thr = -INFINITY;  // score of list slot K-1 (warp-uniform)
  for (int t = 0; t < cnt; ++t) {
    const float2 e = mo[t];
    const float cs = e.x;
    if (cs > thr) {
      list_insert(ls, li, cs, __float_as_int(e.y), K);
      thr = __shfl_sync(SRB_FULL_MASK, ls, K - 1);
    }
  }
  // exactness test
  const float kth = __shfl_sync(SRB_FULL_MASK, ls, K - 1);
  const float thr32 = fmaxf(w.cand_thr[(size_t)q * 2], w.cand_thr[(size_t)q * 2 + 1]);
  int deg = 0;
  if (d.rated_ptr) {
    const int u = d.users[q];
    deg = d.rated_ptr[u + 1] - d.rated_ptr[u];
  }
  const bool unsafe = (d.n_items - deg < K) || !(thr32 + E < kth);
  if (unsafe) {
    if (lane == 0) {
      const int slot = atomicAdd(w.fb_count, 1);
      w.fb_rows[slot] = q;
      w.fb_users[slot] = d.users[q];
    }
    return;
  }
  if (lane < K) {
    d.out_ids[(size_t)q * K + lane] = li;
    d.out_scores[(size_t)q * K + lane] = ls;
  }
}

// sum over the 256 threads of a block (every thread gets it); red: 8 ints of shared memory
__device__ __forceinline__ int tc_block_sum(int v, int* red) {
  v = warp_sum(v);
  __syncthreads();  // red is free again (its previous use has been read)
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  int s = 0;
#pragma unroll
  for (int w = 0; w < 8; ++w) s += red[w];
  return s;
}

constexpr int TC_LONG_CAND = 2 * ((2 * TC_LONG_MAX + 256 + 31) / 32 * 32);  // both halves' buffers at k = 256

// Long lists (k > 32): CTA per user over the candidates of both half buffers.  The same approximate prune as
// tc_rescore_kernel (a_K - 2E), exact fp32 fma-chain scores of the survivors, then the set find_k_largest keeps when it
// visits the items in id order, written score-descending, ties by id descending.  With s* the k-th score, that set is
// every score above s* and, of the scores equal to s*, those among the first k items (in id order) scoring >= s* --
// the ones that found the list not yet full at s* and entered -- minus the smallest ids, which the later, greater
// scores evicted first: the largest (k - #above) ids of them.
// Certificate: every item outside the buffers has approx score <= thr (the larger of the two halves' final running
// thresholds), so the list is exact iff thr + E < the exact k-th score; otherwise, or when a buffer overflowed or
// the user has fewer than k unrated items, the user goes to the exact fallback.
template <int D>
__global__ void __launch_bounds__(256) tc_rescore_long_kernel(const __grid_constant__ srb_topk_desc d, const __grid_constant__ TcWorkspace w) {
  __shared__ float s_ap[TC_LONG_CAND];       // approx scores, then the survivors' exact-score keys
  __shared__ int32_t s_id[TC_LONG_CAND];
  __shared__ int32_t s_sv[TC_LONG_CAND];     // survivor ids
  __shared__ int32_t s_rank[TC_LONG_CAND];   // per survivor: 2 above s*, 1 tied with s* and entered, 0 otherwise
  __shared__ int red[8];
  __shared__ int s_cnt;
  __shared__ float s_kth;
  __shared__ uint32_t s_kkey;
  const int q = blockIdx.x;
  const int tid = threadIdx.x;
  const int K = d.k;
  const int n0 = w.cand_n[(size_t)q * 2], n1 = w.cand_n[(size_t)q * 2 + 1];
  int deg = 0;
  if (d.rated_ptr) {
    const int u = d.users[q];
    deg = d.rated_ptr[u + 1] - d.rated_ptr[u];
  }
  bool unsafe = n0 < 0 || n1 < 0 || n0 + n1 < K || d.n_items - deg < K;
  if (!unsafe) {
    const int n = n0 + n1;
    for (int c = tid; c < n; c += 256) {
      const size_t o = (c < n0) ? (size_t)q * 2 * w.cap + c : ((size_t)q * 2 + 1) * w.cap + (c - n0);
      s_ap[c] = w.buf_s[o];
      s_id[c] = w.buf_i[o];
    }
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    // the K-th largest approximate key, bit by bit
    uint32_t v = 0;
    for (int b = 31; b >= 0; --b) {
      const uint32_t t = v | (1u << b);
      int c = 0;
      for (int p = tid; p < n; p += 256) c += okey(s_ap[p]) >= t;
      if (tc_block_sum(c, red) >= K) v = t;
    }
    const float E = TcShape<D>::E * w.unorm[q] * __uint_as_float(*w.bmax);
    const float cut = ofloat(v) - 2.0f * E;
    for (int p = tid; p < n; p += 256)
      if (s_ap[p] >= cut) s_sv[atomicAdd(&s_cnt, 1)] = s_id[p];
    __syncthreads();
    const int S = s_cnt;
    uint32_t* s_ek = reinterpret_cast<uint32_t*>(s_ap);
    const float4* u = reinterpret_cast<const float4*>(w.ug + (size_t)q * D);
    for (int p = tid; p < S; p += 256) {
      const float4* it = reinterpret_cast<const float4*>(d.item_emb + (size_t)s_sv[p] * D);
      s_ek[p] = okey(exact_score<D>([&](int c) { return u[c]; }, [&](int c) { return __ldg(it + c); }));
    }
    __syncthreads();
    for (int p = tid; p < S; p += 256) {
      const uint32_t ek = s_ek[p];
      const int id = s_sv[p];
      int r = 0;
      for (int j = 0; j < S; ++j) {
        const uint32_t oj = s_ek[j];
        r += (oj > ek) || (oj == ek && s_sv[j] < id);
      }
      if (r == K - 1) {
        s_kth = ofloat(ek);
        s_kkey = ek;
      }
    }
    __syncthreads();
    const float thr = fmaxf(w.cand_thr[(size_t)q * 2], w.cand_thr[(size_t)q * 2 + 1]);
    unsafe = !(thr + E < s_kth);
    if (!unsafe) {
      const uint32_t kk = s_kkey;
      int above = 0;
      for (int p = tid; p < S; p += 256) {
        const uint32_t ek = s_ek[p];
        int st = 0;
        if (ek > kk) {
          st = 2;
          ++above;
        } else if (ek == kk) {  // entered iff fewer than k scores >= s* precede it in id order
          const int id = s_sv[p];
          int before = 0;
          for (int j = 0; j < S; ++j) before += s_ek[j] >= kk && s_sv[j] < id;
          st = before < K ? 1 : 0;
        }
        s_rank[p] = st;
      }
      const int need = K - tc_block_sum(above, red);  // also orders the s_rank writes before the reads below
      int32_t* keep = s_id;                            // free since the survivors were listed
      for (int p = tid; p < S; p += 256) {
        int k_ = s_rank[p] == 2;
        if (s_rank[p] == 1) {
          const int id = s_sv[p];
          int larger = 0;
          for (int j = 0; j < S; ++j) larger += s_rank[j] == 1 && s_sv[j] > id;
          k_ = larger < need;
        }
        keep[p] = k_;
      }
      __syncthreads();
      write_ranked(s_ek, s_sv, S, [&](int j) { return keep[j] != 0; }, d.out_ids + (size_t)q * K, d.out_scores + (size_t)q * K);
      return;
    }
  }
  if (tid == 0) {
    const int slot = atomicAdd(w.fb_count, 1);
    w.fb_rows[slot] = q;
    w.fb_users[slot] = d.users[q];
  }
}

static int64_t tc_align(int64_t x) { return (x + 255) / 256 * 256; }

static int tc_fb_cap(int n_items) {
  long long cap = (64ll << 20) / ((long long)n_items * 4);  // at most 64 MB of scratch
  if (cap > 256) cap = 256;
  if (cap < 8) cap = 8;
  return (int)cap;
}

// The gathered user table is carved last: it is the only part whose size depends on d, so the fallback counter sits
// at the same offset for every width (srb_topk_fallback_count_offset takes no d).  The long-list buffers, the only
// part whose size depends on k, come after the counter too; at k <= 32 they are empty and the layout is unchanged.
static TcWorkspace tc_carve(char* base, int n_q, int n_items, int d, int k) {
  TcWorkspace w;
  const int64_t n_q_pad = ((int64_t)n_q + 255) / 256 * 256 + 256;
  int64_t off = 0;
  auto take = [&](int64_t b) {
    char* p = base ? base + off : nullptr;
    off += tc_align(b);
    return p;
  };
  w.unorm = (float*)take(n_q_pad * 4);
  w.bmax = (unsigned int*)take(16);
  w.cand_s = (float*)take((int64_t)n_q * TC_CAND * 4);
  w.cand_i = (int32_t*)take((int64_t)n_q * TC_CAND * 4);
  w.cand_n = (int32_t*)take((int64_t)n_q * 2 * 4);
  w.cand_thr = (float*)take((int64_t)n_q * 2 * 4);
  w.fb_count = (int32_t*)take(16);
  w.fb_rows = (int32_t*)take((int64_t)n_q * 4);
  w.fb_users = (int32_t*)take((int64_t)n_q * 4);
  w.fb_cap = tc_fb_cap(n_items);
  w.fb_scratch = (float*)take((int64_t)w.fb_cap * n_items * 4);
  w.cap = (k > 32) ? tc_long_cap(k) : 0;
  w.buf_s = (float*)take((int64_t)n_q * 2 * w.cap * 4);
  w.buf_i = (int32_t*)take((int64_t)n_q * 2 * w.cap * 4);
  w.ug = (float*)take(n_q_pad * d * 4);
  w.bytes = off;
  return w;
}

int score_topk_fallback(const srb_topk_desc* d, const int32_t* fb_users, const int32_t* fb_rows, const int32_t* fb_count,
                        float* scratch, int fb_cap, cudaStream_t st);  // score_topk.cu

template <int D, bool LONG>
static int launch_tc_score(const CUtensorMap& tm_users, const CUtensorMap& tm_items, const TcArgs& a, int blocks, cudaStream_t st) {
  const size_t smem = TcSmem<D>::total + 1024;
  static bool attr_done = false;
  if (!attr_done) {
    SRB_TRY(check_cuda(cudaFuncSetAttribute(tc_score_kernel<D, LONG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), "tc smem attr"));
    attr_done = true;
  }
  tc_score_kernel<D, LONG><<<blocks, TC_THREADS, smem, st>>>(tm_users, tm_items, a);
  return post_launch("tc_score_kernel");
}

template <int D>
static int launch_tc(const srb_topk_desc* d, const TcWorkspace& w, cudaStream_t st) {
  const int n_q = d->n_q;
  const int n_q_pad = (n_q + 255) / 256 * 256 + 256;
  SRB_TRY(check_cuda(cudaMemsetAsync(w.bmax, 0, 16, st), "tc memset"));
  SRB_TRY(check_cuda(cudaMemsetAsync(w.fb_count, 0, 16, st), "tc memset"));
  {
    const long long rows = (long long)n_q_pad + d->n_items;
    tc_gather_kernel<D><<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(d->user_emb, d->users, n_q, n_q_pad, w.ug, w.unorm, d->item_emb,
                                                                   d->n_items, w.bmax);
    SRB_TRY(post_launch("tc_gather_kernel"));
  }
  // users per CTA: one wave of SMs when the queries fit (n_q <= TC_UB x SMs), else TC_UB per CTA and several waves
  // (yelp2018: 31 668 users -> 248 CTAs on 132 SMs, one CTA per SM at ~211 KB of shared memory); multiple of 32
  const int sms = sm_count();
  int ub = (n_q + sms - 1) / sms;
  ub = (ub + 31) / 32 * 32;
  if (ub > TC_UB) ub = TC_UB;
  if (ub < 32) ub = 32;
  const int blocks = (n_q + ub - 1) / ub;
  CUtensorMap tm_users, tm_items;
  SRB_REQUIRE(make_tmap_f32_rows(&tm_users, w.ug, (uint64_t)n_q_pad, D, TC_UB) == 0, "topk impl 2: cuTensorMapEncodeTiled(users) failed");
  SRB_REQUIRE(make_tmap_f32_rows(&tm_items, d->item_emb, (uint64_t)d->n_items, D, TC_TN) == 0,
              "topk impl 2: cuTensorMapEncodeTiled(items) failed");
  const TcArgs a{d->users, d->rated_ptr, d->rated_idx, n_q, d->n_items, ub, w.cand_s, w.cand_i, w.cand_n, w.cand_thr, d->k, w.cap,
                 w.buf_s, w.buf_i, w.unorm, w.bmax};
  if (d->k > 32) {
    SRB_TRY((launch_tc_score<D, true>(tm_users, tm_items, a, blocks, st)));
    tc_rescore_long_kernel<D><<<n_q, 256, 0, st>>>(*d, w);
    SRB_TRY(post_launch("tc_rescore_long_kernel"));
  } else {
    SRB_TRY((launch_tc_score<D, false>(tm_users, tm_items, a, blocks, st)));
    tc_rescore_kernel<D><<<(n_q + 7) / 8, 256, 0, st>>>(*d, w);
    SRB_TRY(post_launch("tc_rescore_kernel"));
  }
  return score_topk_fallback(d, w.fb_users, w.fb_rows, w.fb_count, w.fb_scratch, w.fb_cap, st);
}

int score_topk_tc(const srb_topk_desc* d, cudaStream_t st) {
  SRB_REQUIRE(d->d == 16 || d->d == 32 || d->d == 64 || d->d == 128 || d->d == 256,
              "topk impl 2 (tensor cores) supports d = 16, 32, 64, 128 and 256 only (got %d)", d->d);
  SRB_REQUIRE(d->k >= 1 && d->k <= TC_LONG_MAX, "topk impl 2: k=%d unsupported (1..%d)", d->k, TC_LONG_MAX);
  const int n_q = d->n_q;
  const TcWorkspace need = tc_carve(nullptr, n_q, d->n_items, d->d, d->k);
  SRB_REQUIRE(d->workspace && d->workspace_bytes >= need.bytes, "topk impl 2: workspace too small (%lld < %lld)",
              (long long)d->workspace_bytes, (long long)need.bytes);
  SRB_REQUIRE(((uintptr_t)d->workspace & 255) == 0, "topk impl 2: workspace must be 256-byte aligned");
  SRB_REQUIRE(((uintptr_t)d->item_emb & 15) == 0, "topk impl 2: item_emb must be 16-byte aligned");
  const TcWorkspace w = tc_carve((char*)d->workspace, n_q, d->n_items, d->d, d->k);
  switch (d->d) {
    case 16: return launch_tc<16>(d, w, st);
    case 32: return launch_tc<32>(d, w, st);
    case 64: return launch_tc<64>(d, w, st);
    case 128: return launch_tc<128>(d, w, st);
    default: return launch_tc<256>(d, w, st);
  }
}

}  // namespace srb

// byte offset of the int32 fallback counter inside the workspace (diagnostics: how many users the
// exact kernel had to re-run); the same for every width and list length
extern "C" int64_t srb_topk_fallback_count_offset(int32_t n_q, int32_t n_items) {
  if (n_q <= 0 || n_items <= 0) return -1;
  const srb::TcWorkspace w = srb::tc_carve((char*)256, n_q, n_items, 64, 1);
  return (int64_t)((char*)w.fb_count - (char*)256);
}

extern "C" float srb_topk_tc_error_bound(int32_t d) {
  switch (d) {
    case 16: return srb::TcShape<16>::E;
    case 32: return srb::TcShape<32>::E;
    case 64: return srb::TcShape<64>::E;
    case 128: return srb::TcShape<128>::E;
    case 256: return srb::TcShape<256>::E;
    default: return -1.0f;
  }
}

// O(n_q * cap(k) + n_items): the candidate buffers of long lists grow with k, never with the catalogue
extern "C" int64_t srb_topk_workspace_bytes(int32_t n_q, int32_t n_items, int32_t d, int32_t k) {
  if (n_q <= 0 || n_items <= 0 || d <= 0) return 0;
  return srb::tc_carve(nullptr, n_q, n_items, d, k).bytes;
}
