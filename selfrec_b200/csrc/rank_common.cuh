// The ranking contract (include/selfrec_b200.h (iv)), written once for impl 1 (score_topk.cu) and impl 2
// (score_topk_tc.cu):
//   - a score is the oracle's fp32 fma chain over k = 0..d-1 (exact_score);
//   - selection is find_k_largest's (util/algorithm.py:144-156): a candidate enters iff its score is strictly greater
//     than the k-th, and the smallest (score, id) -- what heapq pops -- is evicted (list_insert, list_offer32);
//   - output is score-descending, ties by id descending (write_ranked).
#pragma once
#include "common.cuh"

namespace srb {

constexpr float TK_MASKED = -1e9f;  // -10e8, the score of a rated item (graph_recommender.py:48-50)

// The exact score of one (user, item) pair: acc = fma(u[k], i[k], acc) for k = 0..D-1 from acc = +0, so it is never
// -0.  u4(c) / i4(c) return floats 4c..4c+3 of the user / item row; UNROLL sets how far their loads may run ahead.
// A caller that walks the row in pieces passes the chain so far as acc (the next piece's floats indexed from 0).
template <int D, int UNROLL = 8, class U4, class I4>
__device__ __forceinline__ float exact_score(U4 u4, I4 i4, float acc = 0.f) {
#pragma unroll UNROLL
  for (int c = 0; c < D / 4; ++c) {
    const float4 u = u4(c), i = i4(c);
    const float uk[4] = {u.x, u.y, u.z, u.w}, ik[4] = {i.x, i.y, i.z, i.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) acc = fmaf(uk[j], ik[j], acc);
  }
  return acc;
}

// A warp's top-K list (K <= 32): lane l < K holds entry l, sorted by (score desc, id desc); empty entries are
// (-inf, -1).  list_insert puts (cs, cid), known to the whole warp, at its place and drops the last entry.  The caller
// has checked cs > the K-th score.
__device__ __forceinline__ void list_insert(float& ls, int& li, float cs, int cid, int K) {
  const int lane = threadIdx.x & 31;
  const int pos = __popc(__ballot_sync(SRB_FULL_MASK, lane < K && ls > cs));
  const float ps = __shfl_up_sync(SRB_FULL_MASK, ls, 1);
  const int pi = __shfl_up_sync(SRB_FULL_MASK, li, 1);
  if (lane > pos && lane < K) ls = ps, li = pi;
  if (lane == pos) ls = cs, li = cid;
}

// find_k_largest's step over the warp's 32 lane candidates (sc, id) in lane order: the callers visit items in id
// order, so the final set is the reference's, ties included.
__device__ __forceinline__ void list_offer32(float& ls, int& li, float sc, int id, int K) {
  float thr = __shfl_sync(SRB_FULL_MASK, ls, K - 1);
  unsigned m = __ballot_sync(SRB_FULL_MASK, sc > thr);
  while (m) {
    const int src = __ffs(m) - 1;
    m &= m - 1;
    const float cs = __shfl_sync(SRB_FULL_MASK, sc, src);
    const int cid = __shfl_sync(SRB_FULL_MASK, id, src);
    thr = __shfl_sync(SRB_FULL_MASK, ls, K - 1);
    if (cs > thr) list_insert(ls, li, cs, cid, K);
  }
}

// order-preserving map of a float to uint32 (+0 and -0 map alike) and back
__device__ __forceinline__ uint32_t okey(float s) {
  const uint32_t b = __float_as_uint(s == 0.f ? 0.f : s);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float ofloat(uint32_t key) {
  return __uint_as_float((key & 0x80000000u) ? (key & 0x7fffffffu) : ~key);
}

// is v in the sorted run idx[lo, hi)
__device__ __forceinline__ bool sorted_contains(const int32_t* idx, int lo, int hi, int v) {
  const int end = hi;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (idx[mid] < v) lo = mid + 1;
    else hi = mid;
  }
  return lo < end && idx[lo] == v;
}

// Block-wide: write each of the n entries (key[p], id[p]) with keep(p) at its rank among the kept ones, (key desc,
// id desc), into the user's output row.  The scores written are ofloat(key), the same bits as the exact scores.
template <class Keep>
__device__ __forceinline__ void write_ranked(const uint32_t* key, const int32_t* id, int n, Keep keep, int32_t* out_ids,
                                             float* out_scores) {
  for (int p = threadIdx.x; p < n; p += blockDim.x) {
    if (!keep(p)) continue;
    const uint32_t ek = key[p];
    const int e = id[p];
    int pos = 0;
    for (int j = 0; j < n; ++j) pos += keep(j) && (key[j] > ek || (key[j] == ek && id[j] > e));
    out_ids[pos] = e;
    out_scores[pos] = ofloat(ek);
  }
}

}  // namespace srb
