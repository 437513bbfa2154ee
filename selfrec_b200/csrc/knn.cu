// Neighbourhood baselines (model/graph/ItemKNN.py, model/graph/UserKNN.py): neighbour tables, neighbour-weighted
// float64 score rows, and the float64 find_k_largest of util/algorithm.py:144-156 in the reference's exact order.
//
// Every float64 step the reference rounds on its own (sqrt, product, + 1e-8, quotient, sum) is written with an _rn
// intrinsic, so nvcc cannot contract a product and an add into one FMA and change the bits.
#include <algorithm>

#include "common.cuh"

namespace srb {

constexpr int KNN_THREADS = 512;
constexpr int KNN_BUF = SRB_KNN_MAX_TOPK * 2;  // on-chip candidate buffer of one row: the kept top-k plus one refill

// ItemKNN.py:14-30 with unit ratings: raw = c / (sqrt(deg_a) * sqrt(deg_b) + 1e-8); sim = (c / (c + shrinkage)) * raw
__device__ __forceinline__ double knn_sim(int c, int deg_a, int deg_b, long long shrinkage) {
  const double den = __dadd_rn(__dmul_rn(__dsqrt_rn((double)deg_a), __dsqrt_rn((double)deg_b)), 1e-8);
  const double raw = __ddiv_rn((double)c, den);
  return __dmul_rn(__ddiv_rn((double)c, (double)((long long)c + shrinkage)), raw);
}

// heapq.nlargest over (sim, name) tuples: larger sim first, then the larger name (its host-computed rank)
__device__ __forceinline__ bool knn_better(double sa, int ra, double sb, int rb) { return sa > sb || (sa == sb && ra > rb); }

// Sort the first n entries of the candidate buffer best-first (bitonic, padded to a power of two with entries that lose
// to every real one: a real sim is > 0).  Called by the whole CTA; ends synchronised.
__device__ void knn_sort_buffer(double* s_sim, int* s_rank, int* s_id, int n) {
  int p = 1;
  while (p < n) p <<= 1;
  for (int t = n + threadIdx.x; t < p; t += blockDim.x) {
    s_sim[t] = -1.0;
    s_rank[t] = -1;
    s_id[t] = -1;
  }
  __syncthreads();
  for (int k = 2; k <= p; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < p; i += blockDim.x) {
        const int l = i ^ j;
        if (l > i) {
          const bool desc = (i & k) == 0;
          const bool sw = desc ? knn_better(s_sim[l], s_rank[l], s_sim[i], s_rank[i]) : knn_better(s_sim[i], s_rank[i], s_sim[l], s_rank[l]);
          if (sw) {
            const double ts = s_sim[i];
            s_sim[i] = s_sim[l];
            s_sim[l] = ts;
            int t = s_rank[i];
            s_rank[i] = s_rank[l];
            s_rank[l] = t;
            t = s_id[i];
            s_id[i] = s_id[l];
            s_id[l] = t;
          }
        }
      }
      __syncthreads();
    }
  }
}

// One CTA per row a at a time (rows handed out by an atomic counter).  Phase 1 (Gustavson): walk a's members m and the
// rows b of each member through the transpose, counting c(a, b) in this CTA's count scratch and listing each b once.
// Phase 2: sim of every listed b, filtered against the current k-th best key into the on-chip buffer; whenever the
// buffer holds more than k entries it is sorted and cut back to k, so a row with any number of candidates is exact.
// The counts of the listed rows are reset on the way, which leaves the scratch zero for the next row.
__global__ void __launch_bounds__(KNN_THREADS) knn_neighbors_kernel(const int32_t* __restrict__ a_ptr, const int32_t* __restrict__ a_idx,
                                                                    const int32_t* __restrict__ t_ptr, const int32_t* __restrict__ t_idx,
                                                                    const int32_t* __restrict__ rank, int n_rows, int topk,
                                                                    long long shrinkage, int* __restrict__ cnt_ws, int* __restrict__ list_ws,
                                                                    int* __restrict__ next_row, int32_t* __restrict__ out_id,
                                                                    double* __restrict__ out_sim, int32_t* __restrict__ out_cnt) {
  __shared__ double s_sim[KNN_BUF];
  __shared__ int s_rank[KNN_BUF];
  __shared__ int s_id[KNN_BUF];
  __shared__ int s_row, s_nl, s_nbuf;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n_warps = blockDim.x >> 5;
  int* cnt = cnt_ws + (size_t)blockIdx.x * n_rows;
  int* list = list_ws + (size_t)blockIdx.x * n_rows;
  for (;;) {
    if (tid == 0) {
      s_row = atomicAdd(next_row, 1);
      s_nl = 0;
      s_nbuf = 0;
    }
    __syncthreads();
    const int a = s_row;
    if (a >= n_rows) return;
    const int beg = a_ptr[a], end = a_ptr[a + 1];
    for (int e = beg + warp; e < end; e += n_warps) {
      const int m = a_idx[e];
      const int f1 = t_ptr[m + 1];
      for (int f = t_ptr[m] + lane; f < f1; f += 32) {
        const int b = t_idx[f];
        const bool fresh = b != a && atomicAdd(&cnt[b], 1) == 0;
        const unsigned act = __activemask();
        const unsigned bal = __ballot_sync(act, fresh);
        const int leader = __ffs(act) - 1;
        int base = 0;
        if (lane == leader && bal) base = atomicAdd(&s_nl, __popc(bal));
        base = __shfl_sync(act, base, leader);
        if (fresh) list[base + __popc(bal & ((1u << lane) - 1u))] = b;
      }
    }
    __syncthreads();
    const int nl = s_nl, deg_a = end - beg;
    bool have_thr = false;
    double thr_sim = 0.0;
    int thr_rank = 0;
    for (int r0 = 0; r0 < nl; r0 += KNN_BUF - topk) {
      const int r1 = min(nl, r0 + KNN_BUF - topk);  // the buffer holds <= topk on entry: this round cannot overflow it
      for (int t = r0 + tid; t < r1; t += blockDim.x) {
        const int b = list[t];
        const int c = cnt[b];
        cnt[b] = 0;
        const double s = knn_sim(c, deg_a, a_ptr[b + 1] - a_ptr[b], shrinkage);
        const int rb = rank[b];
        if (!have_thr || knn_better(s, rb, thr_sim, thr_rank)) {
          const int slot = atomicAdd(&s_nbuf, 1);
          s_sim[slot] = s;
          s_rank[slot] = rb;
          s_id[slot] = b;
        }
      }
      __syncthreads();
      const int nb = s_nbuf;
      if (nb > topk || r1 == nl) {
        knn_sort_buffer(s_sim, s_rank, s_id, nb);
        if (nb >= topk) {
          have_thr = true;
          thr_sim = s_sim[topk - 1];
          thr_rank = s_rank[topk - 1];
        }
        if (tid == 0) s_nbuf = min(nb, topk);
      }
      __syncthreads();
    }
    const int keep = s_nbuf;
    for (int t = tid; t < topk; t += blockDim.x) {
      const size_t o = (size_t)a * topk + t;
      out_id[o] = t < keep ? s_id[t] : -1;
      out_sim[o] = t < keep ? s_sim[t] : 0.0;
    }
    if (tid == 0) out_cnt[a] = keep;
    __syncthreads();
  }
}

// One CTA per query user.  The row starts at zero; warp 0 adds the neighbour sims in the reference's order (mode 0,
// ItemKNN.py:58-81: the user's items in training_set_u order, each item's neighbours in list order; mode 1,
// UserKNN.py:59-80: the user's neighbours in list order, each neighbour's items).  Within one step the destinations are
// distinct, and __syncwarp orders consecutive steps, so each destination sums in the reference's order.  Then
// pred = acc / (acc + 1e-8) (an untouched 0 stays 0) and, optionally, rated items -> -10e8 (graph_recommender.py:49-50).
__global__ void __launch_bounds__(256) knn_score_rows_kernel(int mode, const int32_t* __restrict__ users, int n_items,
                                                             const int32_t* __restrict__ nbr_id, const double* __restrict__ nbr_sim,
                                                             const int32_t* __restrict__ nbr_cnt, int topk,
                                                             const int32_t* __restrict__ seq_ptr, const int32_t* __restrict__ seq_idx,
                                                             const int32_t* __restrict__ rated_ptr, const int32_t* __restrict__ rated_idx,
                                                             double* __restrict__ out) {
  const int u = users[blockIdx.x];
  double* row = out + (size_t)blockIdx.x * n_items;
  const int tid = threadIdx.x, lane = tid & 31;
  for (int j = tid; j < n_items; j += blockDim.x) row[j] = 0.0;
  __syncthreads();
  if (tid < 32) {
    if (mode == 0) {
      for (int e = seq_ptr[u]; e < seq_ptr[u + 1]; ++e) {
        const size_t i = seq_idx[e];
        const int n = nbr_cnt[i];
        for (int t = lane; t < n; t += 32) {
          const int j = nbr_id[i * topk + t];
          row[j] = __dadd_rn(row[j], nbr_sim[i * topk + t]);
        }
        __syncwarp();
      }
    } else {
      const int n = nbr_cnt[u];
      for (int t = 0; t < n; ++t) {
        const int v = nbr_id[(size_t)u * topk + t];
        const double s = nbr_sim[(size_t)u * topk + t];
        for (int f = seq_ptr[v] + lane; f < seq_ptr[v + 1]; f += 32) {
          const int j = seq_idx[f];
          row[j] = __dadd_rn(row[j], s);
        }
        __syncwarp();
      }
    }
  }
  __syncthreads();
  for (int j = tid; j < n_items; j += blockDim.x) {
    const double v = row[j];
    row[j] = __ddiv_rn(v, __dadd_rn(v, 1e-8));
  }
  if (rated_ptr) {
    __syncthreads();
    for (int e = rated_ptr[u] + tid; e < rated_ptr[u + 1]; e += blockDim.x) row[rated_idx[e]] = -10e8;
  }
}

// ---- find_k_largest on float64 rows ---------------------------------------------------------------------------
// heapq on (score, id) tuples (CPython Lib/heapq.py _siftdown / _siftup): the id breaks score ties inside the heap.
__device__ __forceinline__ bool knn_ent_lt(double sa, int ia, double sb, int ib) { return sa < sb || (sa == sb && ia < ib); }

__device__ void knn_siftdown(double* hs, int* hi, int start, int pos) {
  const double s = hs[pos];
  const int id = hi[pos];
  while (pos > start) {
    const int parent = (pos - 1) >> 1;
    if (!knn_ent_lt(s, id, hs[parent], hi[parent])) break;
    hs[pos] = hs[parent];
    hi[pos] = hi[parent];
    pos = parent;
  }
  hs[pos] = s;
  hi[pos] = id;
}

__device__ void knn_siftup(double* hs, int* hi, int n, int pos) {
  const int start = pos;
  const double s = hs[pos];
  const int id = hi[pos];
  int child = 2 * pos + 1;
  while (child < n) {
    const int right = child + 1;
    if (right < n && !knn_ent_lt(hs[child], hi[child], hs[right], hi[right])) child = right;
    hs[pos] = hs[child];
    hi[pos] = hi[child];
    pos = child;
    child = 2 * pos + 1;
  }
  hs[pos] = s;
  hi[pos] = id;
  knn_siftdown(hs, hi, start, pos);
}

// numba's list.sort(key=score, reverse=True): the argsort of numba/misc/quicksort.py with LT(a, b) = a > b
// (median-of-three partition while high - low >= 15, insertion sort below, a stack of 100 partitions).
__device__ void knn_argsort_desc(const double* A, int* R, int n) {
  for (int i = 0; i < n; ++i) R[i] = i;
  if (n < 2) return;
  int st_lo[100], st_hi[100];
  st_lo[0] = 0;
  st_hi[0] = n - 1;
  int sp = 1;
  while (sp > 0) {
    --sp;
    int low = st_lo[sp], high = st_hi[sp];
    while (high - low >= 15) {
      const int mid = (low + high) >> 1;
      int t;
      if (A[R[mid]] > A[R[low]]) t = R[low], R[low] = R[mid], R[mid] = t;
      if (A[R[high]] > A[R[mid]]) t = R[high], R[high] = R[mid], R[mid] = t;
      if (A[R[mid]] > A[R[low]]) t = R[low], R[low] = R[mid], R[mid] = t;
      const double pivot = A[R[mid]];
      t = R[high], R[high] = R[mid], R[mid] = t;
      int i = low, j = high - 1;
      for (;;) {
        while (i < high && A[R[i]] > pivot) ++i;
        while (j >= low && pivot > A[R[j]]) --j;
        if (i >= j) break;
        t = R[i], R[i] = R[j], R[j] = t;
        ++i;
        --j;
      }
      t = R[i], R[i] = R[high], R[high] = t;
      if (high - i > i - low) {
        if (high > i) st_lo[sp] = i + 1, st_hi[sp] = high, ++sp;
        high = i - 1;
      } else {
        if (i > low) st_lo[sp] = low, st_hi[sp] = i - 1, ++sp;
        low = i + 1;
      }
    }
    for (int i = low + 1; i <= high; ++i) {  // insertion sort of [low, high]
      const int k = R[i];
      const double v = A[k];
      int j = i;
      while (j > low && v > A[R[j - 1]]) {
        R[j] = R[j - 1];
        --j;
      }
      R[j] = k;
    }
  }
}

// One warp per row.  Lane 0 owns the heap (in the workspace); the lanes test 32 scores at a time against heap[0]
// (strict >, as the reference's `score > n_candidates[0][0]`), and lane 0 replays the passing ids in id order,
// re-testing each against the root the previous replacement left.  A score that fails against a root fails against
// every later one (the root never decreases), so the filter skips nothing the reference would take.
__global__ void __launch_bounds__(256) knn_topk_f64_kernel(const double* __restrict__ rows, int n_q, int n_items, int k,
                                                           double* __restrict__ heap_s, int* __restrict__ heap_id, int* __restrict__ perm,
                                                           int32_t* __restrict__ out_ids, double* __restrict__ out_sc) {
  const int q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (q >= n_q) return;
  const double* A = rows + (size_t)q * n_items;
  double* hs = heap_s + (size_t)q * k;
  int* hi = heap_id + (size_t)q * k;
  int* R = perm + (size_t)q * k;
  for (int t = lane; t < k; t += 32) {
    hs[t] = A[t];
    hi[t] = t;
  }
  __syncwarp();
  double root = 0.0;
  if (lane == 0) {
    for (int i = k / 2 - 1; i >= 0; --i) knn_siftup(hs, hi, k, i);  // heapq.heapify
    root = hs[0];
  }
  root = __shfl_sync(SRB_FULL_MASK, root, 0);
  for (int base = k; base < n_items; base += 32) {
    const int i = base + lane;
    const double v = i < n_items ? A[i] : 0.0;
    unsigned bal = __ballot_sync(SRB_FULL_MASK, i < n_items && v > root);
    while (bal) {
      const int l = __ffs(bal) - 1;
      bal &= bal - 1;
      const double s = __shfl_sync(SRB_FULL_MASK, v, l);
      if (s > root) {  // heapq.heapreplace
        if (lane == 0) {
          hs[0] = s;
          hi[0] = base + l;
          knn_siftup(hs, hi, k, 0);
          root = hs[0];
        }
        root = __shfl_sync(SRB_FULL_MASK, root, 0);
      }
    }
  }
  if (lane == 0) knn_argsort_desc(hs, R, k);
  __syncwarp();
  for (int t = lane; t < k; t += 32) {
    out_ids[(size_t)q * k + t] = hi[R[t]];
    out_sc[(size_t)q * k + t] = hs[R[t]];
  }
}

}  // namespace srb

extern "C" int64_t srb_knn_neighbors_workspace_bytes(int32_t n_rows) {
  if (n_rows < 1) return 0;
  const int64_t ctas = std::min<int64_t>(n_rows, (int64_t)srb::sm_count() * 2);
  return 256 + ctas * (int64_t)n_rows * 8;
}

extern "C" int srb_knn_neighbors(const srb_knn_rows* rows, int32_t topk, int64_t shrinkage, int32_t* out_id, double* out_sim,
                                 int32_t* out_cnt, void* workspace, int64_t workspace_bytes, void* stream) {
  SRB_REQUIRE(rows && out_id && out_sim && out_cnt && workspace, "knn_neighbors: null pointer");
  SRB_REQUIRE(rows->row_ptr && rows->row_idx && rows->t_ptr && rows->t_idx && rows->rank, "knn_neighbors: null CSR pointer");
  SRB_REQUIRE(rows->n_rows >= 1, "knn_neighbors: n_rows=%d must be >= 1", rows->n_rows);
  SRB_REQUIRE(topk >= 1 && topk <= SRB_KNN_MAX_TOPK, "knn_neighbors: topK=%d outside 1..%d", topk, SRB_KNN_MAX_TOPK);
  SRB_REQUIRE(shrinkage >= 0 && shrinkage < (1ll << 52), "knn_neighbors: shrinkage=%lld outside 0..2^52", (long long)shrinkage);
  const int64_t need = srb_knn_neighbors_workspace_bytes(rows->n_rows);
  SRB_REQUIRE(workspace_bytes >= need, "knn_neighbors: workspace of %lld bytes, %lld needed", (long long)workspace_bytes, (long long)need);
  const int n = rows->n_rows;
  const int ctas = (int)std::min<int64_t>(n, (int64_t)srb::sm_count() * 2);
  char* ws = (char*)workspace;
  int* next_row = (int*)ws;
  int* cnt = (int*)(ws + 256);
  int* list = cnt + (size_t)ctas * n;
  cudaStream_t st = (cudaStream_t)stream;
  SRB_TRY(srb::check_cuda(cudaMemsetAsync(ws, 0, 256 + (size_t)ctas * n * 4, st), "knn_neighbors: clear counts"));
  srb::knn_neighbors_kernel<<<ctas, srb::KNN_THREADS, 0, st>>>(rows->row_ptr, rows->row_idx, rows->t_ptr, rows->t_idx, rows->rank, n, topk,
                                                               (long long)shrinkage, cnt, list, next_row, out_id, out_sim, out_cnt);
  return srb::post_launch("knn_neighbors_kernel");
}

extern "C" int srb_knn_score_rows(int32_t mode, const int32_t* users, int32_t n_q, int32_t n_items, const int32_t* nbr_id,
                                  const double* nbr_sim, const int32_t* nbr_cnt, int32_t topk, const int32_t* seq_ptr,
                                  const int32_t* seq_idx, const int32_t* rated_ptr, const int32_t* rated_idx, double* out,
                                  void* stream) {
  SRB_REQUIRE(mode == 0 || mode == 1, "knn_score_rows: mode=%d (0 ItemKNN, 1 UserKNN)", mode);
  SRB_REQUIRE(users && nbr_id && nbr_sim && nbr_cnt && seq_ptr && seq_idx && out, "knn_score_rows: null pointer");
  SRB_REQUIRE(!rated_ptr == !rated_idx, "knn_score_rows: rated_ptr and rated_idx go together");
  SRB_REQUIRE(n_q >= 0 && n_items >= 1 && topk >= 1, "knn_score_rows: bad shape (n_q=%d, n_items=%d, topK=%d)", n_q, n_items, topk);
  if (n_q == 0) return SRB_OK;
  srb::knn_score_rows_kernel<<<n_q, 256, 0, (cudaStream_t)stream>>>(mode, users, n_items, nbr_id, nbr_sim, nbr_cnt, topk, seq_ptr,
                                                                    seq_idx, rated_ptr, rated_idx, out);
  return srb::post_launch("knn_score_rows_kernel");
}

extern "C" int64_t srb_topk_f64_workspace_bytes(int32_t n_q, int32_t k) { return (int64_t)n_q * k * 16; }

extern "C" int srb_topk_rows_f64(const double* rows, int32_t n_q, int32_t n_items, int32_t k, int32_t* out_ids, double* out_scores,
                                 void* workspace, int64_t workspace_bytes, void* stream) {
  SRB_REQUIRE(rows && out_ids && out_scores, "topk_rows_f64: null pointer");
  SRB_REQUIRE(n_q >= 0 && n_items >= 1, "topk_rows_f64: bad shape (n_q=%d, n_items=%d)", n_q, n_items);
  SRB_REQUIRE(k >= 1 && k <= n_items, "topk_rows_f64: k=%d outside 1..n_items=%d", k, n_items);
  if (n_q == 0) return SRB_OK;
  const int64_t need = srb_topk_f64_workspace_bytes(n_q, k);
  SRB_REQUIRE(workspace && workspace_bytes >= need, "topk_rows_f64: workspace of %lld bytes, %lld needed", (long long)workspace_bytes,
              (long long)need);
  double* hs = (double*)workspace;
  int* hi = (int*)(hs + (size_t)n_q * k);
  int* perm = hi + (size_t)n_q * k;
  srb::knn_topk_f64_kernel<<<(n_q + 7) / 8, 256, 0, (cudaStream_t)stream>>>(rows, n_q, n_items, k, hs, hi, perm, out_ids, out_scores);
  return srb::post_launch("knn_topk_f64_kernel");
}
