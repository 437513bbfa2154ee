/*
 * selfrec_b200 -- C ABI of the B200-native hot path behind SELFRec's plugin surface.
 *
 * Every entry point takes plain pointers and sizes (no torch types).  Device pointers
 * are raw CUDA addresses (e.g. tensor.data_ptr()); `stream` is a cudaStream_t passed as
 * void* (NULL = legacy default stream).  All kernels are stream-ordered, never
 * synchronise the device, and are CUDA-graph capturable.  Every function returns
 * SRB_OK (0) or a negative error code; srb_last_error() gives the message.  There is
 * no CPU fallback: device entry points fail with SRB_ERR_CUDA when no GPU is present.
 *
 * The reference (Coder-Yu/SELFRec) has no FFI; each entry point names the reference
 * Python call site it replaces (paths relative to the reference root).
 *
 * Layout conventions
 *   - embedding tables: fp32, row-major [rows, d], rows 0..U-1 users, U..U+I-1 items
 *     (the reference's torch.cat([user_emb, item_emb]), LightGCN.py:69).
 *   - adjacency: CSR, int32 rowptr[n+1], int32 colidx[nnz], fp32 vals[nnz]
 *     (scipy CSR of data/graph.py:10-24, indices sorted within a row).
 *   - d (embedding.size) must be one of 16, 32, 64, 128, 256.
 */
#ifndef SELFREC_B200_H
#define SELFREC_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SRB_OK 0
#define SRB_ERR_ARG (-1)   /* bad argument (shape, null pointer, unsupported d/k) */
#define SRB_ERR_CUDA (-2)  /* CUDA runtime error or no device */
#define SRB_ERR_STATE (-3) /* handle misuse */

const char* srb_last_error(void);
int srb_version(void);
/* Number of kernel launches issued through this library since load (bench `gpu_launches`). */
int64_t srb_launch_count(void);
/* 0 when a CUDA device is usable, SRB_ERR_CUDA otherwise. */
int srb_device_ok(void);

/* ---------------------------------------------------------------------------------------
 * (i) Propagation: Y = A * X with a fused epilogue.
 * Replaces torch.sparse.mm(self.sparse_norm_adj, ego_embeddings)
 *   LightGCN.py:72, SimGCL.py:85, XSimGCL.py:88, SGL.py:104-108
 * and the elementwise ops that follow it in the encoders:
 *   noise      XSimGCL.py:90-91 / SimGCL.py:87-88   y += sign(y) * normalize(noise) * eps
 *   layer sum  LightGCN.py:74-75 / XSimGCL.py:95-96 (torch.stack + torch.mean)
 *   Adam       torch.optim.Adam.step (XSimGCL.py:25,37) when the product is the E0 gradient.
 * ------------------------------------------------------------------------------------- */
/* Split ("huge") rows.  A power-law graph at config-5 scale (10 M x 2 M x 200 M) has rows with millions of
 * non-zeros; rows with at least SRB_HUB_MIN_NNZ non-zeros are cut into chunks of SRB_HUB_CHUNK non-zeros, one CTA
 * per chunk writes its partial sum to `part`, and the row's owner adds the partials in chunk order (deterministic).
 * Static lists (built with the graph): the first n_rows entries of row_order are the split rows, first[r] is the
 * slot of row r's first chunk, work[w] = (row, chunk index), n_work chunks in total.  Device-classified lists
 * (the batch rows of a training step): first / work are written on the device, n_work is the capacity and the live counts come
 * from n_vlong_dev[0] (rows) and n_vlong_dev[4] (chunks). */
#define SRB_HUB_CHUNK 2048
#define SRB_HUB_MIN_NNZ 4096
#define SRB_HUB_WARP_SEG 256
typedef struct srb_hub_split {
  int32_t n_rows;
  int32_t n_work;
  const int32_t* first; /* [n_rows] */
  const int32_t* work;  /* [n_work][2] */
  float* part;          /* [n_work, d] scratch (one product at a time per graph) */
  /* Column-blocked variant of the static lists (optional; seg != NULL selects it).  At config-5 size the split rows
   * hold ~40 % of the non-zeros and their gathers miss L2 (the X table is 6 GB): cutting every split row at column-block
   * boundaries (a block of X rows = a quarter of the L2, 12.5 MB on an H100) and processing ALL rows' segments of one block before the next keeps that
   * block of X in L2, so it is read from HBM once per product instead of once per row.
   *   seg[w] = (begin, end) CSR positions of segment w; a row's segments are consecutive slots (first[r], seg_cnt[r]);
   *   n_work = number of segments (capacity of part);
   *   order_cta / order_warp: segment ids in processing order (column block, then row): segments longer than
   *   SRB_HUB_WARP_SEG non-zeros take a CTA each, the others a warp each. */
  const int32_t* seg;       /* [n_work][2] */
  const int32_t* seg_cnt;   /* [n_rows] */
  const int32_t* order_cta;
  const int32_t* order_warp;
  int32_t n_cta;
  int32_t n_warp;
} srb_hub_split;

typedef struct srb_spmm_desc {
  /* A: CSR [n_rows, n_cols] */
  const int32_t* rowptr;
  const int32_t* colidx;
  const float* vals;
  int32_t n_rows;
  int32_t n_cols;
  int32_t d;
  /* optional processing order of rows (length n_rows), NULL = natural order; when it is sorted by
   * descending degree, the first hub.n_rows entries are split rows (see srb_hub_split), the next n_vlong_rows
   * entries are given a whole CTA each and the next n_long_rows entries a whole warp each (the rest share warps) */
  const int32_t* row_order;
  int32_t n_long_rows;
  int32_t n_vlong_rows;
  srb_hub_split hub;
  /* optional device-side classification (row lists built on the device, e.g. the rows of a batch):
   * n_vlong_dev[0..3] = number of split / very long / long / short rows, [4] = number of chunks; row_order then
   * holds four segments of capacity n_rows each: split, very long, long, short */
  const int32_t* n_vlong_dev;
  /* optional bitmap over columns (bit c of word c/32): a clear bit promises X[c,:] == 0, so the
     non-zero is skipped without touching X (row-sparse X: the first backward product). */
  const uint32_t* col_mask;
  const float* X;     /* [n_cols, d] */
  float* Y;           /* [n_rows, d] or NULL (result only feeds sum/adam) */
  const float* extra; /* optional dense addend [n_rows, d]: y += extra_scale * extra[row] */
  float extra_scale;
  /* noise epilogue: 0 none, 1 tensor (parity mode), 2 in-kernel Philox (perf mode) */
  int32_t noise_mode;
  const float* noise; /* [n_rows, d] uniform [0,1) when noise_mode == 1 */
  float eps;
  uint64_t philox_seed;   /* noise_mode == 2 */
  uint64_t philox_offset; /* distinct per (layer, view) */
  const int32_t* philox_step_dev; /* optional device step counter mixed into the counter */
  /* running layer sum: sum_out[row] = sum_scale * ((sum_in ? sum_in[row] : 0) + y) */
  const float* sum_in;
  float* sum_out;
  float sum_scale;
  /* fused Adam on (p, m, v) with gradient y (after extra); scalars from srb_adam_prepare */
  float* adam_p;
  float* adam_m;
  float* adam_v;
  const float* adam_scalars; /* device: {step_size, bias_correction2_sqrt} */
  double beta1, beta2;       /* doubles: 1 - beta is rounded to fp32 from the double, like torch */
  float adam_eps;
} srb_spmm_desc;

int srb_spmm_csr(const srb_spmm_desc* desc, void* stream);
/* The epilogue alone, row by row: Y[r] = epilogue(X[r]) for r < n_rows -- the product with the identity matrix
 * (rowptr / colidx / vals are not read).  Used for the noise that SimGCL's perturbed encoders add to the shared first
 * product (SimGCL.py:87-88): same Philox keying / noise tensor indexing as the fused SpMM epilogue. */
int srb_spmm_epilogue_rows(const srb_spmm_desc* desc, void* stream);

/* Encoder forward (R4).  Composes srb_spmm_csr launches:
 *   LGCN_Encoder.forward LightGCN.py:68-78, SGL_Encoder.forward SGL.py:98-113  (include_ego=1)
 *   SimGCL_Encoder.forward SimGCL.py:81-93, XSimGCL_Encoder.forward XSimGCL.py:83-101 (include_ego=0)
 * final = mean over layers; cl_view = (perturbed) output of layer layer_cl (1-based), or E0
 * if layer_cl is never reached (XSimGCL.py:86).  work0/work1: [n, d] ping-pong buffers.
 * noise (noise_mode==1): [n_layers, n, d]. */
typedef struct srb_encoder_desc {
  const int32_t* rowptr;
  const int32_t* colidx;
  const float* vals;
  const int32_t* row_order;
  int32_t n_long_rows;
  int32_t n_vlong_rows;
  srb_hub_split hub;
  int32_t n;
  int32_t d;
  int32_t n_layers;
  int32_t include_ego;
  int32_t layer_cl; /* 0 = no CL view requested */
  int32_t noise_mode;
  const float* noise;
  float eps;
  uint64_t philox_seed;
  uint64_t philox_offset;
  const int32_t* philox_step_dev;
  /* optional: the LAST layer is only evaluated for these rows (device list, duplicates allowed), e.g.
   * the batch rows of a training step -- nothing else reads the final mean there.  Refused with n_layers == 0
   * and with cl_out set at layer_cl == n_layers: that last layer is needed in full, so leave last_rows unset and
   * read the mean from final_out */
  const int32_t* last_rows;
  int32_t n_last_rows;
  const int32_t* last_rows_nv_dev; /* device-classified list: counts [5]; last_rows = 4 segments of n_last_rows (see srb_spmm_desc.n_vlong_dev) */
  srb_hub_split last_rows_hub;     /* split rows of that list (device-written first / work) */
  float* last_rows_out; /* [n, d], required with last_rows: receives the final mean of the listed rows
                           (final_out then only holds the running sum; the list may contain duplicates,
                           so the last layer must not update the running sum in place) */
  const float* E0; /* [n, d] parameters */
  float* final_out; /* [n, d] */
  float* cl_out;    /* [n, d] or NULL */
  float* work0;
  float* work1;
  /* optional [n, d]: the output of layer 1 (its noise included), computed by the caller -- SimGCL's three encoders
   * share the product A * E0 (SimGCL.py:85) and differ only in the noise added to it.  The first product is skipped
   * and the layer sum starts from x1.  Needs n_layers >= 2, include_ego == 0 and layer_cl != 1; x1 must not be
   * work0 / work1. */
  const float* x1;
} srb_encoder_desc;

int srb_encoder_forward(const srb_encoder_desc* desc, void* stream);

/* ---------------------------------------------------------------------------------------
 * (ii) Fused (u,i,j) gather + BPR + L2 forward/backward.
 * Replaces   rec_user_emb[user_idx] ...          XSimGCL.py:30 (and peers)
 *            bpr_loss                            util/loss_torch.py:6-10
 *            l2_reg_loss                         util/loss_torch.py:18-22
 * and their autograd backward.  Two launches (the un-squared Frobenius norm needs a
 * grid-wide reduction before its gradient).
 *   emb      [n, d] table the (u,i,j) rows are gathered from (item rows offset by n_users)
 *   l2_emb   table the L2 term gathers from (== emb except LightGCN.py:25 -> raw params)
 *   l2_terms 2: (u,i)   3: (u,i,j);   l2_div: extra divisor (batch_size or 1)
 * Outputs: losses[0]=bpr mean, losses[1]=l2 term (reg * sum ||.||_F / rows / l2_div)
 *   g_emb   [3, b, d] gradient w.r.t. gathered emb rows (u, i, j)
 *   g_l2    [3, b, d] gradient w.r.t. gathered l2_emb rows (NULL => added into g_emb;
 *           only valid when l2_emb == emb)
 *   scratch [8] floats device workspace (zeroed by the call)
 * ------------------------------------------------------------------------------------- */
typedef struct srb_bpr_desc {
  const float* emb;
  const float* l2_emb;
  int32_t n_users;
  int32_t d;
  const int32_t* u_idx;
  const int32_t* i_idx;
  const int32_t* j_idx;
  const int32_t* b_dev; /* optional device batch size (<= b); NULL => b */
  int32_t b;
  float emb_scale; /* gathered rows are emb_scale * emb[row] (lazy layer mean); g_emb is the gradient w.r.t. these
                    * scaled rows.  With l2_emb == emb the L2 term regularises the scaled rows; a separate l2_emb is
                    * read unscaled */
  float reg;
  int32_t l2_terms;
  float l2_div;
  float grad_scale; /* upstream dLoss (1.0): scales g_emb and g_l2, not losses */
  float* losses;    /* [2] device */
  float* g_emb;
  float* g_l2;
  float* scratch;
} srb_bpr_desc;

int srb_bpr_l2_fwd_bwd(const srb_bpr_desc* desc, void* stream);

/* ---------------------------------------------------------------------------------------
 * (iii) Fused InfoNCE forward/backward over in-batch negatives.
 * Replaces InfoNCE(view1[idx], view2[idx], temperature) util/loss_torch.py:35-50 as used by
 *   XSimGCL.py:45-50, SimGCL.py:43-50, SGL.py:115-125 (and its autograd backward).
 * The n x n logit matrix never reaches HBM.  A "problem" is one InfoNCE call; several
 * problems run in one launch sequence (user + item terms).
 *   view rows are gathered: v1 = scale1 * table1[idx[i] + row_off1], v2 likewise.
 *   loss_p = mean_i(logsumexp_j S_ij - S_ii),  S = normalize(v1) normalize(v2)^T / tau
 *   losses[p] device output; g1/g2 [n, d] gradients w.r.t. the gathered rows times weight.
 * workspace: srb_infonce_workspace_bytes(max_n, d, n_problems) bytes, device.
 * ------------------------------------------------------------------------------------- */
typedef struct srb_infonce_problem {
  const float* table1;
  const float* table2;
  int32_t row_off1;
  int32_t row_off2;
  float scale1;
  float scale2;
  const int32_t* idx;   /* [n] device row ids */
  const int32_t* n_dev; /* optional device count (<= n) */
  int32_t n;
  float weight; /* gradient/loss weight (lambda); loss output is unweighted */
  float* g1;    /* [n, d] */
  float* g2;    /* [n, d] */
  float* loss;  /* [1] */
} srb_infonce_problem;

typedef struct srb_infonce_desc {
  int32_t n_problems; /* <= 4 */
  int32_t d;
  int32_t b_cos;
  float temperature;
  srb_infonce_problem prob[4];
  void* workspace;
  int64_t workspace_bytes;
} srb_infonce_desc;

int64_t srb_infonce_workspace_bytes(int32_t max_n, int32_t d, int32_t n_problems);
int srb_infonce_fwd_bwd(const srb_infonce_desc* desc, void* stream);

/* In-batch softmax loss, on the InfoNCE kernels and descriptor.
 * Replaces batch_softmax_loss(user_emb, item_emb, temperature) util/loss_torch.py:25-32 as used by
 *   SSL4Rec.py:33 (and imported by CL4SRec.py:7), plus its autograd backward:
 *   loss_p = mean_i(-log(p_i + 1e-5)),  p_i = softmax(S)_ii,  S = normalize(v1) normalize(v2)^T / tau
 * with v1 = user rows, v2 = item rows.  Same fields and workspace (srb_infonce_workspace_bytes) as
 * srb_infonce_fwd_bwd; b_cos must be 1.  p_i comes from the row's log-sum-exp, so the loss stays
 * finite where the reference's unshifted exp(S) overflows (1/tau > 88.7). */
int srb_batch_softmax_fwd_bwd(const srb_infonce_desc* desc, void* stream);

/* Standalone l2_reg_loss (util/loss_torch.py:18-22) on already-gathered embeddings, for the
 * op-level drop-in: loss = reg * sum_t ||x_t||_F / rows_t.  sumsq_dev: [4] device scratch kept
 * for the backward; gout_dev: device scalar upstream gradient. */
int srb_l2_reg_fwd(int32_t n_terms, const float* const* x, const int64_t* n_elems, const int32_t* rows,
                   float reg, float* sumsq_dev, float* loss_dev, void* stream);
int srb_l2_reg_bwd(int32_t n_terms, const float* const* x, float* const* g, const int64_t* n_elems,
                   const int32_t* rows, float reg, const float* sumsq_dev, const float* gout_dev,
                   void* stream);

/* ---------------------------------------------------------------------------------------
 * Sparse-row scatter: dst[rows[r] + row_off] += scale * src[r]  (atomic; duplicates sum).
 * Replaces the index_put_(accumulate=True) autograd backward of tensor[list] gathers
 *   (MF.py:20, LightGCN.py:24, XSimGCL.py:30).
 * ------------------------------------------------------------------------------------- */
int srb_scatter_add_rows(float* dst, int32_t d, const float* src, const int32_t* rows,
                         int32_t n, const int32_t* n_dev, int32_t row_off, float scale,
                         void* stream);

/* Up to 8 such scatters into the same table in ONE launch (the gradient of several gathers of
 * one tensor).  n_dev (optional, device) overrides n with min(*n_dev, n). */
typedef struct srb_scatter_seg {
  const float* src;     /* [n, d] compact rows */
  const int32_t* rows;  /* [n] destination rows */
  const int32_t* n_dev;
  int32_t n;
  int32_t row_off;
  float scale;
} srb_scatter_seg;
int srb_scatter_add_segments(float* dst, int32_t d, int32_t n_segs, const srb_scatter_seg* segs,
                             void* stream);

/* ---------------------------------------------------------------------------------------
 * Adam (R10): torch.optim.Adam defaults, dense (MF.py:15 ... XSimGCL.py:25).
 * srb_adam_prepare: one tiny launch; increments the device step counter and writes
 *   scalars = {lr / (1 - beta1^t), sqrt(1 - beta2^t)} (double arithmetic, like torch's
 *   Python-float bias corrections).
 * srb_adam_step: p,m,v update from dense gradient g over n elements.  It and the SpMM's Adam epilogue round every
 *   element as torch.optim.Adam's CUDA kernels do (bit for bit).
 * ------------------------------------------------------------------------------------- */
int srb_adam_prepare(int32_t* step_dev, float* scalars_dev, double lr, double beta1,
                     double beta2, void* stream);
int srb_adam_step(float* p, float* m, float* v, const float* g, int64_t n,
                  const float* scalars_dev, double beta1, double beta2, float eps,
                  void* stream);

/* ---------------------------------------------------------------------------------------
 * (iv) Full-catalog scoring + rated-item mask + top-k.
 * Replaces the per-user loop of GraphRecommender.test() base/graph_recommender.py:38-58:
 *   predict (XSimGCL.py:57-60), mask -10e8 (graph_recommender.py:48-50),
 *   find_k_largest util/algorithm.py:144-156.
 *   user_emb [n_users_total, d], item_emb [n_items, d]
 *   users    [n_q] user ids to score (test_set order)
 *   rated_ptr/rated_idx: CSR over ALL users of sorted rated item ids (interaction_mat)
 *   out_ids  [n_q, k] int32, out_scores [n_q, k] fp32, score-descending
 * Selection follows find_k_largest's sequential semantics (strict > threshold, evict the
 * lexicographically smallest (score, id)); scores are exact fp32 fma chains over d.
 * k: 1..32 on impl 1; 1..256 on impl 2 (d = 16, 32, 64, 128 or 256).  Longer lists, and lists over 32
 * that auto does not send to impl 2, are extracted 32 at a time from dense score rows
 * (selfrec_b200/ops.py _score_topk_wide).
 * ------------------------------------------------------------------------------------- */
typedef struct srb_topk_desc {
  const float* user_emb;
  const float* item_emb;
  int32_t n_items;
  int32_t d;
  const int32_t* users;
  int32_t n_q;
  const int32_t* rated_ptr;
  const int32_t* rated_idx;
  int32_t k;
  int32_t* out_ids;
  float* out_scores;
  int32_t impl; /* 0 auto (impl 2 when n_items >= 1024, a workspace is given and either k <= 32 or d is 64 or
                   128, else impl 1);
                   1 CUDA cores, exact fp32, k <= 32 (k > 32 is refused);
                   2 (d = 16, 32, 64, 128 or 256, k <= 256) wgmma TF32 candidates + exact fp32 rescoring + a per-user exactness
                   certificate, uncertified users re-run by the exact path.  k <= 32: candidate lists of 2 x 24 per
                   user; 33 <= k <= 256: per-half candidate buffers behind a running threshold (DESIGN 4.4) */
  void* workspace; /* impl 2: srb_topk_workspace_bytes(n_q, n_items, d, k) bytes, 256-byte aligned;
                      O(n_q * k + n_items), never a dense [n_q, n_items] buffer */
  int64_t workspace_bytes;
} srb_topk_desc;

int64_t srb_topk_workspace_bytes(int32_t n_q, int32_t n_items, int32_t d, int32_t k);
/* byte offset (inside the impl-2 workspace) of the int32 count of users the exact fallback re-ran; the same at
   every d and k */
int64_t srb_topk_fallback_count_offset(int32_t n_q, int32_t n_items);
/* impl 2's error bound at width d: |approximate - exact score| <= E(d) * ||u|| * max_i ||item_i|| (DESIGN 4.4), the
   constant of its certificate; -1 at a width impl 2 does not rank */
float srb_topk_tc_error_bound(int32_t d);
int srb_score_topk(const srb_topk_desc* desc, void* stream);
/* Dense score rows out[q, i] = <user_emb[users[q]], item_emb[i]>, the reference's predict()
 * (XSimGCL.py:57-60); same fp32 fma chain as srb_score_topk. */
int srb_score_rows(const float* user_emb, const float* item_emb, int32_t d, const int32_t* users,
                   int32_t n_q, int32_t n_items, float* out, void* stream);
/* Mask-free top-k of precomputed score rows [n_q, n_items] (models whose predict() is not one
 * dot product, e.g. BUIR.py); same selection rule.  The caller applies the -10e8 mask. */
int srb_topk_rows(const float* scores, int32_t n_q, int32_t n_items, int32_t k, int32_t* out_ids,
                  float* out_scores, void* stream);

/* random.sample(range(n), k) on a CPython MT19937 state (624 words + index, as random.getstate()[1]):
 * the draw behind GraphAugmentor.node_dropout / edge_dropout (data/augmentor.py:16-17, 28).  use_pool
 * selects CPython's pool-list variant (n <= setsize) or its selected-set variant; the state is advanced
 * exactly as CPython would. */
int srb_random_sample_range(uint32_t* mt625, int64_t n, int64_t k, int32_t use_pool, int64_t* out);


/* ---------------------------------------------------------------------------------------
 * Native dataset -> CSR builder (host C++; SURVEY 8(f) row 1).  Replaces the Python loops of
 *   FileIO.load_data_set (data/loader.py:23-33), Interaction.__generate_set (data/ui_graph.py:29-45),
 *   __create_sparse_bipartite_adjacency / __create_sparse_interaction_matrix (data/ui_graph.py:47-72)
 *   and the scaling half of normalize_graph_mat (data/graph.py:16-18)
 * with identical results: ids in order of first appearance in the training file, duplicate lines
 * summed, test pairs kept only when both user and item are known, adjacency values the fp32
 * products (d[r] * a) * d[c].  A malformed line fails the load (the reference raises IndexError /
 * ValueError there).  Handles are host objects; nothing here touches the GPU.
 * ------------------------------------------------------------------------------------- */
typedef struct srb_dataset srb_dataset;
srb_dataset* srb_dataset_load(const char* train_path, const char* test_path /* may be NULL */);
void srb_dataset_free(srb_dataset* d);
/* out[8] = n_users, n_items, n_train_lines, n_test_pairs_kept, n_distinct_train_pairs,
 *          total bytes of user names, total bytes of item names, n_test_lines (kept or not) */
int srb_dataset_counts(const srb_dataset* d, int64_t* out);
/* names of ids 0..n-1 (which: 0 users, 1 items), concatenated; offsets[n+1] */
int srb_dataset_names(const srb_dataset* d, int32_t which, char* blob, int64_t* offsets);
/* (user id, item id, weight) in file order; which: 0 training lines, 1 kept test lines */
int srb_dataset_pairs(const srb_dataset* d, int32_t which, int32_t* u, int32_t* i, double* w);
/* users x items, duplicates summed, columns ascending: rowptr[U+1], colidx/vals[n_distinct] */
int srb_dataset_interaction_csr(const srb_dataset* d, int32_t* rowptr, int32_t* colidx, float* vals);
/* (U+I) x (U+I) bipartite adjacency, rows = users then items, columns ascending:
 * rowptr[N+1], colidx/vals[2 n_distinct].  d_inv == NULL: raw counts; else vals = (d_inv[r]*a)*d_inv[c].
 * rowsum (optional, [N]) receives the fp32 row sums of the raw counts. */
int srb_dataset_adjacency_csr(const srb_dataset* d, const float* d_inv, int32_t* rowptr,
                              int32_t* colidx, float* vals, float* rowsum);

/* The same adjacency for arbitrary (user, item) pairs with unit weights (duplicates summed): the CSR assembly of
 * Interaction.convert_to_laplacian_mat (data/ui_graph.py:58-65) for SGL's dropped graphs.  colidx / vals have
 * capacity 2 * n_pairs; *nnz_out receives the number of stored entries; rowsum is optional. */
int srb_bipartite_adjacency_csr(const int32_t* users, const int32_t* items, int64_t n_pairs, int32_t n_users,
                                int32_t n_items, int32_t* rowptr, int32_t* colidx, float* vals, float* rowsum,
                                int64_t* nnz_out);

/* ---------------------------------------------------------------------------------------
 * Device-side assembly of the normalised (U+I) x (U+I) adjacency (SURVEY 8(f) row 3, R2, R11):
 *   Interaction.__create_sparse_bipartite_adjacency / convert_to_laplacian_mat  data/ui_graph.py:47-65
 *   Graph.normalize_graph_mat                                                  data/graph.py:10-24
 * for the interaction edges that survive GraphAugmentor.edge_dropout / node_dropout (data/augmentor.py:11-40,
 * SGL.py:80-96) -- or all of them (a config-5 sized graph is built this way: no scipy at 200 M edges).
 * Inputs (device): the users x items CSR of distinct pairs, columns ascending (ui_ptr[U+1], ui_col[nnz], ui_val[nnz]
 * = multiplicities, NULL = 1), its transpose (iu_ptr[I+1], iu_col[nnz] user ids ascending, iu_perm[nnz] = position
 * in the ui order of each entry of the iu order), the kept edges as byte flags over the ui order (keep_flags) or as
 * a list of positions (keep_idx, n_keep; e.g. srb_random_sample_range's output) or neither (all edges);
 * reset_weights != 0 gives kept edges weight 1 (augmentor.py:36 np.ones_like).
 * dinv_table[k] = float32 power(k, -0.5) with inf -> 0 for k = 0 .. dinv_table_n-1, computed by the caller with
 * numpy so that the rounding is the reference's (row sums are small integers).
 * Outputs (device): rowptr[N+1], colidx / vals[out_cap >= 2 * kept] (columns ascending, values the fp32 products
 * (d[r] * a) * d[c] of graph.py:16-18), dinv[N], *nnz_out (optional) = stored entries.  Results are bit-identical
 * to the scipy route (tests/test_gpu_graphbuild.py).  Stream-ordered; workspace from
 * srb_graph_assemble_workspace_bytes, 256-byte aligned.
 * ------------------------------------------------------------------------------------- */
typedef struct srb_graph_assemble_desc {
  int32_t n_users, n_items;
  int64_t nnz;
  const int32_t* ui_ptr;
  const int32_t* ui_col;
  const float* ui_val;
  const int32_t* iu_ptr;
  const int32_t* iu_col;
  const int32_t* iu_perm;
  const uint8_t* keep_flags;
  const int64_t* keep_idx;
  int64_t n_keep;
  int32_t reset_weights;
  const float* dinv_table;
  int32_t dinv_table_n;
  int32_t* rowptr;
  int32_t* colidx;
  float* vals;
  float* dinv;
  int64_t out_cap;
  int64_t* nnz_out;
  void* workspace;
  int64_t workspace_bytes;
} srb_graph_assemble_desc;
int64_t srb_graph_assemble_workspace_bytes(int32_t n_users, int32_t n_items, int64_t nnz);
int srb_graph_assemble(const srb_graph_assemble_desc* desc, void* stream);

/* ---------------------------------------------------------------------------------------
 * Ranking metrics, device part (SURVEY 8(f) row 2; util/evaluation.py:9-15 `hits`, :85-97 NDCG):
 * hit_mask[q * W + r / 64] bit r % 64 = 1 iff topk_ids[q, r] is in the test set of users[q]
 * (r < k <= 256, W = ceil(k / 64) words per row: one word for k <= 64).
 * test_ptr / test_idx: CSR over user ids of the test items that have a training id, sorted per
 * user.  Hit Ratio / Precision / Recall / NDCG follow on the host from the masks with the
 * reference's own float expressions (selfrec_b200/util/evaluation.py), so they match bit for bit.
 * ------------------------------------------------------------------------------------- */
int srb_rank_hit_masks(const int32_t* topk_ids, int32_t n_q, int32_t k, const int32_t* users,
                       const int32_t* test_ptr, const int32_t* test_idx, uint64_t* hit_mask,
                       void* stream);

/* ---------------------------------------------------------------------------------------
 * One whole training step (R3-R8, R10) as a single call: forward propagation, gather +
 * BPR + L2, InfoNCE, Horner backward through the propagation, Adam in the epilogue of the
 * last backward SpMM.  Replaces the body of <Model>.train()'s batch loop:
 *   MF.py:17-25  LightGCN.py:21-29  SimGCL.py:25-36  XSimGCL.py:27-37  SGL.py:30-41
 * The call only enqueues work (graph-capturable); batch indices live in one device
 * buffer laid out by srb_sampler_next_batch (header + u,i,j + unique lists).
 * ------------------------------------------------------------------------------------- */
enum { SRB_MODEL_MF = 0, SRB_MODEL_LIGHTGCN = 1, SRB_MODEL_SIMGCL = 2, SRB_MODEL_XSIMGCL = 3, SRB_MODEL_SGL = 4 };

typedef struct srb_graph_csr {
  const int32_t* rowptr;
  const int32_t* colidx;
  const float* vals;
  const int32_t* row_order;
  int32_t n_long_rows;
  int32_t n_vlong_rows;
  srb_hub_split hub;
} srb_graph_csr;

typedef struct srb_step_desc {
  int32_t model;
  int32_t n_users, n_items, d, n_layers;
  int32_t batch_cap;       /* B: capacity of the batch buffer sections */
  int32_t layer_cl;        /* XSimGCL l_star */
  float eps, tau, cl_rate; /* noise magnitude, temperature, lambda */
  float reg;
  double lr, beta1, beta2;
  float adam_eps;
  float l2_div;            /* configured batch.size where the model divides by it, else 1 */
  int32_t noise_mode;      /* 1 tensor, 2 philox */
  const float* noise;      /* mode 1: [views, n_layers, n, d] */
  uint64_t philox_seed;
  srb_graph_csr adj;       /* clean normalised adjacency */
  srb_graph_csr adj_view[2]; /* SGL: the two dropped graphs */
  const int32_t* batch;    /* device batch buffer (see srb_batch_layout) */
  float* params;           /* [n, d] E0 (updated in place) */
  float* adam_m;
  float* adam_v;
  int32_t* step_dev;       /* device step counter */
  float* scalars;          /* [16] device scratch for adam scalars + loss accumulators */
  float* losses;           /* [4] device: rec (bpr), l2, cl (weighted), total */
  void* workspace;
  int64_t workspace_bytes; /* >= srb_step_workspace_bytes */
  /* optional (all three or none): a cudaStream_t and two cudaEvent_t (timing disabled) owned by the caller, used to run
   * BPR + L2 beside InfoNCE.  Without them one set per device is shared by every step on that device, which is only
   * safe while steps on that device are enqueued one after the other. */
  void* fork_stream;
  void* fork_event;
  void* join_event;
} srb_step_desc;

/* n_hub_work: adj.hub.n_work of the clean graph (chunks of its split rows; 0 when it has none) */
int64_t srb_step_workspace_bytes(int32_t model, int32_t n, int32_t d, int32_t batch_cap, int32_t n_hub_work);
int srb_train_step(const srb_step_desc* desc, void* stream);

/* batch buffer layout (int32 words): [0]=b [1]=n_uniq_u [2]=n_uniq_i [3]=reserved
 * then 5 sections of batch_cap words: u_idx, i_idx, j_idx, uniq_u, uniq_i. */
#define SRB_BATCH_HEADER 4
static inline int64_t srb_batch_words(int32_t batch_cap) { return SRB_BATCH_HEADER + 5ll * batch_cap; }

/* ---------------------------------------------------------------------------------------
 * (R1) Pairwise sampler, host side, bit-exact with CPython's `random` stream.
 * Replaces next_batch_pairwise util/sampler.py:5-28 : random.shuffle (in place, persists
 * across epochs) + per positive `choice(item_list)` re-drawn while (u, j) in train.
 * The MT19937 state is imported from / exported to random.getstate() (625 words:
 * 624 state + index) so the Python-visible stream stays identical to the reference's.
 * ------------------------------------------------------------------------------------- */
typedef struct srb_sampler srb_sampler;

/* users/items: the training pairs (internal ids) in training_data order; copied. */
srb_sampler* srb_sampler_create(const int32_t* users, const int32_t* items, int64_t n_pairs,
                                int32_t n_users, int32_t n_items);
void srb_sampler_destroy(srb_sampler* s);
int srb_sampler_set_state(srb_sampler* s, const uint32_t* mt625);
int srb_sampler_get_state(const srb_sampler* s, uint32_t* mt625);
/* Start an epoch: shuffles the pair order exactly like random.shuffle(training_data).
 * perm_out (optional, n_pairs int64): new_order[k] = index into the PREVIOUS order. */
int srb_sampler_begin_epoch(srb_sampler* s, int64_t* perm_out);
/* Next batch into `out` (srb_batch_words(batch_cap) int32 words, host).  Returns the
 * batch size b (0 when the epoch is exhausted), negative on error.  n_negs == 1. */
int srb_sampler_next_batch(srb_sampler* s, int32_t batch_size, int32_t batch_cap, int32_t* out);
/* General form: n_negs >= 1, separate arrays u[b], i[b], j[b * n_negs] (sampler.py:23-27). */
int srb_sampler_next_batch_negs(srb_sampler* s, int32_t batch_size, int32_t n_negs, int32_t* u,
                                int32_t* i, int32_t* j);
/* Whole-epoch variant: fills out[n_batches * srb_batch_words(batch_cap)]; returns n_batches. */
int64_t srb_sampler_epoch(srb_sampler* s, int32_t batch_size, int32_t batch_cap, int32_t* out,
                          int64_t out_words);
int64_t srb_sampler_pairs(const srb_sampler* s);
/* Sample-ahead ring: after srb_sampler_begin_epoch, one native thread fills up to `depth` batches ahead of the
 * consumer (same layout and -- the producer being the only reader of the MT19937 state -- the same batches as
 * srb_sampler_next_batch would return).  srb_sampler_ring_pop blocks for the next batch and returns its size, 0 at
 * the end of the epoch.  srb_sampler_ring_stop joins the producer and puts the generator back to the state after the
 * last batch the caller popped (batches sampled ahead but never read are un-drawn), so srb_sampler_get_state returns
 * the reference's stream position whenever the ring is stopped. */
int srb_sampler_ring_start(srb_sampler* s, int32_t batch_size, int32_t batch_cap, int32_t depth);
int srb_sampler_ring_pop(srb_sampler* s, int32_t* out);
int srb_sampler_ring_stop(srb_sampler* s);
/* Position, for checkpoints (refused while a ring runs: stop it first, which un-draws what was not popped).
 * get/set_order: the current pair order (n_pairs users and items); set_order range-checks and copies.
 * srb_sampler_cursor: *cursor = the pairs already consumed in the open epoch, -1 when no epoch is open.
 * srb_sampler_seek: reopen an epoch at `cursor` (0..n_pairs) without shuffling, or close it (-1); with the order and
 * the MT19937 state restored, the next batches -- sequential calls or a ring started now -- are the ones the
 * uninterrupted epoch would have drawn. */
int srb_sampler_get_order(const srb_sampler* s, int32_t* users, int32_t* items);
int srb_sampler_set_order(srb_sampler* s, const int32_t* users, const int32_t* items, int64_t n_pairs);
int srb_sampler_cursor(const srb_sampler* s, int64_t* cursor);
int srb_sampler_seek(srb_sampler* s, int64_t cursor);

/* ---------------------------------------------------------------------------------------
 * Bipartite-sharded training step (SURVEY 8e; selfrec_b200/csrc/sharded.cu).  One process per GPU.
 * Rank g owns the users u with u % world == g, stored as local row u / world (n_local_users = ceil((n_users - g) / world))
 * -- their rows of every [U, d] table stay on that GPU -- and the item tables are replicated; per propagation layer only the item half is exchanged: each rank's partial
 * product R_g^T X_u is stored by the SpMM epilogue into the staging area of the rank that owns the item slice
 * (P2P stores, reduce-scatter), the owner adds the partials in rank order, applies the epilogue and stores the
 * finished rows into every rank's copy (all-gather; one multicast store per row when sym_mc is given).  With sym_mc the
 * reduce-scatter goes through the NVSwitch instead (NVLS): partial products stay in the rank's own copy of the
 * staging buffer and the owner reads their sum with multimem.ld_reduce -- one reduced row of ingress instead of
 * world - 1 partial rows.  Item slice of rank g: [g * I / world, (g+1) * I / world).
 *   Ru  CSR [n_local_users x n_items]: rows = this rank's users (local rows), columns = item ids
 *   Rt  CSR [n_items x n_local_users]: its transpose (columns = local user ids); values = the rank's block of the
 *       normalised adjacency (data/graph.py:10-24)
 *   sym[q]   base of rank q's symmetric region (torch.distributed._symmetric_memory), sym_bytes each, zero-filled
 *            once before the first step; item parameters live at srb_shard_layout.item_params inside it
 *   workspace local, zero-filled once before the first step (it holds the barrier epoch)
 * Models: LightGCN, SimGCL, XSimGCL, SGL (same arithmetic as srb_train_step; noise from the in-kernel Philox stream,
 * keyed by GLOBAL row id, so a sharded run draws the noise the single-GPU engine draws).  SGL also propagates over the
 * epoch's two view graphs, given as this rank's blocks of each (Ru_view / Rt_view, same layout as Ru / Rt; their split-row
 * chunk counts must not exceed those of Ru / Rt, which size the plan).  world == 1 is valid.
 * ------------------------------------------------------------------------------------- */
typedef struct srb_shard_desc {
  int32_t model;
  int32_t world, rank;
  int32_t n_users, n_items, d, n_layers, batch_cap, layer_cl;
  float eps, tau, cl_rate, reg;
  double lr, beta1, beta2;
  float adam_eps;
  float l2_div;
  int32_t noise_mode; /* 0 (LightGCN) or 2 */
  uint64_t philox_seed;
  srb_graph_csr Ru;
  srb_graph_csr Rt;
  const int32_t* batch; /* device batch buffer, identical on every rank */
  float* pu;            /* [n_local_users, d] parameters of the owned users */
  float* mu;
  float* vu;
  float* mi;            /* [n_items, d] Adam moments of the items (only the owned slice is used) */
  float* vi;
  int32_t* step_dev;
  float* scalars;
  float* losses;        /* [4] rec, l2, cl, total (replicated) */
  void* sym[8];
  void* sym_mc;         /* multicast mapping of the symmetric region, or NULL */
  int64_t sym_bytes;
  void* workspace;
  int64_t workspace_bytes;
  /* optional (all three or none): a cudaStream_t and two cudaEvent_t (timing disabled) of the caller.  With them the
   * owner-side reduction of a layer (NVLink-bound) runs on fork_stream beside the user-side product (local compute). */
  void* fork_stream;
  void* fork_event;
  void* join_event;
  int32_t nvls; /* != 0 (needs sym_mc): reduce-scatter through the NVSwitch (multimem.ld_reduce) instead of P2P partial pushes */
  srb_graph_csr Ru_view[2]; /* SGL: this rank's blocks of the epoch's two dropped, re-normalised graphs (else unused) */
  srb_graph_csr Rt_view[2];
} srb_shard_desc;

typedef struct srb_shard_layout {
  int64_t sym_bytes;       /* size of the symmetric region */
  int64_t workspace_bytes; /* size of the local workspace */
  int64_t item_params;     /* byte offset of the [n_items, d] item parameters inside the symmetric region */
  int64_t item_final;      /* byte offset of the [n_items, d] item output of srb_shard_forward */
  int64_t ctrl;            /* byte offset inside the workspace of int32 {barrier epoch, peer-timeout flag} */
} srb_shard_layout;

/* model: SRB_MODEL_* of the step (SGL needs more workspace: a third seed table per side, the batch-row lists of its views
 * and a larger InfoNCE workspace; the other three share one layout).
 * hub_chunks_u / hub_chunks_t: Ru.hub.n_work / Rt.hub.n_work of the rank's blocks (capacity of the per-batch split-row
 * lists of the last forward layer, which is evaluated on the batch rows only) */
int srb_shard_plan(int32_t model, int32_t n_users, int32_t n_items, int32_t n_local_users, int32_t d, int32_t batch_cap,
                   int32_t world, int32_t hub_chunks_u, int32_t hub_chunks_t, srb_shard_layout* out);
int srb_shard_step(const srb_shard_desc* desc, void* stream);
/* clean forward (evaluation / save(), XSimGCL.py:40-41,53-55): out_user [n_local_users, d]; the complete item half
 * lands in every rank's symmetric region at item_final */
int srb_shard_forward(const srb_shard_desc* desc, float* out_user, void* stream);

/* ---- neighbourhood baselines: ItemKNN / UserKNN (model/graph/ItemKNN.py, model/graph/UserKNN.py) ---------------- */
#define SRB_KNN_MAX_TOPK 1024

/* Rows of a binary CSR A (ItemKNN: items -> users; UserKNN: users -> items) compared with each other through the
 * transpose T.  rank[r]: position of row r's name in Python's sorted() of the row names, the second key of
 * heapq.nlargest over (sim, name) tuples (ItemKNN.py:51, UserKNN.py:53).  Device pointers, int32. */
typedef struct srb_knn_rows {
  const int32_t* row_ptr; /* [n_rows + 1] */
  const int32_t* row_idx;
  const int32_t* t_ptr;   /* [n_cols + 1] */
  const int32_t* t_idx;
  const int32_t* rank;    /* [n_rows] */
  int32_t n_rows;
} srb_knn_rows;

int64_t srb_knn_neighbors_workspace_bytes(int32_t n_rows);
/* ItemKNN.py:14-56 / UserKNN.py:14-57, train(): for every row a, c(a, b) = |A[a] ∩ A[b]| over b != a, and
 *   sim = (c / (c + shrinkage)) * (c / (sqrt(|A[a]|) * sqrt(|A[b]|) + 1e-8)),
 * each operation one correctly rounded float64 step in that order.  Candidates are the b with c >= 1; the row keeps
 * the topk best by (sim desc, rank desc).  out_id / out_sim: [n_rows, topk], entries past out_cnt[a] are -1 / 0.
 * topk in 1..SRB_KNN_MAX_TOPK, shrinkage in 0..2^52; workspace: srb_knn_neighbors_workspace_bytes (a count and a
 * candidate list of n_rows int32 per CTA, no n_rows^2 buffer). */
int srb_knn_neighbors(const srb_knn_rows* rows, int32_t topk, int64_t shrinkage, int32_t* out_id, double* out_sim,
                      int32_t* out_cnt, void* workspace, int64_t workspace_bytes, void* stream);
/* ItemKNN.py:58-81 (mode 0) / UserKNN.py:59-80 (mode 1), predict(u) for the listed user ids: out[q] = float64
 * [n_items] row.  Mode 0: seq = each user's items in training_set_u order, the neighbour table is the items'; the
 * sims of item i's neighbours are added for every i in seq[u], in that order.  Mode 1: seq = each user's items, the
 * table is the users'; for each neighbour v of u in list order its sim is added to every item of seq[v].  Then
 * out = acc / (acc + 1e-8).  With rated_ptr / rated_idx (both or neither) rated items become -10e8
 * (base/graph_recommender.py:49-50). */
int srb_knn_score_rows(int32_t mode, const int32_t* users, int32_t n_q, int32_t n_items, const int32_t* nbr_id,
                       const double* nbr_sim, const int32_t* nbr_cnt, int32_t topk, const int32_t* seq_ptr,
                       const int32_t* seq_idx, const int32_t* rated_ptr, const int32_t* rated_idx, double* out,
                       void* stream);
int64_t srb_topk_f64_workspace_bytes(int32_t n_q, int32_t k);
/* find_k_largest(k, row) of util/algorithm.py:144-156 on float64 rows [n_q, n_items], k in 1..n_items: heapify of the
 * first k (score, id) tuples, heapreplace iff score > heap[0] score, then numba's quicksort argsort by score,
 * descending.  Ties come out in the reference's order, which depends on the heap's array layout. */
int srb_topk_rows_f64(const double* rows, int32_t n_q, int32_t n_items, int32_t k, int32_t* out_ids, double* out_scores,
                      void* workspace, int64_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SELFREC_B200_H */
