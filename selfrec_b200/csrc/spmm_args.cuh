// Kernel-argument block of the SpMM family (spmm.cu), shared with the sharded step (sharded.cu).
#pragma once
#include "common.cuh"

namespace srb {

// Cross-GPU synchronisation folded into a kernel of the bipartite-sharded step (no separate barrier launch):
//   wait   -- at kernel start every CTA polls this rank's flag array until all ranks have sent signal number *epoch
//             (the peers' stores this kernel is about to read, or whose buffers it is about to overwrite, are done);
//   signal -- at kernel end the last CTA to finish bumps *epoch and stores it into every rank's flag array
//             (st.release.sys after a system fence: this kernel's peer stores are visible before the flag).
// Every rank runs the same kernel sequence, so signal numbers agree; a peer that never arrives trips *err after ~30 s.
struct PeerSync {
  int* flags[8];  // every rank's flags [8]; flags[rank] is local
  int* epoch;     // local: signals sent so far
  int* counter;   // local: CTAs of the signalling kernel that are done
  int* err;
  int world, rank;
  int wait, signal;
};

__device__ __forceinline__ void st_release_sys(int* p, int v) { asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ int ld_acquire_sys(const int* p) {
  int v;
  asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ int ld_relaxed_sys(const int* p) {
  int v;
  asm volatile("ld.relaxed.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ void peer_wait(const PeerSync& s) {
  if (!s.wait) return;
  if ((int)threadIdx.x < s.world) {
    const int target = *reinterpret_cast<volatile int*>(s.epoch);
    const int* f = s.flags[s.rank] + threadIdx.x;
    const long long t0 = clock64();
    while (ld_relaxed_sys(f) < target) {  // relaxed polls; one acquire fence once the flag is there
      if (clock64() - t0 > 60000000000ll) {  // ~30 s: a peer died; do not hang the GPU
        *s.err = 1;
        break;
      }
      __nanosleep(20);
    }
    (void)ld_acquire_sys(f);  // relaxed polls, then one acquiring read of the flag that is there
  }
  __syncthreads();
}

__device__ __forceinline__ void peer_signal(const PeerSync& s) {
  if (!s.signal) return;
  __syncthreads();  // every store of this CTA has been issued (and is observed by thread 0: its fence is cumulative)
  if (threadIdx.x == 0) {
    __threadfence();  // device scope is enough here: the ONE system-scope fence is the last CTA's, after the counter
    if (atomicAdd(s.counter, 1) == (int)gridDim.x - 1) {  // last CTA of the grid
      *s.counter = 0;
      __threadfence_system();
      const int e = *s.epoch + 1;
      *s.epoch = e;
      for (int q = 0; q < s.world; ++q) st_release_sys(s.flags[q] + s.rank, e);
    }
  }
}

struct SpmmArgs {
  const int32_t* rowptr;
  const int32_t* colidx;
  const float* vals;
  const int32_t* row_order;
  int32_t n_rows;
  const int32_t* n_vlong_dev;  // optional device-side class split (see srb_spmm_desc)
  const uint32_t* col_mask;    // optional: clear bit = X row is zero
  int32_t n_huge;  // leading entries of row_order that are split into SRB_HUB_CHUNK-sized chunks (spmm_hub_kernel)
  int32_t n_vlong; // following entries that get a whole CTA
  int32_t n_long;  // following entries that get a whole warp
  const int32_t* hub_first;  // [n_huge] first chunk slot of each split row
  const int32_t* hub_work;   // [n_work][2] (row, chunk index)
  int32_t n_work;
  float* hub_part;           // [n_work, D] partial sums of the chunks
  // column-blocked static lists (srb_hub_split.seg): segment w = CSR positions [seg[2w], seg[2w+1])
  const int32_t* seg;
  const int32_t* seg_cnt;
  const int32_t* order_cta;
  const int32_t* order_warp;
  int32_t n_cta;
  int32_t n_warp;
  const float* X;
  float* Y;
  const float* extra;
  float extra_scale;
  // optional backward seed table (engine.cu, run_chain): y += seed[row] where seed_mask has the row's bit; the
  // table holds nothing elsewhere
  const uint32_t* seed_mask;
  const float* seed;
  int32_t noise_mode;
  const float* noise;
  float eps;
  uint2 pkey;
  uint2 poff;
  const int32_t* pstep;
  const float* sum_in;
  const float* sum_add[3];  // optional: earlier layer outputs, added onto sum_in in this order before the row's own value
  float* sum_out;
  float sum_scale;
  float* ap;
  float* am;
  float* av;
  const float* ascal;
  float b2, w1, w2, aeps;  // beta2, 1 - beta1, 1 - beta2 (rounded from double like torch's Python floats)
  int32_t world;
  float* peer[8];      // layer output -> every rank's buffer
  float* peer_sum[8];  // running sum  -> every rank's buffer
  float* peer_p[8];    // updated parameters (Adam epilogue) -> every rank's copy
  int32_t stream;          // tables larger than L2: CSR arrays and outputs are touched once per product -> evict-first accesses
  int32_t peer_mc;         // the one peer address is an NVSwitch multicast mapping: stores go out as multimem.st
  int32_t noise_row_base;  // Philox row id = noise_row_base + row * noise_row_stride: the GLOBAL id of a row of a
  int32_t noise_row_stride;  // sharded table (cyclic user blocks: base = rank, stride = world)
  // partial-sum push (bipartite sharding, item-side product): row r of this rank's partial product goes to the
  // staging area of the rank that owns item r: stage_peer[o] + ((size_t)stage_rank * stage_cap + r - stage_bounds[o]) * D
  float* stage_peer[8];
  int32_t stage_bounds[9];
  int32_t stage_rank;
  int32_t stage_cap;
  PeerSync ps;
};

// rows of an item slice summed over the ranks' staged partial products (fixed rank order), then the common epilogue
struct ReduceArgs {
  const float* stage;  // this rank's staging area: [world][stage_cap, D]
  int32_t world;
  int32_t stage_cap;
  int32_t slice_begin;  // item id of slice row 0 (epilogue tensors are indexed by item id)
  int32_t n_slice;
  const uint32_t* mask; // optional bitmap over item ids: only the rows whose bit is set are reduced (batch rows of the last layer)
  // NVLS route: every rank left its partial product in ITS OWN copy of a multicast-mapped [n_items, D] buffer; mc_part is
  // the multicast address of that buffer, and one multimem.ld_reduce per 16 bytes returns the sum over all ranks, added
  // inside the NVSwitch -- the owner receives one reduced row instead of world - 1 partial rows
  const float* mc_part;
  int32_t small_grid;   // the kernel runs beside the user-side SpMM and is NVLink-bound: a CTA or two per SM
};

int launch_spmm(const SpmmArgs& a, int d, cudaStream_t st);
int launch_reduce_rows(const SpmmArgs& a, const ReduceArgs& r, int d, cudaStream_t st);
int launch_rows_epilogue(const SpmmArgs& a, int d, cudaStream_t st);  // Y[r] = epilogue(X[r]), r < n_rows
int fill_args(const srb_spmm_desc* d, SpmmArgs& a);
// the product Y = g X (g: n_rows x n_cols) with a neutral epilogue (scales 1; no output, noise, sum or Adam yet)
int graph_args(const srb_graph_csr& g, int n_rows, int n_cols, int d, const float* X, SpmmArgs& a);

// Philox offset of the noise that layer `layer` (0-based) of view `view` adds: both training steps draw the same stream
inline uint64_t noise_offset(int view, int layer) { return ((uint64_t)view << 32) | (uint64_t)(0x10 + layer); }

// Appends one batch row of degree deg to a device-classified row list of the last forward layer (the format of
// srb_spmm_desc.n_vlong_dev): rows holds four segments of capacity cap -- split rows (only with hub_first; their
// chunks go to hub_work), a CTA per row of >= 128 non-zeros, a warp per other row; the lane-group class stays empty.
// A batch has only a few thousand rows, so parallelism is scarce and no row shares a warp.  counters[c] counts class c,
// counters[4] the chunks.  Slots are allocated per warp among the threads with the same class + key_off, so lists
// filled by one warp take different key offsets.
__device__ __forceinline__ void list_batch_row(int row, int deg, int key_off, int32_t* rows, int cap, int32_t* counters,
                                               int32_t* hub_first, int32_t* hub_work, int hub_cap) {
  const int cls = (hub_first && deg >= SRB_HUB_MIN_NNZ) ? 0 : (deg >= 128 ? 1 : 2);
  const unsigned mine = __match_any_sync(__activemask(), cls + key_off);
  const int lane = threadIdx.x & 31;
  const int leader = __ffs(mine) - 1;
  int base = 0;
  if (lane == leader) base = atomicAdd(counters + cls, __popc(mine));
  base = __shfl_sync(mine, base, leader);
  const int slot = base + __popc(mine & ((1u << lane) - 1));
  rows[cls * cap + slot] = row;
  if (cls == 0) {
    const int nch = (deg + SRB_HUB_CHUNK - 1) / SRB_HUB_CHUNK;
    const int first = atomicAdd(counters + 4, nch);
    hub_first[slot] = first;
    for (int c = 0; c < nch && first + c < hub_cap; ++c) {
      hub_work[2 * (first + c)] = row;
      hub_work[2 * (first + c) + 1] = c;
    }
  }
}



}  // namespace srb
