// (R1) Pairwise BPR sampler, host side, bit-exact with CPython's `random` module.
//
// Replaces next_batch_pairwise util/sampler.py:5-28:
//   shuffle(training_data)                       :7   in place, persists across epochs
//   batches [ptr, min(ptr + batch_size, n))      :10-17
//   neg_item = choice(item_list) re-drawn while neg_item in training_set_u[user]   :24-27
// item_list is list(data.item.keys()) and item ids are assigned in insertion order
// (data/ui_graph.py:35-38), so item_list[r] has id r and choice() reduces to
// _randbelow(item_num).  RNG: MT19937 exactly as CPython 3.12 uses it
// (Lib/random.py: shuffle, choice, _randbelow_with_getrandbits; Modules/_randommodule.c:
// genrand_uint32, getrandbits(k) = genrand_uint32() >> (32 - k) for k <= 32).
// Also emits torch.unique(user_idx) / torch.unique(pos_idx) (XSimGCL.py:46-47): sorted
// unique ids, computed here because the batch is on the host anyway.
#include <stdint.h>
#include <string.h>
#include <algorithm>
#include <condition_variable>
#include <mutex>
#include <new>
#include <thread>
#include <vector>
#include "selfrec_b200.h"

namespace srb {
void set_error(const char* fmt, ...);
}

struct srb_sampler {
  uint32_t mt[624];
  int mti;
  std::vector<int32_t> pu, pi;  // training pairs in their current (shuffled) order
  std::vector<int64_t> rated_ptr;
  std::vector<int32_t> rated_idx;  // per user sorted unique item ids
  int32_t n_users, n_items;
  int64_t ptr;
  bool epoch_open;
  std::vector<uint64_t> ubits, ibits;  // scratch bitmaps of sorted_unique

  // sample-ahead ring (srb_sampler_ring_*): one native producer thread fills `ring_depth` batch buffers ahead of the
  // consumer.  The producer is the only reader of the MT19937 state while it runs, so the stream of draws -- hence
  // every batch -- is what the sequential calls would produce.
  std::thread ring_thread;
  std::mutex ring_mu;
  std::condition_variable ring_cv;
  std::vector<int32_t> ring_buf;   // [depth][words]
  std::vector<int32_t> ring_b;     // batch size of each slot (0 = end of epoch, < 0 = error code)
  int64_t ring_words = 0;
  int ring_depth = 0;
  int64_t ring_head = 0, ring_tail = 0;  // produced / consumed counts
  bool ring_stop = false, ring_running = false;
  int32_t ring_bs = 0, ring_cap = 0;
  // generator state after each produced batch (625 words + ptr), and after the last CONSUMED one: a ring that is
  // stopped early puts the sampler back there, so the caller sees the stream exactly where it stopped reading
  struct Snap {
    uint32_t mt[624];
    int mti;
    int64_t ptr;
    bool open;
  };
  std::vector<Snap> ring_snap;
  Snap ring_consumed;
  void snap(Snap& d) const {
    memcpy(d.mt, mt, sizeof mt);
    d.mti = mti;
    d.ptr = ptr;
    d.open = epoch_open;
  }

  inline uint32_t genrand() {
    static const uint32_t mag01[2] = {0x0u, 0x9908b0dfu};
    if (mti >= 624) {
      int kk;
      uint32_t y;
      for (kk = 0; kk < 624 - 397; kk++) {
        y = (mt[kk] & 0x80000000u) | (mt[kk + 1] & 0x7fffffffu);
        mt[kk] = mt[kk + 397] ^ (y >> 1) ^ mag01[y & 1u];
      }
      for (; kk < 623; kk++) {
        y = (mt[kk] & 0x80000000u) | (mt[kk + 1] & 0x7fffffffu);
        mt[kk] = mt[kk + (397 - 624)] ^ (y >> 1) ^ mag01[y & 1u];
      }
      y = (mt[623] & 0x80000000u) | (mt[0] & 0x7fffffffu);
      mt[623] = mt[396] ^ (y >> 1) ^ mag01[y & 1u];
      mti = 0;
    }
    uint32_t y = mt[mti++];
    y ^= (y >> 11);
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= (y >> 18);
    return y;
  }

  // Random._randbelow_with_getrandbits(n), n >= 1 and n < 2^32
  inline uint32_t randbelow(uint32_t n) {
    const int k = 32 - __builtin_clz(n);  // n.bit_length()
    uint32_t r = genrand() >> (32 - k);
    while (r >= n) r = genrand() >> (32 - k);
    return r;
  }

  inline bool rated(int32_t u, int32_t item) const {
    const int32_t* b = rated_idx.data() + rated_ptr[u];
    const int32_t* e = rated_idx.data() + rated_ptr[u + 1];
    return std::binary_search(b, e, item);
  }
};

extern "C" srb_sampler* srb_sampler_create(const int32_t* users, const int32_t* items, int64_t n_pairs, int32_t n_users,
                                           int32_t n_items) {
  if (!users || !items || n_pairs < 0 || n_users <= 0 || n_items <= 0) {
    srb::set_error("sampler_create: bad arguments");
    return nullptr;
  }
  srb_sampler* s = new (std::nothrow) srb_sampler();
  if (!s) {
    srb::set_error("sampler_create: out of memory");
    return nullptr;
  }
  s->n_users = n_users;
  s->n_items = n_items;
  s->pu.assign(users, users + n_pairs);
  s->pi.assign(items, items + n_pairs);
  for (int64_t t = 0; t < n_pairs; ++t) {
    if (users[t] < 0 || users[t] >= n_users || items[t] < 0 || items[t] >= n_items) {
      srb::set_error("sampler_create: pair %lld out of range", (long long)t);
      delete s;
      return nullptr;
    }
  }
  // training_set_u as CSR (duplicates collapse, like the dict of dicts ui_graph.py:39)
  std::vector<int64_t> cnt(n_users + 1, 0);
  for (int64_t t = 0; t < n_pairs; ++t) cnt[users[t] + 1]++;
  for (int32_t u = 0; u < n_users; ++u) cnt[u + 1] += cnt[u];
  std::vector<int32_t> tmp(n_pairs);
  {
    std::vector<int64_t> fill(cnt.begin(), cnt.end() - 1);
    for (int64_t t = 0; t < n_pairs; ++t) tmp[fill[users[t]]++] = items[t];
  }
  s->rated_ptr.assign(n_users + 1, 0);
  s->rated_idx.reserve(n_pairs);
  for (int32_t u = 0; u < n_users; ++u) {
    int32_t* b = tmp.data() + cnt[u];
    int32_t* e = tmp.data() + cnt[u + 1];
    std::sort(b, e);
    e = std::unique(b, e);
    s->rated_idx.insert(s->rated_idx.end(), b, e);
    s->rated_ptr[u + 1] = (int64_t)s->rated_idx.size();
  }
  // default state = init_genrand(19650218) is irrelevant: callers import random.getstate()
  memset(s->mt, 0, sizeof s->mt);
  s->mt[0] = 0x80000000u;
  s->mti = 624;
  s->ptr = 0;
  s->epoch_open = false;
  return s;
}

extern "C" int srb_sampler_ring_stop(srb_sampler* s);

extern "C" void srb_sampler_destroy(srb_sampler* s) {
  if (s) srb_sampler_ring_stop(s);
  delete s;
}

extern "C" int srb_sampler_set_state(srb_sampler* s, const uint32_t* mt625) {
  if (!s || !mt625) {
    srb::set_error("sampler_set_state: null");
    return SRB_ERR_ARG;
  }
  if (mt625[624] > 624) {
    srb::set_error("sampler_set_state: invalid index %u", mt625[624]);
    return SRB_ERR_ARG;
  }
  memcpy(s->mt, mt625, 624 * sizeof(uint32_t));
  s->mti = (int)mt625[624];
  return SRB_OK;
}

extern "C" int srb_sampler_get_state(const srb_sampler* s, uint32_t* mt625) {
  if (!s || !mt625) {
    srb::set_error("sampler_get_state: null");
    return SRB_ERR_ARG;
  }
  memcpy(mt625, s->mt, 624 * sizeof(uint32_t));
  mt625[624] = (uint32_t)s->mti;
  return SRB_OK;
}

extern "C" int64_t srb_sampler_pairs(const srb_sampler* s) { return s ? (int64_t)s->pu.size() : -1; }

// ---- position: the pair order and the epoch cursor (checkpoints) --------------------------------------------------
extern "C" int srb_sampler_get_order(const srb_sampler* s, int32_t* users, int32_t* items) {
  if (!s || !users || !items) {
    srb::set_error("sampler_get_order: null");
    return SRB_ERR_ARG;
  }
  if (s->ring_running) {
    srb::set_error("sampler_get_order: a ring is running");
    return SRB_ERR_STATE;
  }
  memcpy(users, s->pu.data(), s->pu.size() * sizeof(int32_t));
  memcpy(items, s->pi.data(), s->pi.size() * sizeof(int32_t));
  return SRB_OK;
}

extern "C" int srb_sampler_set_order(srb_sampler* s, const int32_t* users, const int32_t* items, int64_t n_pairs) {
  if (!s || !users || !items) {
    srb::set_error("sampler_set_order: null");
    return SRB_ERR_ARG;
  }
  if (s->ring_running) {
    srb::set_error("sampler_set_order: a ring is running");
    return SRB_ERR_STATE;
  }
  if (n_pairs != (int64_t)s->pu.size()) {
    srb::set_error("sampler_set_order: %lld pairs, the sampler has %lld", (long long)n_pairs, (long long)s->pu.size());
    return SRB_ERR_ARG;
  }
  for (int64_t t = 0; t < n_pairs; ++t) {
    if (users[t] < 0 || users[t] >= s->n_users || items[t] < 0 || items[t] >= s->n_items) {
      srb::set_error("sampler_set_order: pair %lld out of range", (long long)t);
      return SRB_ERR_ARG;
    }
  }
  memcpy(s->pu.data(), users, (size_t)n_pairs * sizeof(int32_t));
  memcpy(s->pi.data(), items, (size_t)n_pairs * sizeof(int32_t));
  return SRB_OK;
}

extern "C" int srb_sampler_cursor(const srb_sampler* s, int64_t* cursor) {
  if (!s || !cursor) {
    srb::set_error("sampler_cursor: null");
    return SRB_ERR_ARG;
  }
  if (s->ring_running) {
    srb::set_error("sampler_cursor: a ring is running");
    return SRB_ERR_STATE;
  }
  *cursor = s->epoch_open ? s->ptr : -1;
  return SRB_OK;
}

extern "C" int srb_sampler_seek(srb_sampler* s, int64_t cursor) {
  if (!s) {
    srb::set_error("sampler_seek: null");
    return SRB_ERR_ARG;
  }
  if (s->ring_running) {
    srb::set_error("sampler_seek: a ring is running");
    return SRB_ERR_STATE;
  }
  if (cursor < -1 || cursor > (int64_t)s->pu.size()) {
    srb::set_error("sampler_seek: cursor %lld outside -1..%lld", (long long)cursor, (long long)s->pu.size());
    return SRB_ERR_ARG;
  }
  s->epoch_open = cursor >= 0;
  s->ptr = cursor >= 0 ? cursor : 0;
  return SRB_OK;
}

extern "C" int srb_sampler_begin_epoch(srb_sampler* s, int64_t* perm_out) {
  if (!s) {
    srb::set_error("sampler_begin_epoch: null");
    return SRB_ERR_ARG;
  }
  const int64_t n = (int64_t)s->pu.size();
  if (n >= (1ll << 32)) {
    srb::set_error("sampler_begin_epoch: more than 2^32 pairs");
    return SRB_ERR_ARG;
  }
  if (perm_out)
    for (int64_t k = 0; k < n; ++k) perm_out[k] = k;
  // random.shuffle: for i in reversed(range(1, n)): j = randbelow(i + 1); swap
  for (int64_t i = n - 1; i >= 1; --i) {
    const int64_t j = (int64_t)s->randbelow((uint32_t)(i + 1));
    std::swap(s->pu[i], s->pu[j]);
    std::swap(s->pi[i], s->pi[j]);
    if (perm_out) std::swap(perm_out[i], perm_out[j]);
  }
  s->ptr = 0;
  s->epoch_open = true;
  return SRB_OK;
}

// sorted unique ids of src (torch.unique, XSimGCL.py:46-47).  Ids are < `universe`: one pass marks a bitmap,
// one pass over its words emits the ids in order -- no comparison sort on the per-batch path.
static int sorted_unique(const int32_t* src, int n, int32_t* dst, std::vector<uint64_t>& bits, int32_t universe) {
  const size_t words = ((size_t)universe + 63) / 64;
  if (bits.size() < words) bits.assign(words, 0);
  if ((size_t)n * 16 < words) {  // tiny batch over a huge id space: sorting is cheaper than scanning the bitmap
    memcpy(dst, src, (size_t)n * sizeof(int32_t));
    std::sort(dst, dst + n);
    return (int)(std::unique(dst, dst + n) - dst);
  }
  for (int t = 0; t < n; ++t) bits[(size_t)src[t] >> 6] |= (uint64_t)1 << (src[t] & 63);
  int m = 0;
  for (size_t w = 0; w < words; ++w) {
    uint64_t b = bits[w];
    if (!b) continue;
    bits[w] = 0;  // leave the bitmap clean for the next call
    while (b) {
      dst[m++] = (int32_t)(w * 64 + (size_t)__builtin_ctzll(b));
      b &= b - 1;
    }
  }
  return m;
}

extern "C" int srb_sampler_next_batch(srb_sampler* s, int32_t batch_size, int32_t batch_cap, int32_t* out) {
  if (!s || !out || batch_size <= 0 || batch_cap < batch_size) {
    srb::set_error("sampler_next_batch: bad arguments");
    return SRB_ERR_ARG;
  }
  if (!s->epoch_open) {
    srb::set_error("sampler_next_batch: begin_epoch was not called");
    return SRB_ERR_STATE;
  }
  const int64_t n = (int64_t)s->pu.size();
  if (s->ptr >= n) {
    s->epoch_open = false;
    return 0;
  }
  const int64_t end = (s->ptr + batch_size < n) ? s->ptr + batch_size : n;
  const int b = (int)(end - s->ptr);
  int32_t* u = out + SRB_BATCH_HEADER;
  int32_t* i = u + batch_cap;
  int32_t* j = i + batch_cap;
  int32_t* uu = j + batch_cap;
  int32_t* ui = uu + batch_cap;
  for (int t = 0; t < b; ++t) {
    // the rated list of a user is a random place in memory: fetch the ones a few positives ahead
    if (t + 16 < b) __builtin_prefetch(&s->rated_ptr[s->pu[s->ptr + t + 16]]);
    if (t + 8 < b) __builtin_prefetch(&s->rated_idx[(size_t)s->rated_ptr[s->pu[s->ptr + t + 8]]]);
    const int32_t user = s->pu[s->ptr + t];
    u[t] = user;
    i[t] = s->pi[s->ptr + t];
    if (s->rated_ptr[user + 1] - s->rated_ptr[user] >= s->n_items) {
      srb::set_error("sampler_next_batch: user %d has rated every item; no negative exists", user);
      return SRB_ERR_STATE;
    }
    int32_t neg = (int32_t)s->randbelow((uint32_t)s->n_items);
    while (s->rated(user, neg)) neg = (int32_t)s->randbelow((uint32_t)s->n_items);
    j[t] = neg;
  }
  for (int t = b; t < batch_cap; ++t) u[t] = i[t] = j[t] = 0;
  const int nu = sorted_unique(u, b, uu, s->ubits, s->n_users);
  const int ni = sorted_unique(i, b, ui, s->ibits, s->n_items);
  for (int t = nu; t < batch_cap; ++t) uu[t] = 0;
  for (int t = ni; t < batch_cap; ++t) ui[t] = 0;
  out[0] = b;
  out[1] = nu;
  out[2] = ni;
  out[3] = 0;
  s->ptr = end;
  return b;
}

// General form (n_negs >= 1, separate output arrays): j has b * n_negs entries, the n_negs
// negatives of positive t at j[t * n_negs ...] exactly like sampler.py:23-27.
extern "C" int srb_sampler_next_batch_negs(srb_sampler* s, int32_t batch_size, int32_t n_negs, int32_t* u, int32_t* i,
                                           int32_t* j) {
  if (!s || !u || !i || !j || batch_size <= 0 || n_negs < 1) {
    srb::set_error("sampler_next_batch_negs: bad arguments");
    return SRB_ERR_ARG;
  }
  if (!s->epoch_open) {
    srb::set_error("sampler_next_batch_negs: begin_epoch was not called");
    return SRB_ERR_STATE;
  }
  const int64_t n = (int64_t)s->pu.size();
  if (s->ptr >= n) {
    s->epoch_open = false;
    return 0;
  }
  const int64_t end = (s->ptr + batch_size < n) ? s->ptr + batch_size : n;
  const int b = (int)(end - s->ptr);
  for (int t = 0; t < b; ++t) {
    const int32_t user = s->pu[s->ptr + t];
    u[t] = user;
    i[t] = s->pi[s->ptr + t];
    if (s->rated_ptr[user + 1] - s->rated_ptr[user] >= s->n_items) {
      srb::set_error("sampler_next_batch_negs: user %d has rated every item; no negative exists", user);
      return SRB_ERR_STATE;
    }
    for (int m = 0; m < n_negs; ++m) {
      int32_t neg = (int32_t)s->randbelow((uint32_t)s->n_items);
      while (s->rated(user, neg)) neg = (int32_t)s->randbelow((uint32_t)s->n_items);
      j[(int64_t)t * n_negs + m] = neg;
    }
  }
  s->ptr = end;
  return b;
}

// ---- sample-ahead ring ---------------------------------------------------------------------------------------------
// The host sampler costs ~0.2 ms per batch on one core; a training step that is faster than that would wait for
// it.  One native thread samples ahead (no GIL, no per-batch Python hand-off), the consumer pops finished batches.
static void ring_producer(srb_sampler* s) {
  while (true) {
    int slot;
    {
      std::unique_lock<std::mutex> lk(s->ring_mu);
      s->ring_cv.wait(lk, [&] { return s->ring_stop || s->ring_head - s->ring_tail < s->ring_depth; });
      if (s->ring_stop) return;
      slot = (int)(s->ring_head % s->ring_depth);
    }
    const int b = srb_sampler_next_batch(s, s->ring_bs, s->ring_cap, s->ring_buf.data() + (size_t)slot * s->ring_words);
    s->snap(s->ring_snap[slot]);
    {
      std::lock_guard<std::mutex> lk(s->ring_mu);
      s->ring_b[slot] = b;
      ++s->ring_head;
    }
    s->ring_cv.notify_all();
    if (b <= 0) return;  // end of the epoch (or an error): the state is final
  }
}

extern "C" int srb_sampler_ring_start(srb_sampler* s, int32_t batch_size, int32_t batch_cap, int32_t depth) {
  if (!s || batch_size <= 0 || batch_cap < batch_size || depth < 1 || depth > 1024) {
    srb::set_error("sampler_ring_start: bad arguments");
    return SRB_ERR_ARG;
  }
  if (s->ring_running) {
    srb::set_error("sampler_ring_start: a ring is already running");
    return SRB_ERR_STATE;
  }
  if (!s->epoch_open) {
    srb::set_error("sampler_ring_start: begin_epoch was not called");
    return SRB_ERR_STATE;
  }
  s->ring_words = srb_batch_words(batch_cap);
  s->ring_depth = depth;
  s->ring_bs = batch_size;
  s->ring_cap = batch_cap;
  s->ring_buf.assign((size_t)depth * s->ring_words, 0);
  s->ring_b.assign(depth, 0);
  s->ring_snap.resize(depth);
  s->snap(s->ring_consumed);
  s->ring_head = s->ring_tail = 0;
  s->ring_stop = false;
  s->ring_running = true;
  s->ring_thread = std::thread(ring_producer, s);
  return SRB_OK;
}

extern "C" int srb_sampler_ring_pop(srb_sampler* s, int32_t* out) {
  if (!s || !out || !s->ring_running) {
    srb::set_error("sampler_ring_pop: no ring is running");
    return SRB_ERR_STATE;
  }
  int slot, b;
  {
    std::unique_lock<std::mutex> lk(s->ring_mu);
    s->ring_cv.wait(lk, [&] { return s->ring_head > s->ring_tail; });
    slot = (int)(s->ring_tail % s->ring_depth);
    b = s->ring_b[slot];
  }
  if (b > 0) memcpy(out, s->ring_buf.data() + (size_t)slot * s->ring_words, (size_t)s->ring_words * sizeof(int32_t));
  {
    std::lock_guard<std::mutex> lk(s->ring_mu);
    s->ring_consumed = s->ring_snap[slot];
    if (b > 0) ++s->ring_tail;  // the end marker stays: every later pop returns it again
  }
  s->ring_cv.notify_all();
  return b;
}

extern "C" int srb_sampler_ring_stop(srb_sampler* s) {
  if (!s) return SRB_ERR_ARG;
  if (!s->ring_running) return SRB_OK;
  {
    std::lock_guard<std::mutex> lk(s->ring_mu);
    s->ring_stop = true;
  }
  s->ring_cv.notify_all();
  if (s->ring_thread.joinable()) s->ring_thread.join();
  s->ring_running = false;
  // batches sampled ahead but never read are un-drawn: back to the state after the last batch the caller consumed
  memcpy(s->mt, s->ring_consumed.mt, sizeof s->mt);
  s->mti = s->ring_consumed.mti;
  s->ptr = s->ring_consumed.ptr;
  s->epoch_open = s->ring_consumed.open;
  return SRB_OK;
}

extern "C" int64_t srb_sampler_epoch(srb_sampler* s, int32_t batch_size, int32_t batch_cap, int32_t* out, int64_t out_words) {
  if (!s || !out) {
    srb::set_error("sampler_epoch: null");
    return SRB_ERR_ARG;
  }
  const int64_t words = srb_batch_words(batch_cap);
  int64_t nb = 0;
  while (true) {
    if ((nb + 1) * words > out_words) {
      const int64_t n = (int64_t)s->pu.size();
      if (s->ptr >= n) break;
      srb::set_error("sampler_epoch: output buffer too small");
      return SRB_ERR_ARG;
    }
    const int b = srb_sampler_next_batch(s, batch_size, batch_cap, out + nb * words);
    if (b < 0) return b;
    if (b == 0) break;
    ++nb;
  }
  s->epoch_open = false;
  return nb;
}


// random.sample(range(n), k) on an MT19937 state (data/augmentor.py:16-17,28: SGL's node / edge dropout draws
// its survivors this way every epoch; 1.1 M draws at yelp2018).  Both CPython strategies (Lib/random.py
// sample()): `use_pool` != 0 -> the pool-list variant (n <= setsize), else the selected-set variant with
// re-draws.  The caller decides which, with CPython's own float expression for setsize.  mt625 is updated.
extern "C" int srb_random_sample_range(uint32_t* mt625, int64_t n, int64_t k, int32_t use_pool, int64_t* out) {
  if (!mt625 || (k > 0 && !out)) {
    srb::set_error("random_sample_range: null pointer");
    return SRB_ERR_ARG;
  }
  if (k < 0 || k > n || n >= (int64_t)1 << 32) {
    srb::set_error("random_sample_range: need 0 <= k <= n < 2^32 (k=%lld n=%lld)", (long long)k, (long long)n);
    return SRB_ERR_ARG;
  }
  if (mt625[624] > 624) {
    srb::set_error("random_sample_range: bad MT index %u", mt625[624]);
    return SRB_ERR_ARG;
  }
  srb_sampler* g = new (std::nothrow) srb_sampler();
  if (!g) {
    srb::set_error("random_sample_range: out of memory");
    return SRB_ERR_ARG;
  }
  memcpy(g->mt, mt625, 624 * 4);
  g->mti = (int)mt625[624];
  if (use_pool) {
    std::vector<int64_t> pool((size_t)n);
    for (int64_t i = 0; i < n; ++i) pool[(size_t)i] = i;
    for (int64_t i = 0; i < k; ++i) {
      const int64_t j = (int64_t)g->randbelow((uint32_t)(n - i));
      out[i] = pool[(size_t)j];
      pool[(size_t)j] = pool[(size_t)(n - i - 1)];  // move a non-selected item into the vacancy
    }
  } else {
    std::vector<uint64_t> seen((size_t)((n + 63) / 64), 0);
    for (int64_t i = 0; i < k; ++i) {
      uint32_t j = g->randbelow((uint32_t)n);
      while (seen[j >> 6] >> (j & 63) & 1) j = g->randbelow((uint32_t)n);
      seen[j >> 6] |= (uint64_t)1 << (j & 63);
      out[i] = (int64_t)j;
    }
  }
  memcpy(mt625, g->mt, 624 * 4);
  mt625[624] = (uint32_t)g->mti;
  delete g;
  return SRB_OK;
}
