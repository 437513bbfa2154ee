"""Drop-in for util/sampler.py:5-28 (next_batch_pairwise) on the native sampler.

Bit-exact with the reference given the same `random` state: the MT19937 state is pulled
from random.getstate() before every native call and pushed back afterwards, so the global
stream advances exactly as with the Python implementation; data.training_data is permuted
in place like random.shuffle would.
"""
import ctypes as C
import random

import numpy as np

from .. import _lib
from ..data.data import _PendingShuffles


class NativePairSampler:
    """Owns a srb_sampler for one Interaction object."""

    def __init__(self, data, track_order=False):
        lib = _lib.load()
        pu = np.ascontiguousarray(data.pair_users if hasattr(data, "pair_users") else [data.user[p[0]] for p in data.training_data], dtype=np.int32)
        pi = np.ascontiguousarray(data.pair_items if hasattr(data, "pair_items") else [data.item[p[1]] for p in data.training_data], dtype=np.int32)
        self._lib = lib
        self.n_pairs = len(pu)
        self.handle = lib.srb_sampler_create(pu.ctypes.data_as(_lib.c_i32p), pi.ctypes.data_as(_lib.c_i32p), self.n_pairs,
                                             int(data.user_num), int(data.item_num))
        if not self.handle:
            raise _lib.SrbError("srb_sampler_create failed: " + _lib.last_error())
        self._state = (C.c_uint32 * 625)()
        # the pair order as positions in the training file (new_order[k] = file index) while tracked: every epoch's
        # permutation is composed into it (track_order; one n_pairs gather per epoch).  Nothing pending = the file
        # order; None = unknown (an epoch was shuffled untracked)
        self._tracking = bool(track_order)
        self._shuffles = _PendingShuffles(fold=2)
        self._ring = None     # (batch_size, batch_cap, depth) of the running ring
        self._resume = False  # restore() reopened an epoch: the next stream_epoch continues it

    def __del__(self):
        if getattr(self, "handle", None):
            self._lib.srb_sampler_destroy(self.handle)
            self.handle = None

    def pull_state(self):
        st = random.getstate()
        self._gauss = st[2]
        self._state[:] = st[1]
        _lib.check(self._lib.srb_sampler_set_state(self.handle, self._state), "srb_sampler_set_state")

    def push_state(self):
        _lib.check(self._lib.srb_sampler_get_state(self.handle, self._state), "srb_sampler_get_state")
        random.setstate((3, tuple(self._state), self._gauss))

    def begin_epoch(self, want_perm=True):
        perm = np.empty(self.n_pairs, dtype=np.int64) if want_perm else None
        ptr = perm.ctypes.data_as(_lib.c_i64p) if want_perm else None
        _lib.check(self._lib.srb_sampler_begin_epoch(self.handle, ptr), "srb_sampler_begin_epoch")
        if self._shuffles is not None:
            if want_perm and self._tracking:
                self._shuffles.add(perm)
            else:
                self._shuffles = None
        return perm

    def track_order(self):
        """Keep the pair order from here on (file_order()).  Only an order never shuffled untracked is known."""
        self._tracking = True

    # ---- position (checkpoints) ----------------------------------------------------------
    def file_order(self):
        """The current pair order as int64 positions in the training file (pair_users / pair_items order)."""
        if self._shuffles is None:
            raise _lib.SrbError("sampler: an epoch was shuffled while the pair order was not tracked; it is unknown (enable "
                                "track_order before the first epoch: checkpoint.dir, or HostFeed.track_pair_order())")
        order = self._shuffles.take()
        order = np.arange(self.n_pairs, dtype=np.int64) if order is None else order
        self._shuffles.add(order)
        return order

    def pair_order(self):
        """(users, items) int32 in the sampler's current order (srb_sampler_get_order)."""
        u, i = np.empty(self.n_pairs, dtype=np.int32), np.empty(self.n_pairs, dtype=np.int32)
        ring = self._pause()
        try:
            _lib.check(self._lib.srb_sampler_get_order(self.handle, u.ctypes.data_as(_lib.c_i32p), i.ctypes.data_as(_lib.c_i32p)),
                       "srb_sampler_get_order")
        finally:
            self._unpause(ring)
        return u, i

    def _pause(self):
        ring = self._ring
        if ring is not None:
            self.ring_stop()  # un-draws what the consumer has not popped
        return ring

    def _unpause(self, ring):
        if ring is not None:
            self.ring_start(*ring)  # continues from the cursor

    def position(self):
        """(order, cursor, random_state) at the current batch boundary: the file order of the pairs, the pairs consumed
        in the open epoch (-1 between epochs) and Python's `random` state at that point of the stream (inside an epoch
        the stream lives in the sampler, not in `random`).  A running ring is paused for the read and restarted."""
        ring = self._pause()
        try:
            cur = C.c_int64(0)
            _lib.check(self._lib.srb_sampler_cursor(self.handle, C.byref(cur)), "srb_sampler_cursor")
            cursor = int(cur.value)
            if cursor >= 0:
                _lib.check(self._lib.srb_sampler_get_state(self.handle, self._state), "srb_sampler_get_state")
                st = (3, tuple(self._state), getattr(self, "_gauss", random.getstate()[2]))
            else:
                st = random.getstate()
        finally:
            self._unpause(ring)
        return self.file_order(), cursor, st

    def restore(self, data, order, cursor, random_state):
        """Put the pairs in `order` (file positions, as position() returned them), reopen the epoch at `cursor` (-1:
        between epochs) and set Python's `random` to `random_state`.  `data`'s training_data follows the order.  The
        next stream_epoch() then continues the epoch instead of starting one."""
        if getattr(self, "_open_epoch", None) is not None:  # an abandoned epoch generator: retire it (stream_epoch)
            self._open_epoch, self._ring = None, None
            self.ring_stop()
        order = np.ascontiguousarray(order, dtype=np.int64)
        if order.shape != (self.n_pairs,):
            raise _lib.SrbError(f"sampler.restore: an order of {order.shape} for {self.n_pairs} pairs")
        pu, pi = np.asarray(data.pair_users), np.asarray(data.pair_items)
        u, i = np.ascontiguousarray(pu[order], dtype=np.int32), np.ascontiguousarray(pi[order], dtype=np.int32)
        _lib.check(self._lib.srb_sampler_set_order(self.handle, u.ctypes.data_as(_lib.c_i32p), i.ctypes.data_as(_lib.c_i32p),
                                                   self.n_pairs), "srb_sampler_set_order")
        _lib.check(self._lib.srb_sampler_seek(self.handle, int(cursor)), "srb_sampler_seek")
        # training_data is in the order this sampler's shuffles left it: move it from there to `order`
        cur = self.file_order()
        inv = np.empty_like(cur)
        inv[cur] = np.arange(self.n_pairs, dtype=np.int64)
        permute_training_data(data, inv[order])
        self._shuffles = _PendingShuffles(fold=2)
        self._shuffles.add(order)
        self._tracking = True
        self._resume = int(cursor) >= 0
        random.setstate(random_state)
        self.pull_state()  # the sampler's generator too: position() before the next batch reads it

    def next_batch_negs(self, batch_size, n_negs, u, i, j):
        b = self._lib.srb_sampler_next_batch_negs(self.handle, batch_size, n_negs, u.ctypes.data_as(_lib.c_i32p),
                                                  i.ctypes.data_as(_lib.c_i32p), j.ctypes.data_as(_lib.c_i32p))
        if b < 0:
            _lib.check(b, "srb_sampler_next_batch_negs")
        return b

    def next_batch(self, batch_size, batch_cap, out):
        """Fixed layout (header + u,i,j,uniq_u,uniq_i) into the int32 array `out`."""
        b = self._lib.srb_sampler_next_batch(self.handle, batch_size, batch_cap, out.ctypes.data_as(_lib.c_i32p))
        if b < 0:
            _lib.check(b, "srb_sampler_next_batch")
        return b

    def ring_start(self, batch_size, batch_cap, depth=16):
        _lib.check(self._lib.srb_sampler_ring_start(self.handle, batch_size, batch_cap, depth), "srb_sampler_ring_start")

    def ring_pop(self, out):
        b = self._lib.srb_sampler_ring_pop(self.handle, out.ctypes.data_as(_lib.c_i32p))
        if b < 0:
            _lib.check(b, "srb_sampler_ring_pop")
        return b

    def ring_stop(self):
        _lib.check(self._lib.srb_sampler_ring_stop(self.handle), "srb_sampler_ring_stop")

    def epoch(self, batch_size, batch_cap):
        """All batches of one epoch (after begin_epoch): int32 array [n_batches, words]."""
        words = _lib.BATCH_HEADER + 5 * batch_cap
        nb = (self.n_pairs + batch_size - 1) // batch_size
        out = np.empty((nb, words), dtype=np.int32)
        got = self._lib.srb_sampler_epoch(self.handle, batch_size, batch_cap, out.ctypes.data_as(_lib.c_i32p), out.size)
        if got < 0:
            _lib.check(int(got), "srb_sampler_epoch")
        return out[:got]


def stream_epoch(sampler, data, batch_size, batch_cap, ring_depth=16):
    """One epoch of batch buffers (srb_sampler_next_batch layout) in ONE reused int32 buffer (the consumer copies
    it, e.g. into a pinned slot).  The batches come from the native sample-ahead ring: a C++ thread samples up to
    `ring_depth` batches ahead (0.2 ms each on one core) while Python enqueues GPU work, so the sampler stops being
    the ceiling of a step that is faster than that (a Python producer thread was tried in round 1 and dropped: its
    queue hand-offs under the GIL cost more than they hid).  ring_depth=0: one native call per batch.  Python's
    `random` state is taken at the start and handed back when the epoch ends or the generator is closed (batches the
    ring sampled ahead but nobody read are un-drawn: the state is the reference's at that point of the stream);
    data.training_data gets the epoch's shuffle.  After sampler.restore() reopened an epoch, the generator continues
    that epoch from its cursor instead (no shuffle); sampler.position() may be read between two batches."""
    # an epoch generator that was abandoned without close() (e.g. zip(range(n), gen)) still owns the ring and a
    # pending state hand-back: retire it now -- its own `finally`, whenever the garbage collector gets to it, must
    # neither stop the new ring nor overwrite Python's `random` state with a stale one
    if getattr(sampler, "_open_epoch", None) is not None:
        sampler._ring = None
        sampler.ring_stop()
        sampler.push_state()
    token = object()
    sampler._open_epoch = token
    resume, sampler._resume = getattr(sampler, "_resume", False), False
    sampler.pull_state()
    try:
        if not resume:
            perm = sampler.begin_epoch(want_perm=True)
            permute_training_data(data, perm)
        buf = np.empty(_lib.BATCH_HEADER + 5 * batch_cap, dtype=np.int32)
        if ring_depth > 0:
            sampler.ring_start(batch_size, batch_cap, ring_depth)
            sampler._ring = (batch_size, batch_cap, ring_depth)
            while sampler._open_epoch is token and sampler.ring_pop(buf) > 0:
                yield buf
        else:
            while sampler._open_epoch is token and sampler.next_batch(batch_size, batch_cap, buf) > 0:
                yield buf
    finally:
        if sampler._open_epoch is token:
            sampler._open_epoch = None
            sampler._ring = None
            sampler.ring_stop()
            sampler.push_state()


def _sampler_for(data):
    s = getattr(data, "_srb_sampler", None)
    n = len(data.pair_users) if hasattr(data, "pair_users") else len(data.training_data)
    if s is None or s.n_pairs != n:
        s = NativePairSampler(data)
        data._srb_sampler = s
    return s


def permute_training_data(data, perm):
    """data.training_data[k] <- data.training_data[perm[k]], lazily when the data object supports it."""
    if hasattr(data, "shuffle_training_data"):
        data.shuffle_training_data(perm)
    else:
        td = data.training_data
        td[:] = [td[k] for k in perm]


def next_batch_pairwise(data, batch_size, n_negs=1):
    s = _sampler_for(data)
    s.pull_state()
    perm = s.begin_epoch(want_perm=True)
    s.push_state()
    permute_training_data(data, perm)  # the in-place shuffle side effect (sampler.py:7)
    u = np.empty(batch_size, dtype=np.int32)
    i = np.empty(batch_size, dtype=np.int32)
    j = np.empty(batch_size * n_negs, dtype=np.int32)
    while True:
        s.pull_state()
        b = s.next_batch_negs(batch_size, n_negs, u, i, j)
        s.push_state()
        if b == 0:
            return
        yield u[:b].tolist(), i[:b].tolist(), j[: b * n_negs].tolist()


def next_batch_sequence(data, batch_size, n_negs=1, max_len=50):
    """util/sampler.py:84-112 (SASRec, BERT4Rec, CL4SRec): (seq, pos, y, neg, seq_len) int64 batches over a shuffled
    copy of data.original_seq, with the same `random` draws as the reference.  Each row holds the last max_len - 1
    items before the last one (seq) and the items after them (y); neg is one sample of as many catalogue ids
    (1..item_num), drawn again until it shares no item with seq.  n_negs is accepted and unused, as in the reference.
    Plain Python: shuffle and sample on the global `random` stream.  sample() picks positions, so drawing from
    range(1, item_num + 1) takes the same draws as the reference's list of those ids."""
    sequences = [s for _, s in data.original_seq]
    random.shuffle(sequences)
    catalogue = range(1, data.item_num + 1)
    for ptr in range(0, len(sequences), batch_size):
        rows = sequences[ptr:ptr + batch_size]
        seq, pos, y, neg = (np.zeros((len(rows), max_len), dtype=np.int64) for _ in range(4))
        seq_len = np.zeros(len(rows), dtype=np.int64)
        for r, s in enumerate(rows):
            start, end = (len(s) - max_len, max_len - 1) if len(s) > max_len else (0, len(s) - 1)
            history = s[start:-1]
            seq[r, :end] = history
            pos[r, :end] = np.arange(1, end + 1)
            y[r, :end] = s[start + 1:]
            seen = set(history)
            negatives = random.sample(catalogue, end)
            while not seen.isdisjoint(negatives):
                negatives = random.sample(catalogue, end)
            neg[r, :end] = negatives
            seq_len[r] = end
        yield seq, pos, y, neg, seq_len


def next_batch_sequence_for_test(data, batch_size, max_len=50):
    """util/sampler.py:114-132 (base/seq_recommender.py test()): (seq, pos, seq_len) int64 batches of the last
    max_len items of every sequence, in data.original_seq order.  Draws nothing from `random`."""
    sequences = [s for _, s in data.original_seq]
    for ptr in range(0, len(sequences), batch_size):
        rows = sequences[ptr:ptr + batch_size]
        seq, pos = (np.zeros((len(rows), max_len), dtype=np.int64) for _ in range(2))
        seq_len = np.zeros(len(rows), dtype=np.int64)
        for r, s in enumerate(rows):
            end = min(len(s), max_len)
            seq[r, :end] = s[len(s) - end:]
            pos[r, :end] = np.arange(1, end + 1)
            seq_len[r] = end
        yield seq, pos, seq_len
