"""Neighbourhood baselines (reference model/graph/ItemKNN.py, model/graph/UserKNN.py) on the GPU.

The host side builds what the kernels read from an interaction object (data/ui_graph.py's Interaction mirror,
NativeInteraction or synth.ArrayInteraction):
  insertion_csr()   per user its distinct items in training_set_u order (the order ItemKNN.predict adds them in)
  transpose_csr()   item -> user CSR
  name_ranks()      rank of every name in Python's sorted() order, the tie key of heapq.nlargest over (sim, name)
NeighbourTable holds one model's device neighbour table and computes predict() rows and find_k_largest lists from it,
all in float64 and bit for bit with the reference (DESIGN §11).
"""
import numpy as np
import torch

from . import _lib, ops

# bytes of float64 score rows (plus top-k workspace) ranked per launch: bounds test()'s memory at any catalogue size
RANK_CHUNK_BYTES = 1 << 30


def insertion_csr(pair_users, pair_items, n_users, n_items):
    """(ptr int32 [U+1], idx int32): each user's distinct items in order of the user's first line per item, which is
    the key order of training_set_u[user] (ui_graph.py:39; a repeated line keeps its first position)."""
    pu = np.asarray(pair_users, dtype=np.int64)
    pi = np.asarray(pair_items, dtype=np.int64)
    _, first = np.unique(pu * int(n_items) + pi, return_index=True)
    first = first[np.lexsort((first, pu[first]))]
    ptr = np.zeros(int(n_users) + 1, dtype=np.int32)
    ptr[1:] = np.cumsum(np.bincount(pu[first], minlength=int(n_users)))
    return ptr, pi[first].astype(np.int32)


def transpose_csr(ptr, idx, n_cols):
    """CSR of the transpose of a CSR with unique entries per row; each transposed row is sorted."""
    rows = np.repeat(np.arange(len(ptr) - 1, dtype=np.int32), np.diff(ptr))
    order = np.lexsort((rows, idx))
    tptr = np.zeros(int(n_cols) + 1, dtype=np.int32)
    tptr[1:] = np.cumsum(np.bincount(idx, minlength=int(n_cols)))
    return tptr, rows[order]


def name_ranks(names):
    """int32 rank of names[id] in sorted(names) (names are unique)."""
    order = sorted(range(len(names)), key=names.__getitem__)
    rank = np.empty(len(names), dtype=np.int32)
    rank[order] = np.arange(len(names), dtype=np.int32)
    return rank


def id_names(data, side):
    """Names of the user (side "user") or item ids in id order; an object without name maps (synth.ArrayInteraction)
    is named by its ids, as its training_data is."""
    n = data.user_num if side == "user" else data.item_num
    id2name = getattr(data, "id2user" if side == "user" else "id2item", None)
    return list(range(n)) if id2name is None else [id2name[k] for k in range(n)]


class NeighbourTable:
    """The device neighbour table of ItemKNN (by="item": rows are items, a row's set is its users) or UserKNN
    (by="user": rows are users, a row's set is its items), built by train(), and the ranking that reads it."""

    def __init__(self, data, by, topk, shrinkage, device=None):
        if by not in ("item", "user"):
            raise ValueError(f"by={by!r}: 'item' (ItemKNN) or 'user' (UserKNN)")
        _lib.require_device()
        self.data, self.by = data, by
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        U, I = int(data.user_num), int(data.item_num)
        seq_ptr, seq_idx = insertion_csr(data.pair_users, data.pair_items, U, I)
        iu_ptr, iu_idx = transpose_csr(seq_ptr, seq_idx, I)
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(self.device)
        self.seq = (dev(seq_ptr), dev(seq_idx))
        if by == "item":
            rows, trans, self.mode = (iu_ptr, iu_idx), (seq_ptr, seq_idx), ops.KNN_ITEM
        else:
            rows, trans, self.mode = (seq_ptr, seq_idx), (iu_ptr, iu_idx), ops.KNN_USER
        self.names = id_names(data, by)
        rank = dev(name_ranks(self.names))
        self.table = ops.knn_neighbors(dev(rows[0]), dev(rows[1]), dev(trans[0]), dev(trans[1]), rank, topk, shrinkage)
        rated_ptr, rated_idx = data.rated_csr()
        self.rated = (dev(rated_ptr), dev(rated_idx))
        self.n_items = I

    def score_rows(self, uids, masked=False):
        """Float64 predict() rows [len(uids), item_num] on the device; masked: rated items set to -10e8."""
        rated = self.rated if masked else (None, None)
        return ops.knn_score_rows(self.mode, uids, self.n_items, self.table, *self.seq, *rated)

    def rank(self, uids, max_n):
        """find_k_largest(max_n, masked predict row) for each user id: (ids int32 [n, max_n], scores float64) on the host."""
        uids = np.asarray(uids, dtype=np.int32)
        ids = np.empty((len(uids), max_n), dtype=np.int32)
        scores = np.empty((len(uids), max_n), dtype=np.float64)
        step = max(1, RANK_CHUNK_BYTES // (8 * self.n_items + 16 * max_n))
        for s in range(0, len(uids), step):
            rows = self.score_rows(uids[s:s + step], masked=True)
            i, v = ops.topk_rows_f64(rows, max_n)
            del rows
            ids[s:s + step], scores[s:s + step] = i.cpu().numpy(), v.cpu().numpy()
        return ids, scores

    def neighbours(self):
        """Host copies (ids int32 [n_rows, topK], sims float64 [n_rows, topK], counts int32 [n_rows])."""
        return tuple(t.cpu().numpy() for t in self.table)

    def as_dict(self):
        """The reference's item_sim / user_sim: {row name: [(sim, neighbour name), ...]} in list order."""
        ids, sims, cnt = self.neighbours()
        names = self.names
        return {names[a]: [(sims[a, t], names[ids[a, t]]) for t in range(cnt[a])] for a in range(len(names))}
