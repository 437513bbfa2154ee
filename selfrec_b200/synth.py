"""Synthetic bipartite interaction graphs of a named |U| x |I| x nnz shape (SURVEY 8d).

No dataset travels to the GPU box, so bench.py and the full-size property tests build a
power-law graph with the same shape as the named configuration (yelp2018: 31 668 x 38 048 x
1 237 259).  Ids follow the reference's convention: first-appearance order of the pair list
(ui_graph.py:29-40), every user and item has at least one interaction, pairs are unique.
"""
import numpy as np
import scipy.sparse as sp

from .data.data import Data
from .data.graph import Graph

SHAPES = {
    "douban-book": (12638, 22222, 478730),
    "yelp2018": (31668, 38048, 1237259),
    "amazon-kindle": (138333, 98572, 1525091),
}


def _first_appearance_relabel(x, n):
    _, first = np.unique(x, return_index=True)
    order = np.argsort(first)  # old ids in order of first appearance
    new = np.empty(n, dtype=np.int64)
    new[np.unique(x)[order]] = np.arange(len(order))
    return new[x]


def make_pairs(n_users, n_items, nnz, seed=0, alpha_u=0.42, alpha_i=0.40):
    """Unique (user, item) id pairs, power-law degrees on both sides, shuffled by user blocks."""
    rng = np.random.default_rng(seed)
    pu = (1.0 / np.arange(1, n_users + 1) ** alpha_u)
    pi = (1.0 / np.arange(1, n_items + 1) ** alpha_i)
    pu /= pu.sum()
    pi /= pi.sum()
    # one guaranteed edge per node, then draw until nnz unique pairs
    u0 = np.concatenate([np.arange(n_users), rng.choice(n_users, n_items, p=pu)])
    i0 = np.concatenate([rng.choice(n_items, n_users, p=pi), np.arange(n_items)])
    key = set()
    keys = u0.astype(np.int64) * n_items + i0
    keys = np.unique(keys)
    while len(keys) < nnz:
        need = int((nnz - len(keys)) * 1.3) + 1024
        k = rng.choice(n_users, need, p=pu).astype(np.int64) * n_items + rng.choice(n_items, need, p=pi)
        keys = np.unique(np.concatenate([keys, k]))
    if len(keys) > nnz:
        # drop random extras but never a node's only edge
        u, i = keys // n_items, keys % n_items
        du, di = np.bincount(u, minlength=n_users), np.bincount(i, minlength=n_items)
        perm = rng.permutation(len(keys))
        keep = np.ones(len(keys), dtype=bool)
        extra = len(keys) - nnz
        for t in perm:
            if extra == 0:
                break
            if du[u[t]] > 1 and di[i[t]] > 1:
                keep[t] = False
                du[u[t]] -= 1
                di[i[t]] -= 1
                extra -= 1
        keys = keys[keep]
    u, i = keys // n_items, keys % n_items
    # the training file is grouped by user; users in random order
    uperm = rng.permutation(n_users)
    order = np.lexsort((rng.random(len(u)), uperm[u]))
    u, i = u[order], i[order]
    return _first_appearance_relabel(u, n_users).astype(np.int32), _first_appearance_relabel(i, n_items).astype(np.int32)


class ArrayInteraction(Data, Graph):
    """The subset of data/ui_graph.py's Interaction the CUDA path consumes, built straight
    from id arrays (no name dictionaries).  training_data holds (user_id, item_id, 1.0)."""

    def __init__(self, pair_users, pair_items, n_users, n_items, test_users=None):
        self.pair_users = np.ascontiguousarray(pair_users, dtype=np.int32)
        self.pair_items = np.ascontiguousarray(pair_items, dtype=np.int32)
        self.user_num, self.item_num = int(n_users), int(n_items)
        Data.__init__(self, None, list(zip(self.pair_users.tolist(), self.pair_items.tolist())), [])
        n = self.user_num + self.item_num
        ones = np.ones(len(self.pair_users), dtype=np.float32)
        half = sp.csr_matrix((ones, (self.pair_users, self.pair_items.astype(np.int64) + self.user_num)), shape=(n, n), dtype=np.float32)
        self.ui_adj = half + half.T
        self.norm_adj = self.normalize_graph_mat(self.ui_adj)
        self.interaction_mat = sp.csr_matrix((ones, (self.pair_users, self.pair_items)), shape=(self.user_num, self.item_num), dtype=np.float32)
        self.test_user_ids = np.arange(self.user_num, dtype=np.int32) if test_users is None else np.asarray(test_users, dtype=np.int32)
        self._rated = None

    def rated_csr(self):
        if self._rated is None:
            m = sp.csr_matrix(self.interaction_mat)
            m.sum_duplicates()
            m.sort_indices()
            self._rated = (m.indptr.astype(np.int32), m.indices.astype(np.int32))
        return self._rated

    def convert_to_laplacian_mat(self, adj_mat):
        rows, cols = adj_mat.nonzero()
        n = adj_mat.shape[0] + adj_mat.shape[1]
        half = sp.csr_matrix((adj_mat.data, (rows, cols + adj_mat.shape[0])), shape=(n, n), dtype=np.float32)
        return self.normalize_graph_mat(half + half.T)


def make_interaction(shape="yelp2018", seed=0, scale=1.0):
    """ArrayInteraction of a named shape (optionally scaled down for quick tests)."""
    U, I, nnz = SHAPES[shape] if isinstance(shape, str) else shape
    U, I, nnz = max(8, int(U * scale)), max(8, int(I * scale)), max(16, int(nnz * scale))
    pu, pi = make_pairs(U, I, nnz, seed)
    return ArrayInteraction(pu, pi, U, I)


# ------------------------------------------------------------------------------------------------
# config-5 sized graphs: generated, relabelled and normalised on the GPU (no scipy / no Python lists at 200 M edges)
# ------------------------------------------------------------------------------------------------
SHAPES["synthetic-10M"] = (10_000_000, 2_000_000, 200_000_000)   # BASELINE.json configs[4] (about 100 GB of device memory at d = 128)
SHAPES["synthetic-5M"] = (5_000_000, 1_000_000, 100_000_000)     # the same recipe at half the rows: fits one 80 GB GPU
SHAPES["synthetic-2M"] = (2_000_000, 500_000, 40_000_000)        # mid-size stand-in (same recipe, 1/5 of the rows)


def _zipf_ranks(n, size, alpha, gen, dev):
    """Ranks 0..n-1 with P(rank r) ~ (r+1)^-alpha (bounded-Pareto inverse CDF, float64)."""
    import torch
    r = torch.rand(size, generator=gen, device=dev, dtype=torch.float64)
    a = 1.0 - alpha
    x = (((n + 1.0) ** a - 1.0) * r + 1.0) ** (1.0 / a)
    return torch.clamp(x.floor().to(torch.int64) - 1, 0, n - 1)


def make_pairs_device(n_users, n_items, nnz, seed=0, alpha=1.1, device="cuda"):
    """SURVEY 8(d) recipe for config 5, on the device: user ~ Zipf(alpha) over U, item ~ Zipf(alpha) over I, pairs
    de-duplicated, every node >= 1 edge, exactly nnz distinct pairs, pair list in random ("log") order, ids by
    first appearance in that order (ui_graph.py:29-40).  Returns int32 device tensors (users, items) in file order."""
    import torch
    dev = torch.device(device)
    gen = torch.Generator(device=dev).manual_seed(int(seed))
    U, I = int(n_users), int(n_items)
    # one guaranteed edge per node (never dropped), partner drawn from the other side's Zipf
    gu = torch.cat([torch.arange(U, device=dev), _zipf_ranks(U, I, alpha, gen, dev)])
    gi = torch.cat([_zipf_ranks(I, U, alpha, gen, dev), torch.arange(I, device=dev)])
    kg = torch.unique(gu * I + gi)
    if kg.numel() > nnz:
        raise ValueError("nnz is smaller than the number of nodes")
    kr = torch.empty(0, dtype=torch.int64, device=dev)
    need = nnz - kg.numel()
    while kr.numel() < need:
        m = int((need - kr.numel()) * 1.35) + 4096
        k = _zipf_ranks(U, m, alpha, gen, dev) * I + _zipf_ranks(I, m, alpha, gen, dev)
        kr = torch.unique(torch.cat([kr, k]))
        pos = torch.searchsorted(kg, kr).clamp_(max=kg.numel() - 1)
        kr = kr[kg[pos] != kr]  # the guaranteed edges are counted once
        del k, pos
    if kr.numel() > need:
        sel = torch.randperm(kr.numel(), generator=gen, device=dev)[:need]
        kr = kr[sel]
        del sel
    keys = torch.cat([kg, kr])
    del kg, kr
    keys = keys[torch.randperm(keys.numel(), generator=gen, device=dev)]  # file order: a random interleaving
    u, i = keys // I, keys % I
    del keys
    pos = torch.arange(u.numel(), device=dev)

    def relabel(x, n):
        first = torch.full((n,), u.numel(), dtype=torch.int64, device=dev).scatter_reduce_(0, x, pos, "amin")
        new = torch.empty(n, dtype=torch.int64, device=dev)
        new[torch.sort(first, stable=True).indices] = torch.arange(n, device=dev)
        return new[x].to(torch.int32)

    return relabel(u, U), relabel(i, I)


class DeviceInteraction:
    """What the CUDA path consumes of data/ui_graph.py's Interaction, with the graph resident on the device:
    user_num / item_num, norm_adj (ops.SparseAdj on the device), bip (DeviceBipartite, for SGL views), the
    training pairs in file order (device; host copies are made on first use, for the native sampler)."""

    def __init__(self, pair_users, pair_items, n_users, n_items):
        import torch
        from .data.device_graph import DeviceBipartite
        self.user_num, self.item_num = int(n_users), int(n_items)
        self.pairs_dev = (pair_users.contiguous(), pair_items.contiguous())
        dev = pair_users.device
        key = pair_users.to(torch.int64) * self.item_num + pair_items.to(torch.int64)
        key = torch.sort(key).values
        ui_col = (key % self.item_num).to(torch.int32)
        cnt = torch.bincount(key // self.item_num, minlength=self.user_num)
        del key
        ui_ptr = torch.zeros(self.user_num + 1, dtype=torch.int32, device=dev)
        ui_ptr[1:] = torch.cumsum(cnt, 0).to(torch.int32)
        self.bip = DeviceBipartite.from_device_csr(self.user_num, self.item_num, ui_ptr, ui_col)
        self.norm_adj = self.bip.assemble()
        self.bip.free_workspace()
        self._host_pairs = None
        self._rated = None

    @property
    def pair_users(self):
        return self._pairs()[0]

    @property
    def pair_items(self):
        return self._pairs()[1]

    def _pairs(self):
        if self._host_pairs is None:
            self._host_pairs = tuple(t.cpu().numpy() for t in self.pairs_dev)
        return self._host_pairs

    def training_size(self):
        return int(self.pairs_dev[0].numel())

    def shuffle_training_data(self, perm):
        """The sampler's in-place shuffle of training_data (sampler.py:7): the pair arrays live in the native
        sampler, nothing else reads the order here."""

    def rated_csr(self):
        if self._rated is None:
            self._rated = (self.bip.ui_ptr.cpu().numpy(), self.bip.ui_col.cpu().numpy())
        return self._rated

    def rated_csr_device(self):
        return self.bip.ui_ptr, self.bip.ui_col


def make_device_interaction(shape="synthetic-10M", seed=0, alpha=1.1, device="cuda"):
    U, I, nnz = SHAPES[shape] if isinstance(shape, str) else shape
    pu, pi = make_pairs_device(U, I, nnz, seed, alpha, device)
    return DeviceInteraction(pu, pi, U, I)
