"""Training, evaluation and ranking of a model on the bipartite-sharded engine, one process per GPU (SURVEY 8e).

Every rank must follow one trajectory: broadcast_start_state() hands rank 0's Python `random` state (the sampler
stream, SGL's view draws) and torch's CPU generator state (the initial tables, and torch.initial_seed(), which keys the
device draw of large tables) to every rank before the engine is built.

Ranking: rank g holds the final embeddings of its own users ([Ug, d], local row = the user's position among g's users)
and the whole item table.  Each rank scores and selects the top-k of the queried users it owns, on the existing
kernels (ops.score_topk, ops.rank_hit_masks) against rated / test CSRs cut down to its own rows; no rank ever holds
the full user table.  The per-rank results are all-gathered, padded to the largest rank's count, and put back in query
order on every rank, so every rank computes the same lists, the same measure strings and the same keep-best decision.

The collective plumbing (owned_positions, local_csr, reassemble, gather_in_order) is plain numpy / tensor code that also runs on
CPU tensors under a gloo group (tests/test_shard_rank_cpu.py); which rank owns which user is decided by sharded.py.
"""
import random

import numpy as np

from .sharded import local_row_of, owner_of, user_ids_of


def _dist():
    import torch.distributed as dist
    return dist if dist.is_available() and dist.is_initialized() else None


def process_group():
    """(rank, world) of the default process group, or None when no group is initialised."""
    dist = _dist()
    return None if dist is None else (dist.get_rank(), dist.get_world_size())


def is_main_process():
    """True outside a process group and on rank 0 of one: the process that prints and writes the result files."""
    pg = process_group()
    return pg is None or pg[0] == 0


def broadcast_start_state(group=None):
    """Give every rank rank 0's Python `random` state and torch CPU generator state (which carries
    torch.initial_seed()).  Collective."""
    import torch
    dist = _dist()
    if dist is None:
        return
    state = [random.getstate(), torch.get_rng_state()] if dist.get_rank(group) == 0 else [None, None]
    dist.broadcast_object_list(state, group=group, group_src=0)
    random.setstate(state[0])
    torch.set_rng_state(state[1])


def owned_positions(uids, rank, world):
    """(positions in query order of the queried users `rank` owns, their local rows), numpy int64."""
    uids = np.asarray(uids, dtype=np.int64)
    pos = np.flatnonzero(owner_of(uids, world) == int(rank))
    return pos, local_row_of(uids[pos], world)


def local_csr(ptr, idx, rows):
    """Rows `rows` of the CSR (ptr, idx), renumbered 0..len(rows)-1: (ptr int32, idx int32)."""
    ptr, rows = np.asarray(ptr, dtype=np.int64), np.asarray(rows, dtype=np.int64)
    beg = ptr[rows]
    cnt = ptr[rows + 1] - beg
    lp = np.zeros(rows.size + 1, dtype=np.int64)
    np.cumsum(cnt, out=lp[1:])
    pos = np.arange(int(lp[-1]), dtype=np.int64) + np.repeat(beg - lp[:-1], cnt)
    return lp.astype(np.int32), np.asarray(idx)[pos].astype(np.int32)


def reassemble(parts, uids, world):
    """parts[g]: rank g's results [>= n_g, ...] for its queried users in owned_positions() order (rows past n_g are
    padding).  Returns the [len(uids), ...] results in query order."""
    import torch
    own = owner_of(uids, world)
    out = parts[0].new_empty((own.size,) + tuple(parts[0].shape[1:]))
    for g in range(world):
        pos = np.flatnonzero(own == g)
        out[torch.from_numpy(pos).to(out.device)] = parts[g][: pos.size]
    return out


def gather_in_order(local, uids, rank, world, group=None):
    """`local` [n_rank, ...]: this rank's results for its queried users in owned_positions() order.  Returns the
    [len(uids), ...] results of all ranks in query order, on every rank: one all_gather, padded to the largest rank's
    count, then reassemble().  Collective when world > 1; the tensors stay on local's device (CUDA under NCCL, CPU
    under gloo)."""
    import torch
    counts = np.bincount(owner_of(uids, world), minlength=world)
    if local.shape[0] != counts[rank]:
        raise ValueError(f"gather_in_order: rank {rank} holds {local.shape[0]} rows, it owns {counts[rank]} queried users")
    if world == 1:
        return reassemble([local], uids, 1)
    pad = local.new_zeros((int(counts.max()),) + tuple(local.shape[1:]))
    pad[: local.shape[0]] = local
    parts = [torch.empty_like(pad) for _ in range(world)]
    _dist().all_gather(parts, pad, group=group)
    return reassemble(parts, uids, world)


class ShardRanker:
    """Ranking of rank `rank`'s users: its [Ug, d] user block against the replicated [I, d] item table.  The rated CSR
    of its rows is built at construction, the test CSR on first use; both live on `device`."""

    def __init__(self, data, rank, world, device, group=None):
        import torch
        self.data, self.rank, self.world, self.group, self.dev = data, int(rank), int(world), group, device
        self.rows = user_ids_of(data.user_num, rank, world)
        self.rated = tuple(torch.from_numpy(a).to(device) for a in local_csr(*data.rated_csr(), self.rows))
        self._test = None

    def owner(self, uid):
        return int(owner_of([uid], self.world)[0])

    def local_row(self, uid):
        return int(local_row_of([uid], self.world)[0])

    def local_topk(self, user_block, item_emb, uids, k):
        """(ids [n_rank, k] int32, scores [n_rank, k] fp32) of the queried global ids `uids` this rank owns, in
        owned_positions() order: ops.score_topk on the local rows of the user block and the local rated CSR."""
        import torch
        from . import ops
        _, rows = owned_positions(uids, self.rank, self.world)
        if rows.size == 0:  # no launch on an empty grid
            dev = item_emb.device
            return torch.empty((0, k), dtype=torch.int32, device=dev), torch.empty((0, k), dtype=torch.float32, device=dev)
        return ops.score_topk(user_block, item_emb, rows.astype(np.int32), *self.rated, k)

    def local_hit_masks(self, user_block, item_emb, uids, k):
        """fast_evaluation's hit masks (ops.rank_hit_masks: int64 [n] for k <= 64, [n, ceil(k / 64)] up to 256) of the
        queried users this rank owns."""
        import torch
        from . import ops
        if self._test is None:
            tp, ti, _ = self.data.test_csr()
            self._test = tuple(torch.from_numpy(a).to(self.dev) for a in local_csr(tp, ti, self.rows))
        _, rows = owned_positions(uids, self.rank, self.world)
        ids, _ = self.local_topk(user_block, item_emb, uids, k)
        if rows.size == 0:
            words = (k + 63) // 64
            return torch.empty((0,) if words == 1 else (0, words), dtype=torch.int64, device=ids.device)
        return ops.rank_hit_masks(ids, rows.astype(np.int32), *self._test)

    def gather(self, local, uids):
        return gather_in_order(local, uids, self.rank, self.world, self.group)

    def topk(self, user_block, item_emb, uids, k):
        """(ids [n, k] int32, scores [n, k] fp32) of the global user ids `uids`, in their order, on every rank."""
        ids, sc = self.local_topk(user_block, item_emb, uids, k)
        return self.gather(ids, uids), self.gather(sc, uids)

    def hit_masks(self, user_block, item_emb, uids, k):
        """The hit masks of `uids`, in their order, on every rank."""
        return self.gather(self.local_hit_masks(user_block, item_emb, uids, k), uids)
