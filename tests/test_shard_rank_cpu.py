"""Host logic of training and ranking on the sharded engine, on CPU with real gloo process groups: rank 0's start
state reaches every rank (same sampler batches, SGL view draws and initial tables), the rank-local rated / test CSRs
tile the global ones, the per-rank ranking results reassemble into query order identically on every rank, and the
refusals (MF on more than one rank, predict() of a user another rank owns)."""
import hashlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _spawn(target, world, *args):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    port = 31000 + (os.getpid() * 7 + world) % 2000
    procs = [ctx.Process(target=target, args=(r, world, port, ret) + args) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(180)
        assert p.exitcode == 0
    return ret.get(timeout=5)


def _init(rank, world, port):
    import torch.distributed as dist
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    return dist


def _digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return int.from_bytes(h.digest()[:7], "little")


def _all_same(dist, value):
    """True on every rank iff every rank passed the same integer."""
    import torch
    t = torch.tensor([value, -value], dtype=torch.int64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return int(t[0]) == value and int(-t[1]) == value


def _state_worker(rank, world, port, ret):
    import random

    import torch
    dist = _init(rank, world, port)
    from selfrec_b200 import synth
    from selfrec_b200.data.augmentor import sample_range
    from selfrec_b200.engine import initial_tables
    from selfrec_b200.shard_rank import broadcast_start_state
    from selfrec_b200.util.sampler import NativePairSampler, stream_epoch
    random.seed(1000 + rank)  # the reference seeds nothing: every process starts somewhere else
    torch.manual_seed(2000 + rank)
    differed = not _all_same(dist, _digest(np.array(random.getstate()[1], dtype=np.int64), torch.get_rng_state().numpy()))
    broadcast_start_state()
    data = synth.make_interaction((300, 200, 3000), seed=1)
    ue, ie = initial_tables(data.user_num, data.item_num, torch.empty((data.user_num + data.item_num, 32)))
    views = [sample_range(300, 30), sample_range(200, 20), sample_range(len(data.pair_users), 2400)]  # node, then edge dropout
    s = NativePairSampler(data)
    gen = stream_epoch(s, data, 256, 256)
    batches = [next(gen).copy() for _ in range(3)]
    gen.close()
    same = all(_all_same(dist, _digest(*x)) for x in ([ue.numpy(), ie.numpy()], views, batches))
    ok = differed and same and torch.initial_seed() == 2000 and not np.array_equal(batches[0], batches[1])
    out = torch.tensor([1.0 if ok else 0.0])
    dist.all_reduce(out, op=dist.ReduceOp.MIN)
    if rank == 0:
        ret.put(float(out.item()))
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_start_state_broadcast_gives_one_trajectory(built_lib, world):
    assert _spawn(_state_worker, world) == 1.0


class _Data:
    """rated_csr / test_csr / user_num of a random graph, the parts ShardRanker reads."""

    def __init__(self, U, I, seed):
        rng = np.random.default_rng(seed)
        self.user_num = U

        def csr(lo, hi):
            rows = [np.sort(rng.choice(I, size=rng.integers(lo, hi), replace=False)).astype(np.int32) for _ in range(U)]
            ptr = np.zeros(U + 1, dtype=np.int32)
            ptr[1:] = np.cumsum([len(r) for r in rows])
            return ptr, np.concatenate(rows).astype(np.int32)
        self._rated, self._test = csr(1, 12), csr(0, 5)
        self.n_test = (np.diff(self._test[0]) + rng.integers(0, 2, U)).astype(np.int32)

    def rated_csr(self):
        return self._rated

    def test_csr(self):
        return self._test + (self.n_test,)


def test_local_csrs_tile_the_global_ones():
    from selfrec_b200.shard_rank import ShardRanker, local_csr
    from selfrec_b200.sharded import local_user_count, user_ids_of
    data = _Data(103, 60, 4)
    for ptr, idx in (data.rated_csr(), data.test_csr()[:2]):
        for world in (1, 2, 3, 4):
            seen = np.zeros(data.user_num, dtype=np.int64)
            for g in range(world):
                rows = user_ids_of(data.user_num, g, world)
                lp, li = local_csr(ptr, idx, rows)
                assert lp.dtype == np.int32 and li.dtype == np.int32 and lp.size == local_user_count(data.user_num, g, world) + 1
                for r, u in enumerate(rows):
                    assert np.array_equal(li[lp[r]:lp[r + 1]], idx[ptr[u]:ptr[u + 1]])
                seen[rows] += 1
            assert (seen == 1).all()  # every row on exactly one rank
    for world in (1, 2, 3, 4):  # the ranker's own copy is the same cut
        for g in range(world):
            rk = ShardRanker(data, g, world, "cpu")
            lp, li = local_csr(*data.rated_csr(), user_ids_of(data.user_num, g, world))
            assert np.array_equal(rk.rated[0].numpy(), lp) and np.array_equal(rk.rated[1].numpy(), li)


def _gather_worker(rank, world, port, ret):
    import torch
    dist = _init(rank, world, port)
    from selfrec_b200.shard_rank import gather_in_order, owned_positions
    # test users in a shuffled order; rank world - 1 owns none of them, the others own uneven counts
    U, k = 50, 7
    rng = np.random.default_rng(9)
    uids = rng.permutation([u for u in range(U) if u % world != world - 1 and (u % world != 0 or u < 20)]).astype(np.int32)
    pos, rows = owned_positions(uids, rank, world)
    mine = uids[pos]
    assert np.array_equal(rows, mine // world) and (mine % world == rank).all()
    ids = torch.from_numpy((mine[:, None] * 100 + np.arange(k)).astype(np.int32))
    sc = torch.from_numpy((mine[:, None] + np.arange(k) / 8).astype(np.float32))
    masks = torch.from_numpy((mine.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)).view(np.int64))  # all 64 bits in use
    got = [gather_in_order(t, uids, rank, world).numpy() for t in (ids, sc, masks)]
    want = [(uids[:, None] * 100 + np.arange(k)).astype(np.int32), (uids[:, None] + np.arange(k) / 8).astype(np.float32),
            (uids.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)).view(np.int64)]
    ok = all(g.dtype == w.dtype and np.array_equal(g, w) for g, w in zip(got, want)) and _all_same(dist, _digest(*got))
    ok = ok and len(mine) == 0 if rank == world - 1 else ok
    out = torch.tensor([1.0 if ok else 0.0])
    dist.all_reduce(out, op=dist.ReduceOp.MIN)
    if rank == 0:
        ret.put(float(out.item()))
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3, 4])
def test_ranking_results_reassemble_in_test_order_on_every_rank(world):
    assert _spawn(_gather_worker, world) == 1.0


def test_reassemble_single_process_matches_gather_layout():
    import torch
    from selfrec_b200.shard_rank import gather_in_order, owned_positions, reassemble
    uids = np.array([5, 0, 3, 8, 1, 6], dtype=np.int32)
    world = 3
    parts = []
    for g in range(world):
        pos, _ = owned_positions(uids, g, world)
        p = torch.zeros((4, 2), dtype=torch.int32)  # padded past the owned count
        p[: pos.size] = torch.from_numpy(uids[pos])[:, None]
        parts.append(p)
    assert reassemble(parts, uids, world)[:, 0].tolist() == uids.tolist()
    one = torch.from_numpy(uids)
    assert gather_in_order(one, uids, 0, 1).tolist() == uids.tolist()
    with pytest.raises(ValueError):
        gather_in_order(one[:3], uids, 0, 1)


class _Conf:
    """The configuration keys the model classes read."""

    def __init__(self, model, extra):
        self.config = {"training.set": "train.txt", "test.set": "test.txt", "model": {"name": model, "type": "graph"},
                       "item.ranking.topN": [5, 10], "embedding.size": 64, "max.epoch": 1, "batch.size": 128,
                       "learning.rate": 0.001, "reg.lambda": 0.0001, "output": "./results/", model: extra}

    def __getitem__(self, k):
        return self.config[k]

    def contain(self, k):
        return k in self.config


def _refusal_worker(rank, world, port, ret, cwd):
    import torch
    dist = _init(rank, world, port)
    os.chdir(cwd)
    from selfrec_b200._lib import SrbError
    from selfrec_b200.data.loader import FileIO
    from selfrec_b200.data.ui_graph import Interaction
    from selfrec_b200.model.graph.LightGCN import LightGCN
    from selfrec_b200.model.graph.MF import MF
    from selfrec_b200.shard_rank import ShardRanker
    train = FileIO.load_data_set(os.path.join(ROOT, "tests", "golden", "tiny_train.txt"))
    test = FileIO.load_data_set(os.path.join(ROOT, "tests", "golden", "tiny_test.txt"))
    ok = True
    try:  # refused before anything touches a device
        MF(_Conf("MF", {}), [list(t) for t in train], [list(t) for t in test])
        ok = False
    except SrbError as e:
        ok = ok and "MF" in str(e)
    m = object.__new__(LightGCN)
    m.data = Interaction(_Conf("LightGCN", {"n_layer": 2}), [list(t) for t in train], [list(t) for t in test])
    m.shard_ranker = ShardRanker(m.data, rank, world, "cpu")
    other = (rank + 1) % world
    name = next(n for n, u in m.data.user.items() if u % world == other)
    try:
        m.predict(name)
        ok = False
    except SrbError as e:
        ok = ok and f"rank {other}" in str(e)
    out = torch.tensor([1.0 if ok else 0.0])
    dist.all_reduce(out, op=dist.ReduceOp.MIN)
    if rank == 0:
        ret.put(float(out.item()))
    dist.destroy_process_group()


def test_mf_on_two_ranks_and_predict_of_another_ranks_user_are_refused(built_lib, tmp_path):
    assert _spawn(_refusal_worker, 2, str(tmp_path)) == 1.0


def test_install_without_torchrun_starts_no_process_group(monkeypatch):
    import torch.distributed as dist
    import selfrec_b200
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    selfrec_b200.install()
    assert not dist.is_initialized()
