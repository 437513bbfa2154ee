"""Checkpoints without a GPU: the native sampler paused and resumed mid-epoch in a fresh process state, and the on-disk
format (manifest refusals, atomic saves, re-sharding between world sizes)."""
import json
import os
import random

import numpy as np
import pytest

B = 512
SHAPE = (300, 400, 5000)  # 10 batches of 512, the last one short
NB = -(-SHAPE[2] // B)


def _fresh():
    from selfrec_b200 import synth
    from selfrec_b200.util.sampler import NativePairSampler
    data = synth.make_interaction(SHAPE, seed=9)
    return NativePairSampler(data, track_order=True), data


def _reference(seed, depth):
    """Three uninterrupted epochs: their batches, the final `random` state and training_data."""
    from selfrec_b200.util.sampler import stream_epoch
    smp, data = _fresh()
    random.seed(seed)
    out = [[w.copy() for w in stream_epoch(smp, data, B, B, ring_depth=depth)] for _ in range(3)]
    return out, random.getstate(), list(data.training_data)


@pytest.mark.parametrize("depth", [0, 4])
@pytest.mark.parametrize("epoch,n", [(0, 0), (0, 3), (0, NB), (1, 0), (1, 7), (2, NB - 1), (1, "between")])
def test_sampler_resumes_mid_epoch_bit_exact(built_lib, depth, epoch, n):
    """Stop after n batches of an epoch (or between two epochs), read the order, cursor and MT state, rebuild a fresh
    sampler and data object, restore into them: every later batch, the final `random` state and training_data are the
    uninterrupted run's.  The interrupted run itself also continues unchanged after the read (the ring is paused)."""
    from selfrec_b200.util.sampler import stream_epoch
    ref, ref_state, ref_td = _reference(1234, depth)
    smp, data = _fresh()
    random.seed(1234)
    for e in range(epoch):
        whole = [w.copy() for w in stream_epoch(smp, data, B, B, ring_depth=depth)]
        assert len(whole) == NB and all(np.array_equal(a, w) for a, w in zip(ref[e], whole))
    cont = []
    if n == "between":
        for w in stream_epoch(smp, data, B, B, ring_depth=depth):
            pass
        order, cursor, st = smp.position()
        assert cursor == -1 and st == random.getstate()
        tail = [b for e in range(epoch + 1, 3) for b in ref[e]]
    else:
        g = stream_epoch(smp, data, B, B, ring_depth=depth)
        for k in range(n):
            assert np.array_equal(next(g), ref[epoch][k])
        order, cursor, st = smp.position()
        assert cursor == (min(n * B, SHAPE[2]) if n > 0 else -1)  # a generator not yet started has opened no epoch
        u, i = smp.pair_order()
        assert np.array_equal(u, data.pair_users[order]) and np.array_equal(i, data.pair_items[order])
        cont = [w.copy() for w in g]  # the interrupted run goes on after the read
        assert len(cont) == NB - n and all(np.array_equal(a, b) for a, b in zip(cont, ref[epoch][n:]))
        tail = ref[epoch][n:] + [b for e in range(epoch + 1, 3) for b in ref[e]]
    # a new process state: fresh objects, `random` scrambled, then the restore
    smp2, data2 = _fresh()
    random.seed(999)
    smp2.restore(data2, order, cursor, st)
    got = []
    n_epochs = 3 - epoch - (1 if (n == "between" or cursor >= 0) else 0)  # whole epochs after the restored position
    if cursor >= 0:
        got += [w.copy() for w in stream_epoch(smp2, data2, B, B, ring_depth=depth)]
    for _ in range(n_epochs):
        got += [w.copy() for w in stream_epoch(smp2, data2, B, B, ring_depth=depth)]
    assert len(got) == len(tail) and all(np.array_equal(a, b) for a, b in zip(got, tail))
    assert random.getstate() == ref_state
    assert list(data2.training_data) == ref_td


def test_sampler_restore_mid_epoch_with_exact_lazy_feed(built_lib):
    """The per-batch feed (HostFeed.batches(exact_lazy=True)) continues a restored epoch too."""
    from selfrec_b200.engine import HostFeed
    from selfrec_b200.util.sampler import NativePairSampler

    class Feed(HostFeed):
        def __init__(self, data):
            self.data, self.B, self.words, self.sampler = data, B, 4 + 5 * B, None
            self.track_pair_order()

    ref, ref_state, _ = _reference(77, 0)
    smp, data = _fresh()
    f = Feed(data)
    random.seed(77)
    g = f.batches(exact_lazy=True)
    for k in range(4):
        assert np.array_equal(next(g), ref[0][k])
    pos = f.feed_state()
    assert pos["random"] == random.getstate()  # the lazy feed hands the state back after every batch
    f2 = Feed(_fresh()[1])
    random.seed(3)
    f2.load_feed_state(pos)
    got = [w.copy() for w in f2.batches(exact_lazy=True)] + [w.copy() for e in (1, 2) for w in f2.batches(exact_lazy=True)]
    want = ref[0][4:] + ref[1] + ref[2]
    assert len(got) == len(want) and all(np.array_equal(a, b) for a, b in zip(got, want))
    assert random.getstate() == ref_state
    assert isinstance(f2.sampler, NativePairSampler)


def test_sampler_native_position_entry_points(built_lib):
    """srb_sampler_seek / cursor / set_order refuse bad input and a running ring."""
    from selfrec_b200 import _lib
    smp, data = _fresh()
    with pytest.raises(_lib.SrbError, match="cursor"):
        _lib.check(smp._lib.srb_sampler_seek(smp.handle, SHAPE[2] + 1), "srb_sampler_seek")
    bad = np.full(SHAPE[2], SHAPE[0], dtype=np.int32)
    ok = np.zeros(SHAPE[2], dtype=np.int32)
    with pytest.raises(_lib.SrbError, match="out of range"):
        _lib.check(smp._lib.srb_sampler_set_order(smp.handle, bad.ctypes.data_as(_lib.c_i32p), ok.ctypes.data_as(_lib.c_i32p), SHAPE[2]), "set_order")
    with pytest.raises(_lib.SrbError, match="pairs"):
        _lib.check(smp._lib.srb_sampler_set_order(smp.handle, ok.ctypes.data_as(_lib.c_i32p), ok.ctypes.data_as(_lib.c_i32p), 3), "set_order")
    random.seed(1)
    smp.pull_state()
    smp.begin_epoch()
    smp.ring_start(B, B, 2)
    try:
        with pytest.raises(_lib.SrbError, match="ring"):
            _lib.check(smp._lib.srb_sampler_seek(smp.handle, 0), "srb_sampler_seek")
    finally:
        smp.ring_stop()


# ---------------------------------------------------------------------------------------------------------------------
# the on-disk format
# ---------------------------------------------------------------------------------------------------------------------
U, I, D = 37, 23, 8


def _tables(seed=0):
    rng = np.random.default_rng(seed)
    return {k: rng.standard_normal((U + I, D)).astype(np.float32) for k in ("params", "m", "v")}


def _shard_state(t, rank, world, bounds):
    ids = np.arange(rank, U, world, dtype=np.int64)
    lo, hi = bounds[rank], bounds[rank + 1]
    return {"step": 5, "user_ids": ids, "user": {k: t[k][:U][ids] for k in ("params", "m", "v")}, "item_params": t["params"][U:],
            "item_rows": (lo, hi), "item": {k: t[k][U + lo:U + hi] for k in ("m", "v")}}


def _manifest(world, epoch=1, batch=0):
    from selfrec_b200 import checkpoint
    man = {"format": checkpoint.FORMAT_VERSION, "model": "LightGCN", "U": U, "I": I, "nnz": 2 * 100, "pairs": 100,
           "pairs_fingerprint": "ab" * 16, "d": D, "L": 2, "B": 16, "lr": 1e-3, "reg": 1e-4, "eps": 0.0, "tau": 0.2, "cl_rate": 0.0,
           "layer_cl": 0, "l2_div": 1.0, "philox_seed": 24301}
    man.update(epoch=epoch, batch=batch, step=5, cursor=-1, bestPerformance=[], rng=checkpoint.rng_states())
    return man


def _save_world(root, t, world, epoch=1, batch=0):
    from selfrec_b200 import checkpoint
    from selfrec_b200.sharded import item_bounds
    bounds = [int(x) for x in item_bounds(I, world)]
    man = dict(_manifest(world, epoch, batch), item_bounds=bounds)
    # one process holds every shard here, as a loopback world does: it writes them all as rank 0
    shards = {r: (_shard_state(t, r, world, bounds), t["params"][:U][r::world] * 2) for r in range(world)}
    return checkpoint.save(str(root), man, shards, {"item_params.npy": t["params"][U:], "pair_order.npy": np.arange(100)},
                           world=world)


@pytest.mark.parametrize("w1", range(1, 9))
def test_resharding_every_world_to_every_world(tmp_path, w1):
    """Shards written at world W1 read back at every world W2 in 1..8: every rank gets exactly its own users' rows, and
    the item tables and moments are the global ones."""
    from selfrec_b200 import checkpoint
    t = _tables(w1)
    path = _save_world(tmp_path / f"w{w1}", t, w1)
    man = checkpoint.read_manifest(path)
    assert man["world"] == w1
    for w2 in range(1, 9):
        got = {k: np.empty((U, D), dtype=np.float32) for k in ("params", "m", "v", "best")}
        for r in range(w2):
            ids = np.arange(r, U, w2, dtype=np.int64)
            st = checkpoint.engine_state(path, man, ids)
            for k in ("params", "m", "v"):
                got[k][ids] = st["user"][k]
            got["best"][ids] = checkpoint.read_user_rows(path, man, "best", ids)
            assert np.array_equal(st["item_params"], t["params"][U:])
            for k in ("m", "v"):
                assert np.array_equal(st["item"][k], t[k][U:])
        for k in ("params", "m", "v"):
            assert np.array_equal(got[k], t[k][:U]), (w1, w2, k)
        assert np.array_equal(got["best"], t["params"][:U] * 2)


def test_every_manifest_mismatch_is_refused_by_name(tmp_path):
    from selfrec_b200 import checkpoint
    from selfrec_b200._lib import SrbError
    path = _save_world(tmp_path, _tables(), 2)
    man = checkpoint.read_manifest(path)
    want = {k: man[k] for k in checkpoint.IDENTITY}
    checkpoint.verify(man, want, path)
    for key in checkpoint.IDENTITY:
        other = dict(want)
        v = want[key]
        other[key] = v + "x" if isinstance(v, str) else (v * 2 + 1 if isinstance(v, int) else v * 2 + 0.5)
        with pytest.raises(SrbError, match=rf"\b{key} is {v!r} in the checkpoint, {other[key]!r} here"):
            checkpoint.verify(man, other, path)
    with pytest.raises(SrbError, match="format"):
        checkpoint.verify(dict(man, format=checkpoint.FORMAT_VERSION + 1), want, path)


def _snapshot(root):
    out = {}
    for dirpath, _dirs, files in os.walk(root):
        for f in files:
            p = os.path.join(dirpath, f)
            out[os.path.relpath(p, root)] = open(p, "rb").read()
    return out


def test_interrupted_save_leaves_the_previous_checkpoint(tmp_path, monkeypatch):
    """An exception after every file is written but before the rename: the previous checkpoint is still the latest,
    byte for byte, and loads; the next save cleans up and succeeds, and then only the newest checkpoint is kept."""
    from selfrec_b200 import checkpoint
    t = _tables(3)
    first = _save_world(tmp_path, t, 2, epoch=1, batch=0)
    before = _snapshot(tmp_path)

    def boom(tmp, final):
        assert os.path.exists(os.path.join(tmp, checkpoint.MANIFEST))  # everything was written
        raise KeyboardInterrupt("killed between the writes and the rename")

    monkeypatch.setattr(checkpoint, "_publish", boom)
    with pytest.raises(KeyboardInterrupt):
        _save_world(tmp_path, _tables(4), 3, epoch=1, batch=40)
    monkeypatch.undo()
    assert checkpoint.latest(str(tmp_path)) == first
    assert _snapshot(tmp_path) == before
    man = checkpoint.read_manifest(first)
    st = checkpoint.engine_state(first, man, np.arange(U))
    assert np.array_equal(st["user"]["params"], t["params"][:U])
    # a save killed half way (temporary directory left behind) is cleaned up by the next one
    os.makedirs(tmp_path / ".ckpt-000001-0000000040.tmp")
    second = _save_world(tmp_path, _tables(5), 3, epoch=1, batch=40)
    assert checkpoint.latest(str(tmp_path)) == second
    assert sorted(os.listdir(tmp_path)) == [os.path.basename(second)]
    assert checkpoint.resolve("latest", str(tmp_path)) == second


def test_rng_states_round_trip_through_json():
    import torch
    from selfrec_b200 import checkpoint
    random.seed(5)
    np.random.seed(6)
    torch.manual_seed(7)
    random.random(), np.random.rand(), torch.rand(1)
    saved = json.loads(json.dumps(checkpoint.rng_states()))
    want = (random.random(), np.random.rand(), float(torch.rand(1)))
    random.seed(0)
    np.random.seed(0)
    torch.manual_seed(0)
    checkpoint.set_rng_states(saved)
    assert (random.random(), np.random.rand(), float(torch.rand(1))) == want


def test_pair_order_is_tracked_only_on_request(built_lib):
    """Without track_order the sampler keeps no permutation (nothing changes for runs that do not checkpoint); a
    position() after an untracked shuffle is refused instead of recording a wrong order."""
    from selfrec_b200 import _lib, synth
    from selfrec_b200.util.sampler import NativePairSampler, stream_epoch
    data = synth.make_interaction(SHAPE, seed=9)
    smp = NativePairSampler(data)
    random.seed(2)
    assert np.array_equal(smp.file_order(), np.arange(SHAPE[2]))  # never shuffled: the file order
    for _ in stream_epoch(smp, data, B, B):
        pass
    assert smp._shuffles is None
    with pytest.raises(_lib.SrbError, match="not tracked"):
        smp.position()


def test_position_saved_twice_survives_a_kill_between_the_renames(tmp_path, monkeypatch):
    """Saving a position that already exists moves the old directory aside before the new one takes its name; a process
    killed between those two renames leaves the old one, which latest() still finds and which loads."""
    from selfrec_b200 import checkpoint
    t = _tables(6)
    first = _save_world(tmp_path, t, 1, epoch=2, batch=0)
    real, calls = os.replace, []

    def replace(a, b):
        calls.append((a, b))
        if len(calls) == 2:  # the first rename (final -> final.old) done, the second one (tmp -> final) not
            raise KeyboardInterrupt("killed between the renames")
        return real(a, b)

    monkeypatch.setattr(checkpoint.os, "replace", replace)
    with pytest.raises(KeyboardInterrupt):
        _save_world(tmp_path, _tables(7), 1, epoch=2, batch=0)
    monkeypatch.undo()
    found = checkpoint.latest(str(tmp_path))
    assert found == first + ".old" and not os.path.exists(first)
    st = checkpoint.engine_state(found, checkpoint.read_manifest(found), np.arange(U))
    assert np.array_equal(st["user"]["params"], t["params"][:U])
    # the next save of that position publishes normally and clears the leftover
    again = _save_world(tmp_path, _tables(8), 1, epoch=2, batch=0)
    assert checkpoint.latest(str(tmp_path)) == again == first and sorted(os.listdir(tmp_path)) == [os.path.basename(first)]


@pytest.mark.parametrize("phase", [0, 1])
def test_a_failed_rank_stops_the_save_everywhere(tmp_path, phase):
    """agree(ok) is where the ranks compare notes: when another rank reports a failure while the directory is created
    or while the shards are written, this rank raises too, nothing is published and the previous checkpoint stays the
    latest, byte for byte.  (The last phase, manifest and rename, is rank 0's alone: its outcome is what the others
    hear.)"""
    from selfrec_b200 import checkpoint
    from selfrec_b200._lib import SrbError
    from selfrec_b200.sharded import item_bounds
    t = _tables(9)
    first = _save_world(tmp_path, t, 2, epoch=1, batch=0)
    before = _snapshot(tmp_path)
    seen = []

    def agree(ok):
        seen.append(ok)
        return ok and len(seen) != phase + 1  # another rank failed in this phase

    bounds = [int(x) for x in item_bounds(I, 2)]
    with pytest.raises(SrbError, match="another rank failed"):
        checkpoint.save(str(tmp_path), dict(_manifest(2, 1, 9), item_bounds=bounds), {0: (_shard_state(t, 0, 2, bounds), None)},
                        {"item_params.npy": t["params"][U:]}, rank=0, world=2, agree=agree)
    assert len(seen) == phase + 1
    assert checkpoint.latest(str(tmp_path)) == first
    assert _snapshot(tmp_path) == before
