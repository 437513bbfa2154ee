"""On-disk checkpoints of the fused engines: save a run, resume it at any world size, rank from a saved model.

One directory per checkpoint, `ckpt-<epoch>-<batch>` (the epoch and batch the run continues at):
  manifest.json            format version, model, shapes, data fingerprint, hyperparameters, world size at save, the
                           position (epoch, batch, step, sampler cursor), bestPerformance, Python / numpy / torch RNG states
  pair_order.npy           int64: the sampler's pair order as positions in the training file
  item_params.npy          [I, d] replicated item table;  best_item.npy: the keep-best item table (when there is one)
  user_ids.<g>.npy         int64 global user ids of shard g, ascending; user_{params,m,v}.<g>.npy and best_user.<g>.npy
                           their rows.  A single-process save is one shard holding users 0..U-1.
  item_{m,v}.<g>.npy       the Adam moments of item rows manifest["item_bounds"][g] .. [g + 1] (each rank owns one slice)
  extra files              what the model adds (SGL: the draws of the epoch's two view graphs)
Every table holds rows in global id order, so a checkpoint does not depend on the world size that wrote it: a reader at
any world takes the rows it owns out of every shard file through a memory map.

Saving is atomic: the files go to a hidden sibling directory, are fsynced, and the directory is renamed into place;
older checkpoints are removed only after that.  A process killed while saving leaves the previous checkpoint whole.
"""
import base64
import hashlib
import json
import os
import random
import shutil

import numpy as np

from ._lib import SrbError

FORMAT_VERSION = 1
MANIFEST = "manifest.json"
PREFIX = "ckpt-"
HYPER = ("d", "L", "B", "lr", "reg", "eps", "tau", "cl_rate", "layer_cl", "l2_div", "philox_seed")
IDENTITY = ("format", "model", "U", "I", "nnz", "pairs", "pairs_fingerprint") + HYPER


def checkpoint_name(epoch, batch):
    return f"{PREFIX}{int(epoch):06d}-{int(batch):010d}"


def pairs_fingerprint(pair_users, pair_items):
    """blake2b of the training pairs in file order (int32 users, then int32 items)."""
    h = hashlib.blake2b(digest_size=16)
    h.update(np.ascontiguousarray(pair_users, dtype=np.int32).tobytes())
    h.update(np.ascontiguousarray(pair_items, dtype=np.int32).tobytes())
    return h.hexdigest()


def identity(model, engine, data, fingerprint=None):
    """The manifest fields a checkpoint must match to be loaded into `engine` training `model` on `data`."""
    nnz = int(engine.nnzA) if hasattr(engine, "nnzA") else (int(engine.adj.nnz) if getattr(engine, "adj", None) is not None else 0)
    pu, pi = data.pair_users, data.pair_items
    out = {"format": FORMAT_VERSION, "model": str(model), "U": int(engine.U), "I": int(engine.I), "nnz": nnz, "pairs": int(len(pu)),
           "pairs_fingerprint": fingerprint or pairs_fingerprint(pu, pi), "d": int(engine.d), "L": int(engine.L), "B": int(engine.B)}
    out.update(engine.hyper)
    return out


# ---- RNG states as JSON ----------------------------------------------------------------------------------------------
def rng_states(random_state=None):
    """Python `random` (or the given state), numpy's global and torch's CPU generator states, JSON-serialisable."""
    import torch
    st = random.getstate() if random_state is None else random_state
    ns = np.random.get_state()
    return {"random": [st[0], list(st[1]), st[2]],
            "numpy": [ns[0], np.asarray(ns[1]).tolist(), int(ns[2]), int(ns[3]), float(ns[4])],
            "torch": base64.b64encode(torch.get_rng_state().numpy().tobytes()).decode()}


def python_random_state(saved):
    return (int(saved["random"][0]), tuple(int(x) for x in saved["random"][1]), saved["random"][2])


def set_rng_states(saved, python=True):
    """Restore rng_states() (`python=False`: leave Python's `random` to the caller, e.g. the sampler's restore)."""
    import torch
    if python:
        random.setstate(python_random_state(saved))
    n = saved["numpy"]
    np.random.set_state((n[0], np.asarray(n[1], dtype=np.uint32), n[2], n[3], n[4]))
    torch.set_rng_state(torch.from_numpy(np.frombuffer(base64.b64decode(saved["torch"]), dtype=np.uint8).copy()))


# ---- writing -----------------------------------------------------------------------------------------------------------
def _fsync_dir(path):
    fd = os.open(path, os.O_RDONLY)
    try:
        os.fsync(fd)
    finally:
        os.close(fd)


def write_array(directory, name, arr):
    """np.save + fsync of one file."""
    with open(os.path.join(directory, name), "wb") as f:
        np.save(f, np.ascontiguousarray(arr))
        f.flush()
        os.fsync(f.fileno())


def _publish(tmp, final):
    """The step that makes a checkpoint visible: one rename of the finished directory."""
    if os.path.exists(final):  # the same position saved again (e.g. after a resume): replace it
        old = final + ".old"
        shutil.rmtree(old, ignore_errors=True)
        os.replace(final, old)
        os.replace(tmp, final)
        shutil.rmtree(old, ignore_errors=True)
    else:
        os.replace(tmp, final)


def write_shard(directory, shard, state, best_user=None):
    """Shard `shard`'s files of an engine state_dict(): its user rows with their ids, its slice of item moments."""
    ids = np.asarray(state["user_ids"], dtype=np.int64)
    order = np.argsort(ids, kind="stable")
    sorted_rows = not (order.size and np.any(order != np.arange(order.size)))
    pick = (lambda a: a) if sorted_rows else (lambda a: np.asarray(a)[order])
    write_array(directory, f"user_ids.{shard}.npy", pick(ids))
    for name in ("params", "m", "v"):
        write_array(directory, f"user_{name}.{shard}.npy", pick(state["user"][name]))
    if best_user is not None:
        write_array(directory, f"best_user.{shard}.npy", pick(best_user))
    for name in ("m", "v"):
        write_array(directory, f"item_{name}.{shard}.npy", state["item"][name])


def _phase(fn, agree):
    """Run fn() on this rank, then agree on the outcome with every rank: a rank that failed re-raises its own error, the
    others raise SrbError, and nobody is left waiting in a barrier for a rank that gave up."""
    err = None
    try:
        fn()
    except BaseException as e:  # noqa: BLE001 -- re-raised below, after the other ranks have heard of it
        err = e
    ok = agree(err is None)
    if err is not None:
        raise err
    if not ok:
        raise SrbError("checkpoint save: another rank failed; nothing was published")


def save(root, manifest, shards, common, rank=0, world=1, agree=lambda ok: ok):
    """Write one checkpoint atomically under `root` and remove the older ones.  Returns the checkpoint's path.

    manifest: the JSON fields (epoch and batch name the directory); shards: {g: (state_dict, best_user or None)} of the
    shards this process writes; common: {file name: array} written by rank 0 (item_params, pair_order, best_item, the
    model's extra files).  Under a process group every rank calls save() with its own shard, and `agree(ok)` (True when
    `ok` holds on every rank; collective) separates the creation of the temporary directory, the writes and the rename,
    so a failure on any rank stops every rank and publishes nothing."""
    name = checkpoint_name(manifest["epoch"], manifest["batch"])
    final = os.path.join(root, name)
    tmp = os.path.join(root, "." + name + ".tmp")

    def begin():
        if rank == 0:
            os.makedirs(root, exist_ok=True)
            for entry in os.listdir(root):  # what a killed save left behind
                if entry.startswith(".") and entry.endswith(".tmp"):
                    shutil.rmtree(os.path.join(root, entry), ignore_errors=True)
            os.makedirs(tmp)

    def write():
        for g, (state, best_user) in shards.items():
            write_shard(tmp, g, state, best_user)
        if rank == 0:
            for fname, arr in common.items():
                write_array(tmp, fname, arr)

    def finish():
        if rank == 0:
            man = dict(manifest, world=int(world))
            with open(os.path.join(tmp, MANIFEST), "w") as f:
                json.dump(man, f, indent=1)
                f.flush()
                os.fsync(f.fileno())
            _fsync_dir(tmp)
            _publish(tmp, final)
            _fsync_dir(root)
            for entry in os.listdir(root):  # the new checkpoint is good: the older ones can go
                if entry.startswith(PREFIX) and entry != name:
                    shutil.rmtree(os.path.join(root, entry), ignore_errors=True)

    _phase(begin, agree)
    try:
        _phase(write, agree)
        _phase(finish, agree)
    except BaseException:
        if rank == 0:
            shutil.rmtree(tmp, ignore_errors=True)
        raise
    return final


# ---- reading -----------------------------------------------------------------------------------------------------------
def latest(root):
    """The newest complete checkpoint under `root` (None if there is none).  A `<name>.old` directory is the previous
    checkpoint of a position saved twice (_publish); it counts when the save that replaces it was killed between its two
    renames, i.e. when `<name>` itself is missing."""
    if not os.path.isdir(root):
        return None
    entries = set(os.listdir(root))
    names = []
    for e in entries:
        base = e[:-len(".old")] if e.endswith(".old") else e
        if not base.startswith(PREFIX) or not os.path.exists(os.path.join(root, e, MANIFEST)):
            continue
        if e != base and base in entries and os.path.exists(os.path.join(root, base, MANIFEST)):
            continue  # the replacement was published
        names.append((base, e))
    return os.path.join(root, max(names)[1]) if names else None


def resolve(spec, root=None):
    """`checkpoint.resume`: a checkpoint directory, or "latest" in `root` (checkpoint.dir)."""
    if str(spec) == "latest":
        if root is None:
            raise SrbError("checkpoint.resume: latest needs checkpoint.dir")
        path = latest(root)
        if path is None:
            raise SrbError(f"checkpoint.resume: latest, but {root} holds no checkpoint")
        return path
    if not os.path.exists(os.path.join(str(spec), MANIFEST)):
        raise SrbError(f"checkpoint.resume: {spec} is not a checkpoint (no {MANIFEST})")
    return str(spec)


def read_manifest(path):
    with open(os.path.join(path, MANIFEST)) as f:
        return json.load(f)


def verify(manifest, want, path=""):
    """Raise SrbError naming the first field where the checkpoint and this run differ (nothing is loaded before)."""
    if manifest.get("format") != FORMAT_VERSION:
        raise SrbError(f"checkpoint {path}: format is {manifest.get('format')!r} in the checkpoint, {FORMAT_VERSION!r} here")
    for key in IDENTITY:
        if manifest.get(key) != want.get(key):
            raise SrbError(f"checkpoint {path}: {key} is {manifest.get(key)!r} in the checkpoint, {want.get(key)!r} here")


def _shards(path, manifest):
    return range(int(manifest["world"]))


def _mmap(path, fname):
    return np.load(os.path.join(path, fname), mmap_mode="r")


def read_user_rows(path, manifest, name, user_ids, chunk=1 << 20):
    """Rows of the users `user_ids` (global ids, in the reader's local order) of the per-shard user table `name`
    (params, m, v, best): only those rows are read out of each shard file's memory map."""
    U = int(manifest["U"])
    user_ids = np.asarray(user_ids, dtype=np.int64)
    where = np.full(U, -1, dtype=np.int64)
    where[user_ids] = np.arange(user_ids.size, dtype=np.int64)
    out = None
    seen = 0
    fname = "best_user" if name == "best" else "user_" + name
    for g in _shards(path, manifest):
        ids = np.load(os.path.join(path, f"user_ids.{g}.npy"))
        sel = np.flatnonzero(where[ids] >= 0)
        mm = _mmap(path, f"{fname}.{g}.npy")
        if out is None:
            out = np.empty((user_ids.size, mm.shape[1]), dtype=np.float32)
        for lo in range(0, sel.size, chunk):
            s = sel[lo:lo + chunk]
            out[where[ids[s]]] = mm[s]
        seen += sel.size
        del mm
    if seen != user_ids.size:
        raise SrbError(f"checkpoint {path}: {seen} of the {user_ids.size} requested user rows of {name} are in the checkpoint")
    return out


def read_item_moment(path, manifest, name):
    """The [I, d] item moment `name` (m or v) put together from every shard's slice."""
    b = manifest["item_bounds"]
    parts = [_mmap(path, f"item_{name}.{g}.npy") for g in _shards(path, manifest)]
    for g, p in enumerate(parts):
        if p.shape[0] != b[g + 1] - b[g]:
            raise SrbError(f"checkpoint {path}: item_{name}.{g}.npy has {p.shape[0]} rows, the bounds say {b[g + 1] - b[g]}")
    return np.concatenate(parts) if parts else None


class _Rows:
    """Mapping name -> array, read when asked for (one table in host memory at a time)."""

    def __init__(self, read):
        self._read = read

    def __getitem__(self, name):
        return self._read(name)


def engine_state(path, manifest, user_ids):
    """What load_state_dict() of an engine holding the users `user_ids` (global ids in its local-row order) takes."""
    return {"step": int(manifest["step"]),
            "user": _Rows(lambda name: read_user_rows(path, manifest, name, user_ids)),
            "item_params": _mmap(path, "item_params.npy"),
            "item": _Rows(lambda name: read_item_moment(path, manifest, name))}


def engine_user_ids(engine):
    """Global ids of the engine's user rows, in its local-row order."""
    ids = getattr(engine, "user_ids", None)
    if ids is None:
        return np.arange(engine.U, dtype=np.int64)
    return ids.cpu().numpy().astype(np.int64)


def save_engines(root, manifest, engines, common=None, best_users=None):
    """save() of the ranks `engines` of one world held by this process (a single engine, or every rank of a loopback
    world); rank 0's item table and feed are the shared ones."""
    states = [e.state_dict() for e in engines]
    bounds = [0] * (len(engines) + 1)
    for g, st in enumerate(states):
        bounds[g], bounds[g + 1] = st["item_rows"]
    common = dict(common or {}, item_params=states[0]["item_params"])
    e0 = engines[0]
    man = dict({"U": int(e0.U), "I": int(e0.I), "d": int(e0.d)}, **manifest)
    man.update(step=states[0]["step"], item_bounds=[int(x) for x in bounds])
    shards = {g: (st, None if best_users is None else best_users[g]) for g, st in enumerate(states)}
    return save(root, man, shards, {k if k.endswith(".npy") else k + ".npy": v for k, v in common.items()}, world=len(engines))
