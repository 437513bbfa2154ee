"""Export every user's top-N recommendation list of a trained (or resumed) model to disk, and read it back.

    path = model.export_recommendations(out_dir, top_n=None, users=None)
    names, ids, scores = export.read(path)

One directory `<out_dir>/<model>-top<N>`:
  manifest.json     format version, model, U, I, d (null for models without embedding tables), N, world (number of
                    parts), the training-pair fingerprint (checkpoint.pairs_fingerprint), the score dtype
  items.txt         item names, line i = item id i;  users.txt: user names, line u = user id u
  users.<g>.npy     int64 [n_g]      global user ids of part g, ascending
  ids.<g>.npy       int32 [n_g, N]   item ids, score-descending (ties by id descending), rated items masked as in test()
  scores.<g>.npy    float32 [n_g, N] (float64 for ItemKNN / UserKNN)
A single process writes one part; under torchrun each rank of a sharded model ranks only the users it owns, from its
own [Ug, d] user block and rated rows (shard_rank.ShardRanker), and writes its own part -- nothing is all-gathered.

Users go through the ranker in chunks; each chunk's lists are copied to pinned host buffers on a side stream and from
there into the memory-mapped part files, so the copy and file write of chunk k overlap the ranking of chunk k + 1 and
host memory stays proportional to the chunk.  Lists of 33..256 at d = 64 / 128 are ranked on the tensor cores like the
short ones (ops.long_list_route): no score rows, only per-user candidate buffers, whose workspace cuts the chunk so it
stays under LONG_WS_BYTES.  Other lists longer than 32 come from dense [chunk, I] score rows (the 32-at-a-time path of
ops.score_topk); their chunk is cut so those rows stay under WIDE_ROWS_BYTES.

Publishing is atomic, as for checkpoints: the part files go to a hidden sibling `.<name>.tmp`, are fsynced, and the
directory is renamed into place in one os.replace (an older export of the same name is replaced only then).  Under a
process group every phase ends in an all-reduced success flag, so a rank that fails stops every rank and nothing is
published.
"""
import json
import os
import shutil

import numpy as np

from . import checkpoint, ops
from ._lib import SrbError
from .shard_rank import is_main_process, owned_positions, process_group

FORMAT_VERSION = 1
MANIFEST = "manifest.json"
EXPORT_CHUNK = 1 << 16            # users per ranking call
WIDE_ROWS_BYTES = 1 << 30         # cap on the dense [chunk, I] fp32 score rows of lists longer than 32
LONG_WS_BYTES = 1 << 30           # cap on the ranking workspace of a chunk of long lists on the tensor cores


def export_name(model_name, n):
    return f"{model_name}-top{int(n)}"


class _Job:
    """One process's share of an export: which users it ranks, how, and where the files go.  begin() / write() /
    finish() are the three phases of the atomic publish; begin() and finish() act on rank 0 only."""

    def __init__(self, model, out_dir, top_n=None, users=None, chunk=None):
        from .knn import RANK_CHUNK_BYTES
        data = model.data
        U, I = int(data.user_num), int(data.item_num)
        n = int(model.max_N if top_n is None else top_n)
        if not 1 <= n <= I:
            raise SrbError(f"export: topN={top_n} must be in 1..item_num={I}")
        if users is None:
            uids = np.arange(U, dtype=np.int64)
        else:
            unknown = [u for u in users if u not in data.user]
            if unknown:
                raise SrbError(f"export: {len(unknown)} unknown user name(s), first {unknown[0]!r}")
            uids = np.unique(np.fromiter((data.user[u] for u in users), dtype=np.int64, count=len(users)))
        chunk = int(EXPORT_CHUNK if chunk is None else chunk)
        if chunk < 1:
            raise SrbError(f"export: chunk={chunk} must be >= 1")
        self.model, self.n, self.d = model, n, None
        self.rank, self.world, self.agree = 0, 1, (lambda ok: ok)
        self.score_dtype = np.float32
        ranker, table = getattr(model, "shard_ranker", None), getattr(model, "neighbour_table", None)
        if ranker is not None:
            import torch
            self.rank, self.world = ranker.rank, ranker.world
            eng = getattr(model, "engine", None)
            if self.world > 1 and eng is not None and hasattr(eng, "all_ok"):
                self.agree = eng.all_ok
            pos, rows = owned_positions(uids, self.rank, self.world)
            uids = uids[pos]
            ue, ie = model.user_emb.detach(), model.item_emb.detach()
            self.d = int(ie.shape[1])
            rows_d = torch.from_numpy(rows.astype(np.int32)).to(ie.device)
            self._fn = lambda lo, hi: ops.score_topk(ue, ie, rows_d[lo:hi], *ranker.rated, n)
        elif table is not None:  # ItemKNN / UserKNN: float64 scores
            self.score_dtype = np.float64
            chunk = min(chunk, max(1, RANK_CHUNK_BYTES // (8 * I + 16 * n)))

            def fn(lo, hi):
                return ops.topk_rows_f64(table.score_rows(uids[lo:hi].astype(np.int32), masked=True), n)
            self._fn = fn
        elif model._has_embedding_tables():
            import torch
            ue, ie = model.user_emb.detach(), model.item_emb.detach()
            self.d = int(ie.shape[1])
            rp, ri = data.rated_csr()
            rated = (torch.from_numpy(rp).to(ie.device), torch.from_numpy(ri).to(ie.device))
            uids_d = torch.from_numpy(uids.astype(np.int32)).to(ie.device)
            self._fn = lambda lo, hi: ops.score_topk(ue, ie, uids_d[lo:hi], *rated, n)
        else:  # any other model: its own predict() rows
            names = [data.id2user[int(u)] for u in uids]
            self._fn = lambda lo, hi: model._predict_topk(names[lo:hi], uids[lo:hi].astype(np.int32), n)
        if n > ops.TOPK_KERNEL_MAX and self.score_dtype == np.float32:
            if self.d is not None and ops.long_list_route(self.d, I, n):
                chunk = long_list_chunk(chunk, I, self.d, n)
            else:
                chunk = min(chunk, max(1, WIDE_ROWS_BYTES // (4 * I)))
        self.uids, self.chunk = uids, chunk
        self.name = export_name(model.model_name, n)
        self.out_dir = out_dir
        self.final = os.path.join(out_dir, self.name)
        self.tmp = os.path.join(out_dir, "." + self.name + ".tmp")

    # ---- phases ----
    def begin(self):
        if self.rank == 0:
            os.makedirs(self.out_dir, exist_ok=True)
            shutil.rmtree(self.tmp, ignore_errors=True)  # what a killed export left behind
            os.makedirs(self.tmp)

    def write(self):
        _write_part(self.tmp, self.rank, self.uids, self._fn, self.n, self.score_dtype, self.chunk)

    def finish(self):
        if self.rank != 0:
            return
        data = self.model.data
        man = {"format": FORMAT_VERSION, "model": self.model.model_name, "U": int(data.user_num), "I": int(data.item_num),
               "d": self.d, "N": self.n, "world": int(self.world),
               "pairs_fingerprint": checkpoint.pairs_fingerprint(data.pair_users, data.pair_items),
               "score_dtype": np.dtype(self.score_dtype).name}
        _write_names(self.tmp, "items.txt", data.id2item, int(data.item_num))
        _write_names(self.tmp, "users.txt", data.id2user, int(data.user_num))
        with open(os.path.join(self.tmp, MANIFEST), "w") as f:
            json.dump(man, f, indent=1)
            f.flush()
            os.fsync(f.fileno())
        checkpoint._fsync_dir(self.tmp)
        checkpoint._publish(self.tmp, self.final)
        checkpoint._fsync_dir(self.out_dir)

    def abort(self):
        if self.rank == 0:
            shutil.rmtree(self.tmp, ignore_errors=True)


def long_list_chunk(chunk, n_items, d, n):
    """The largest chunk <= `chunk` whose tensor-core ranking workspace of lists of n stays under LONG_WS_BYTES
    (halving; at least 1)."""
    from . import _lib
    lib = _lib.load()
    while chunk > 1 and lib.srb_topk_workspace_bytes(chunk, n_items, d, n) > LONG_WS_BYTES:
        chunk //= 2
    return chunk


def _write_names(directory, fname, id2name, n):
    with open(os.path.join(directory, fname), "w") as f:
        for i in range(n):
            f.write(f"{id2name[i]}\n")
        f.flush()
        os.fsync(f.fileno())


def _fsync_file(path):
    fd = os.open(path, os.O_RDONLY)
    try:
        os.fsync(fd)
    finally:
        os.close(fd)


def _write_part(directory, g, uids, fn, n, score_dtype, chunk):
    """Rank the part's users chunk by chunk through fn(lo, hi) -> (ids, scores) device tensors and stream the lists
    into ids.<g>.npy / scores.<g>.npy: device -> pinned host buffer on a side stream, then into the memory map while
    the device ranks the next chunk."""
    import torch
    m = len(uids)
    checkpoint.write_array(directory, f"users.{g}.npy", np.asarray(uids, dtype=np.int64))
    ids_path, sc_path = os.path.join(directory, f"ids.{g}.npy"), os.path.join(directory, f"scores.{g}.npy")
    if m == 0:
        checkpoint.write_array(directory, f"ids.{g}.npy", np.empty((0, n), np.int32))
        checkpoint.write_array(directory, f"scores.{g}.npy", np.empty((0, n), score_dtype))
        return
    ids_mm = np.lib.format.open_memmap(ids_path, mode="w+", dtype=np.int32, shape=(m, n))
    sc_mm = np.lib.format.open_memmap(sc_path, mode="w+", dtype=score_dtype, shape=(m, n))
    rows = min(chunk, m)
    tdt = torch.float64 if score_dtype == np.float64 else torch.float32
    bufs = [(torch.empty((rows, n), dtype=torch.int32, pin_memory=True), torch.empty((rows, n), dtype=tdt, pin_memory=True))
            for _ in range(2)]
    main, side = torch.cuda.current_stream(), torch.cuda.Stream()
    pending = None

    def flush(p):
        ev, (hi_ids, hi_sc), lo, hi = p
        ev.synchronize()
        ids_mm[lo:hi] = hi_ids[: hi - lo].numpy()
        sc_mm[lo:hi] = hi_sc[: hi - lo].numpy()

    for k, lo in enumerate(range(0, m, chunk)):
        hi = min(m, lo + chunk)
        ids_d, sc_d = fn(lo, hi)  # enqueued on the current stream
        buf = bufs[k % 2]        # last used by chunk k - 2, already flushed
        side.wait_stream(main)
        with torch.cuda.stream(side):
            buf[0][: hi - lo].copy_(ids_d, non_blocking=True)
            buf[1][: hi - lo].copy_(sc_d, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(side)
        ids_d.record_stream(side)
        sc_d.record_stream(side)
        if pending is not None:
            flush(pending)       # the host writes chunk k - 1 while the device ranks chunk k
        pending = (ev, buf, lo, hi)
    flush(pending)
    ids_mm.flush()
    sc_mm.flush()
    del ids_mm, sc_mm
    _fsync_file(ids_path)
    _fsync_file(sc_path)


def run(jobs, agree):
    """The three phases of every job of this process, each followed by agree(ok) across the process group."""
    def phase(step):
        err = None
        try:
            for j in jobs:
                getattr(j, step)()
        except BaseException as e:  # noqa: BLE001 -- re-raised below, after the other ranks have heard of it
            err = e
        ok = agree(err is None)
        if err is not None:
            raise err
        if not ok:
            raise SrbError("export: another rank failed; nothing was published")

    phase("begin")
    try:
        phase("write")
        phase("finish")
    except BaseException:
        for j in jobs:
            j.abort()
        raise
    return jobs[0].final


def export_recommendations(model, out_dir, top_n=None, users=None, chunk=None):
    """Write the top-N lists of `users` (names; default every training user) of a trained model under out_dir and
    return the export's path.  Collective for a sharded model under a process group; a model that is not sharded is
    exported by the main process alone."""
    if getattr(model, "shard_ranker", None) is None and process_group() is not None and not is_main_process():
        return os.path.join(out_dir, export_name(model.model_name, model.max_N if top_n is None else top_n))
    job = _Job(model, out_dir, top_n, users, chunk)
    return run([job], job.agree)


def read(path):
    """(user names [n], ids int32 [n, N], scores [n, N]) of an export, users in ascending global id order.  With one
    part ids and scores are the memory-mapped files; parts of a sharded export are merged into memory."""
    with open(os.path.join(path, MANIFEST)) as f:
        man = json.load(f)
    if man.get("format") != FORMAT_VERSION:
        raise SrbError(f"{path}: export format {man.get('format')} (this reader reads {FORMAT_VERSION})")
    with open(os.path.join(path, "users.txt")) as f:
        user_names = f.read().split("\n")[: man["U"]]
    load = lambda name: np.load(os.path.join(path, name), mmap_mode="r")
    parts = [(load(f"users.{g}.npy"), load(f"ids.{g}.npy"), load(f"scores.{g}.npy")) for g in range(man["world"])]
    if len(parts) == 1:
        uids, ids, scores = parts[0]
    else:
        uids = np.concatenate([p[0] for p in parts])
        order = np.argsort(uids, kind="stable")
        uids = uids[order]
        ids = np.concatenate([p[1] for p in parts])[order]
        scores = np.concatenate([p[2] for p in parts])[order]
    return [user_names[int(u)] for u in uids], ids, scores


def read_items(path):
    """Item names by id (items.txt)."""
    with open(os.path.join(path, "items.txt")) as f:
        return f.read().split("\n")[:-1]
