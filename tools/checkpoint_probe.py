"""Time checkpoint save and load of a TrainEngine at the yelp2018 shape and at the config-5 shape (synthetic-5M).

For each shape: build the engine (SimGCL, L = 2; d = 64 at yelp2018, d = 128 at synthetic-5M as in the README's config-5 row),
run a few steps, then time, with the device idle:
  * state_dict()            device -> host copy of the tables and moments
  * checkpoint.save()       the .npy writes, fsyncs and the rename (save_engines(): the engine's own state only)
  * engine_state + load     memory-mapped reads into the engine's existing tensors
  * the sampler position    position() at the shape's pair count (the pair order composed from the epoch shuffles)
and prints one JSON line per shape with the sizes, the seconds, the GB/s and the filesystem the directory is on.
Usage: python tools/checkpoint_probe.py [--dir DIR] [--shapes yelp2018,synthetic-5M]   (DIR defaults to a temporary one)"""
import argparse
import json
import os
import random
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _fs(path):
    """(filesystem type, mount point) of `path` from /proc/mounts (longest matching mount point)."""
    best = ("?", "/")
    try:
        with open("/proc/mounts") as f:
            for line in f:
                dev, mnt, typ = line.split()[:3]
                if os.path.abspath(path).startswith(mnt) and len(mnt) >= len(best[1]):
                    best = (typ, mnt)
    except OSError:
        pass
    return best


def probe(shape, root):
    import numpy as np
    import torch
    from selfrec_b200 import checkpoint, synth
    from selfrec_b200.engine import TrainEngine
    dev = torch.device("cuda", 0)
    d = 64 if shape == "yelp2018" else 128
    data = synth.make_interaction(shape, seed=0) if shape == "yelp2018" else synth.make_device_interaction(shape, seed=0)
    random.seed(0)
    torch.manual_seed(0)
    eng = TrainEngine("SimGCL", data, d, 2, 2048, 1e-3, 1e-4, eps=0.1, tau=0.2, cl_rate=0.5, device=dev)
    eng.track_pair_order()  # what checkpoint.dir turns on: the sampler keeps the pair order
    gen = eng.batches()
    for _ in range(3):
        eng.step(next(gen))
    torch.cuda.synchronize()
    out = {"shape": shape, "U": eng.U, "I": eng.I, "d": d, "pairs": int(len(data.pair_users))}
    t0 = time.perf_counter()
    pos = eng.feed_state()
    out["position_s"] = time.perf_counter() - t0
    gen.close()
    t0 = time.perf_counter()
    st = eng.state_dict()
    out["state_dict_s"] = time.perf_counter() - t0
    nbytes = sum(a.nbytes for a in (*st["user"].values(), st["item_params"], *st["item"].values())) + pos["order"].nbytes
    out["bytes"] = int(nbytes)
    man = {"format": checkpoint.FORMAT_VERSION, "epoch": 0, "batch": 3, "cursor": int(pos["cursor"])}
    t0 = time.perf_counter()
    state = {"step": st["step"], "user_ids": st["user_ids"], "user": st["user"], "item_params": st["item_params"],
             "item_rows": st["item_rows"], "item": st["item"]}
    path = checkpoint.save(root, dict(man, U=eng.U, I=eng.I, d=d, step=st["step"], item_bounds=[0, eng.I]), {0: (state, None)},
                           {"item_params.npy": st["item_params"], "pair_order.npy": pos["order"]})
    out["save_s"] = time.perf_counter() - t0
    del st, state
    t0 = time.perf_counter()
    eng.load_state_dict(checkpoint.engine_state(path, checkpoint.read_manifest(path), np.arange(eng.U)))
    out["load_s"] = time.perf_counter() - t0
    out["save_GBps"] = nbytes / out["save_s"] / 1e9
    out["load_GBps"] = nbytes / out["load_s"] / 1e9  # page cache warm: the files were just written
    out["filesystem"], out["mount"] = _fs(root)
    out["gpu"] = torch.cuda.get_device_name(0)
    shutil.rmtree(path, ignore_errors=True)
    del eng, data
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir", default=None)
    ap.add_argument("--shapes", default="yelp2018,synthetic-5M")
    args = ap.parse_args()
    root = args.dir or tempfile.mkdtemp(prefix="srb-ckpt-probe-")
    try:
        for shape in args.shapes.split(","):
            print(json.dumps(probe(shape, os.path.join(root, shape))), flush=True)
    finally:
        if args.dir is None:
            shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
