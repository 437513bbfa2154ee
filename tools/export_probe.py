"""Time the full-catalog ranker at embedding size 64 and 128 and the export of every user's top-N lists.

1. Rank every user of the yelp2018 shape (synth.make_interaction) with k = 20, for d = 64 / 128 x impl 1 (CUDA cores) /
   impl 2 (tensor cores), CUDA events over --reps calls after a warm-up call; for impl 2 also the number of users the
   exact fallback re-ran.  Both impls must return the same lists.
2. Export every user's top-N of a model of the --export-shape (default synthetic-5M: 5 M users x 1 M items, 100 M
   training pairs on the device) at d = 128 with random N(0, 0.1) tables: wall time, GB written, peak device memory
   (torch) and peak host memory (ru_maxrss) of the export.
Prints the card's name and power limit, then one JSON line per measurement.

    python tools/export_probe.py [--reps 5] [--export-shape synthetic-5M] [--top-n 20] [--out-dir DIR] [--skip-export]"""
import argparse
import json
import os
import resource
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def rank_times(reps):
    import numpy as np
    import torch
    from selfrec_b200 import ops, synth
    data = synth.make_interaction("yelp2018", seed=0)
    U, I = data.user_num, data.item_num
    rp, ri = (torch.from_numpy(a).cuda() for a in data.rated_csr())
    users = torch.arange(U, dtype=torch.int32, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    for d in (64, 128):
        ue = torch.randn((U, d), device="cuda", generator=g) * 0.1
        ie = torch.randn((I, d), device="cuda", generator=g) * 0.1
        lists = {}
        for impl in (1, 2):
            st = {}
            ids, sc = ops.score_topk(ue, ie, users, rp, ri, 20, impl=impl, stats=st)  # warm-up
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                ops.score_topk(ue, ie, users, rp, ri, 20, impl=impl)
            e1.record()
            torch.cuda.synchronize()
            lists[impl] = (ids.cpu().numpy(), sc.cpu().numpy())
            row = dict(what="rank_all_users", shape="yelp2018", users=U, items=I, d=d, k=20, impl=impl,
                       ms=e0.elapsed_time(e1) / reps, reps=reps)
            if impl == 2:
                row["fallback_users"] = int(st["fallback_count"].item())
            print(json.dumps(row), flush=True)
        same = np.array_equal(lists[1][0], lists[2][0]) and np.array_equal(lists[1][1].view(np.uint32), lists[2][1].view(np.uint32))
        print(json.dumps(dict(what="impl2_equals_impl1", d=d, equal=bool(same))), flush=True)
        del ue, ie


class _Names:
    def __getitem__(self, i):
        return str(i)


class _Model:
    """What export reads of a trained fused model: its data, tables and list length."""

    def __init__(self, data, user_emb, item_emb, n):
        self.data, self.user_emb, self.item_emb, self.max_N = data, user_emb, item_emb, n
        self.model_name, self.shard_ranker, self.neighbour_table = "SimGCL", None, None

    def _has_embedding_tables(self):
        return True


def export_time(shape, top_n, out_dir):
    import torch
    from selfrec_b200 import export, synth
    t0 = time.perf_counter()
    data = synth.make_device_interaction(shape, seed=0)
    data.id2user, data.id2item = _Names(), _Names()
    data.rated_csr(), data.pair_users  # host copies, as a trained model already has them
    U, I = data.user_num, data.item_num
    g = torch.Generator(device="cuda").manual_seed(1)
    ue = torch.randn((U, 128), device="cuda", generator=g) * 0.1
    ie = torch.randn((I, 128), device="cuda", generator=g) * 0.1
    data.bip = data.norm_adj = None  # a ranked model keeps only its tables and the rated lists
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    setup_s = time.perf_counter() - t0
    m = _Model(data, ue, ie, top_n)
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    rss0 = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss
    t0 = time.perf_counter()
    path = export.export_recommendations(m, out_dir, top_n=top_n)
    export_s = time.perf_counter() - t0
    nbytes = sum(os.path.getsize(os.path.join(path, f)) for f in os.listdir(path))
    print(json.dumps(dict(what="export", shape=shape, users=U, items=I, d=128, N=top_n, seconds=export_s, setup_seconds=setup_s,
                          gb_written=nbytes / 1e9, peak_device_gb_above_tables=(torch.cuda.max_memory_allocated() - base) / 1e9,
                          peak_host_rss_gb=resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1e6, host_rss_gb_before=rss0 / 1e6,
                          chunk=export.EXPORT_CHUNK)), flush=True)
    shutil.rmtree(path, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--export-shape", default="synthetic-5M")
    ap.add_argument("--top-n", type=int, default=20)
    ap.add_argument("--out-dir", default=None, help="where the export is written (default: a temporary directory), removed after")
    ap.add_argument("--skip-export", action="store_true")
    args = ap.parse_args()
    from selfrec_b200 import _lib
    _lib.require_device()
    print(json.dumps(dict(card=card())), flush=True)
    rank_times(args.reps)
    if not args.skip_export:
        out = args.out_dir or tempfile.mkdtemp(prefix="export_probe_")
        try:
            export_time(args.export_shape, args.top_n, out)
        finally:
            if args.out_dir is None:
                shutil.rmtree(out, ignore_errors=True)


if __name__ == "__main__":
    main()
