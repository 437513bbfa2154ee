"""Time ItemKNN and UserKNN on the GPU: train() (host inputs, copies and the neighbour-table kernel), the kernel alone
(CUDA events), and a full test() (float64 score rows and the find_k_largest replay for every user, lists copied to the
host), with the peak device memory of each, at the douban-book, yelp2018 and amazon-kindle shapes (synth.make_interaction)
or on a real training file.  Prints the card's name and power limit, then one JSON line per (shape, model).

    python tools/knn_probe.py [--shapes douban-book,yelp2018,amazon-kindle] [--train FILE] [--topk 50] [--shrinkage 100]
                              [--max-n 20] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def probe(name, data, topk, shrinkage, max_n):
    import numpy as np
    import torch
    from selfrec_b200 import ops
    from selfrec_b200.knn import NeighbourTable, insertion_csr, name_ranks, transpose_csr
    out = []
    uids = np.arange(data.user_num, dtype=np.int32)
    for model, by in (("ItemKNN", "item"), ("UserKNN", "user")):
        NeighbourTable(data, by, topk, shrinkage)  # warm-up: module load, allocator
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        t0 = time.perf_counter()
        t = NeighbourTable(data, by, topk, shrinkage)
        torch.cuda.synchronize()
        train_s = time.perf_counter() - t0
        train_peak = torch.cuda.max_memory_allocated() - base
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        # the kernel alone, on the same device inputs
        sp, si = insertion_csr(data.pair_users, data.pair_items, data.user_num, data.item_num)
        tp, ti = transpose_csr(sp, si, data.item_num)
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).cuda()
        a, b = ((tp, ti), (sp, si)) if by == "item" else ((sp, si), (tp, ti))
        args = (dev(a[0]), dev(a[1]), dev(b[0]), dev(b[1]), dev(name_ranks(t.names)), topk, shrinkage)
        ops.knn_neighbors(*args)
        e0.record()
        ops.knn_neighbors(*args)
        e1.record()
        torch.cuda.synchronize()
        kernel_ms = e0.elapsed_time(e1)
        del args
        t.rank(uids[:64], max_n)  # warm-up
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        t0 = time.perf_counter()
        ids, sc = t.rank(uids, max_n)
        torch.cuda.synchronize()
        test_s = time.perf_counter() - t0
        test_peak = torch.cuda.max_memory_allocated() - base
        deg_u = np.diff(sp).astype(np.int64)
        deg_i = np.diff(tp).astype(np.int64)
        out.append(dict(shape=name, model=model, U=int(data.user_num), I=int(data.item_num), nnz=int(len(si)), topK=topk,
                        shrinkage=shrinkage, max_N=max_n, accumulations=int((deg_u ** 2).sum() if by == "item" else (deg_i ** 2).sum()),
                        train_s=round(train_s, 4), neighbors_kernel_ms=round(kernel_ms, 3), train_peak_MB=round(train_peak / 2 ** 20, 1),
                        test_users=int(len(uids)), test_s=round(test_s, 4), test_peak_MB=round(test_peak / 2 ** 20, 1)))
        del t, ids, sc
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="douban-book,yelp2018,amazon-kindle")
    ap.add_argument("--train", default=None, help="a training file in the reference's format instead of the synthetic shapes")
    ap.add_argument("--topk", type=int, default=50)
    ap.add_argument("--shrinkage", type=int, default=100)
    ap.add_argument("--max-n", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from selfrec_b200 import _lib, synth
    _lib.require_device()
    torch.cuda.set_device(0)
    print("card:", card(), flush=True)
    if args.train:
        from selfrec_b200.data.native import NativeInteraction
        cases = [(os.path.basename(args.train), lambda: NativeInteraction(None, args.train))]
    else:
        cases = [(s, lambda s=s: synth.make_interaction(s, seed=0)) for s in args.shapes.split(",")]
    results = []
    for name, make in cases:
        data = make()
        for r in probe(name, data, args.topk, args.shrinkage, args.max_n):
            r["card"] = card()
            print(json.dumps(r), flush=True)
            results.append(r)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
