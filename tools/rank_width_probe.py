"""Rank every user of the yelp2018 shape at embedding sizes 16, 32 and 256 (and 64 / 128 with --dims) on both routes:

* k = 20: the CUDA-core kernel (impl 1) against the tensor-core ranker (impl 2);
* k = 50, 100, 256: the dense-row route (ops._score_topk_wide, what impl 0 takes there) against impl 2.

Two kinds of tables per width: N(0, 0.1) and LightGCN's tables after --epochs epochs of the fused training step.  Per
case: the mean time of --reps calls after a warm-up call (CUDA events), the users impl 2's exact fallback re-ran,
whether both routes return the same scores, bit for bit, and in how many rows their ids differ (only possible among
exactly tied scores).  Prints the card's name and power limit first, then one JSON line per case.

    python tools/rank_width_probe.py [--dims 16,32,256] [--reps 5] [--epochs 3] [--ks 20,50,100,256]"""
import argparse
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from export_probe import card  # noqa: E402


def _time(fn, reps):
    import torch
    out = fn()  # warm-up
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1) / reps


def trained_tables(data, d, epochs):
    """LightGCN's final tables after `epochs` epochs of the fused step (batch 2048, lr 1e-3, reg 1e-4, 3 layers)."""
    import torch
    from selfrec_b200.engine import TrainEngine
    random.seed(1234)
    torch.manual_seed(1234)
    eng = TrainEngine("LightGCN", data, d, 3, 2048, 1e-3, 1e-4, philox_seed=2026, l2_div=2048.0)
    for _ in range(epochs):
        for words in eng.batches():
            eng.step(words)
    torch.cuda.synchronize()
    ue, ie = eng.forward_clean()
    return ue.contiguous(), ie.contiguous()


def measure(ue, ie, users, rp, ri, ks, reps, row):
    import torch
    from selfrec_b200 import ops
    for k in ks:
        st = {}
        (i2, s2), ms2 = _time(lambda: ops.score_topk(ue, ie, users, rp, ri, k, impl=2, stats=st), reps)
        if k <= 32:
            (i1, s1), ms1 = _time(lambda: ops.score_topk(ue, ie, users, rp, ri, k, impl=1), reps)
            other = "impl1"
        else:
            (i1, s1), ms1 = _time(lambda: ops._score_topk_wide(ue, ie, users, rp, ri, k), reps)
            other = "dense_rows"
        same_sc = bool(torch.equal(s1.view(torch.int32), s2.view(torch.int32)))
        # where the scores agree, ids can only differ among exactly tied items: the dense-row route selects 32 entries
        # at a time and may keep other tied items than find_k_largest (tests/test_gpu_rank_long.py)
        rows_ids_differ = int((i1 != i2).any(1).sum().item())
        print(json.dumps(dict(row, k=k, impl2_ms=ms2, **{f"{other}_ms": ms1}, impl2_fallback_users=int(st["fallback_count"].item()),
                              scores_equal=same_sc, rows_ids_differ=rows_ids_differ, reps=reps)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dims", default="16,32,256")
    ap.add_argument("--ks", default="20,50,100,256")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--epochs", type=int, default=3)
    args = ap.parse_args()
    import torch
    from selfrec_b200 import _lib, synth
    _lib.require_device()
    print(json.dumps(dict(card=card())), flush=True)
    data = synth.make_interaction("yelp2018", seed=0)
    U, I = data.user_num, data.item_num
    rp, ri = (torch.from_numpy(a).cuda() for a in data.rated_csr())
    users = torch.arange(U, dtype=torch.int32, device="cuda")
    ks = [int(x) for x in args.ks.split(",")]
    g = torch.Generator(device="cuda").manual_seed(0)
    for d in (int(x) for x in args.dims.split(",")):
        ue = torch.randn((U, d), device="cuda", generator=g) * 0.1
        ie = torch.randn((I, d), device="cuda", generator=g) * 0.1
        measure(ue, ie, users, rp, ri, ks, args.reps, dict(shape="yelp2018", users=U, items=I, d=d, tables="N(0,0.1)"))
        del ue, ie
        ue, ie = trained_tables(data, d, args.epochs)
        measure(ue, ie, users, rp, ri, ks, args.reps,
                dict(shape="yelp2018", users=U, items=I, d=d, tables=f"LightGCN, {args.epochs} epochs"))
        del ue, ie
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
