"""Embedding width on the yelp2018 shape: XSimGCL and LightGCN steps/s, workspace size and full-catalogue rank time at
the widths of --dims (any of 16, 32, 64, 128, 256), with the card's name and power limit read in the same run.  One
JSON line on stdout.

    python tools/wide_probe.py [--dims 64,128,256] [--window 1.0]

Steps: 64 pre-sampled batches resident in HBM, one captured step replayed (CUDA graph), warm-up replays, then a window
of at least --window seconds bracketed by CUDA events.  Ranking: ops.score_topk over every user with the rated mask,
top-20 (impl 0 picks the tensor-core kernel at d = 64 and the exact CUDA-core kernel elsewhere), same timing.  The
"algorithmic" fields are computed from the shapes, not measured: compulsory bytes of one SpMM and of the XSimGCL step
(3 forward + 3 backward products and Adam), InfoNCE FLOP of the first batch, ranking FLOP, and the least time each
needs at the data sheet's 3.35 TB/s and 67 TFLOP/s FP32 (H100 SXM, 700 W)."""
import argparse
import json
import os
import random
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BPS, FP32_FLOPS = 3.35e12, 67e12
L, B, LR, REG = 3, 2048, 1e-3, 1e-4
XS = dict(eps=0.2, tau=0.2, cl_rate=0.2, layer_cl=1)


def card():
    import torch
    out = dict(device=torch.cuda.get_device_name(0))
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        out.update(power_limit_w=float(q[0]), sm_max_mhz=float(q[1]))
    except Exception as e:  # noqa: BLE001 -- the probe still reports what it measured
        out.update(power_limit_w=None, power_limit_error=str(e))
    return out


def timed(fn, window_s, torch):
    """Mean ms per call of fn over a window of at least window_s seconds (CUDA events), after three warm-up calls."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    est = max(e0.elapsed_time(e1), 1e-3)
    while True:  # a first call is slower than the steady state: grow the count until the window is long enough
        n = max(10, int(window_s * 1e3 / est * 1.1) + 1)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        if ms >= window_s * 1e3:
            return ms / n, n, ms
        est = ms / n


def steps_per_s(model, data, d, window_s, torch):
    from selfrec_b200.engine import TrainEngine
    random.seed(1234)
    torch.manual_seed(1234)
    kw = XS if model == "XSimGCL" else dict(l2_div=float(B))
    eng = TrainEngine(model, data, d, L, B, LR, REG, philox_seed=2026, **kw)
    pool = torch.from_numpy(np.stack([w.copy() for _, w in zip(range(64), eng.batches())])).cuda()
    eng.batch_dev.copy_(pool[0])
    graph = eng.capture()
    k = [0]

    def step():
        eng.batch_dev.copy_(pool[k[0] % 64], non_blocking=True)
        graph.replay()
        k[0] += 1

    ms, n, win = timed(step, window_s, torch)
    assert np.isfinite(eng.losses.cpu().numpy()).all()
    first = pool[0].cpu().numpy()
    out = dict(steps_per_s=1e3 / ms, ms_per_step=ms, steps_timed=n, window_ms=win, workspace_bytes=int(eng.workspace.numel()))
    return out, eng, (int(first[1]), int(first[2]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dims", default="64,128,256")
    ap.add_argument("--window", type=float, default=1.0)
    args = ap.parse_args()
    import torch
    from selfrec_b200 import _lib, build, ops, synth
    build.build()
    _lib.require_device()
    torch.cuda.set_device(0)
    data = synth.make_interaction("yelp2018")
    U, I = int(data.user_num), int(data.item_num)
    N, nnz = U + I, int(data.norm_adj.nnz)
    rp, ri = data.rated_csr()
    rp_d, ri_d = torch.from_numpy(rp).cuda(), torch.from_numpy(ri).cuda()
    users = torch.arange(U, device="cuda", dtype=torch.int32)
    res = dict(probe="wide_probe", shape=f"yelp2018 {U}x{I}, {nnz} adjacency non-zeros", L=L, B=B, **card(), widths={})
    for d in (int(x) for x in args.dims.split(",")):
        row = {}
        row["LightGCN"], _, _ = steps_per_s("LightGCN", data, d, args.window, torch)
        row["XSimGCL"], eng, (nu, ni) = steps_per_s("XSimGCL", data, d, args.window, torch)
        ue, ie = eng.forward_clean()
        impl = 2 if d == 64 else 1
        rank_ms, n, _ = timed(lambda: ops.score_topk(ue, ie, users, rp_d, ri_d, 20, impl=impl), args.window, torch)
        row["rank"] = dict(ms=rank_ms, impl=impl, calls_timed=n, users=U, items=I, k=20)
        del eng, ue, ie
        torch.cuda.empty_cache()
        spmm = 2 * N * d * 4 + nnz * 8 + (N + 1) * 4
        adam = 7 * N * d * 4
        step = 6 * spmm + adam
        nce = 8 * d * (nu * nu + ni * ni)
        rank = 2 * U * I * d
        row["algorithmic"] = dict(spmm_bytes=spmm, x_table_bytes=N * d * 4, gather_bytes=nnz * d * 4, adam_bytes=adam,
                                  xsimgcl_step_bytes=step, xsimgcl_step_floor_us=step / HBM_BPS * 1e6, infonce_flop=nce,
                                  infonce_floor_us=nce / FP32_FLOPS * 1e6, rank_flop=rank, rank_floor_ms=rank / FP32_FLOPS * 1e3,
                                  first_batch_unique=(nu, ni))
        res["widths"][str(d)] = row
        print(f"d={d}: {json.dumps(row)}", file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
