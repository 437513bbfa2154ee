#!/usr/bin/env python
"""Probe of the bipartite-sharded step at any world size (torchrun or plain python); prints one JSON line.

    [torchrun --nproc-per-node N] tools/shard_probe.py [shape] [--model SimGCL] [--d 128] [--steps 5] [--parity]
    tools/shard_probe.py amazon-kindle --model SGL --dim 64 --layers 3

SGL draws two edge-dropout views (--drop) on the device, the same on every rank.  At world 1 the probe also times the
single-GPU TrainEngine on the same graph, views and batches, alternating the two engines over --rounds rounds.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("shape", nargs="?", default="synthetic-2M")
    ap.add_argument("--model", default="SimGCL")
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--layers", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--alpha", type=float, default=1.1)
    ap.add_argument("--eager", action="store_true")
    ap.add_argument("--parity", action="store_true")
    ap.add_argument("--hubstats", action="store_true")
    ap.add_argument("--drop", type=float, default=0.1, help="SGL: edge dropout rate of the two views")
    ap.add_argument("--rounds", type=int, default=3, help="timed rounds (world 1: alternating with the single-GPU engine)")
    args = ap.parse_args()
    import torch
    import torch.distributed as dist
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank, local = int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)
    from selfrec_b200 import build, synth
    build.build()
    from selfrec_b200.shard_check import device_batches, sharded_vs_single
    from selfrec_b200.sharded import ShardedEngine
    rec = {"shape": args.shape, "model": args.model, "d": args.dim, "L": args.layers, "world": world, "gpu": torch.cuda.get_device_name(dev)}
    try:
        rec["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(local)],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        rec["power_limit"] = "unknown"
    t0 = time.perf_counter()
    if args.shape in ("yelp2018", "amazon-kindle", "douban-book"):
        data = synth.make_interaction(args.shape, seed=0)
    else:
        shape = synth.SHAPES[args.shape] if args.shape in synth.SHAPES else tuple(int(x) for x in args.shape.split("x"))
        data = synth.make_device_interaction(shape, seed=0, alpha=args.alpha, device=dev)
    torch.cuda.synchronize()
    rec["graph_s"] = time.perf_counter() - t0
    B = 2048
    kw = {"LightGCN": dict(l2_div=float(B)), "SGL": dict(tau=0.2, cl_rate=0.1)}.get(args.model, dict(eps=0.1, tau=0.2, cl_rate=0.5, layer_cl=1))
    views = None
    if args.model == "SGL":
        from selfrec_b200.data.device_graph import DeviceBipartite
        bip = data.bip if hasattr(data, "bip") else DeviceBipartite.from_interaction_mat(data.interaction_mat, dev)
        g = torch.Generator(device=dev).manual_seed(11)  # the same views on every rank
        views = [bip.assemble(keep_idx=torch.sort(torch.randperm(bip.nnz, generator=g, device=dev)[: int(bip.nnz * (1 - args.drop))]).values,
                              reset_weights=True) for _ in range(2)]
        rec.update(drop=args.drop, view_nnz=views[0].nnz, tau=0.2, cl_rate=0.1)
    pool = device_batches(data, B, 8, seed=3, dev=dev)
    if args.hubstats and rank == 0 and hasattr(data, "bip"):
        bip = data.bip
        for K in (128, 256, 432, 864, 2048):
            fi = float((bip.ui_col < K).float().mean().item())
            fu = float((bip.iu_col < K).float().mean().item())
            rec[f"share_cols_lt_{K}"] = {"item_cols_of_user_rows": fi, "user_cols_of_item_rows": fu}
    if args.parity:
        rec["parity"] = sharded_vs_single(args.model, data, args.dim, args.layers, B, pool, steps=3, dev=dev, views=views, **kw)
        torch.cuda.empty_cache()
    sh = ShardedEngine(args.model, data, args.dim, args.layers, B, 1e-3, 1e-4, device=dev, **kw)
    if views is not None:
        sh.set_view_graphs(*views)
    rec["mem_gb"] = torch.cuda.memory_allocated() / 1e9
    rec["nvlink_bytes_per_layer_out"] = sh.nvlink_bytes_per_layer()
    rec["route"] = "multicast" if sh.use_multicast else "unicast"
    rec["Ug"] = sh.Ug
    rec["nnz_Ru"], rec["nnz_Rt"] = sh.Ru.nnz, sh.Rt.nnz
    if not args.eager:
        sh.capture()
    ref = None
    if world == 1 and args.model == "SGL":  # the single-GPU engine on the same graph, views and batches
        from selfrec_b200.engine import TrainEngine
        ref = TrainEngine(args.model, data, args.dim, args.layers, B, 1e-3, 1e-4, device=dev, **kw)
        ref.set_view_graphs(*views)
        if not args.eager:
            ref.capture()

    def timed(eng):
        def step(k):
            eng.batch_dev.copy_(pool[k % pool.shape[0]], non_blocking=True)
            if eng.graph is not None:
                eng.graph.replay()
            else:
                eng.step_resident()

        for k in range(2):
            step(k)
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for k in range(args.steps):
            step(k)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    ms_sh, ms_ref = [], []
    for _ in range(args.rounds):
        ms_sh.append(timed(sh))
        if ref is not None:
            ms_ref.append(timed(ref))
    t = torch.tensor([statistics.median(ms_sh)], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    sh.check_peers()
    rec["step_ms"] = float(t.item())
    rec["step_ms_rounds"] = ms_sh
    rec["steps_per_s"] = 1e3 / rec["step_ms"]
    if ref is not None:
        rec["single_gpu_step_ms"] = statistics.median(ms_ref)
        rec["single_gpu_step_ms_rounds"] = ms_ref
    rec["loss"] = sh.losses.cpu().tolist()
    rec["mem_peak_gb"] = torch.cuda.max_memory_allocated() / 1e9
    if rank == 0:
        print(json.dumps(rec), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
