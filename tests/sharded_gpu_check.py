"""Launched by torchrun (one rank per GPU) or directly (world 1): the bipartite-sharded step must follow the
single-GPU fused engine -- same losses, same Adam moments, same clean forward -- on the same batches and the same
Philox noise, for XSimGCL, SimGCL and LightGCN, on both peer-store routes (unicast P2P and NVSwitch multicast) and, at
2 ranks, with the optional NVLS reduce-scatter (multimem.ld_reduce).

Two passes per case.  eps = 0: strict, every compared quantity within 1e-4.  eps as configured: the perturbation
sign(y) * noise * eps (XSimGCL.py:90-91) is discontinuous at y = 0, so an element within fp32 rounding of zero flips
under the sharded summation order (item rows are sums of per-rank partial sums); the losses must still agree to
1e-4 and only a small fraction of rows (the flipped ones and their neighbours) may differ."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TOL = 1e-4


def main():
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank, local = int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from selfrec_b200 import synth
    from selfrec_b200.shard_check import device_batches, sharded_vs_single
    ok = True
    cases = [("XSimGCL", 64, 3, dict(eps=0.2, tau=0.2, cl_rate=0.2, layer_cl=1)),
             ("XSimGCL", 64, 2, dict(eps=0.2, tau=0.2, cl_rate=0.2, layer_cl=2)),
             ("SimGCL", 128, 2, dict(eps=0.1, tau=0.2, cl_rate=0.5)),
             ("LightGCN", 64, 3, dict(l2_div=512.0)),
             # where the backward's second seed table G enters: XSimGCL at L = 1 gathers it in the only product, which
             # also applies Adam; LightGCN at L = 1 adds it at the ego level of that product; XSimGCL with layer_cl = 0
             # holds only view 2's gradient in G and adds it at the ego level
             ("XSimGCL", 64, 1, dict(eps=0.2, tau=0.2, cl_rate=0.2, layer_cl=1)),
             ("LightGCN", 64, 1, dict(l2_div=512.0)),
             ("XSimGCL", 64, 3, dict(eps=0.2, tau=0.2, cl_rate=0.2, layer_cl=0))]
    graphs = {"powerlaw": synth.make_interaction((3000, 4000, 60000), seed=3),
              "zipf-split-rows": synth.make_device_interaction((30000, 8000, 1200000), seed=2, alpha=1.1)}
    # P2P stores | multicast stores | + in-switch reduce-scatter (the optional NVLS route, exercised at 2 ranks)
    routes = [None] if world == 1 else ([False, True, "nvls"] if world == 2 else [False, True])
    for gname, data in graphs.items():
        B = 512
        batches = device_batches(data, B, 3, seed=5)
        for model, d, L, kw0 in cases:
            for mc, strict in [(m, s) for m in routes for s in ((True, False) if "eps" in kw0 else (True,))]:
                kw = dict(kw0, eps=0.0) if (strict and "eps" in kw0) else kw0
                r = sharded_vs_single(model, data, d, L, B, batches, steps=3, multicast=bool(mc), nvls=(mc == "nvls"), **kw) if mc is not None else \
                    sharded_vs_single(model, data, d, L, B, batches, steps=3, **kw)
                if strict:
                    good = r["max_rel"] <= TOL and r["m_rows_off_frac"] == 0.0
                else:
                    good = r["loss_rel"] <= TOL and r["m_rows_off_frac"] <= 0.05 and max(r["final_user_rel"], r["final_item_rel"]) <= 0.05
                if rank == 0:
                    print(f"{gname} {model} d={d} L={L} route={r['route']} {'eps=0 strict' if strict and 'eps' in kw0 else 'as configured'}: max_rel {r['max_rel']:.2e} rows off {r['m_rows_off_frac']:.1e} "
                          f"(loss {r['loss_rel']:.1e} m {r['m_user_rel']:.1e}/{r['m_item_rel']:.1e} v {r['v_user_rel']:.1e}/{r['v_item_rel']:.1e} "
                          f"final {r['final_user_rel']:.1e}/{r['final_item_rel']:.1e} params {r['user_rel']:.1e}/{r['item_rel']:.1e} "
                          f"updates off {r['upd_off_frac']:.1e}) {'ok' if good else 'FAIL'}",
                          flush=True)
                ok = ok and good
    if rank == 0:
        print("SHARDED_CHECK", "PASS" if ok else "FAIL", f"world={world}", flush=True)
    if world > 1:
        dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
