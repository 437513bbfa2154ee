"""Launched by torchrun (one rank per GPU) or directly (world 1): the bipartite-sharded SGL step must follow the
single-GPU fused engine on the same batches and the same two view graphs -- same losses, same Adam moments, same clean
forward within 1e-4 and no row off (SGL adds no noise) -- on a power-law graph and on a zipf graph whose blocks and views
have split rows, with edge- and node-dropout views, full and partial batches, and on every peer-store route (unicast
P2P, NVSwitch multicast and, at 2 ranks, the NVLS reduce-scatter)."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TOL = 1e-4
SGL_KW = dict(tau=0.2, cl_rate=0.1)


def view_graphs(data, kind, rate, seed, dev):
    """SGL's two dropped, re-normalised graphs (edge or node dropout at `rate`), drawn on the device from a seeded
    generator, so every rank builds the same two."""
    from selfrec_b200.data.device_graph import DeviceBipartite
    bip = data.bip if hasattr(data, "bip") else DeviceBipartite.from_interaction_mat(data.interaction_mat, dev)
    g = torch.Generator(device=dev).manual_seed(int(seed))
    out = []
    for _ in range(2):
        if kind == "edge":
            keep = torch.sort(torch.randperm(bip.nnz, generator=g, device=dev)[: int(bip.nnz * (1 - rate))]).values
            out.append(bip.assemble(keep_idx=keep, reset_weights=True))
        else:  # node dropout: every edge of a dropped user or item goes, leaving empty rows
            ku = (torch.rand(bip.U, generator=g, device=dev) >= rate).to(torch.uint8)
            ki = (torch.rand(bip.I, generator=g, device=dev) >= rate).to(torch.uint8)
            rows = torch.repeat_interleave(torch.arange(bip.U, device=dev), (bip.ui_ptr[1:] - bip.ui_ptr[:-1]).long())
            out.append(bip.assemble(keep_flags=ku[rows] & ki[bip.ui_col.long()], reset_weights=True))
    return out


def partial_batches(data, b, B, n, seed, dev=None):
    """n batch buffers of capacity B holding b < B rows each (an epoch's last batch)."""
    from selfrec_b200 import _lib
    from selfrec_b200.shard_check import device_batches
    H = _lib.BATCH_HEADER
    src = device_batches(data, b, n, seed=seed, dev=dev)
    out = torch.zeros((n, H + 5 * B), dtype=torch.int32, device=src.device)
    out[:, :H] = src[:, :H]
    for s in range(5):
        out[:, H + s * B: H + s * B + b] = src[:, H + s * b: H + (s + 1) * b]
    return out


# (graph, d, L, view kind, partial batch)
CASES = [("powerlaw", 64, 3, "edge", False), ("powerlaw", 32, 1, "node", False), ("powerlaw", 128, 2, "edge", True),
         ("zipf-split-rows", 64, 3, "edge", False), ("zipf-split-rows", 128, 1, "node", True), ("zipf-split-rows", 32, 2, "edge", False)]


def graphs():
    from selfrec_b200 import synth
    return {"powerlaw": synth.make_interaction((3000, 4000, 60000), seed=3),
            "zipf-split-rows": synth.make_device_interaction((30000, 8000, 1200000), seed=2, alpha=1.1)}


def main():
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank, local = int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    from selfrec_b200.shard_check import device_batches, sharded_vs_single
    ok = True
    routes = [None] if world == 1 else ([False, True, "nvls"] if world == 2 else [False, True])
    B = 512
    for gname, data in graphs().items():
        full = device_batches(data, B, 3, seed=5)
        part = partial_batches(data, 300, B, 3, seed=6)
        for g, d, L, kind, partial in CASES:
            if g != gname:
                continue
            views = view_graphs(data, kind, 0.1, seed=9, dev=dev)
            for mc in routes:
                route = {} if mc is None else dict(multicast=bool(mc), nvls=(mc == "nvls"))
                r = sharded_vs_single("SGL", data, d, L, B, part if partial else full, steps=3, views=views, **route, **SGL_KW)
                good = r["max_rel"] <= TOL and r["m_rows_off_frac"] == 0.0
                if rank == 0:
                    print(f"{gname} SGL d={d} L={L} {kind}-dropout views{' partial batch' if partial else ''} route={r['route']}: "
                          f"max_rel {r['max_rel']:.2e} rows off {r['m_rows_off_frac']:.1e} (loss {r['loss_rel']:.1e} "
                          f"m {r['m_user_rel']:.1e}/{r['m_item_rel']:.1e} v {r['v_user_rel']:.1e}/{r['v_item_rel']:.1e} "
                          f"final {r['final_user_rel']:.1e}/{r['final_item_rel']:.1e}) {'ok' if good else 'FAIL'}", flush=True)
                ok = ok and good
    if rank == 0:
        print("SHARDED_SGL_CHECK", "PASS" if ok else "FAIL", f"world={world}", flush=True)
    if world > 1:
        dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
