"""Time batch_softmax_loss forward + backward (ops.batch_softmax_loss, srb_batch_softmax_fwd_bwd) against its torch
restatement (util/loss_torch.py:25-32 under autograd) at n = 2048 (SSL4Rec's batch size), d = 64 and 128, tau = 0.07
(SSL4Rec's) and 0.2.  d = 64 takes the tensor-core route at these taus, d = 128 the CUDA-core kernels.  CUDA events
over --reps calls after --warmup calls, in windows of at least --min-ms; the two are timed alternately, twice each.
Each line also gives the loss of both and their relative difference.  Prints the card's name and power limit, then
one JSON line per measurement.

    python tools/batch_softmax_probe.py [--reps 200] [--warmup 20] [--min-ms 1000]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from export_probe import card  # noqa: E402


def torch_batch_softmax_loss(user_emb, item_emb, temperature):
    import torch
    import torch.nn.functional as F
    user_emb, item_emb = F.normalize(user_emb, dim=1), F.normalize(item_emb, dim=1)
    pos_score = torch.exp((user_emb * item_emb).sum(dim=-1) / temperature)
    ttl_score = torch.exp(torch.matmul(user_emb, item_emb.transpose(0, 1)) / temperature).sum(dim=1)
    return torch.mean(-torch.log(pos_score / ttl_score + 10e-6))


def time_ms(fn, reps, warmup, min_ms):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    while True:
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        if ms >= min_ms:
            return ms / reps, reps
        reps *= 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--min-ms", type=float, default=1000.0)
    args = ap.parse_args()
    import torch
    from selfrec_b200 import ops
    print("card:", card(), flush=True)
    n = 2048
    g = torch.Generator(device="cuda").manual_seed(0)
    for d in (64, 128):
        for tau in (0.07, 0.2):
            u = (torch.randn((n, d), device="cuda", generator=g) * 0.1).requires_grad_(True)
            i = (u.detach() + 0.05 * torch.randn((n, d), device="cuda", generator=g)).requires_grad_(True)

            def step(fn):
                loss = fn(u, i, tau)
                loss.backward()
                return loss

            mine, ref = step(ops.batch_softmax_loss).item(), step(torch_batch_softmax_loss).item()
            times = {"kernels": [], "torch": []}
            for _ in range(2):
                for name, fn in (("kernels", ops.batch_softmax_loss), ("torch", torch_batch_softmax_loss)):
                    times[name].append(time_ms(lambda: step(fn), args.reps, args.warmup, args.min_ms))
            row = dict(what="batch_softmax_fwd_bwd", n=n, d=d, tau=tau, route="tensor_cores" if d == 64 and tau >= 1 / 40 else "cuda_cores",
                       kernels_ms=[round(t, 4) for t, _ in times["kernels"]], torch_ms=[round(t, 4) for t, _ in times["torch"]],
                       reps=[r for _, r in times["kernels"] + times["torch"]], loss=mine, torch_loss=ref,
                       rel_diff=abs(mine - ref) / abs(ref))
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
