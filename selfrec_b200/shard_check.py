"""Parity of the bipartite-sharded step against the single-GPU engine, usable inside a run (bench.py prints the
result in its JSON line, tests assert on it): both engines get the same initial tables, Philox seed and batches,
so they compute the same trajectory up to fp32 summation order (the sharded item rows are sums of per-rank
partial sums)."""
import numpy as np


def max_rel(a, b):
    """max |a - b| / max |b| over a tensor pair (scale-relative: Adam's first steps move every entry by ~lr)."""
    import torch
    den = float(b.abs().max().item())
    return float((a - b).abs().max().item()) / max(den, 1e-30)


def sharded_vs_single(model, data, d, L, B, batches, *, steps=3, lr=1e-3, reg=1e-4, seed=7, dev=None, multicast=None, nvls=None, views=None,
                      **kw):
    """Collective over the default process group (or single-process).  Runs `steps` steps of ShardedEngine on all
    ranks and of TrainEngine on every rank (the reference replica), on batches[k] (device int32 rows).  views: SGL's two
    view graphs, given to both engines.
    Returns dict(loss_rel, m_*_rel, v_*_rel, final_*_rel, user_rel, item_rel, upd_off_frac, max_rel, ...) -- maxima
    over steps and ranks; max_rel covers the losses, the Adam moments and the clean forward."""
    import torch
    import torch.distributed as dist
    from .engine import TrainEngine
    from .sharded import ShardedEngine
    dev = torch.device("cuda", torch.cuda.current_device()) if dev is None else dev
    U, I = int(data.user_num), int(data.item_num)
    g = torch.Generator(device=dev).manual_seed(1234)
    iu = torch.empty((U, d), device=dev).uniform_(-0.1, 0.1, generator=g)
    ii = torch.empty((I, d), device=dev).uniform_(-0.1, 0.1, generator=g)
    sh = ShardedEngine(model, data, d, L, B, lr, reg, init_user=iu, init_item=ii, philox_seed=seed, device=dev, multicast=multicast, nvls=nvls, **kw)
    ref = TrainEngine(model, data, d, L, B, lr, reg, init_user=iu, init_item=ii, philox_seed=seed, device=dev, **kw)
    if views is not None:
        sh.set_view_graphs(*views)
        ref.set_view_graphs(*views)
    # Parity is asserted on well-conditioned quantities: the losses, Adam's first moment m (linear in the gradient:
    # after step 1, m = 0.1 g) and second moment, and the clean forward.  The PARAMETERS themselves are compared in two
    # ways that say what they mean: relative to the table (`user_rel` / `item_rel`), and as the fraction of entries
    # whose update differs by more than 5 % of lr -- Adam's first steps move every entry by ~lr * sign(g), so entries
    # whose gradient is within fp32 summation noise of zero legitimately flip (the sharded item rows are sums of
    # per-rank partial sums, a different order than the single-GPU row sum).
    out = dict(loss_rel=0.0, user_rel=0.0, item_rel=0.0, m_user_rel=0.0, m_item_rel=0.0, v_user_rel=0.0, v_item_rel=0.0, upd_off_frac=0.0,
               m_rows_off_frac=0.0)
    uid = sh.user_ids  # global ids of this rank's users (cyclic assignment)
    ilo, ihi = int(sh.ib[sh.rank]), int(sh.ib[sh.rank + 1])  # the item slice whose moments this rank owns
    for k in range(steps):
        w = batches[k % len(batches)]
        pu0, pi0 = sh.user_emb.clone(), sh.item_emb.clone()
        pr0 = ref.params.clone()
        ref.batch_dev.copy_(w)
        ref.step_resident()
        sh.step(words_dev=w)
        torch.cuda.synchronize()
        la, lb = sh.losses, ref.losses
        out["loss_rel"] = max(out["loss_rel"], float(((la - lb).abs() / lb.abs().clamp_min(1e-12)).max().item()))
        out["user_rel"] = max(out["user_rel"], max_rel(sh.user_emb, ref.params[uid]))
        out["item_rel"] = max(out["item_rel"], max_rel(sh.item_emb, ref.params[U:]))
        out["m_user_rel"] = max(out["m_user_rel"], max_rel(sh.mu, ref.m[uid]))
        out["m_item_rel"] = max(out["m_item_rel"], max_rel(sh.mi[ilo:ihi], ref.m[U + ilo:U + ihi]))
        # rows whose first moment is off by more than 1e-4 of the largest entry.  With eps > 0 a few are expected:
        # the perturbation is sign(y) * noise * eps (XSimGCL.py:90-91), and an element y that is within fp32 rounding
        # of zero takes the opposite sign under a different summation order (~1e-7 of the elements, i.e. a handful
        # per step at yelp2018 size); the flipped rows and their graph neighbours then differ by ~1 %
        off = 0
        for a_, b_ in ((sh.mu, ref.m[uid]), (sh.mi[ilo:ihi], ref.m[U + ilo:U + ihi])):
            off += int(((a_ - b_).abs().max(1).values > 1e-4 * float(b_.abs().max().item())).sum().item())
        out["m_rows_off_frac"] = max(out["m_rows_off_frac"], off / float(sh.Ug + (ihi - ilo)))
        out["v_user_rel"] = max(out["v_user_rel"], max_rel(sh.vu, ref.v[uid]))
        out["v_item_rel"] = max(out["v_item_rel"], max_rel(sh.vi[ilo:ihi], ref.v[U + ilo:U + ihi]))
        du = (sh.user_emb - pu0) - (ref.params[uid] - pr0[uid])
        di = (sh.item_emb - pi0) - (ref.params[U:] - pr0[U:])
        off = float(((du.abs() > 0.05 * lr).sum() + (di.abs() > 0.05 * lr).sum()).item()) / float(du.numel() + di.numel())
        out["upd_off_frac"] = max(out["upd_off_frac"], off)
        del pu0, pi0, pr0, du, di
    fu, fi = sh.forward_clean()
    ru, ri = ref.forward_clean()
    torch.cuda.synchronize()
    out["final_user_rel"] = max_rel(fu, ru[uid])
    out["final_item_rel"] = max_rel(fi, ri)
    sh.check_peers()
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        t = torch.tensor([out[k] for k in sorted(out)], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        out = {k: float(v) for k, v in zip(sorted(out), t.tolist())}
    out["world"] = sh.world
    out["route"] = ("nvls" if sh.use_nvls else "multicast") if sh.use_multicast else ("unicast" if sh.world > 1 else "single")
    out["steps"] = steps
    out["max_rel"] = max(out["loss_rel"], out["m_user_rel"], out["m_item_rel"], out["v_user_rel"], out["v_item_rel"],
                         out["final_user_rel"], out["final_item_rel"])
    del sh, ref
    torch.cuda.empty_cache()
    return out


def device_batches(data, B, n, seed=0, dev=None):
    """n batch buffers (srb_sampler_next_batch layout) sampled on the device: uniformly drawn training pairs,
    uniform negatives re-drawn (a few rounds) while they hit a rated item.  Identical on every rank for a seed."""
    import torch
    from . import _lib
    if hasattr(data, "pairs_dev"):
        pu, pi = data.pairs_dev
        rp, ri = data.rated_csr_device()
    else:
        dev = torch.device("cuda", torch.cuda.current_device()) if dev is None else dev
        pu, pi = torch.from_numpy(np.asarray(data.pair_users)).to(dev), torch.from_numpy(np.asarray(data.pair_items)).to(dev)
        rp, ri = (torch.from_numpy(a).to(dev) for a in data.rated_csr())
    dev = pu.device
    g = torch.Generator(device=dev).manual_seed(int(seed))
    H = _lib.BATCH_HEADER
    I = int(data.item_num)
    key = None
    out = torch.zeros((n, H + 5 * B), dtype=torch.int32, device=dev)
    for k in range(n):
        sel = torch.randint(0, pu.numel(), (B,), generator=g, device=dev)
        u, i = pu[sel].to(torch.int64), pi[sel].to(torch.int64)
        j = torch.randint(0, I, (B,), generator=g, device=dev)
        for _ in range(8):  # rejection rounds: is (u, j) a training pair?  (binary search in the user's sorted item list)
            lo, hi = rp[u].to(torch.int64), rp[u + 1].to(torch.int64)
            for _s in range(32):
                mid = (lo + hi) // 2
                go = (mid < hi) & (ri[mid.clamp(max=ri.numel() - 1)].to(torch.int64) < j)
                lo = torch.where(go, mid + 1, lo)
                hi = torch.where(go, hi, mid)
                if bool((lo >= hi).all()):
                    break
            hit = (lo < rp[u + 1].to(torch.int64)) & (ri[lo.clamp(max=ri.numel() - 1)].to(torch.int64) == j)
            if not bool(hit.any()):
                break
            j = torch.where(hit, torch.randint(0, I, (B,), generator=g, device=dev), j)
        uq, iq = torch.unique(u), torch.unique(i)
        w = out[k]
        w[0], w[1], w[2] = B, uq.numel(), iq.numel()
        w[H:H + B], w[H + B:H + 2 * B], w[H + 2 * B:H + 3 * B] = u.to(torch.int32), i.to(torch.int32), j.to(torch.int32)
        w[H + 3 * B:H + 3 * B + uq.numel()] = uq.to(torch.int32)
        w[H + 4 * B:H + 4 * B + iq.numel()] = iq.to(torch.int32)
    return out
