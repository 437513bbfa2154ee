"""Generate tests/golden/*.npz by running the REFERENCE itself (imported from a checkout of it).

    python oracle/gen_golden.py --ref <reference checkout> [--out tests/golden]

The reference has no tests and seeds nothing (SURVEY 4), so the golden vectors are produced
here: a small synthetic dataset is written in the reference's text format, the reference's
own modules are imported unmodified and driven with fixed seeds, and inputs + outputs are
stored.  Harness-side shims only (no edits to the reference): cwd = scratch dir holding the
dataset and ./log; Tensor.cuda / Module.cuda patched to identity (the reference hard-codes
.cuda(), XSimGCL.py:24,46-47,73,90); torch.rand_like hooked so the noise becomes a recorded
input.  Versions and seeds are written into each fixture.
"""
import argparse
import os
import random
import sys
import tempfile

import numpy as np

SEED = 20260923


def make_dataset(rng, n_users=48, n_items=60, n_train=520, n_test=120, dup=3):
    """Power-law-ish bipartite interactions; string ids deliberately NOT equal to internal ids."""
    users = [f"u{1000 + 7 * k}" for k in range(n_users)]
    items = [f"i{500 + 3 * k}" for k in range(n_items)]
    pu = rng.zipf(1.4, size=4 * n_train) % n_users
    pi = rng.zipf(1.3, size=4 * n_train) % n_items
    pairs, seen = [], set()
    for a, b in zip(pu, pi):
        if (a, b) not in seen:
            seen.add((a, b))
            pairs.append((a, b))
    for u in range(n_users):  # every user and item appears
        if not any(p[0] == u for p in pairs):
            pairs.append((u, int(rng.integers(n_items))))
    for i in range(n_items):
        if not any(p[1] == i for p in pairs):
            pairs.append((int(rng.integers(n_users)), i))
    rng.shuffle(pairs)
    train = pairs[:n_train] + pairs[:dup]  # a few duplicate lines (amazon-kindle has them)
    rest = pairs[n_train:n_train + n_test]
    test = rest + [(n_users + 5, 2)]  # a test user unknown to training is filtered (ui_graph.py:43)
    fmt = lambda ps: [f"{users[a] if a < n_users else 'ghost'} {items[b]} {int(rng.integers(1, 6))}\n" for a, b in ps]
    return fmt(train), fmt(test)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", required=True, help="root of a Coder-Yu/SELFRec checkout")
    ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden"))
    args = ap.parse_args()
    out = os.path.abspath(args.out)
    os.makedirs(out, exist_ok=True)
    scratch = tempfile.mkdtemp(prefix="srb_golden_")
    os.makedirs(os.path.join(scratch, "dataset", "tiny"))
    rng = np.random.default_rng(SEED)
    train_lines, test_lines = make_dataset(rng)
    with open(os.path.join(scratch, "dataset", "tiny", "train.txt"), "w") as f:
        f.writelines(train_lines)
    with open(os.path.join(scratch, "dataset", "tiny", "test.txt"), "w") as f:
        f.writelines(test_lines)
    # the dataset itself is a fixture (tests rebuild everything from it)
    with open(os.path.join(out, "tiny_train.txt"), "w") as f:
        f.writelines(train_lines)
    with open(os.path.join(out, "tiny_test.txt"), "w") as f:
        f.writelines(test_lines)

    os.chdir(scratch)
    sys.path.insert(0, args.ref)
    import torch

    torch.set_num_threads(1)
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.nn.Module.cuda = lambda self, *a, **k: self
    import scipy
    import numba

    meta = dict(torch=torch.__version__, numpy=np.__version__, scipy=scipy.__version__, numba=numba.__version__,
                python=sys.version.split()[0], seed=SEED)

    from data.loader import FileIO
    from data.ui_graph import Interaction
    from util.conf import ModelConf

    def conf_for(model, extra):
        cfg = {
            "training.set": "./dataset/tiny/train.txt", "test.set": "./dataset/tiny/test.txt",
            "model": {"name": model, "type": "graph"}, "item.ranking.topN": [5, 10], "embedding.size": 64,
            "max.epoch": 1, "batch.size": 128, "learning.rate": 0.001, "reg.lambda": 0.0001, "output": "./results/",
        }
        if extra is not None:
            cfg[model] = extra
        c = ModelConf.__new__(ModelConf)
        c.config = cfg
        return c

    training = FileIO.load_data_set("./dataset/tiny/train.txt", "graph")
    test = FileIO.load_data_set("./dataset/tiny/test.txt", "graph")

    # ---------------- R2: Interaction -------------------------------------------------
    data = Interaction(conf_for("MF", None), [list(t) for t in training], [list(t) for t in test])
    na = data.norm_adj.tocsr()
    na.sort_indices()
    ua = data.ui_adj.tocsr()
    ua.sort_indices()
    im = data.interaction_mat.tocsr()
    im.sort_indices()
    np.savez_compressed(
        os.path.join(out, "graph.npz"), meta=str(meta), user_num=data.user_num, item_num=data.item_num,
        user_names=np.array([data.id2user[k] for k in range(data.user_num)]),
        item_names=np.array([data.id2item[k] for k in range(data.item_num)]),
        norm_indptr=na.indptr, norm_indices=na.indices, norm_data=na.data,
        ui_indptr=ua.indptr, ui_indices=ua.indices, ui_data=ua.data,
        im_indptr=im.indptr, im_indices=im.indices, im_data=im.data,
        test_users=np.array(list(data.test_set)), test_sizes=np.array([len(data.test_set[u]) for u in data.test_set]),
        sizes=np.array(list(data.training_size()) + list(data.test_size())),
    )

    # ---------------- R1: sampler -------------------------------------------------------
    from util.sampler import next_batch_pairwise

    sdata = Interaction(conf_for("MF", None), [list(t) for t in training], [list(t) for t in test])
    random.seed(4242)
    rec = {}
    for epoch in range(2):  # the shuffle persists across epochs (sampler.py:7)
        us, is_, js = [], [], []
        for u, i, j in next_batch_pairwise(sdata, 100):
            us.append(u), is_.append(i), js.append(j)
        rec[f"e{epoch}_u"] = np.concatenate(us)
        rec[f"e{epoch}_i"] = np.concatenate(is_)
        rec[f"e{epoch}_j"] = np.concatenate(js)
        rec[f"e{epoch}_sizes"] = np.array([len(x) for x in us])
    us, is_, js = [], [], []
    for u, i, j in next_batch_pairwise(sdata, 64, n_negs=3):
        us.append(u), is_.append(i), js.append(j)
    rec["n3_u"], rec["n3_i"], rec["n3_j"] = np.concatenate(us), np.concatenate(is_), np.concatenate(js)
    rec["final_state"] = np.array(random.getstate()[1], dtype=np.uint32)
    rec["final_order_users"] = np.array([sdata.user[p[0]] for p in sdata.training_data])
    rec["final_order_items"] = np.array([sdata.item[p[1]] for p in sdata.training_data])
    np.savez_compressed(os.path.join(out, "sampler.npz"), meta=str(meta), seed=4242, **rec)

    # ---------------- R6-R8: losses + autograd ------------------------------------------
    from util.loss_torch import InfoNCE, bpr_loss, l2_reg_loss

    torch.manual_seed(7)
    lo = {}
    for tag, (b, d) in {"a": (37, 64), "b": (128, 32)}.items():
        u, p, n = (torch.randn(b, d, requires_grad=True) for _ in range(3))
        loss = bpr_loss(u, p, n)
        gu, gp, gn = torch.autograd.grad(loss, (u, p, n))
        lo.update({f"bpr_{tag}_u": u.detach().numpy(), f"bpr_{tag}_p": p.detach().numpy(), f"bpr_{tag}_n": n.detach().numpy(),
                   f"bpr_{tag}_loss": loss.item(), f"bpr_{tag}_gu": gu.numpy(), f"bpr_{tag}_gp": gp.numpy(), f"bpr_{tag}_gn": gn.numpy()})
        l2 = l2_reg_loss(1e-2, u, p, n)
        g2 = torch.autograd.grad(l2, (u, p, n))
        lo.update({f"l2_{tag}_loss": l2.item(), f"l2_{tag}_gu": g2[0].numpy(), f"l2_{tag}_gp": g2[1].numpy(), f"l2_{tag}_gn": g2[2].numpy()})
    for tag, (n_, d, tau, cos) in {"a": (50, 64, 0.2, True), "b": (131, 64, 0.15, True), "c": (64, 32, 0.5, False), "d": (1, 64, 0.2, True)}.items():
        v1 = (0.1 * torch.randn(n_, d)).requires_grad_(True)
        v2 = (0.1 * torch.randn(n_, d)).requires_grad_(True)
        loss = InfoNCE(v1, v2, tau, cos)
        g1, g2 = torch.autograd.grad(loss, (v1, v2))
        lo.update({f"nce_{tag}_v1": v1.detach().numpy(), f"nce_{tag}_v2": v2.detach().numpy(), f"nce_{tag}_tau": tau, f"nce_{tag}_cos": cos,
                   f"nce_{tag}_loss": loss.item(), f"nce_{tag}_g1": g1.numpy(), f"nce_{tag}_g2": g2.numpy()})
    np.savez_compressed(os.path.join(out, "losses.npz"), meta=str(meta), **lo)

    # ---------------- R3/R4/R10: encoders and whole train steps ---------------------------
    import importlib

    noise_log = []
    real_rand_like = torch.rand_like
    noise_gen = torch.Generator().manual_seed(99)

    def rand_like_hook(t, *a, **k):
        nz = torch.rand(t.shape, generator=noise_gen, dtype=t.dtype)
        noise_log.append(nz.numpy().copy())
        return nz

    torch.rand_like = rand_like_hook

    model_cfg = {
        "MF": None,
        "LightGCN": {"n_layer": 3},
        "SimGCL": {"n_layer": 2, "lambda": 0.5, "eps": 0.1},
        "XSimGCL": {"n_layer": 3, "l_star": 1, "lambda": 0.2, "eps": 0.2, "tau": 0.2},
        "SGL": {"n_layer": 2, "lambda": 0.1, "drop_rate": 0.1, "aug_type": 1, "temp": 0.2},
    }
    n_steps = 3
    for name, extra in model_cfg.items():
        mod = importlib.import_module(f"model.graph.{name}")
        cls = getattr(mod, name)
        random.seed(1000 + len(name))
        torch.manual_seed(2000 + len(name))
        noise_log.clear()
        m = cls(conf_for(name, extra), [list(t) for t in training], [list(t) for t in test])
        enc = m.model
        init_u = enc.embedding_dict["user_emb"].detach().numpy().copy()
        init_i = enc.embedding_dict["item_emb"].detach().numpy().copy()
        fx = dict(meta=str(meta), init_user=init_u, init_item=init_i, n_steps=n_steps,
                  cfg=str(extra), batch_size=128, lr=0.001, reg=0.0001)
        # clean forward of the freshly initialised encoder
        with torch.no_grad():
            outs = enc() if name != "MF" else enc()
        fx["clean_user"], fx["clean_item"] = outs[0].detach().numpy().copy(), outs[1].detach().numpy().copy()

        batches, losses, params = [], [], []
        orig_sampler = mod.next_batch_pairwise

        def limited(data_, bs, n_negs=1, _orig=orig_sampler):
            for k, b in enumerate(_orig(data_, bs, n_negs)):
                if k >= n_steps:
                    return
                batches.append([np.array(x) for x in b])
                yield b

        mod.next_batch_pairwise = limited
        for fn_name in ("bpr_loss", "l2_reg_loss", "InfoNCE"):
            if hasattr(mod, fn_name):
                def wrap(f, tag):
                    def g(*a, **k):
                        r = f(*a, **k)
                        losses.append((tag, float(r.detach())))
                        return r
                    return g
                setattr(mod, fn_name, wrap(getattr(mod, fn_name), fn_name))
        orig_step = torch.optim.Adam.step

        def step_hook(self_, *a, **k):
            r = orig_step(self_, *a, **k)
            params.append(np.concatenate([enc.embedding_dict["user_emb"].detach().numpy(), enc.embedding_dict["item_emb"].detach().numpy()]).copy())
            return r

        torch.optim.Adam.step = step_hook
        m.fast_evaluation = lambda epoch, _m=m: _m.save()
        view_graphs = []
        if name == "SGL":
            orig_aug = enc.random_graph_augment

            def aug_hook():
                from data.augmentor import GraphAugmentor
                dropped = GraphAugmentor.edge_dropout(enc.data.interaction_mat, enc.drop_rate)
                lap = enc.data.convert_to_laplacian_mat(dropped).tocsr()
                lap.sort_indices()
                view_graphs.append(lap)
                from base.torch_interface import TorchGraphInterface
                return TorchGraphInterface.convert_sparse_mat_to_tensor(lap)

            enc.random_graph_augment = aug_hook
        m.save()  # SGL only evaluates from epoch 5 on; make sure best_* exists
        noise_log.clear()
        m.train()
        torch.optim.Adam.step = orig_step
        mod.next_batch_pairwise = orig_sampler
        for k, b in enumerate(batches):
            fx[f"b{k}_u"], fx[f"b{k}_i"], fx[f"b{k}_j"] = b
        for k, p in enumerate(params):
            fx[f"params_after_{k}"] = p
        fx["loss_tags"] = np.array([t for t, _ in losses])
        fx["loss_vals"] = np.array([v for _, v in losses])
        if noise_log:
            # training noise only: the post-train clean forwards draw none (perturbed=False)
            fx["noise"] = np.stack(noise_log)
        for k, g in enumerate(view_graphs):
            fx[f"view{k}_indptr"], fx[f"view{k}_indices"], fx[f"view{k}_data"] = g.indptr, g.indices, g.data
        fx["final_user"], fx["final_item"] = m.user_emb.detach().numpy(), m.item_emb.detach().numpy()
        np.savez_compressed(os.path.join(out, f"train_{name}.npz"), **fx)
        print(name, "steps", len(params), "loss records", len(losses), "noise tensors", len(noise_log), "views", len(view_graphs))
        if name == "XSimGCL":
            keep_model = m
    torch.rand_like = real_rand_like

    # ---------------- R9: find_k_largest, test(), ranking_evaluation ------------------------
    from util.algorithm import find_k_largest
    from util.evaluation import ranking_evaluation

    r2 = np.random.default_rng(5)
    tk = {}
    cases = {
        "rand": r2.standard_normal(500).astype(np.float32),
        "ties": r2.integers(0, 6, 300).astype(np.float32),
        "survey": np.array([1, 3, 3, 3, 2, 3, 3, 0, 3, 3], dtype=np.float32),
        "const": np.zeros(64, dtype=np.float32),
        "masked": np.where(r2.random(200) < 0.4, -10e8, r2.standard_normal(200)).astype(np.float32),
        "asc": np.arange(100, dtype=np.float32),
        "desc": np.arange(100, dtype=np.float32)[::-1].copy(),
    }
    for tag, v in cases.items():
        for K in (3, 10, 20):
            ids, sc = find_k_largest(K, v)
            tk[f"{tag}_K{K}_ids"], tk[f"{tag}_K{K}_scores"] = np.array(ids), np.array(sc, dtype=np.float32)
        tk[f"{tag}_in"] = v
    np.savez_compressed(os.path.join(out, "topk.npz"), meta=str(meta), **tk)

    m = keep_model
    rec_list = m.test()
    users = list(rec_list)
    measure = ranking_evaluation(m.data.test_set, rec_list, [5, 10])
    np.savez_compressed(
        os.path.join(out, "rank.npz"), meta=str(meta), user_emb=m.user_emb.detach().numpy(), item_emb=m.item_emb.detach().numpy(),
        users=np.array(users), items=np.array([[it for it, _ in rec_list[u]] for u in users]),
        scores=np.array([[s for _, s in rec_list[u]] for u in users], dtype=np.float32), measure=np.array(measure),
    )
    print("golden fixtures written to", out)
    print("\n".join(f"{f}: {os.path.getsize(os.path.join(out, f))} B" for f in sorted(os.listdir(out))))


if __name__ == "__main__":
    main()
