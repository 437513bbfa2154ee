"""The launcher flow on the sharded engine: `execute()` of LightGCN, XSimGCL, SimGCL and SGL, started by torchrun (any
world size, 1 included) after selfrec_b200.install(), against the same flow in one plain process (`--ref`, which
trains on TrainEngine and saves what the sharded run is compared with).

Every rank seeds `random` and torch differently, as unseeded processes would; install() + the model's start-state
broadcast must put every rank on rank 0's trajectory, which is the plain run's when rank 0 has its seeds.  Checked:
the engine is ShardedEngine; the logged losses agree with the plain run within 1e-4; the final clean tables within
the strict bound of sharded_gpu_check.py (1e-4 of the table; the noisy models run at eps = 0); test() equals
ops.score_topk on the model's own tables; every rank returns the same rec list and bestPerformance; one set of result
files is written.  At world > 1 also: MF and predict() of another rank's user are refused."""
import hashlib
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TOL = 1e-4
EPOCHS = 7  # SGL evaluates from epoch 5 on, LightGCN every 5th: fast_evaluation fires at least twice for each
MODELS = {
    "LightGCN": {"n_layer": 2},
    "XSimGCL": {"n_layer": 2, "lambda": 0.2, "eps": 0.0, "tau": 0.2, "l_star": 1},
    "SimGCL": {"n_layer": 2, "lambda": 0.5, "eps": 0.0},
    "SGL": {"n_layer": 2, "lambda": 0.1, "drop_rate": 0.1, "aug_type": 1, "temp": 0.2},
}


class Conf:
    def __init__(self, model, out):
        self.config = {"training.set": "train.txt", "test.set": "test.txt", "model": {"name": model, "type": "graph"},
                       "item.ranking.topN": [10, 20], "embedding.size": 64, "max.epoch": EPOCHS, "batch.size": 32,
                       "learning.rate": 0.001, "reg.lambda": 0.0001, "output": out, model: MODELS[model]}

    def __getitem__(self, k):
        return self.config[k]

    def contain(self, k):
        return k in self.config


def triples():
    """~3300 training pairs (103 batches of 32: one logged loss line per epoch) and one held-out item per user."""
    from selfrec_b200 import synth
    pu, pi = synth.make_pairs(700, 500, 4000, seed=4)
    train, test = [], []
    last = {}
    for k, u in enumerate(pu.tolist()):
        last[u] = k
    deg = np.bincount(pu, minlength=700)
    for k, (u, i) in enumerate(zip(pu.tolist(), pi.tolist())):
        (test if (deg[u] >= 3 and last[u] == k) else train).append([f"u{u}", f"i{i}", 1.0])
    return train, test


def digest(obj):
    return int.from_bytes(hashlib.sha256(repr(obj).encode()).digest()[:7], "little")


def run(name, out_dir, rank):
    """execute() of one model; returns (model, logged losses, rec_list)."""
    import importlib
    cls = getattr(importlib.import_module(f"model.graph.{name}"), name)
    train, test = triples()
    m = cls(Conf(name, os.path.join(out_dir, "results", name) + "/"), train, test)
    logged, got = [], {}
    base_log = m._log_line
    m._log_line = lambda epoch, n, losses: (logged.append(list(losses)), base_log(epoch, n, losses))
    base_eval = m.evaluate
    m.evaluate = lambda rec_list: (got.setdefault("rec", rec_list), base_eval(rec_list))
    m.execute()
    return m, logged, got["rec"]


def main():
    ref = "--ref" in sys.argv
    out = sys.argv[sys.argv.index("--out") + 1]
    import torch
    import selfrec_b200
    selfrec_b200.install()  # under torchrun: the NCCL group, one GPU per rank
    import torch.distributed as dist
    from selfrec_b200 import ops
    from selfrec_b200.shard_check import max_rel
    grouped = dist.is_available() and dist.is_initialized()
    rank, world = (dist.get_rank(), dist.get_world_size()) if grouped else (0, 1)
    work = os.path.join(out, "ref" if ref else f"w{world}")
    os.makedirs(work, exist_ok=True)
    os.chdir(work)
    ok = True
    for k, name in enumerate(MODELS):
        random.seed(11 + k + 1000 * rank)  # different on every rank; rank 0's are the plain run's
        torch.manual_seed(22 + k + 1000 * rank)
        m, logged, rec = run(name, work, rank)
        fu, fi = m.engine.forward_clean()
        if ref:
            np.savez(os.path.join(out, f"ref_{name}.npz"), losses=np.array(logged, dtype=np.float64), user=fu.cpu().numpy(),
                     item=fi.cpu().numpy())
            print(f"{name}: {len(logged)} logged losses, {type(m.engine).__name__}", flush=True)
            continue
        want = np.load(os.path.join(out, f"ref_{name}.npz"))
        eng = m.engine
        good = type(eng).__name__ == "ShardedEngine" and eng.world == world and m.bestPerformance
        la = np.array(logged, dtype=np.float64) if rank == 0 else want["losses"]
        loss_rel = float(np.max(np.abs(la - want["losses"]) / np.maximum(np.abs(want["losses"]), 1e-12))) if la.size else 1.0
        good = good and la.shape == want["losses"].shape and la.shape[0] >= EPOCHS
        wu = torch.from_numpy(want["user"]).cuda()[rank::world]
        u_rel, i_rel = max_rel(fu, wu), max_rel(fi, torch.from_numpy(want["item"]).cuda())
        # test() is the ranking of the model's own (best) tables
        full_u = eng.all_user_rows(m.user_emb)
        names = list(m.data.test_set)
        uids = np.fromiter((m.data.user[u] for u in names), dtype=np.int32, count=len(names))
        ids, sc = ops.score_topk(full_u, m.item_emb, uids, *m.data.rated_csr(), m.max_N)
        ids, sc = ids.cpu().numpy(), sc.cpu().numpy()
        id2item = m.data.id2item
        same_test = list(rec) == names and all(
            [it for it, _ in rec[u]] == [id2item[i] for i in ids[r].tolist()] and [s for _, s in rec[u]] == sc[r].tolist()
            for r, u in enumerate(names))
        stats = torch.tensor([loss_rel, u_rel, i_rel, 0.0 if same_test else 1.0, 0.0 if good else 1.0], dtype=torch.float64, device="cuda")
        d_rec, d_best = digest(sorted(rec.items())), digest(m.bestPerformance)
        dig = torch.tensor([d_rec, -d_rec, d_best, -d_best], dtype=torch.int64, device="cuda")
        if world > 1:
            dist.all_reduce(stats, op=dist.ReduceOp.MAX)
            dist.all_reduce(dig, op=dist.ReduceOp.MAX)
            dist.barrier()
        loss_rel, u_rel, i_rel, bad_test, bad = stats.tolist()
        agree = int(dig[0]) == d_rec and int(-dig[1]) == d_rec and int(dig[2]) == d_best and int(-dig[3]) == d_best
        files = sorted(os.listdir(os.path.join(work, "results", name)))
        logs = [f for f in os.listdir(os.path.join(work, "log")) if f.startswith(name + " ")]
        one_set = len(files) == 2 and any(f.endswith("-performance.txt") for f in files) and len(logs) == 1
        case_ok = not bad and not bad_test and agree and one_set and loss_rel <= TOL and max(u_rel, i_rel) <= TOL
        if rank == 0:
            print(f"{name} world={world}: {la.shape[0]} logged losses, loss_rel {loss_rel:.2e}, final tables {u_rel:.2e}/{i_rel:.2e}, "
                  f"test()==score_topk {not bad_test}, ranks agree {agree}, result files {files} logs {len(logs)}, "
                  f"best {m.bestPerformance[0]} {'ok' if case_ok else 'FAIL'}", flush=True)
        ok = ok and case_ok
        del m, eng, full_u
        torch.cuda.empty_cache()
    if not ref and world > 1:
        from selfrec_b200._lib import SrbError
        from selfrec_b200.model.graph.LightGCN import LightGCN
        from selfrec_b200.model.graph.MF import MF
        train, test = triples()
        refused = 0
        try:
            MF(_mf_conf(work), train, test)
        except SrbError:
            refused += 1
        m = LightGCN(Conf("LightGCN", os.path.join(work, "results", "p") + "/"), train, test)
        other = next(u for u, i in m.data.user.items() if i % world != rank)
        try:
            m.predict(other)
        except SrbError:
            refused += 1
        mine = next(u for u, i in m.data.user.items() if i % world == rank)
        m.user_emb, m.item_emb = m.engine.forward_clean()
        sc = m.predict(mine)
        good = refused == 2 and sc.shape == (m.data.item_num,)
        t = torch.tensor([0.0 if good else 1.0], device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        if rank == 0:
            print(f"refusals (MF at world {world}, predict of another rank's user): {'ok' if t.item() == 0 else 'FAIL'}", flush=True)
        ok = ok and t.item() == 0
    if rank == 0:
        print("SHARD_LAUNCH", "REF" if ref else ("PASS" if ok else "FAIL"), f"world={world}", flush=True)
    sys.exit(0 if ok else 1)


def _mf_conf(work):
    c = Conf("LightGCN", os.path.join(work, "mf") + "/")
    c.config["model"] = {"name": "MF", "type": "graph"}
    c.config["MF"] = {}
    return c


if __name__ == "__main__":
    main()
