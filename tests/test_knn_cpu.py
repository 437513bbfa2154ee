"""ItemKNN / UserKNN without a GPU: the float64 oracle (tests/knn_oracle.py) against the golden vectors of the unmodified
reference (tests/golden/knn.npz, tools/gen_golden_knn.py), the host-side inputs of the kernels (training_set_u order,
item -> user CSR, name ranks) against the reference's dicts, and the models' refusals."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, os.path.join(ROOT, "tests"))
import knn_oracle  # noqa: E402

DATASETS = {"tiny": ("tiny_train.txt", "tiny_test.txt"), "crafted": ("knn_crafted_train.txt", "knn_crafted_test.txt")}
CASES = [(ds, model, k, s) for ds in DATASETS for model in ("ItemKNN", "UserKNN") for k, s in ((50, 100), (5, 2))]


def read_triples(name):
    out = []
    with open(os.path.join(GOLDEN, name)) as f:
        for line in f:
            a, b, w = line.strip().split(" ")
            out.append([a, b, float(w)])
    return out


class Conf:
    def __init__(self, model, topk=50, shrinkage=100, top_n=(10, 20)):
        self.config = {"training.set": "train.txt", "test.set": "test.txt", "model": {"name": model, "type": "graph"},
                       "item.ranking.topN": list(top_n), "topK": topk, "shrinkage": shrinkage, "embedding.size": 64,
                       "max.epoch": 1, "batch.size": 2048, "learning.rate": 0.001, "reg.lambda": 0.0001, "output": "./results/"}

    def __getitem__(self, k):
        return self.config[k]

    def contain(self, k):
        return k in self.config


def mirror(ds):
    from selfrec_b200.data.ui_graph import Interaction
    tr, te = DATASETS[ds]
    return Interaction(None, read_triples(tr), read_triples(te))


def oracle_inputs(d):
    un = [d.id2user[k] for k in range(d.user_num)]
    inn = [d.id2item[k] for k in range(d.item_num)]
    return knn_oracle.model_inputs(d.pair_users, d.pair_items, d.user_num, d.item_num, un, inn)


@pytest.fixture(scope="module")
def knn_golden():
    return np.load(os.path.join(GOLDEN, "knn.npz"), allow_pickle=False)


@pytest.mark.parametrize("ds,model,topk,shrink", CASES)
def test_oracle_matches_reference(knn_golden, ds, model, topk, shrink):
    from selfrec_b200.util.evaluation import ranking_evaluation
    g = knn_golden
    tag = f"{ds}_{model}_{topk}_{shrink}"
    d = mirror(ds)
    inp = oracle_inputs(d)
    kind = "item" if model == "ItemKNN" else "user"
    table = knn_oracle.model_table(kind, inp, d.user_num, d.item_num, topk, shrink)
    assert np.array_equal(table[2], g[tag + "_nbr_cnt"])
    assert np.array_equal(table[0], g[tag + "_nbr_ids"])
    assert np.array_equal(table[1], g[tag + "_nbr_sims"])  # float64 bits
    rows = np.stack([knn_oracle.score_row(kind, u, d.item_num, table, inp["seq_ptr"], inp["seq_idx"]) for u in range(d.user_num)])
    assert np.array_equal(rows, g[tag + "_predict"])
    users = g[tag + "_test_users"]
    assert users.tolist() == [d.user[u] for u in d.test_set]
    rated_ptr, rated_idx = d.rated_csr()
    ids, sc = knn_oracle.rank_users(kind, users, d.item_num, table, inp["seq_ptr"], inp["seq_idx"], rated_ptr, rated_idx, 20)
    assert np.array_equal(ids, g[tag + "_rec_ids"])
    assert np.array_equal(sc, g[tag + "_rec_scores"])
    rec = {d.id2user[int(u)]: [(d.id2item[int(i)], float(s)) for i, s in zip(ids[q], sc[q])] for q, u in enumerate(users)}
    assert ranking_evaluation(d.test_set, rec, [10, 20]) == g[tag + "_metrics"].tolist()


def test_golden_cases_reach_the_edges(knn_golden):
    """The crafted set has what the issue of tie order needs: equal sims, empty rows, zero-score ties in the lists."""
    g = knn_golden
    sims = g["crafted_ItemKNN_5_2_nbr_sims"]
    cnt = g["crafted_ItemKNN_5_2_nbr_cnt"]
    assert (cnt == 0).any()
    assert any(len(set(r[:c].tolist())) < c for r, c in zip(sims, cnt))  # equal sims inside one list
    assert (g["crafted_UserKNN_5_2_nbr_cnt"] == 0).any()
    assert (g["crafted_ItemKNN_5_2_rec_scores"] == 0.0).sum(1).max() > 1  # zero ties inside a top-20 list


@pytest.mark.parametrize("ds", list(DATASETS))
def test_host_inputs_follow_the_reference_dicts(ds):
    from selfrec_b200 import knn
    d = mirror(ds)
    ptr, idx = knn.insertion_csr(d.pair_users, d.pair_items, d.user_num, d.item_num)
    for name, uid in d.user.items():
        assert [d.id2item[i] for i in idx[ptr[uid]:ptr[uid + 1]].tolist()] == list(d.training_set_u[name])
    tptr, tidx = knn.transpose_csr(ptr, idx, d.item_num)
    for name, iid in d.item.items():
        assert sorted(d.id2user[u] for u in tidx[tptr[iid]:tptr[iid + 1]].tolist()) == sorted(d.training_set_i[name])
    for side, names in (("user", d.user), ("item", d.item)):
        ordered = knn.id_names(d, side)
        rank = knn.name_ranks(ordered)
        assert [ordered[k] for k in np.argsort(rank)] == sorted(names)
    inp = oracle_inputs(d)
    assert np.array_equal(ptr, inp["seq_ptr"]) and np.array_equal(idx, inp["seq_idx"])
    assert np.array_equal(tptr, inp["iu_ptr"]) and np.array_equal(tidx, inp["iu_idx"])


def test_host_inputs_of_native_interaction(built_lib):
    """The file-built NativeInteraction gives the same lists and ranks as the dict mirror (duplicate lines included)."""
    from selfrec_b200 import knn
    from selfrec_b200.data.native import NativeInteraction
    tr, te = DATASETS["crafted"]
    nat = NativeInteraction(None, os.path.join(GOLDEN, tr), os.path.join(GOLDEN, te))
    d = mirror("crafted")
    a = knn.insertion_csr(nat.pair_users, nat.pair_items, nat.user_num, nat.item_num)
    b = knn.insertion_csr(d.pair_users, d.pair_items, d.user_num, d.item_num)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    for side in ("user", "item"):
        assert knn.id_names(nat, side) == knn.id_names(d, side)


def test_name_ranks_of_synthetic_ids():
    from selfrec_b200 import knn, synth
    d = synth.ArrayInteraction([0, 1, 2, 2], [0, 1, 1, 2], 3, 3)
    assert knn.id_names(d, "user") == [0, 1, 2]
    assert knn.name_ranks([10, 9, 100]).tolist() == [1, 0, 2]
    assert knn.name_ranks(["i10", "i9", "i100"]).tolist() == [0, 2, 1]


@pytest.mark.parametrize("model", ["ItemKNN", "UserKNN"])
@pytest.mark.parametrize("topk,shrink,what", [(0, 100, "topK"), (-3, 100, "topK"), (50, -1, "shrinkage")])
def test_bad_settings_are_refused(model, topk, shrink, what, tmp_path, monkeypatch):
    import importlib
    from selfrec_b200._lib import SrbError
    monkeypatch.chdir(tmp_path)
    cls = getattr(importlib.import_module(f"selfrec_b200.model.graph.{model}"), model)
    tr, te = DATASETS["tiny"]
    with pytest.raises(SrbError, match=what):
        cls(Conf(model, topk, shrink), read_triples(tr), read_triples(te))


def _spawn(target, world, *args):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    port = 33000 + (os.getpid() * 7 + world) % 2000
    procs = [ctx.Process(target=target, args=(r, world, port, ret) + args) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(180)
        assert p.exitcode == 0
    return ret.get(timeout=5)


def _refusal_worker(rank, world, port, ret, cwd):
    import torch
    import torch.distributed as dist
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    os.chdir(cwd)
    from selfrec_b200._lib import SrbError
    from selfrec_b200.model.graph.ItemKNN import ItemKNN
    from selfrec_b200.model.graph.UserKNN import UserKNN
    tr, te = DATASETS["tiny"]
    ok = True
    for cls in (ItemKNN, UserKNN):
        try:  # refused before anything touches a device
            cls(Conf(cls.__name__), read_triples(tr), read_triples(te))
            ok = False
        except SrbError as e:
            ok = ok and cls.__name__ in str(e) and f"{world} ranks" in str(e)
    out = torch.tensor([1.0 if ok else 0.0])
    dist.all_reduce(out, op=dist.ReduceOp.MIN)
    if rank == 0:
        ret.put(float(out.item()))
    dist.destroy_process_group()


def test_knn_models_on_two_ranks_are_refused(tmp_path):
    assert _spawn(_refusal_worker, 2, str(tmp_path)) == 1.0


def test_install_resolves_the_knn_models():
    import selfrec_b200
    names = selfrec_b200.install()
    assert "model.graph.ItemKNN" in names and "model.graph.UserKNN" in names
    assert sys.modules["model.graph.ItemKNN"].ItemKNN.__module__ == "selfrec_b200.model.graph.ItemKNN"
    assert "model.graph.ItemKNN" not in selfrec_b200.install(fused_models=False)
