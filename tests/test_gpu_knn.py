"""ItemKNN / UserKNN on the GPU, bit for bit (`==` on float64) against the golden vectors of the unmodified reference
(tests/golden/knn.npz) and the float64 oracle (tests/knn_oracle.py): neighbour tables, predict() rows, test() lists
with their tie order and scores, the ranking_evaluation strings, execute() from a ModelConf, a power-law graph whose
hubs overflow the kernel's on-chip candidate buffer, and the edges of the float64 top-k."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, os.path.join(ROOT, "tests"))
import knn_oracle  # noqa: E402
from test_knn_cpu import CASES, DATASETS, mirror, oracle_inputs  # noqa: E402

pytestmark = pytest.mark.gpu
KNN_BUF = 2048  # knn.cu: candidates the neighbour kernel keeps on chip per row (kept top-k plus one refill)


@pytest.fixture(scope="module")
def knn_golden(built_lib):
    return np.load(os.path.join(GOLDEN, "knn.npz"), allow_pickle=False)


@pytest.mark.parametrize("ds,model,topk,shrink", CASES)
def test_tables_rows_and_lists_match_reference(knn_golden, ds, model, topk, shrink):
    from selfrec_b200.knn import NeighbourTable
    from selfrec_b200.util.evaluation import ranking_evaluation
    g = knn_golden
    tag = f"{ds}_{model}_{topk}_{shrink}"
    d = mirror(ds)
    t = NeighbourTable(d, "item" if model == "ItemKNN" else "user", topk, shrink)
    ids, sims, cnt = t.neighbours()
    assert np.array_equal(cnt, g[tag + "_nbr_cnt"])
    assert np.array_equal(ids, g[tag + "_nbr_ids"])
    assert np.array_equal(sims, g[tag + "_nbr_sims"])
    rows = t.score_rows(np.arange(d.user_num)).cpu().numpy()
    assert rows.dtype == np.float64 and np.array_equal(rows, g[tag + "_predict"])
    users = g[tag + "_test_users"]
    rid, rsc = t.rank(users, 20)
    assert np.array_equal(rid, g[tag + "_rec_ids"])
    assert np.array_equal(rsc, g[tag + "_rec_scores"])
    rec = {d.id2user[int(u)]: [(d.id2item[int(i)], float(s)) for i, s in zip(rid[q], rsc[q])] for q, u in enumerate(users)}
    assert ranking_evaluation(d.test_set, rec, [10, 20]) == g[tag + "_metrics"].tolist()


def test_edges_of_the_crafted_set(knn_golden):
    """topK above a row's candidate count, rows without candidates, a user whose row is zero apart from the mask."""
    from selfrec_b200.knn import NeighbourTable
    d = mirror("crafted")
    item = NeighbourTable(d, "item", 50, 100)
    _, _, cnt = item.neighbours()
    assert cnt[d.item["i999"]] == 0 and (cnt < 50).all()
    user = NeighbourTable(d, "user", 5, 2)
    _, _, ucnt = user.neighbours()
    u = d.user["u999"]
    assert ucnt[u] == 0
    assert not user.score_rows([u]).cpu().numpy().any()
    masked = user.score_rows([u], masked=True).cpu().numpy()[0]
    assert masked[d.item["i999"]] == -10e8 and np.count_nonzero(masked) == 1


@pytest.mark.parametrize("model", ["ItemKNN", "UserKNN"])
def test_execute_from_model_conf(knn_golden, model, tmp_path, monkeypatch):
    from selfrec_b200.data.loader import FileIO
    from selfrec_b200.util.conf import ModelConf
    import importlib
    monkeypatch.chdir(tmp_path)
    tr, te = (os.path.join(GOLDEN, f) for f in DATASETS["tiny"])
    conf = ModelConf(config={"training.set": tr, "test.set": te, "model": {"name": model, "type": "graph"},
                             "item.ranking.topN": [10, 20], "topK": 50, "shrinkage": 100, "embedding.size": 64,
                             "max.epoch": 20, "batch.size": 2048, "learning.rate": 0.001, "reg.lambda": 0.0001,
                             "output": str(tmp_path / "results") + "/"})
    cls = getattr(importlib.import_module(f"selfrec_b200.model.graph.{model}"), model)
    m = cls(conf, FileIO.load_data_set(tr, "graph"), FileIO.load_data_set(te, "graph"))
    m.execute()
    assert m.result == knn_golden[f"tiny_{model}_50_100_metrics"].tolist()
    assert any(f.endswith("-top-20items.txt") for f in os.listdir(tmp_path / "results"))
    sim = m.item_sim if model == "ItemKNN" else m.user_sim
    g_ids, g_sims, g_cnt = (knn_golden[f"tiny_{model}_50_100_{k}"] for k in ("nbr_ids", "nbr_sims", "nbr_cnt"))
    names = m.neighbour_table.names
    for a, name in enumerate(names):
        assert [(float(s), o) for s, o in sim[name]] == [(float(s), names[j]) for s, j in zip(g_sims[a, :g_cnt[a]], g_ids[a, :g_cnt[a]])]
    u = next(iter(m.data.test_set))
    assert np.array_equal(m.predict(u), knn_golden[f"tiny_{model}_50_100_predict"][m.data.user[u]])


@pytest.fixture(scope="module")
def hub_graph(built_lib):
    from selfrec_b200 import synth
    U, I = 6000, 3000
    pu, pi = synth.make_pairs(U, I, 90000, seed=3)
    d = synth.ArrayInteraction(pu, pi, U, I)
    return d, knn_oracle.model_inputs(pu, pi, U, I, list(range(U)), list(range(I)))


@pytest.mark.parametrize("model,topk,shrink", [("UserKNN", 50, 100), ("UserKNN", 1000, 0), ("ItemKNN", 20, 2)])
def test_power_law_graph_matches_oracle(hub_graph, model, topk, shrink):
    import scipy.sparse as sp
    from selfrec_b200.knn import NeighbourTable
    d, inp = hub_graph
    kind = "item" if model == "ItemKNN" else "user"
    want = knn_oracle.model_table(kind, inp, d.user_num, d.item_num, topk, shrink)
    if kind == "user":  # hubs: rows with more candidates than the buffer holds beside the kept top-k
        A = sp.csr_matrix((np.ones(len(inp["seq_idx"])), inp["seq_idx"], inp["seq_ptr"]), shape=(d.user_num, d.item_num))
        assert (np.diff((A @ A.T).tocsr().indptr) - 1).max() > KNN_BUF
    t = NeighbourTable(d, kind, topk, shrink)
    got = t.neighbours()
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    users = np.arange(0, d.user_num, 37, dtype=np.int32)
    rows = t.score_rows(users).cpu().numpy()
    for q, u in enumerate(users):
        assert np.array_equal(rows[q], knn_oracle.score_row(kind, u, d.item_num, want, inp["seq_ptr"], inp["seq_idx"]))
    rated_ptr, rated_idx = d.rated_csr()
    ids, sc = t.rank(users, 20)
    wid, wsc = knn_oracle.rank_users(kind, users, d.item_num, want, inp["seq_ptr"], inp["seq_idx"], rated_ptr, rated_idx, 20)
    assert np.array_equal(ids, wid) and np.array_equal(sc, wsc)


@pytest.mark.parametrize("k", [1, 33, 64, 100, "all"])
def test_topk_f64_lengths(hub_graph, k):
    import torch
    from selfrec_b200 import ops
    from selfrec_b200.knn import NeighbourTable
    d, _ = hub_graph
    t = NeighbourTable(d, "item", 5, 2)
    users = np.arange(0, d.user_num, 151, dtype=np.int32)
    rows = t.score_rows(users, masked=True)
    K = d.item_num if k == "all" else k
    ids, sc = ops.topk_rows_f64(rows, K)
    host = rows.cpu().numpy()
    for q in range(len(users)):
        wi, ws = knn_oracle.find_k_largest(K, host[q])
        assert np.array_equal(ids[q].cpu().numpy(), wi) and np.array_equal(sc[q].cpu().numpy(), ws)
    small = torch.zeros((3, 7), dtype=torch.float64, device="cuda")
    small[1, 2] = -10e8
    ids, sc = ops.topk_rows_f64(small, 7)
    for q in range(3):
        wi, ws = knn_oracle.find_k_largest(7, small[q].cpu().numpy())
        assert np.array_equal(ids[q].cpu().numpy(), wi) and np.array_equal(sc[q].cpu().numpy(), ws)


def test_ops_refuse_bad_arguments(built_lib):
    import torch
    from selfrec_b200 import ops
    from selfrec_b200._lib import SrbError
    rows = torch.zeros((2, 5), dtype=torch.float64, device="cuda")
    for k in (0, 6):
        with pytest.raises(SrbError):
            ops.topk_rows_f64(rows, k)
    with pytest.raises(SrbError):
        ops.topk_rows_f64(rows.float(), 2)
    z = torch.zeros(3, dtype=torch.int32, device="cuda")
    for topk, shrink in ((0, 1), (1025, 1), (5, -1)):
        with pytest.raises(SrbError):
            ops.knn_neighbors(z, z[:1], z, z[:1], z[:2], topk, shrink)
    with pytest.raises(SrbError):
        ops.knn_neighbors(z.cpu(), z[:1], z, z[:1], z[:2], 5, 1)
