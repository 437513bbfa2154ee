"""Export of every user's top-N lists (selfrec_b200/export.py) on the GPU: the export of every fused model equals
rank_all() and the float64 oracle, at any chunk size; the parts of a sharded export (loopback ranks: one ShardRanker per
rank, each holding only its own user rows) reassemble into the single-process export bit for bit; ItemKNN / UserKNN
exports equal the float64 oracle lists; a resumed checkpoint exports what the trained run exported; and execute() with
export.dir writes the same result files as without it."""
import copy
import filecmp
import importlib
import os
import random
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
for _p in (ROOT, TESTS):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import knn_oracle  # noqa: E402
import test_gpu_checkpoint as ck  # noqa: E402  (model construction on the golden tiny and synthetic sets)

FUSED = ["MF", "LightGCN", "SimGCL", "XSimGCL", "SGL"]


def _trained(name, tmp_path, data, **over):
    import torch
    random.seed(5)
    torch.manual_seed(6)
    m = ck._model(name, str(tmp_path / "out") + "/", None, data, **{"max.epoch": 1, **over})
    m.train()
    return m


def _all_names(m):
    return [m.data.id2user[u] for u in range(m.data.user_num)]


def _check_against_rank_all(orc, m, ids, scores, n):
    names = _all_names(m)
    keep = m.max_N
    m.max_N = n
    try:
        _, want_ids, want_sc = m.rank_all(names)
    finally:
        m.max_N = keep
    assert np.array_equal(np.asarray(ids), want_ids)
    assert np.array_equal(np.asarray(scores).view(np.uint32), want_sc.view(np.uint32))
    rp, ri = m.data.rated_csr()
    ue, ie = m.user_emb.detach().cpu().numpy(), m.item_emb.detach().cpu().numpy()
    _, osc = orc.score_topk(ue, ie, np.arange(m.data.user_num, dtype=np.int32), rp, ri, n)
    assert np.array_equal(np.asarray(scores).view(np.uint32), osc.view(np.uint32))


@pytest.mark.parametrize("name", FUSED)
def test_fused_export_equals_rank_all(built_lib, orc, tmp_path, name):
    from selfrec_b200 import export
    m = _trained(name, tmp_path, "golden")
    U = m.data.user_num
    for chunk in (1, 7, U):
        path = m.export_recommendations(str(tmp_path / f"exp{chunk}"), chunk=chunk)
        assert os.path.basename(path) == f"{name}-top{m.max_N}"
        names, ids, scores = export.read(path)
        assert names == _all_names(m)
        _check_against_rank_all(orc, m, ids, scores, m.max_N)
    man = __import__("json").load(open(os.path.join(path, "manifest.json")))
    assert (man["U"], man["I"], man["d"], man["N"], man["world"], man["score_dtype"]) == (U, m.data.item_num, 64, m.max_N, 1, "float32")
    assert export.read_items(path) == [m.data.id2item[i] for i in range(m.data.item_num)]


@pytest.mark.parametrize("name,d,n", [("LightGCN", 64, 20), ("XSimGCL", 128, 20), ("SimGCL", 128, 50)])
def test_synthetic_export(built_lib, orc, tmp_path, name, d, n):
    """A synthetic graph at d = 64 and 128 (the tensor-core ranker at both widths), a list longer than 32, and a
    subset of users given by name in any order."""
    from selfrec_b200 import export
    m = _trained(name, tmp_path, "synthetic", **{"embedding.size": d})
    path = m.export_recommendations(str(tmp_path / "exp"), top_n=n, chunk=97)
    names, ids, scores = export.read(path)
    _check_against_rank_all(orc, m, ids, scores, n)
    some = _all_names(m)[::-5]
    names2, ids2, sc2 = export.read(m.export_recommendations(str(tmp_path / "some"), top_n=n, users=some))
    pos = sorted(m.data.user[u] for u in some)
    assert names2 == [m.data.id2user[u] for u in pos]
    assert np.array_equal(ids2, np.asarray(ids)[pos]) and np.array_equal(sc2, np.asarray(scores)[pos])


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_parts_reassemble(built_lib, tmp_path, world):
    """Each loopback rank holds only its own [Ug, d] user rows and ranks only its users; the parts it writes
    reassemble into the single-process export bit for bit."""
    import torch
    from selfrec_b200 import export, shard_rank
    from selfrec_b200.sharded import user_ids_of
    m = _trained("LightGCN", tmp_path, "synthetic")
    single = export.read(m.export_recommendations(str(tmp_path / "one"), chunk=50))
    ue = m.user_emb.detach()
    dev = ue.device
    jobs = []
    for g in range(world):
        mg = copy.copy(m)
        mg.user_emb = ue[torch.from_numpy(user_ids_of(m.data.user_num, g, world)).to(dev).long()].contiguous()
        mg.shard_ranker = shard_rank.ShardRanker(m.data, g, world, dev)
        jobs.append(export._Job(mg, str(tmp_path / "parts"), chunk=50))
    path = export.run(jobs, lambda ok: ok)
    names, ids, scores = export.read(path)
    man = __import__("json").load(open(os.path.join(path, "manifest.json")))
    assert man["world"] == world
    assert sum(len(np.load(os.path.join(path, f"users.{g}.npy"))) for g in range(world)) == m.data.user_num
    assert names == single[0]
    assert np.array_equal(ids, single[1]) and np.array_equal(scores, single[2])


def _knn_model(name, tmp_path, **over):
    from selfrec_b200.data.loader import FileIO
    from selfrec_b200.util.conf import ModelConf
    tr, te = (os.path.join(TESTS, "golden", f) for f in ("tiny_train.txt", "tiny_test.txt"))
    conf = ModelConf(config={"training.set": tr, "test.set": te, "model": {"name": name, "type": "graph"},
                             "item.ranking.topN": [10, 20], "topK": 50, "shrinkage": 100, "embedding.size": 64,
                             "max.epoch": 20, "batch.size": 2048, "learning.rate": 0.001, "reg.lambda": 0.0001,
                             "output": str(tmp_path / "results") + "/", **over})
    cls = getattr(importlib.import_module(f"selfrec_b200.model.graph.{name}"), name)
    return cls(conf, FileIO.load_data_set(tr, "graph"), FileIO.load_data_set(te, "graph"))


@pytest.mark.parametrize("name", ["ItemKNN", "UserKNN"])
def test_knn_export_equals_oracle(built_lib, tmp_path, name):
    from selfrec_b200 import export
    m = _knn_model(name, tmp_path)
    m.train()
    d = m.data
    U, I = d.user_num, d.item_num
    inp = knn_oracle.model_inputs(d.pair_users, d.pair_items, U, I, [d.id2user[u] for u in range(U)], [d.id2item[i] for i in range(I)])
    kind = "item" if name == "ItemKNN" else "user"
    table = knn_oracle.model_table(kind, inp, U, I, 50, 100)
    rp, ri = d.rated_csr()
    for n, chunk in ((20, None), (7, 3)):
        names, ids, scores = export.read(m.export_recommendations(str(tmp_path / f"exp{n}"), top_n=n, chunk=chunk))
        assert scores.dtype == np.float64
        wid, wsc = knn_oracle.rank_users(kind, np.arange(U), I, table, inp["seq_ptr"], inp["seq_idx"], rp, ri, n)
        assert np.array_equal(ids, wid) and np.array_equal(scores, wsc)


def test_knn_launcher_result_files_unchanged_by_export(built_lib, tmp_path, monkeypatch):
    """execute() with export.dir writes the same result files, byte for byte, as without it, plus the export."""
    from selfrec_b200 import export
    monkeypatch.chdir(tmp_path)
    outs = []
    for k, over in enumerate(({}, {"export.dir": str(tmp_path / "exp"), "export.topN": 15})):
        m = _knn_model("UserKNN", tmp_path / f"run{k}", **over)
        m.execute()
        res = str(tmp_path / f"run{k}" / "results")
        outs.append({f.split("@", 1)[1].split("-", 3)[-1]: os.path.join(res, f) for f in os.listdir(res)})
    assert sorted(outs[0]) == sorted(outs[1]) and len(outs[0]) == 2
    for key in outs[0]:
        assert filecmp.cmp(outs[0][key], outs[1][key], shallow=False), key
    names, ids, scores = export.read(str(tmp_path / "exp" / "UserKNN-top15"))
    assert ids.shape == (m.data.user_num, 15)


@pytest.mark.parametrize("name", ["LightGCN", "MF"])
def test_resumed_checkpoint_exports_what_the_run_exported(built_lib, tmp_path, monkeypatch, name):
    """execute() with checkpoint.dir and export.dir, then execute() resuming the latest checkpoint with max.epoch at
    the trained epoch count: both exports hold the same lists and scores."""
    import torch
    from selfrec_b200 import export
    monkeypatch.chdir(tmp_path)
    ckd = str(tmp_path / "ck")
    paths = []
    for k, over in enumerate(({"checkpoint.dir": ckd}, {"checkpoint.dir": ckd, "checkpoint.resume": "latest"})):
        random.seed(41 + k)
        torch.manual_seed(42 + k)
        exp = str(tmp_path / f"exp{k}")
        m = ck._model(name, str(tmp_path / f"out{k}") + "/", None, **{"max.epoch": 2, "export.dir": exp, **over})
        del m.EVAL_FROM
        m.execute()
        paths.append(os.path.join(exp, f"{name}-top{m.max_N}"))
    a, b = export.read(paths[0]), export.read(paths[1])
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
