"""Save and resume on the GPU: every fused model stopped mid-epoch or at an epoch end, resumed in this process and in a
fresh one; a captured CUDA graph after load_state_dict(); resuming across world sizes on loopback ranks; ranking from a
checkpoint through execute().

An uninterrupted run is the reference.  The resumed run must restore the saved state bit for bit (tables, moments, step
counter, sampler position, RNG states, SGL's view graphs), consume word for word the batches the reference consumed after
the save, and then agree with it within TOL of each table's scale: the L2 term sums with float atomics, so two runs of
the same batches are not bit-identical (the strict bound of shard_check.sharded_vs_single)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
for _p in (ROOT, TESTS):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import shard_launch_gpu_check as chk  # noqa: E402  (the launcher tests' synthetic triples and configuration)

TOL = 1e-4
MODELS = dict(chk.MODELS, MF={})
MID, END = (0, 40), (1, 0)  # (epoch, batch) to continue at: 40 batches into epoch 0, or the start of epoch 1


def _golden_triples():
    """The golden tiny set (tests/golden/tiny_{train,test}.txt) as [user, item, weight] rows."""
    def read(fn):
        with open(os.path.join(TESTS, "golden", fn)) as f:
            return [[a, b, float(w)] for a, b, w in (line.split() for line in f if line.strip())]
    return read("tiny_train.txt"), read("tiny_test.txt")


def _model(name, out, extra=None, data="synthetic", **over):
    import importlib
    conf = chk.Conf("LightGCN", out)
    conf.config.update({"model": {"name": name, "type": "graph"}, name: dict(MODELS[name], **(extra or {}))})
    conf.config.update(over)
    train, test = chk.triples() if data == "synthetic" else _golden_triples()
    m = getattr(importlib.import_module(f"selfrec_b200.model.graph.{name}"), name)(conf, train, test)
    m.EVAL_FROM = 0  # keep-best tables from the first epoch on, for every model
    return m


def _record(m):
    """Wrap engine.step: every batch's words and the losses after it."""
    eng, log = m.engine, {"words": [], "losses": []}
    base = eng.step

    def step(words, fetch_loss=False):
        log["words"].append(np.array(words, copy=True))
        h = base(words, fetch_loss=True)
        log["losses"].append(h.get())
        return h if fetch_loss else None

    eng.step = step
    return log


def _snapshot(m):
    """Everything a checkpoint carries, as host arrays / plain values."""
    import torch
    eng = m.engine
    st = eng.state_dict()
    pos = eng.feed_state()
    out = {"step": st["step"], "order": pos["order"], "cursor": pos["cursor"], "random": json.dumps(pos["random"]),
           "numpy": json.dumps([np.random.get_state()[1].tolist(), int(np.random.get_state()[2])]),
           "torch": torch.get_rng_state().numpy(), "best": json.dumps(m.bestPerformance)}
    for k in ("params", "m", "v"):
        out["user_" + k] = st["user"][k]
    out["item_params"] = st["item_params"]
    for k in ("m", "v"):
        out["item_" + k] = st["item"][k]
    if pos["cursor"] >= 0:  # between epochs the next epoch draws new views
        for k, a in enumerate(getattr(eng, "view_adj", [])):
            if a is not None:
                for f in ("rowptr", "colidx", "vals"):
                    out[f"view{k}_{f}"] = getattr(a, f).cpu().numpy()
        for k, blocks in enumerate(getattr(eng, "view_blocks", None) or []):  # ShardedEngine: this rank's blocks
            for b, a in zip(("Ru", "Rt"), blocks):
                for f in ("rowptr", "colidx", "vals"):
                    out[f"view{k}_{b}_{f}"] = getattr(a, f).cpu().numpy()
    return out


def _final(m, log):
    st = m.engine.state_dict()
    return {"words": np.stack(log["words"]) if log["words"] else np.zeros((0, 0), np.int32), "losses": np.array(log["losses"]),
            "params": np.concatenate([st["user"]["params"], st["item_params"]]),
            "m": np.concatenate([st["user"]["m"], st["item"]["m"]]), "v": np.concatenate([st["user"]["v"], st["item"]["v"]])}


def _run_reference(name, work, target, epochs, extra, data="synthetic"):
    """The uninterrupted run; it writes the one checkpoint at `target` and snapshots its state there."""
    import random
    import torch
    random.seed(31)
    torch.manual_seed(32)
    np.random.seed(33)
    over = {"max.epoch": epochs, "checkpoint.dir": os.path.join(work, "ck")}
    if target[1]:
        over["checkpoint.every"] = target[1]
    m = _model(name, os.path.join(work, "ref") + "/", extra, data, **over)
    log = _record(m)
    base_save, snap = m.save_checkpoint, {}

    def save(epoch, batch):
        if (epoch, batch) == tuple(target):
            snap["path"] = base_save(epoch, batch)
            snap["state"] = _snapshot(m)
            snap["at"] = len(log["words"])
            snap["engine"] = type(m.engine).__name__

    m.save_checkpoint = save
    m.train()
    return snap, _final(m, log)


def _resume(name, path, work, epochs, extra, data="synthetic"):
    """A new model and engine from other seeds, load(), the snapshot right after it, then train() to the end."""
    import random
    import torch
    random.seed(7)
    torch.manual_seed(8)
    np.random.seed(9)
    m = _model(name, os.path.join(work, "res") + "/", extra, data, **{"max.epoch": epochs, "checkpoint.resume": path})
    m.build()
    snap = _snapshot(m)
    log = _record(m)
    m.train()
    return snap, _final(m, log)


def _same(a, b, what):
    assert set(a) == set(b), (what, sorted(set(a) ^ set(b)))
    for k in a:
        x, y = a[k], b[k]
        if isinstance(x, np.ndarray):
            assert x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x.view(np.uint8), y.view(np.uint8)), (what, k)
        else:
            assert x == y, (what, k, x, y)


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _compare(name, ref_snap, ref_final, snap, final, keys=None):
    """keys: compare only these entries of the restored state (a resume on another engine type has other view blocks)."""
    pick = (lambda d: d) if keys is None else (lambda d: {k: d[k] for k in keys if k in d})
    _same(pick(ref_snap["state"]), pick(snap), f"{name}: state after the load")
    at = ref_snap["at"]
    want = ref_final["words"][at:]
    assert final["words"].shape == want.shape and np.array_equal(final["words"], want), f"{name}: batches after the resume"
    rel = {"losses": _rel(final["losses"], ref_final["losses"][at:])}
    for k in ("params", "m", "v"):
        rel[k] = _rel(final[k], ref_final[k])
    print(f"{name}: resumed at batch {at}, {len(want)} batches word for word, max_rel {rel}", flush=True)
    assert max(rel.values()) <= TOL, (name, rel)


CASES = ([(n, "mid") for n in MODELS] + [(n, "end") for n in MODELS] + [("SGL", "mid-node"), ("SimGCL", "mid-eps"),
          ("XSimGCL", "mid-eps"), ("XSimGCL", "tiny"), ("SGL", "tiny")])
EXTRA = {"mid-node": {"aug_type": 0}, "mid-eps": {"eps": 0.1}, "tiny": {"eps": 0.1}}


@pytest.mark.parametrize("name,where", CASES, ids=[f"{n}-{w}" for n, w in CASES])
def test_resume_in_process_matches_uninterrupted_run(built_lib, tmp_path, monkeypatch, name, where):
    """mid: 40 batches into epoch 0; end: after epoch 0's evaluation; mid-node: SGL on node-dropout views; mid-eps:
    SimGCL / XSimGCL with in-kernel Philox noise (eps = 0.1), whose stream the restored step counter keys; tiny: the
    golden tiny set (17 batches of 32), 8 batches in, then a second whole epoch."""
    monkeypatch.chdir(tmp_path)  # the models' log files
    extra = EXTRA.get(where)
    data = "tiny" if where == "tiny" else "synthetic"
    target, epochs = {"end": (END, 2), "tiny": ((0, 8), 2)}.get(where, (MID, 1))
    ref_snap, ref_final = _run_reference(name, str(tmp_path), target, epochs, extra, data)
    assert ref_snap["state"]["cursor"] == (-1 if where == "end" else target[1] * 32)
    if name == "SGL" and where != "end":
        assert "view0_rowptr" in ref_snap["state"] and "view1_vals" in ref_snap["state"]
    snap, final = _resume(name, ref_snap["path"], str(tmp_path), epochs, extra, data)
    _compare(name, ref_snap, ref_final, snap, final)


_RESUME_SCRIPT = r'''
import sys
sys.path[:0] = [{root!r}, {tests!r}]
import numpy as np
import test_gpu_checkpoint as t
snap, final = t._resume({name!r}, {path!r}, {work!r}, {epochs!r}, None)
np.savez({out!r}, **{{"snap_" + k: (v if isinstance(v, np.ndarray) else np.array(v)) for k, v in snap.items()}}, **final)
print("RESUMED", flush=True)
'''


@pytest.mark.parametrize("name", list(MODELS))
def test_resume_in_a_new_process_matches_uninterrupted_run(built_lib, tmp_path, monkeypatch, name):
    """The same mid-epoch resume in a fresh Python process: nothing but the checkpoint carries the state over."""
    monkeypatch.chdir(tmp_path)
    ref_snap, ref_final = _run_reference(name, str(tmp_path), MID, 1, None)
    out = str(tmp_path / "resumed.npz")
    script = tmp_path / "resume.py"
    script.write_text(_RESUME_SCRIPT.format(root=ROOT, tests=TESTS, name=name, path=ref_snap["path"], work=str(tmp_path), epochs=1, out=out))
    r = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=600, cwd=str(tmp_path),
                       env={k: v for k, v in os.environ.items() if k not in ("WORLD_SIZE", "RANK", "LOCAL_RANK")})
    assert "RESUMED" in r.stdout, r.stdout[-3000:] + r.stderr[-5000:]
    z = np.load(out)
    snap = {k[5:]: (z[k] if z[k].dtype != object and z[k].ndim > 0 else z[k].item()) for k in z.files if k.startswith("snap_")}
    snap = {k: (v.item() if isinstance(v, np.ndarray) and v.ndim == 0 else v) for k, v in snap.items()}
    final = {k: z[k] for k in ("words", "losses", "params", "m", "v")}
    _compare(name, ref_snap, ref_final, snap, final)


def test_captured_graph_replays_after_load_state_dict(built_lib, tmp_path):
    """load_state_dict() copies into the engine's tensors: a graph captured before the load replays the loaded state,
    with no re-capture, and follows the engine it was saved from."""
    import random
    import torch
    from selfrec_b200 import checkpoint, synth
    from selfrec_b200.engine import TrainEngine
    from selfrec_b200.util.sampler import NativePairSampler, stream_epoch
    data = synth.make_interaction((600, 900, 9000), seed=3)
    random.seed(5)
    words = [w.copy() for w in stream_epoch(NativePairSampler(data), data, 256, 256)]
    kw = dict(eps=0.1, tau=0.2, cl_rate=0.2, layer_cl=1, philox_seed=77)
    torch.manual_seed(1)
    a = TrainEngine("XSimGCL", data, 64, 2, 256, 1e-3, 1e-4, **kw)
    torch.manual_seed(2)
    b = TrainEngine("XSimGCL", data, 64, 2, 256, 1e-3, 1e-4, **kw)
    b.batch_dev.copy_(torch.from_numpy(words[0]))
    g = b.capture()
    ptrs = [t.data_ptr() for t in (b.params, b.m, b.v, b.step_dev)]
    for w in words[:10]:
        a.step(w)
    path = checkpoint.save_engines(str(tmp_path), {"epoch": 0, "batch": 10, "cursor": -1}, [a])
    b.load_state_dict(checkpoint.engine_state(path, checkpoint.read_manifest(path), np.arange(a.U)))
    assert b.graph is g and [t.data_ptr() for t in (b.params, b.m, b.v, b.step_dev)] == ptrs
    assert torch.equal(a.params, b.params) and torch.equal(a.m, b.m) and torch.equal(a.v, b.v) and int(b.step_dev.item()) == 10
    for w in words[10:25]:
        a.step(w)
        b.step(w)  # graph replay
    torch.cuda.synchronize()
    assert int(b.step_dev.item()) == int(a.step_dev.item()) == 25
    for x, y in ((b.params, a.params), (b.m, a.m), (b.v, a.v), (b.losses, a.losses)):
        r = _rel(x.cpu().numpy(), y.cpu().numpy())
        assert r <= TOL, r


LOOPBACK = [(2, 1), (2, 2), (2, 3), (0, 2), (2, 0)]


@pytest.mark.parametrize("src,dst", LOOPBACK, ids=[f"W{s}-to-W{d}".replace("W0", "single") for s, d in LOOPBACK])
def test_resume_across_world_sizes_on_loopback_ranks(built_lib, tmp_path, src, dst):
    """Saved by 2 loopback ranks and resumed at 1, 2 and 3; saved by TrainEngine and resumed at 2; saved at 2 and
    resumed on TrainEngine (tests/checkpoint_loopback.py)."""
    from shard_loopback import LOOPBACK_ENV
    env = dict(os.environ, **LOOPBACK_ENV)
    case = json.dumps({"src": src, "dst": dst, "root": str(tmp_path / "ck")})
    r = subprocess.run([sys.executable, os.path.join(TESTS, "checkpoint_loopback.py"), case], capture_output=True, text=True,
                       timeout=300, env=env, cwd=ROOT)
    assert r.returncode == 0 and "CHECKPOINT_CASE PASS" in r.stdout, r.stdout[-3000:] + r.stderr[-5000:]
    print(r.stdout)


@pytest.mark.parametrize("name", ["LightGCN", "XSimGCL", "MF"])
def test_rank_a_saved_model_through_execute(built_lib, tmp_path, monkeypatch, name):
    """execute() with checkpoint.dir writes checkpoints; a second execute() resuming the latest one with max.epoch at
    the saved epoch count trains nothing and ranks from the restored keep-best tables: the same lists, the same
    metric strings."""
    import random
    import torch
    monkeypatch.chdir(tmp_path)
    ck = str(tmp_path / "ck")
    runs = []
    for k, over in enumerate(({"checkpoint.dir": ck}, {"checkpoint.dir": ck, "checkpoint.resume": "latest"})):
        random.seed(41 + k)
        torch.manual_seed(42 + k)
        m = _model(name, str(tmp_path / f"out{k}") + "/", None, **{"max.epoch": 2, **over})
        del m.EVAL_FROM  # the model's own evaluation schedule
        got = {}
        base_eval = m.evaluate
        m.evaluate = lambda rec_list, m=m, base=base_eval: (got.setdefault("rec", rec_list), base(rec_list))
        log = _record(m)
        m.execute()
        runs.append((m, got["rec"], len(log["words"])))
        if k == 0:
            from selfrec_b200 import checkpoint
            assert checkpoint.latest(ck).endswith(checkpoint.checkpoint_name(2, 0))
    (m1, rec1, n1), (m2, rec2, n2) = runs
    assert n1 > 0 and n2 == 0
    assert list(rec1) == list(rec2)
    assert all([it for it, _ in rec1[u]] == [it for it, _ in rec2[u]] for u in rec1)
    assert m1.result == m2.result and m1.bestPerformance == m2.bestPerformance


_TORCHRUN_SCRIPT = r'''
import json, os, sys
sys.path[:0] = [{root!r}, {tests!r}]
import numpy as np
import selfrec_b200
selfrec_b200.install()  # the process group: the graph models train on ShardedEngine
import test_gpu_checkpoint as t
out = {{}}
for name, where, extra in {cases!r}:
    work = os.path.join(os.getcwd(), name + "-" + where)
    target, epochs = (t.MID, 1) if where.startswith("mid") else (t.END, 2)
    ref_snap, ref_final = t._run_reference(name, work, target, epochs, extra)
    assert ref_snap["engine"] == "ShardedEngine", ref_snap["engine"]
    if name == "SGL" and where.startswith("mid"):
        assert "view0_Ru_colidx" in ref_snap["state"] and "view1_Rt_vals" in ref_snap["state"]
    snap, final = t._resume(name, ref_snap["path"], work, epochs, extra)
    t._compare(name, ref_snap, ref_final, snap, final)
    np.savez(os.path.join(work, "ref.npz"), **ref_final, **{{"state_" + k: v for k, v in ref_snap["state"].items()
                                                          if isinstance(v, np.ndarray)}})
    out[name + "-" + where] = {{"path": ref_snap["path"], "at": ref_snap["at"], "work": work,
                               "state": {{k: v for k, v in ref_snap["state"].items() if not isinstance(v, np.ndarray)}}}}
json.dump(out, open("cases.json", "w"))
print("TORCHRUN_CKPT PASS", flush=True)
'''
TORCHRUN_CASES = [("SGL", "mid", None), ("SimGCL", "mid-eps", {"eps": 0.1}), ("LightGCN", "end", None)]
TABLE_KEYS = ("step", "order", "cursor", "random", "numpy", "torch", "best", "user_params", "user_m", "user_v", "item_params",
              "item_m", "item_v")


def test_model_checkpoints_on_the_sharded_engine_under_torchrun(built_lib, tmp_path, monkeypatch):
    """The model-level save and load on ShardedEngine: a torchrun world of one rank (install() starts the group) saves
    through FusedGraphModel.save_checkpoint -- per-rank user and best-user shards, the collective save, SGL's views
    through the collective set_view_graphs on load -- and resumes there; then a plain process resumes the same
    checkpoints on TrainEngine.  Both resumes must follow the uninterrupted sharded run."""
    monkeypatch.chdir(tmp_path)
    script = tmp_path / "torchrun_ckpt.py"
    script.write_text(_TORCHRUN_SCRIPT.format(root=ROOT, tests=TESTS, cases=TORCHRUN_CASES))
    env = {k: v for k, v in os.environ.items() if k not in ("WORLD_SIZE", "RANK", "LOCAL_RANK")}
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=1", "--master-addr", "127.0.0.1",
           "--master-port", "29817", str(script)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env, cwd=str(tmp_path))
    print("\n".join(line for line in r.stdout.splitlines() if "resumed at" in line))
    assert "TORCHRUN_CKPT PASS" in r.stdout, r.stdout[-3000:] + r.stderr[-5000:]
    cases = json.load(open(tmp_path / "cases.json"))
    for name, where, extra in TORCHRUN_CASES:
        c = cases[f"{name}-{where}"]
        z = np.load(os.path.join(c["work"], "ref.npz"))
        ref_final = {k: z[k] for k in ("words", "losses", "params", "m", "v")}
        state = dict(c["state"], **{k[6:]: z[k] for k in z.files if k.startswith("state_")})
        ref_snap = {"state": state, "at": c["at"]}
        epochs = 1 if where.startswith("mid") else 2
        snap, final = _resume(name, c["path"], str(tmp_path / f"single-{name}"), epochs, extra)
        _compare(name + " sharded -> single", ref_snap, ref_final, snap, final, keys=TABLE_KEYS)
