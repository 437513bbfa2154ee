"""SGL on the bipartite-sharded step against the single-GPU engine.  World 1 runs on any box (the parity sweep in a
subprocess, view swaps, the kindle shape and the error paths in-process); worlds 2, 4 and 8 are launched with torchrun
when the box has the GPUs."""
import importlib.util
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHECK = os.path.join(ROOT, "tests", "sharded_sgl_gpu_check.py")
TOL = 1e-4


def _check_module():
    spec = importlib.util.spec_from_file_location("sharded_sgl_gpu_check", CHECK)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_sharded_sgl_world1_matches_single_gpu(built_lib):
    r = subprocess.run([sys.executable, CHECK], capture_output=True, text=True, timeout=900)
    assert "SHARDED_SGL_CHECK PASS" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


@pytest.mark.parametrize("world", [2, 4, 8])
def test_sharded_sgl_matches_single_gpu(built_lib, world):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs at least {world} GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(29711 + world), CHECK]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
    assert "SHARDED_SGL_CHECK PASS" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def _pair(data, d, L, B, **kw):
    import torch
    from selfrec_b200.engine import TrainEngine
    from selfrec_b200.sharded import ShardedEngine
    dev = torch.device("cuda", torch.cuda.current_device())
    g = torch.Generator(device=dev).manual_seed(1234)
    iu = torch.empty((data.user_num, d), device=dev).uniform_(-0.1, 0.1, generator=g)
    ii = torch.empty((data.item_num, d), device=dev).uniform_(-0.1, 0.1, generator=g)
    kw = dict(dict(tau=0.2, cl_rate=0.1), **kw)
    sh = ShardedEngine("SGL", data, d, L, B, 1e-3, 1e-4, init_user=iu, init_item=ii, device=dev, **kw)
    ref = TrainEngine("SGL", data, d, L, B, 1e-3, 1e-4, init_user=iu, init_item=ii, device=dev, **kw)
    return sh, ref


def _compare(sh, ref):
    from selfrec_b200.shard_check import max_rel
    U = ref.U
    return max(max_rel(sh.losses, ref.losses), max_rel(sh.mu, ref.m[:U]), max_rel(sh.mi, ref.m[U:]), max_rel(sh.vu, ref.v[:U]),
               max_rel(sh.vi, ref.v[U:]), max_rel(sh.user_emb, ref.params[:U]), max_rel(sh.item_emb, ref.params[U:]))


@pytest.mark.parametrize("captured", [False, True])
def test_sharded_sgl_view_swap_between_steps(built_lib, captured):
    """New views between steps (an epoch boundary): the sharded step must pick them up like the single-GPU engine, both
    eagerly and through a CUDA graph captured again after the swap."""
    import torch
    from selfrec_b200 import synth
    from selfrec_b200.shard_check import device_batches
    chk = _check_module()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    data = synth.make_device_interaction((30000, 8000, 1200000), seed=2, alpha=1.1)
    B = 512
    batches = device_batches(data, B, 4, seed=5)
    sh, ref = _pair(data, 64, 3, B)
    for epoch, kind in enumerate(("edge", "node")):
        views = chk.view_graphs(data, kind, 0.1, seed=20 + epoch, dev=dev)
        sh.set_view_graphs(*views)
        ref.set_view_graphs(*views)
        assert sh.graph is None
        if captured:
            sh.capture()
        for k in range(2):
            w = batches[2 * epoch + k]
            ref.batch_dev.copy_(w)
            ref.step_resident()
            sh.step(words_dev=w)
        torch.cuda.synchronize()
        assert _compare(sh, ref) <= TOL, (epoch, kind)
    fu, fi = sh.forward_clean()
    ru, ri = ref.forward_clean()
    from selfrec_b200.shard_check import max_rel
    assert max(max_rel(fu, ru), max_rel(fi, ri)) <= TOL


def test_sharded_sgl_kindle_shape_step(built_lib):
    """One step at the amazon-kindle shape (L = 3, d = 64, B = 2048, edge dropout 0.1, tau 0.2, lambda 0.1)."""
    import torch
    from selfrec_b200 import synth
    from selfrec_b200.shard_check import device_batches, sharded_vs_single
    chk = _check_module()
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    data = synth.make_device_interaction(synth.SHAPES["amazon-kindle"], seed=4, alpha=1.1)
    views = chk.view_graphs(data, "edge", 0.1, seed=4, dev=dev)
    r = sharded_vs_single("SGL", data, 64, 3, 2048, device_batches(data, 2048, 1, seed=4), steps=1, views=views, tau=0.2, cl_rate=0.1)
    assert r["max_rel"] <= TOL and r["m_rows_off_frac"] == 0.0, r


def test_sharded_sgl_error_paths(built_lib):
    """A step without views is refused with a message; so is a view whose shape is not the graph's."""
    import scipy.sparse as sp
    import torch
    from selfrec_b200 import _lib, synth
    from selfrec_b200.shard_check import device_batches
    torch.cuda.set_device(0)
    data = synth.make_interaction((300, 400, 5000), seed=3)
    sh, _ref = _pair(data, 32, 2, 64)
    with pytest.raises(_lib.SrbError, match="view"):
        sh.step(words_dev=device_batches(data, 64, 1, seed=1)[0])
    n = data.user_num + data.item_num
    wrong = sp.eye(n + 1, dtype="float32", format="csr")
    with pytest.raises(ValueError, match="view 2"):
        sh.set_view_graphs(data.norm_adj, wrong)
    from selfrec_b200.sharded import ShardedEngine
    lg = ShardedEngine("LightGCN", data, 32, 2, 64, 1e-3, 1e-4)
    with pytest.raises(_lib.SrbError, match="no view graphs"):
        lg.set_view_graphs(data.norm_adj, data.norm_adj)
