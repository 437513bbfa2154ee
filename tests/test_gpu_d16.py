"""Embedding size 16 on every path that runs at 32: the SpMM family with two-lane rows (16 rows per warp), the Philox
noise of its epilogue, BPR + L2, InfoNCE on CUDA cores, the fused training step of all five models, the sharded step,
checkpoints across world sizes, and ranking -- each against the float64 oracle within the suites' tolerances (1e-4
relative in fp32; bit-exact for item ids, scores and Philox noise).  Widths 8 and 24 stay refused.  The helpers of the
other GPU files are imported, not restated; those of test_gpu_d256 that read its module width are run with it set to 16."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp

import test_gpu_d256 as w256
import test_gpu_parity as parity
import test_gpu_philox as phx
import test_gpu_step_edges as edges
from philox_model import philox_noise

pytestmark = pytest.mark.gpu

D = 16
RTOL = 1e-4
TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)

_rand = w256._rand
_every_class_graph = w256._every_class_graph
_check_product = w256._check_product


@pytest.fixture(scope="module")
def torch_cuda(built_lib):
    import torch
    assert torch.cuda.is_available()
    from selfrec_b200 import _lib
    _lib.require_device()
    return torch


@pytest.fixture(scope="module")
def hub(torch_cuda):
    """test_gpu_step_edges' hub graph (split rows of 2 and 3 chunks, CTA, warp and lane-group rows) with its device
    handles at d = 16: split rows in chunk lists, and in column-blocked lists (blocks of 4096 columns)."""
    from selfrec_b200 import ops
    h = edges.make_hub_graph(edges.U, edges.I, edges.HUB_USERS, edges.HUB_ITEMS, 20261016)
    chunked = ops.SparseAdj(h["A"]).cuda()
    blocked = ops.SparseAdj(h["A"]).cuda()
    assert not chunked.hub_struct(D).seg
    saved = ops.HUB_BLOCK_BYTES
    try:
        ops.HUB_BLOCK_BYTES = 2048 * 4 * D
        assert blocked.hub_struct(D).seg
    finally:
        ops.HUB_BLOCK_BYTES = saved
    h["adj"] = dict(chunked=chunked, colblocked=blocked)
    return h


def _run_engine(monkeypatch, *args):
    """test_gpu_d256's oracle-checked step loop; its noise tensors take the module width."""
    monkeypatch.setattr(w256, "D", D)
    w256._run_engine(*args)


# ---------------------------------------------------------------------------------------------------------------------
# SpMM
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("blocked", [False, True], ids=["chunked", "colblocked"])
def test_spmm_every_row_class_plain_and_masked_at_16(torch_cuda, orc, monkeypatch, blocked):
    """Plain and batch-masked products over split, CTA, warp, short and empty rows, with the split rows in chunk
    lists or column-blocked lists.  At d = 16 a warp holds 16 short rows, so the short class spans many warps."""
    torch = torch_cuda
    from selfrec_b200 import ops
    if blocked:
        monkeypatch.setattr(ops, "HUB_BLOCK_BYTES", 2048 * 4 * D)  # blocks of 4096 columns
    rng = np.random.default_rng(16)
    A = _every_class_graph(rng)
    h = ops.SparseAdj(A).cuda()
    assert h.n_huge == 2 and h.n_vlong == 3 and h.n_long == 2
    assert bool(h.hub_struct(D).seg) == blocked
    X = rng.standard_normal((A.shape[1], D)).astype(np.float32)
    y = torch.sparse.mm(h, torch.from_numpy(X).cuda()).cpu().numpy()
    _check_product(y, A, X, orc.spmm(A, X))
    assert (y[np.diff(A.indptr) == 0] == 0).all()
    # masked: only the columns whose bit is set are gathered; the other rows of X hold NaN and must not leak
    keep = rng.random(A.shape[1]) < 0.3
    Xm = np.where(keep[:, None], X, np.float32(np.nan)).astype(np.float32)
    words = np.zeros((A.shape[1] + 31) // 32, dtype=np.uint32)  # bit c & 31 of word c >> 5
    c = np.nonzero(keep)[0]
    np.bitwise_or.at(words, c >> 5, np.left_shift(np.uint32(1), (c & 31).astype(np.uint32)))
    mask = torch.from_numpy(words.view(np.int32)).cuda()
    ym = torch.empty((A.shape[0], D), device="cuda")
    ops._spmm_raw(h, torch.from_numpy(Xm).cuda(), ym, col_mask=mask)
    Ak = A @ sp.diags(keep.astype(np.float32))
    X0 = np.where(keep[:, None], X, 0).astype(np.float32)
    _check_product(ym.cpu().numpy(), abs(Ak), X0, orc.spmm(Ak.tocsr(), X0))


def test_spmm_autograd_at_16(torch_cuda, orc):
    torch = torch_cuda
    from selfrec_b200 import ops
    rng = np.random.default_rng(3)
    A = parity.rand_graph(rng, 300, 200, 8, hub=180)
    X = _rand(torch, rng, (200, D)).requires_grad_(True)
    G = rng.standard_normal((300, D)).astype(np.float32)
    y = torch.sparse.mm(ops.SparseAdj(A).cuda(), X)
    y.backward(torch.from_numpy(G).cuda())
    np.testing.assert_allclose(X.grad.cpu().numpy(), orc.spmm(A.T.tocsr(), G), rtol=RTOL, atol=1e-5)


def test_epilogue_rows_equals_identity_product_at_16(torch_cuda):
    """srb_spmm_epilogue_rows is the SpMM with the identity matrix at d = 16 too: same noise, same running sum."""
    torch = torch_cuda
    from selfrec_b200 import ops
    rng = np.random.default_rng(11)
    n = 1000
    eye = ops.SparseAdj(sp.identity(n, dtype=np.float32, format="csr")).cuda()
    x, base = _rand(torch, rng, (n, D)), _rand(torch, rng, (n, D))
    noise = torch.from_numpy(rng.random((n, D), dtype=np.float32)).cuda()
    step = torch.tensor([7], dtype=torch.int32, device="cuda")
    for epi in (dict(noise_mode=2, eps=0.1, philox_seed=99, philox_offset=(1 << 32) | 0x10, philox_step_dev=step),
                dict(noise_mode=1, noise=noise, eps=0.2)):
        outs = []
        for entry in ("srb_spmm_csr", "srb_spmm_epilogue_rows"):
            y, sm = torch.empty_like(x), torch.empty_like(x)
            ops._spmm_raw(eye, x, y, _entry=entry, sum_in=base, sum_out=sm, sum_scale=0.5, **epi)
            outs.append((y.cpu().numpy(), sm.cpu().numpy()))
        assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
        assert not np.array_equal(outs[1][0], x.cpu().numpy())


# ---------------------------------------------------------------------------------------------------------------------
# Philox noise: the column blocks gl and gl + 2 of a two-lane row
# ---------------------------------------------------------------------------------------------------------------------
def test_spmm_philox_noise_equals_host_model_at_16(torch_cuda, hub):
    torch = torch_cuda
    N = hub["A"].shape[0]
    rng = np.random.default_rng(D)
    x, base = _rand(torch, rng, (N, D), 0.1), _rand(torch, rng, (N, D), 0.1)
    for seed in phx.SEEDS:
        for off in phx.OFFSETS[::3]:
            for step in phx.STEPS:
                noise = torch.from_numpy(philox_noise(seed, off, step, N, D)).cuda()
                sp_ = phx._step_ptr(torch, step)
                for kind, adj in hub["adj"].items():
                    for entry in ("srb_spmm_csr", "srb_spmm_epilogue_rows"):
                        y2, s2 = phx._spmm(torch, adj, x, base, entry, noise_mode=2, philox_seed=seed, philox_offset=off, philox_step_dev=sp_)
                        y1, s1 = phx._spmm(torch, adj, x, base, entry, noise_mode=1, noise=noise)
                        where = (kind, entry, hex(seed), hex(off), step)
                        assert torch.equal(y2, y1), (where, int((y2 != y1).any(1).sum()))
                        assert torch.equal(s2, s1), where


def test_spmm_philox_wrong_keys_differ_at_16(torch_cuda, hub):
    torch = torch_cuda
    from philox_model import noise_offset
    N = hub["A"].shape[0]
    x = _rand(torch, np.random.default_rng(D + 1), (N, D), 0.1)
    base = torch.zeros_like(x)
    off, step = noise_offset(1, 2), 2
    wrong = [(phx.SEED, off, step - 1), (phx.SEED, noise_offset(0, 2), step), (phx.SEED, off + 1, step), (phx.SEED & 0xFFFFFFFF, off, step)]
    sp_ = phx._step_ptr(torch, step)
    adj = hub["adj"]["chunked"]
    y2, _ = phx._spmm(torch, adj, x, base, "srb_spmm_csr", noise_mode=2, philox_seed=phx.SEED, philox_offset=off, philox_step_dev=sp_)
    clean, _ = phx._spmm(torch, adj, x, base, "srb_spmm_csr")
    noisy = (y2 != clean).any(1)
    assert int(noisy.sum()) > 0.9 * N
    for s, o, t in wrong:
        y1, _ = phx._spmm(torch, adj, x, base, "srb_spmm_csr", noise_mode=1, noise=torch.from_numpy(philox_noise(s, o, t, N, D)).cuda())
        assert not ((y1 == y2).all(1) & noisy).any(), (hex(s), hex(o), t)


def test_encoder_forward_philox_equals_host_model_at_16(torch_cuda, hub):
    torch = torch_cuda
    from selfrec_b200 import ops
    N = hub["A"].shape[0]
    e0 = _rand(torch, np.random.default_rng(D + 2), (N, D), 0.1)
    for kind, adj in hub["adj"].items():
        for L in (1, 3):
            noise = torch.from_numpy(np.stack([philox_noise(phx.SEED, k, None, N, D) for k in range(L)])).cuda()
            for ego, lcl in ((False, 1), (False, L), (True, L)):
                f2, c2 = ops.encoder_forward(adj, e0, L, ego, philox_seed=phx.SEED, eps=phx.EPS, layer_cl=lcl, want_cl=True)
                f1, c1 = ops.encoder_forward(adj, e0, L, ego, noise=noise, eps=phx.EPS, layer_cl=lcl, want_cl=True)
                assert torch.equal(f2, f1) and torch.equal(c2, c1), (kind, L, ego, lcl)


@pytest.mark.parametrize("captured", [False, True], ids=["eager", "captured"])
@pytest.mark.parametrize("name,L,lcl", [("XSimGCL", 3, 1), ("SimGCL", 2, 0)])
def test_train_step_philox_equals_noise_tensor_twin_at_16(torch_cuda, hub, name, L, lcl, captured):
    """test_gpu_philox's twin check at d = 16: Philox mode against step_noise() fed as a tensor, with a wrongly keyed
    control."""
    torch = torch_cuda
    N = hub["A"].shape[0]
    E0 = phx._E0(N, D, L)
    noise, wrong = phx.twin_noise(name, L, N, D)
    engines = dict(P=phx.make_engine(torch, hub, name, D, L, lcl, E0, None), T=phx.make_engine(torch, hub, name, D, L, lcl, E0, noise),
                   W=phx.make_engine(torch, hub, name, D, L, lcl, E0, wrong))
    for r in phx.run_twins(torch, hub, captured, engines):
        where = (name, D, L, "step", r["step"], "b", r["b"])
        for t, bar in phx.BAR.items():
            assert r["dist"]["T"][t] <= bar, (where, t, r["dist"]["T"][t])
        assert r["dist"]["T"]["m_fro"] <= phx.M_FRO_BAR, (where, "m_fro", r["dist"]["T"]["m_fro"])
        assert r["dist"]["W"]["m_fro"] >= phx.CONTROL_MARGIN * phx.M_FRO_BAR, (where, "control", r["dist"]["W"]["m_fro"])


# ---------------------------------------------------------------------------------------------------------------------
# losses
# ---------------------------------------------------------------------------------------------------------------------
def test_bpr_l2_forward_backward_at_16(torch_cuda, orc):
    torch = torch_cuda
    from selfrec_b200.util.loss_torch import bpr_loss, l2_reg_loss
    rng = np.random.default_rng(5)
    a, b, c = (rng.standard_normal((300, D)).astype(np.float32) * 0.1 for _ in range(3))
    ta, tb, tc = (torch.from_numpy(x).cuda().requires_grad_(True) for x in (a, b, c))
    loss = bpr_loss(ta, tb, tc)
    l2 = l2_reg_loss(1e-3, ta, tb, tc)
    (loss + l2).backward()
    l1, du, dp, dn = orc.bpr_loss(a, b, c)
    l2r, g2 = orc.l2_reg_loss(1e-3, a, b, c)
    assert abs(loss.item() - l1) <= RTOL * abs(l1) and abs(l2.item() - l2r) <= RTOL * abs(l2r)
    for got, want in ((ta, du + g2[0]), (tb, dp + g2[1]), (tc, dn + g2[2])):
        np.testing.assert_allclose(got.grad.cpu().numpy(), want, rtol=RTOL, atol=1e-7)


@pytest.mark.parametrize("tau", [0.05, 0.2])
@pytest.mark.parametrize("n", [1, 63, 64, 65, 777, 2048, 4096])
def test_infonce_sizes_and_problem_counts_at_16(torch_cuda, orc, n, tau):
    """srb_infonce_fwd_bwd at d = 16 with 1 to 4 problems of sizes n, n - 1, n // 2, 1 in one launch (the padded
    capacity follows the largest): loss and both gradients of every problem against the oracle."""
    torch = torch_cuda
    from selfrec_b200 import ops
    rng = np.random.default_rng(n + int(tau * 100))
    for n_prob in (1, 2, 3, 4):
        sizes = [n, max(n - 1, 1), max(n // 2, 1), 1][:n_prob]
        probs, host = [], []
        for q, m in enumerate(sizes):
            v1 = (rng.standard_normal((m, D)) * 0.1).astype(np.float32)
            v2 = (v1 + 0.05 * rng.standard_normal((m, D))).astype(np.float32)
            t1, t2 = torch.from_numpy(v1).cuda(), torch.from_numpy(v2).cuda()
            probs.append(dict(table1=t1, table2=t2, idx=torch.arange(m, device="cuda", dtype=torch.int32), n=m, weight=1.0))
            host.append((v1, v2))
        losses, outs = ops.infonce_raw(probs, D, tau)
        losses = losses.cpu().numpy()
        for q, ((v1, v2), (g1, g2)) in enumerate(zip(host, outs)):
            ref, r1, r2 = orc.infonce(v1, v2, tau)
            where = (n_prob, q, sizes[q], tau)
            # S_ii is formed twice in fp32, in prep (the diagonal) and in the tile (the row's lse), in different orders
            logit_err = 8 * 1.2e-7 / tau
            assert abs(losses[q] - ref) <= RTOL * abs(ref) + logit_err, (where, losses[q], ref)
            m = sizes[q]
            vmin = min(np.linalg.norm(v1, axis=1).min(), np.linalg.norm(v2, axis=1).min())
            cond = logit_err / (m * tau) / np.sqrt(D) / vmin
            s = np.abs(r1).max()
            np.testing.assert_allclose(g1.cpu().numpy(), r1, rtol=RTOL, atol=2e-5 * s + cond, err_msg=str(where))
            np.testing.assert_allclose(g2.cpu().numpy(), r2, rtol=RTOL, atol=2e-5 * s + cond, err_msg=str(where))


# ---------------------------------------------------------------------------------------------------------------------
# the fused training step
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("captured", [False, True], ids=["eager", "captured"])
@pytest.mark.parametrize("name", ["MF", "LightGCN", "SimGCL", "XSimGCL", "SGL"])
def test_model_steps_on_golden_tiny_graph_at_16(torch_cuda, orc, golden, tiny_conf, tiny_triples, in_tmp_cwd, monkeypatch, name, captured):
    """The model classes built from a config with embedding.size 16, stepped through the golden fixture's batches (and
    SGL's view graphs) from random tables and noise, every step against the oracle's train_step."""
    torch = torch_cuda
    import importlib
    fx = golden(f"train_{name}.npz")
    train, test = tiny_triples
    cls = getattr(importlib.import_module(f"selfrec_b200.model.graph.{name}"), name)
    conf = tiny_conf(name, parity.CFG[name][0], **{"embedding.size": D})
    m = cls(conf, [list(t) for t in train], [list(t) for t in test])
    eng = m.engine
    assert eng.d == D
    N = eng.U + eng.I
    E0 = (np.random.default_rng(7).standard_normal((N, D)) * 0.1).astype(np.float32)
    eng.params.copy_(torch.from_numpy(E0))
    cfg = parity.CFG[name][0] or {}
    L = eng.L
    kw = dict(lr=float(conf["learning.rate"]), reg=float(conf["reg.lambda"]))
    lcl = 0
    if name in ("SimGCL", "XSimGCL"):
        kw.update(eps=cfg["eps"], tau=cfg.get("tau", 0.2), cl_rate=cfg["lambda"])
        lcl = cfg.get("l_star", 0)
    if name == "SGL":
        kw.update(tau=cfg["temp"], cl_rate=cfg["lambda"])
    view_csr = None
    A = m.data.norm_adj.tocsr()
    if name == "SGL":
        view_csr = [parity._csr(fx, f"view{k}", (N, N)) for k in range(2)]
        eng.set_view_graphs(*view_csr)
    batches = [(fx[f"b{k}_u"], fx[f"b{k}_i"], fx[f"b{k}_j"]) for k in range(int(fx["n_steps"]))]
    _run_engine(monkeypatch, torch, orc, eng, name, A, batches, L, lcl, kw, view_csr, captured, f"{name}-d16")


@pytest.mark.parametrize("name,L,lcl", [("XSimGCL", 3, 0), ("XSimGCL", 3, 1), ("XSimGCL", 3, 3), ("SimGCL", 2, 0), ("SGL", 2, 0),
                                        ("LightGCN", 3, 0), ("MF", 0, 0)])
def test_engine_steps_layer_cl_and_short_batches_at_16(torch_cuda, orc, monkeypatch, name, L, lcl):
    """TrainEngine at d = 16 on a random graph: XSimGCL's contrastive layer at 0 (the ego view), 1 and L, a full
    batch, a short one, an empty one and a full one again."""
    torch = torch_cuda
    from selfrec_b200.engine import TrainEngine
    rng = np.random.default_rng(L * 10 + lcl)
    U, I, B = 150, 220, 64
    data = parity._SynthData(rng, U, I, 3000)
    E0 = (rng.standard_normal((U + I, D)) * 0.1).astype(np.float32)
    kw = dict(lr=1e-2, reg=1e-3)
    if name in ("XSimGCL", "SimGCL"):
        ekw = dict(eps=0.2, tau=0.2, cl_rate=0.3, layer_cl=lcl)
    elif name == "SGL":
        ekw = dict(tau=0.2, cl_rate=0.3)
    else:
        ekw = dict(l2_div=float(B))
    kw.update({k: v for k, v in ekw.items() if k in ("eps", "tau", "cl_rate")})
    eng = TrainEngine(name, data, D, L, B, kw["lr"], kw["reg"], init_user=torch.from_numpy(E0[:U]), init_item=torch.from_numpy(E0[U:]), **ekw)
    view_csr = None
    if name == "SGL":
        keep = [rng.random(len(data.pair_users)) >= 0.1 for _ in range(2)]
        view_csr = [parity._norm_adj(data.pair_users[k], data.pair_items[k], U, I) for k in keep]
        eng.set_view_graphs(*view_csr)
    batches = [tuple(rng.integers(0, n, b).astype(np.int32) for n in (U, I, I)) for b in (B, 17, 0, B)]
    _run_engine(monkeypatch, torch, orc, eng, name, data.norm_adj, batches, L, lcl, kw, view_csr, False, f"{name}-d16-L{L}-lcl{lcl}")


@pytest.mark.parametrize("name,L,lcl,views", [("LightGCN", 2, 0, None), ("SimGCL", 2, 0, None), ("XSimGCL", 3, 1, None),
                                              ("SGL", 2, 0, "edge")])
def test_step_from_poisoned_workspace_at_16(torch_cuda, orc, hub, name, L, lcl, views):
    """test_gpu_step_edges' poison step and batch sequence (hubs, 17 triples, one hub triple, empty, one hub triple B
    times) at d = 16."""
    torch = torch_cuda
    from selfrec_b200.engine import TrainEngine
    U, I, B = edges.U, edges.I, edges.B
    rng = np.random.default_rng(D + L)
    E0 = (rng.standard_normal((U + I, D)) * 0.1).astype(np.float32)
    kw = dict(eps=edges.EPS, tau=edges.TAU, cl_rate=edges.CL_RATE, layer_cl=lcl) if name in ("XSimGCL", "SimGCL") else {}
    if name == "LightGCN":
        kw["l2_div"] = float(B)
    if name == "SGL":
        kw = dict(tau=edges.TAU, cl_rate=edges.CL_RATE)
    eng = TrainEngine(name, hub["data"], D, L, B, edges.LR, edges.REG, init_user=torch.from_numpy(E0[:U]), init_item=torch.from_numpy(E0[U:]), **kw)
    view_csr = None
    if name == "SGL":
        view_csr = hub["views"][views]
        eng.set_view_graphs(*view_csr)
    noise_dev = None
    if name in ("XSimGCL", "SimGCL"):
        noise_dev = torch.from_numpy(rng.random((2 if name == "SimGCL" else 1, L, U + I, D), dtype=np.float32)).cuda()
        eng.set_noise_tensor(noise_dev)
    edges._poison(torch, eng, hub["poison"], (eng.params, eng.m, eng.v, eng.step_dev, eng.losses), (eng.params,))

    def read_state():
        return tuple(t.cpu().numpy().copy() for t in (eng.params, eng.m, eng.v, eng.losses))

    edges._run_sequence(torch, orc, hub, name, D, L, lcl, view_csr, eng.step, read_state, noise_dev, f"{name}-d16-L{L}")


# ---------------------------------------------------------------------------------------------------------------------
# ranking
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k,n_items,n_q", [(1, 129, 3), (20, 1000, 70), (32, 640, 40), (20, 2000, 33)])
def test_score_topk_bit_exact_at_16(torch_cuda, orc, k, n_items, n_q):
    torch = torch_cuda
    from selfrec_b200 import ops
    rng = np.random.default_rng(k)
    ue = rng.standard_normal((90, D)).astype(np.float32)
    ie = rng.standard_normal((n_items, D)).astype(np.float32)
    users = rng.integers(0, 90, n_q).astype(np.int32)
    rated = sp.random(90, n_items, density=0.05, random_state=7, format="csr")
    rated.sort_indices()
    oi, os_, full = orc.score_topk(ue, ie, users, rated.indptr, rated.indices, k, want_scores=True)
    for impl in (0, 1):  # auto picks the CUDA-core kernel at d = 16, also past 1024 items
        ids, sc = ops.score_topk(torch.from_numpy(ue).cuda(), torch.from_numpy(ie).cuda(), users, rated.indptr, rated.indices, k, impl=impl)
        assert np.array_equal(ids.cpu().numpy(), oi) and np.array_equal(sc.cpu().numpy(), os_), impl
    dense = ops.score_rows(torch.from_numpy(ue).cuda(), torch.from_numpy(ie).cuda(), users)
    assert np.array_equal(dense.cpu().numpy(), full)


def test_topk_ties_and_long_lists_at_16(torch_cuda, orc):
    """Integer-valued embeddings make every dot product exact, so ties are real (and at d = 16 they are many): the
    selected set equals find_k_largest's.  topN 50 goes through the 32-at-a-time path, ids and scores equal to the
    oracle's."""
    torch = torch_cuda
    from selfrec_b200 import ops
    rng = np.random.default_rng(0)
    ue = rng.integers(-2, 3, (40, D)).astype(np.float32)
    ie = rng.integers(-2, 3, (900, D)).astype(np.float32)
    users = np.arange(40, dtype=np.int32)
    oi, os_ = orc.score_topk(ue, ie, users, None, None, 20)
    ids, sc = ops.score_topk(torch.from_numpy(ue).cuda(), torch.from_numpy(ie).cuda(), users, None, None, 20)
    assert np.array_equal(sc.cpu().numpy(), os_)
    assert all(sorted(a) == sorted(b) for a, b in zip(ids.cpu().numpy().tolist(), oi.tolist()))
    ue = rng.standard_normal((40, D)).astype(np.float32)
    ie = rng.standard_normal((700, D)).astype(np.float32)
    deg = rng.integers(0, 60, 40)
    ptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int32)
    idx = np.concatenate([np.sort(rng.choice(700, k, replace=False)) for k in deg]).astype(np.int32)
    ids, sc = ops.score_topk(torch.from_numpy(ue).cuda(), torch.from_numpy(ie).cuda(), users, ptr, idx, 50)
    oi, os_ = orc.score_topk(ue, ie, users, ptr, idx, 50)
    assert np.array_equal(ids.cpu().numpy(), oi) and np.array_equal(sc.cpu().numpy(), os_)


def test_graph_recommender_test_and_fast_evaluation_at_16(torch_cuda, orc, tiny_conf, tiny_triples, in_tmp_cwd):
    """GraphRecommender.test() at d = 16: every user's list equals the oracle's ranking of the same tables, and
    fast_evaluation's measure equals ranking_evaluation over test()'s output."""
    torch = torch_cuda
    import importlib
    from selfrec_b200.util.evaluation import ranking_evaluation
    train, test = tiny_triples
    cls = getattr(importlib.import_module("selfrec_b200.model.graph.XSimGCL"), "XSimGCL")
    m = cls(tiny_conf("XSimGCL", parity.CFG["XSimGCL"][0], **{"embedding.size": D}), [list(t) for t in train], [list(t) for t in test])
    rng = np.random.default_rng(1)
    ue = rng.standard_normal((m.data.user_num, D)).astype(np.float32)
    ie = rng.standard_normal((m.data.item_num, D)).astype(np.float32)
    m.user_emb, m.item_emb = torch.from_numpy(ue).cuda(), torch.from_numpy(ie).cuda()
    rec = m.test()
    assert list(rec) == list(m.data.test_set)
    users = np.array([m.data.user[u] for u in rec], dtype=np.int32)
    rp, ri = m.data.rated_csr()
    oi, os_ = orc.score_topk(ue, ie, users, rp, ri, m.max_N)
    for q, u in enumerate(rec):
        assert [it for it, _ in rec[u]] == [m.data.id2item[int(x)] for x in oi[q]], u
        assert [s for _, s in rec[u]] == [float(x) for x in os_[q]], u
    assert m.fast_evaluation(0) == ranking_evaluation(m.data.test_set, rec, [m.max_N])


# ---------------------------------------------------------------------------------------------------------------------
# sharded step (loopback ranks in one process; every step checks that each rank's item table is bit-identical to
# rank 0's)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("name,L,lcl,views", [("LightGCN", 2, 0, None), ("SimGCL", 2, 0, None), ("XSimGCL", 2, 1, None),
                                              ("SGL", 2, 0, "edge")])
def test_loopback_step_vs_oracle_at_16(built_lib, orc, name, world, L, lcl, views):
    from test_gpu_shard_loopback import _run
    _run(dict(kind="oracle", name=name, world=world, d=D, L=L, lcl=lcl, views=views))


@pytest.mark.parametrize("name,L,views", [("LightGCN", 2, None), ("SGL", 2, "node")])
def test_sharded_step_world1_at_16(torch_cuda, orc, hub, name, L, views):
    """World 1 of the sharded step: test_gpu_step_edges' world-1 check at d = 16.  SimGCL and XSimGCL run at world 1
    in the launcher test below."""
    edges.test_sharded_step_world1_from_poisoned_workspace_vs_oracle(torch_cuda, orc, hub, name, D, L, views)


@pytest.mark.parametrize("name,world,L,lcl", [("SimGCL", 2, 2, 0), ("XSimGCL", 3, 3, 1)])
def test_loopback_philox_matches_single_gpu_at_16(built_lib, name, world, L, lcl):
    from test_gpu_shard_loopback import _run
    _run(dict(kind="philox", name=name, world=world, d=D, L=L, lcl=lcl))


# ---------------------------------------------------------------------------------------------------------------------
# checkpoints across world sizes
# ---------------------------------------------------------------------------------------------------------------------
_CKPT_SCRIPT = r'''
import json, sys
sys.path.insert(0, {tests!r})
import torch
import checkpoint_loopback as ck
import shard_loopback as lb
ck.D = {d}
torch.cuda.set_device(0)
lb.install()
case = json.loads(sys.argv[1])
ck.run(case["src"], case["dst"], case["root"])
print("CHECKPOINT_CASE PASS", flush=True)
'''


@pytest.mark.parametrize("src,dst", [(0, 2), (2, 0)], ids=["single-to-W2", "W2-to-single"])
def test_resume_across_world_sizes_at_16(built_lib, tmp_path, src, dst):
    """tests/checkpoint_loopback.py at d = 16: saved by TrainEngine and resumed by 2 loopback ranks, and the reverse.
    The loaded state is bit-identical to the saved one, and 6 more steps on both sides agree within 1e-4."""
    from shard_loopback import LOOPBACK_ENV
    script = tmp_path / "ckpt16.py"
    script.write_text(_CKPT_SCRIPT.format(tests=TESTS, d=D))
    env = dict(os.environ, **LOOPBACK_ENV)
    case = json.dumps({"src": src, "dst": dst, "root": str(tmp_path / "ck")})
    r = subprocess.run([sys.executable, str(script), case], capture_output=True, text=True, timeout=300, env=env, cwd=ROOT)
    assert r.returncode == 0 and "CHECKPOINT_CASE PASS" in r.stdout, r.stdout[-3000:] + r.stderr[-5000:]
    print(r.stdout)


# ---------------------------------------------------------------------------------------------------------------------
# refused widths
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [8, 24])
def test_widths_below_and_between_stay_refused(torch_cuda, monkeypatch, d):
    torch = torch_cuda
    import shard_loopback as lb
    from selfrec_b200 import _lib, ops
    from selfrec_b200.engine import TrainEngine
    from selfrec_b200.sharded import ShardedEngine
    h = ops.SparseAdj(sp.eye(10, format="csr")).cuda()
    with pytest.raises(_lib.SrbError):
        torch.sparse.mm(h, torch.zeros(10, d, device="cuda"))
    with pytest.raises(_lib.SrbError):
        ops.InfoNCE(torch.ones(10, d, device="cuda"), torch.ones(10, d, device="cuda"), 0.2)
    pu = np.arange(40, dtype=np.int32)
    data = edges._HubData(pu, pu % 3, 40, 3)
    with pytest.raises(_lib.SrbError):
        TrainEngine("LightGCN", data, d, 1, 8, 1e-3, 1e-4)
    dev = torch.device("cuda", torch.cuda.current_device())
    lb.install(monkeypatch.setattr)
    pool = lb._Pool(2, dev)
    for r in range(2):  # every loopback rank refuses before it allocates or launches anything
        with pytest.raises(_lib.SrbError):
            ShardedEngine("LightGCN", data, d, 1, 8, 1e-3, 1e-4, group=lb.FakeGroup(pool, r), device=dev)


# ---------------------------------------------------------------------------------------------------------------------
# the reference's launcher flow at embedding.size 16
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("launcher", ["plain", "torchrun1"])
def test_one_epoch_of_each_model_through_the_launcher_at_16(built_lib, tmp_path, launcher):
    """install() + the model classes at embedding.size 16: one epoch of each model trains, evaluates and writes its
    results -- all five on TrainEngine in a plain process, the four graph models on ShardedEngine under torchrun.  SGL
    runs six epochs: like the reference (SGL.py:45-46) it evaluates, and keeps best tables, from epoch index 5 on."""
    tests = TESTS
    script = tmp_path / "epoch16.py"
    script.write_text(w256._EPOCH_SCRIPT.replace('"embedding.size": 256', f'"embedding.size": {D}').replace("m.engine.d == 256", f"m.engine.d == {D}")
                      .replace("EPOCH256", "EPOCH16").format(tests=tests))
    assert f'"embedding.size": {D}' in script.read_text() and "256" not in script.read_text()
    env = {k: v for k, v in os.environ.items() if k not in ("WORLD_SIZE", "RANK", "LOCAL_RANK")}
    cmd = [sys.executable, str(script)]
    if launcher == "torchrun1":
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=1", "--master-addr", "127.0.0.1",
               "--master-port", "29793", str(script)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=env, cwd=str(tmp_path))
    print(r.stdout[-3000:])
    assert "EPOCH16 PASS" in r.stdout, r.stdout[-3000:] + r.stderr[-5000:]
    want = "ShardedEngine" if launcher == "torchrun1" else "TrainEngine"
    assert sum(want in line for line in r.stdout.splitlines() if line.startswith("EPOCH16 ")) == (4 if launcher == "torchrun1" else 5)
