"""Parity of the CUDA path (through the C ABI) against the oracle and the reference-generated
golden fixtures.  Tolerances: 1e-4 relative fp32 on embeddings / losses (north_star), bit-exact
on sampler indices and top-k item ids."""
import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu

RTOL = 1e-4


def _csr(g, prefix, shape):
    return sp.csr_matrix((g[prefix + "_data"], g[prefix + "_indices"], g[prefix + "_indptr"]), shape=shape)


@pytest.fixture(scope="module")
def torch_cuda(built_lib):
    import torch
    assert torch.cuda.is_available()
    from selfrec_b200 import _lib
    _lib.require_device()
    return torch


@pytest.fixture(scope="module")
def tiny(golden):
    g = golden("graph.npz")
    U, I = int(g["user_num"]), int(g["item_num"])
    return dict(g=g, U=U, I=I, norm=_csr(g, "norm", (U + I, U + I)), im=_csr(g, "im", (U, I)))


def rand_graph(rng, n_rows, n_cols, avg_deg, hub=0):
    deg = np.minimum(rng.zipf(1.6, n_rows) + rng.integers(0, avg_deg, n_rows), n_cols)
    if hub:
        deg[rng.integers(0, n_rows, 3)] = min(hub, n_cols)
    deg[rng.integers(0, n_rows, 5)] = 0  # empty rows
    rows = np.repeat(np.arange(n_rows), deg)
    cols = np.concatenate([rng.choice(n_cols, k, replace=False) for k in deg]) if len(rows) else np.zeros(0, int)
    vals = rng.standard_normal(len(rows)).astype(np.float32)
    return sp.csr_matrix((vals, (rows, cols)), shape=(n_rows, n_cols), dtype=np.float32)


# ------------------------------------------------------------------------------------------
# (i) SpMM
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [32, 64, 128])
def test_spmm_matches_oracle(torch_cuda, orc, d):
    torch = torch_cuda
    from selfrec_b200 import ops
    rng = np.random.default_rng(d)
    A = rand_graph(rng, 700, 500, 12, hub=450)
    X = rng.standard_normal((500, d)).astype(np.float32)
    ref = orc.spmm(A, X)
    h = ops.SparseAdj(A).cuda()
    y = torch.sparse.mm(h, torch.from_numpy(X).cuda())
    scale = np.abs(A).dot(np.abs(X))  # |A||X|: the natural rounding scale of each entry
    err = np.abs(y.cpu().numpy() - ref)
    assert (err <= 4e-6 * scale + 1e-30).all(), err.max()
    assert (y.cpu().numpy()[np.diff(A.indptr) == 0] == 0).all()  # empty rows give exact zeros


def test_spmm_autograd_symmetric_and_rectangular(torch_cuda, orc):
    torch = torch_cuda
    from selfrec_b200 import ops
    rng = np.random.default_rng(3)
    A = rand_graph(rng, 300, 200, 8)
    X = torch.from_numpy(rng.standard_normal((200, 64)).astype(np.float32)).cuda().requires_grad_(True)
    G = rng.standard_normal((300, 64)).astype(np.float32)
    h = ops.SparseAdj(A).cuda()
    y = torch.sparse.mm(h, X)
    y.backward(torch.from_numpy(G).cuda())
    ref = orc.spmm(A.T.tocsr(), G)  # dL/dX = A^T G
    np.testing.assert_allclose(X.grad.cpu().numpy(), ref, rtol=RTOL, atol=1e-5)
    S = (A[:200, :200] + A[:200, :200].T).tocsr()  # symmetric: backward reuses the same CSR
    hs = ops.SparseAdj(S).cuda()
    assert hs.is_symmetric() and hs.transposed() is hs
    X2 = torch.from_numpy(rng.standard_normal((200, 64)).astype(np.float32)).cuda().requires_grad_(True)
    torch.sparse.mm(hs, X2).sum().backward()
    np.testing.assert_allclose(X2.grad.cpu().numpy(), orc.spmm(S, np.ones((200, 64), np.float32)), rtol=RTOL, atol=1e-5)


def test_spmm_rejects_bad_input(torch_cuda):
    torch = torch_cuda
    from selfrec_b200 import ops, _lib
    h = ops.SparseAdj(sp.eye(10, format="csr")).cuda()
    with pytest.raises(_lib.SrbError):
        torch.sparse.mm(h, torch.zeros(10, 48, device="cuda"))  # unsupported d
    with pytest.raises(ValueError):
        torch.sparse.mm(h, torch.zeros(11, 64, device="cuda"))
    with pytest.raises(_lib.SrbError):
        torch.sparse.mm(h, torch.zeros(10, 64))  # CPU tensor: no fallback


@pytest.mark.parametrize("name,L,ego,lcl", [("LightGCN", 3, True, 0), ("XSimGCL", 3, False, 1), ("SimGCL", 2, False, 0), ("SGL", 2, True, 0)])
def test_encoder_forward_matches_reference(torch_cuda, orc, golden, tiny, name, L, ego, lcl):
    torch = torch_cuda
    from selfrec_b200 import ops
    fx = golden(f"train_{name}.npz")
    U = tiny["U"]
    E = np.concatenate([fx["init_user"], fx["init_item"]]).astype(np.float32)
    h = ops.SparseAdj(tiny["norm"]).cuda()
    final, _ = ops.encoder_forward(h, torch.from_numpy(E).cuda(), L, ego)
    np.testing.assert_allclose(final[:U].cpu().numpy(), fx["clean_user"], rtol=RTOL, atol=1e-7)
    np.testing.assert_allclose(final[U:].cpu().numpy(), fx["clean_item"], rtol=RTOL, atol=1e-7)
    # perturbed forward with the noise as an input (the reference's torch.rand_like draws)
    rng = np.random.default_rng(11)
    noise = rng.random((L, E.shape[0], E.shape[1]), dtype=np.float32)
    want_cl = lcl > 0
    f2, cl = ops.encoder_forward(h, torch.from_numpy(E).cuda(), L, ego, noise=torch.from_numpy(noise).cuda(), eps=0.2,
                                 layer_cl=lcl, want_cl=want_cl)
    rf, rcl, _ = orc.encoder_forward(tiny["norm"], E, L, ego, noise, 0.2, lcl)
    np.testing.assert_allclose(f2.cpu().numpy(), rf, rtol=RTOL, atol=2e-7)
    if want_cl:
        np.testing.assert_allclose(cl.cpu().numpy(), rcl, rtol=RTOL, atol=2e-7)


def test_encoder_cl_view_defaults_to_ego(torch_cuda, orc, tiny):
    """XSimGCL.py:86: with l_star out of range the CL view is the ego embedding."""
    torch = torch_cuda
    from selfrec_b200 import ops
    rng = np.random.default_rng(2)
    E = rng.standard_normal((tiny["U"] + tiny["I"], 64)).astype(np.float32)
    h = ops.SparseAdj(tiny["norm"]).cuda()
    _, cl = ops.encoder_forward(h, torch.from_numpy(E).cuda(), 2, False, layer_cl=5, want_cl=True)
    assert np.array_equal(cl.cpu().numpy(), E)


def test_philox_noise_statistics(torch_cuda, tiny):
    """Perf-mode noise cannot replay torch.rand_like's stream (SURVEY hard part 8): check the
    distribution instead -- perturbation has L2 norm eps per row, follows sign(E), differs per layer."""
    torch = torch_cuda
    from selfrec_b200 import ops
    rng = np.random.default_rng(4)
    n = tiny["U"] + tiny["I"]
    E = torch.from_numpy(rng.standard_normal((n, 64)).astype(np.float32)).cuda()
    h = ops.SparseAdj(tiny["norm"]).cuda()
    clean, _ = ops.encoder_forward(h, E, 1, False)
    a, _ = ops.encoder_forward(h, E, 1, False, philox_seed=123, eps=0.2)
    b, _ = ops.encoder_forward(h, E, 1, False, philox_seed=124, eps=0.2)
    da, db = (a - clean).cpu().numpy(), (b - clean).cpu().numpy()
    c = clean.cpu().numpy()
    nz = np.abs(c).sum(1) > 0
    # every coordinate of a non-zero row moves by a positive amount in the direction of its sign
    np.testing.assert_allclose(np.sqrt((da[nz] ** 2).sum(1)), 0.2, rtol=2e-3)
    assert (np.sign(da[nz]) == np.sign(c[nz])).mean() > 0.999
    assert not np.allclose(da, db)
    u = np.abs(da[nz]) / 0.2  # = normalised uniform noise: mean of u_i / ||u||
    assert 0.09 < u.mean() < 0.12  # E[u]/sqrt(64 E[u^2]) = 0.5 / sqrt(64/3) = 0.108


def test_epilogue_rows_equals_identity_product(torch_cuda):
    """srb_spmm_epilogue_rows (the noise SimGCL's perturbed encoders add to the shared first product, SimGCL.py:87-88)
    is the SpMM with the identity matrix: same Philox stream / noise tensor, same running sum -- bit for bit."""
    torch = torch_cuda
    import scipy.sparse as sp
    from selfrec_b200 import ops
    rng = np.random.default_rng(11)
    n = 1000
    eye = ops.SparseAdj(sp.identity(n, dtype=np.float32, format="csr")).cuda()
    for d in (32, 64, 128):
        x = torch.from_numpy(rng.standard_normal((n, d)).astype(np.float32)).cuda()
        noise = torch.from_numpy(rng.random((n, d), dtype=np.float32)).cuda()
        base = torch.from_numpy(rng.standard_normal((n, d)).astype(np.float32)).cuda()
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


# ------------------------------------------------------------------------------------------
# (ii)(iii) losses, op-level drop-in
# ------------------------------------------------------------------------------------------
def test_bpr_l2_infonce_ops_match_reference(torch_cuda, golden):
    torch = torch_cuda
    from selfrec_b200.util.loss_torch import InfoNCE, bpr_loss, l2_reg_loss
    lo = golden("losses.npz")
    for tag in ("a", "b"):
        u, p, n = (torch.from_numpy(lo[f"bpr_{tag}_{k}"]).cuda().requires_grad_(True) for k in ("u", "p", "n"))
        loss = bpr_loss(u, p, n)
        assert loss.dim() == 0
        gu, gp, gn = torch.autograd.grad(loss, (u, p, n))
        assert abs(loss.item() - lo[f"bpr_{tag}_loss"]) <= RTOL * abs(lo[f"bpr_{tag}_loss"])
        for mine, k in ((gu, "gu"), (gp, "gp"), (gn, "gn")):
            np.testing.assert_allclose(mine.cpu().numpy(), lo[f"bpr_{tag}_{k}"], rtol=RTOL, atol=1e-8)
        l2 = l2_reg_loss(1e-2, u, p, n)
        g2 = torch.autograd.grad(l2, (u, p, n))
        assert abs(l2.item() - lo[f"l2_{tag}_loss"]) <= RTOL * abs(lo[f"l2_{tag}_loss"])
        for mine, k in zip(g2, ("gu", "gp", "gn")):
            np.testing.assert_allclose(mine.cpu().numpy(), lo[f"l2_{tag}_{k}"], rtol=RTOL, atol=1e-10)
    for tag in ("a", "b", "c", "d"):
        v1 = torch.from_numpy(lo[f"nce_{tag}_v1"]).cuda().requires_grad_(True)
        v2 = torch.from_numpy(lo[f"nce_{tag}_v2"]).cuda().requires_grad_(True)
        loss = InfoNCE(v1, v2, float(lo[f"nce_{tag}_tau"]), bool(lo[f"nce_{tag}_cos"]))
        g1, g2 = torch.autograd.grad(loss, (v1, v2))
        ref = float(lo[f"nce_{tag}_loss"])
        # the loss is a mean of (lse - S_ii) with |S| up to 1/tau: fp32 resolution of the terms bounds the abs error
        assert abs(loss.item() - ref) <= RTOL * max(abs(ref), 1e-3) + 2e-7 / float(lo[f"nce_{tag}_tau"]), tag
        scale = max(np.abs(lo[f"nce_{tag}_g1"]).max(), 1e-12)
        # absolute floor: fp32 resolution of a logit (eps32 / tau) through 1/(n tau), a unit-vector entry and 1/||v||
        # (the n = 1 case has an exactly-zero reference gradient, where only an absolute bound is meaningful)
        tau, n_, d_ = float(lo[f"nce_{tag}_tau"]), v1.shape[0], v1.shape[1]
        vmin = float(min(v1.detach().norm(dim=1).min(), v2.detach().norm(dim=1).min())) if bool(lo[f"nce_{tag}_cos"]) else 1.0
        cond = 3 * 1.2e-7 / tau / (n_ * tau) / np.sqrt(d_) / vmin
        np.testing.assert_allclose(g1.cpu().numpy(), lo[f"nce_{tag}_g1"], rtol=RTOL, atol=1e-5 * scale + cond, err_msg=tag)
        np.testing.assert_allclose(g2.cpu().numpy(), lo[f"nce_{tag}_g2"], rtol=RTOL, atol=1e-5 * scale + cond, err_msg=tag)


def test_losses_compose_like_the_reference(torch_cuda, orc):
    """batch_loss = rec + l2 + lambda * cl composes by + and * and backpropagates (XSimGCL.py:31-36)."""
    torch = torch_cuda
    from selfrec_b200.util.loss_torch import InfoNCE, bpr_loss, l2_reg_loss
    rng = np.random.default_rng(8)
    a, b, c = (rng.standard_normal((300, 64)).astype(np.float32) * 0.3 for _ in range(3))
    ta, tb, tc = (torch.from_numpy(x).cuda().requires_grad_(True) for x in (a, b, c))
    total = bpr_loss(ta, tb, tc) + l2_reg_loss(1e-3, ta, tb) / 2048 + 0.2 * InfoNCE(ta, tb, 0.2)
    total.backward()
    l1, du, dp, dn = orc.bpr_loss(a, b, c)
    l2, g2 = orc.l2_reg_loss(1e-3, a, b)
    l3, d1, d2 = orc.infonce(a, b, 0.2)
    assert abs(total.item() - (l1 + l2 / 2048 + 0.2 * l3)) <= RTOL * abs(total.item())
    np.testing.assert_allclose(ta.grad.cpu().numpy(), du + g2[0] / 2048 + 0.2 * d1, rtol=RTOL, atol=1e-7)
    np.testing.assert_allclose(tb.grad.cpu().numpy(), dp + g2[1] / 2048 + 0.2 * d2, rtol=RTOL, atol=1e-7)
    np.testing.assert_allclose(tc.grad.cpu().numpy(), dn, rtol=RTOL, atol=1e-7)


@pytest.mark.parametrize("n,d,tau", [(2048, 64, 0.2), (1900, 64, 0.15), (777, 128, 0.2), (4096, 64, 0.2), (65, 32, 0.05)])
def test_infonce_batch_sizes(torch_cuda, orc, n, d, tau):
    torch = torch_cuda
    from selfrec_b200.util.loss_torch import InfoNCE
    rng = np.random.default_rng(n)
    v1 = (rng.standard_normal((n, d)) * 0.1).astype(np.float32)
    v2 = (v1 + 0.05 * rng.standard_normal((n, d))).astype(np.float32)
    t1, t2 = (torch.from_numpy(x).cuda().requires_grad_(True) for x in (v1, v2))
    loss = InfoNCE(t1, t2, tau)
    loss.backward()
    ref, g1, g2 = orc.infonce(v1, v2, tau)
    # the loss is a mean of (lse - S_ii) with |S| up to 1/tau: fp32 resolution of the terms bounds the abs error
    assert abs(loss.item() - ref) <= RTOL * abs(ref) + 2e-7 / tau
    # fp32 conditioning: G_ii = P_ii - 1 is formed from logits of size 1/tau, so it carries an absolute
    # error ~ eps32 / tau; through 1/(n tau), a unit-vector entry (1/sqrt(d)) and 1/||v|| this bounds the
    # gradient error of ANY fp32 evaluation (torch's included) when the loss is close to zero
    vmin = min(np.linalg.norm(v1, axis=1).min(), np.linalg.norm(v2, axis=1).min())
    cond = 3 * 1.2e-7 / tau / (n * tau) / np.sqrt(d) / vmin
    s = np.abs(g1).max()
    np.testing.assert_allclose(t1.grad.cpu().numpy(), g1, rtol=RTOL, atol=2e-5 * s + cond)
    np.testing.assert_allclose(t2.grad.cpu().numpy(), g2, rtol=RTOL, atol=2e-5 * s + cond)


def test_adam_matches_torch_arithmetic(torch_cuda, orc):
    torch = torch_cuda
    from selfrec_b200 import ops
    rng = np.random.default_rng(1)
    p = rng.standard_normal(10007).astype(np.float32)
    m = np.zeros_like(p)
    v = np.zeros_like(p)
    tp, tm, tv = (torch.from_numpy(x.copy()).cuda() for x in (p, m, v))
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    scal = torch.zeros(16, device="cuda")
    for k in range(1, 6):
        g = (rng.standard_normal(10007) * 10.0 ** rng.integers(-6, 1)).astype(np.float32)
        ops.adam_prepare(step, scal, 1e-3)
        ops.adam_step(tp, tm, tv, torch.from_numpy(g).cuda(), scal)
        p, m, v = orc.adam_step(p, g, m, v, k, 1e-3)
        # p -= lr * m_hat / (sqrt(v_hat) + eps): for |g| near eps=1e-8 the quotient amplifies 1-ulp differences
        # (fma contraction) by up to 1/eps, so allow lr * 2e-5 absolute on top of the relative bound
        np.testing.assert_allclose(tp.cpu().numpy(), p, rtol=2e-6, atol=2e-8)
        np.testing.assert_allclose(tv.cpu().numpy(), v, rtol=2e-6, atol=1e-30)
    assert int(step.item()) == 5


# ------------------------------------------------------------------------------------------
# whole training steps (fused engine) against the reference's own train() loop
# ------------------------------------------------------------------------------------------
CFG = {
    "MF": (None, dict()),
    "LightGCN": ({"n_layer": 3}, dict()),
    "SimGCL": ({"n_layer": 2, "lambda": 0.5, "eps": 0.1}, dict()),
    "XSimGCL": ({"n_layer": 3, "l_star": 1, "lambda": 0.2, "eps": 0.2, "tau": 0.2}, dict()),
    "SGL": ({"n_layer": 2, "lambda": 0.1, "drop_rate": 0.1, "aug_type": 1, "temp": 0.2}, dict()),
}


def _batch_words(u, i, j, cap):
    w = np.zeros(4 + 5 * cap, dtype=np.int32)
    b = len(u)
    uu, ui = np.unique(u), np.unique(i)
    w[0], w[1], w[2] = b, len(uu), len(ui)
    w[4:4 + b] = u
    w[4 + cap:4 + cap + b] = i
    w[4 + 2 * cap:4 + 2 * cap + b] = j
    w[4 + 3 * cap:4 + 3 * cap + len(uu)] = uu
    w[4 + 4 * cap:4 + 4 * cap + len(ui)] = ui
    return w


def _make_model(name, tiny_conf, tiny_triples, fx):
    import importlib
    import torch
    train, test = tiny_triples
    cls = getattr(importlib.import_module(f"selfrec_b200.model.graph.{name}"), name)
    m = cls(tiny_conf(name, CFG[name][0]), [list(t) for t in train], [list(t) for t in test])
    eng = m.engine
    eng.params[: eng.U].copy_(torch.from_numpy(fx["init_user"]))
    eng.params[eng.U:].copy_(torch.from_numpy(fx["init_item"]))
    return m, eng


@pytest.mark.parametrize("name", ["MF", "LightGCN", "SimGCL", "XSimGCL", "SGL"])
@pytest.mark.parametrize("graph_mode", [False, True])
def test_fused_train_steps_match_reference(torch_cuda, golden, tiny, tiny_conf, tiny_triples, in_tmp_cwd, name, graph_mode):
    torch = torch_cuda
    fx = golden(f"train_{name}.npz")
    m, eng = _make_model(name, tiny_conf, tiny_triples, fx)
    U, I = tiny["U"], tiny["I"]
    L = eng.L
    n_steps = int(fx["n_steps"])
    tags, vals = list(fx["loss_tags"]), list(fx["loss_vals"])
    per = len(tags) // n_steps
    if name == "SGL":
        eng.set_view_graphs(*[_csr(fx, f"view{k}", (U + I, U + I)) for k in range(2)])
    views = 2 if name == "SimGCL" else 1
    noise_dev = None
    if "noise" in fx.files:
        noise_dev = torch.empty((views, L, U + I, 64), device="cuda")
        eng.set_noise_tensor(noise_dev)
    g = None
    for k in range(n_steps):
        if noise_dev is not None:
            nz = fx["noise"][k * views * L:(k + 1) * views * L].reshape(views, L, U + I, 64)
            noise_dev.copy_(torch.from_numpy(nz))
        words = _batch_words(fx[f"b{k}_u"], fx[f"b{k}_i"], fx[f"b{k}_j"], eng.B)
        if graph_mode:
            eng.batch_dev.copy_(torch.from_numpy(words))
            if g is None:
                snap = [t.clone() for t in (eng.params, eng.m, eng.v, eng.step_dev)]
                g = eng.capture()  # capture() runs warm-up steps: restore the state afterwards
                for t, s in zip((eng.params, eng.m, eng.v, eng.step_dev), snap):
                    t.copy_(s)
            g.replay()
        else:
            eng.step(words)
        torch.cuda.synchronize()
        rec = dict()
        for t, val in zip(tags[k * per:(k + 1) * per], vals[k * per:(k + 1) * per]):
            rec.setdefault(t, []).append(val)
        los = eng.losses.cpu().numpy()
        assert abs(los[0] - rec["bpr_loss"][0]) <= RTOL * abs(rec["bpr_loss"][0]), (name, k)
        div = 128.0 if name in ("MF", "LightGCN") else 1.0
        assert abs(los[1] - rec["l2_reg_loss"][0] / div) <= RTOL * abs(rec["l2_reg_loss"][0] / div), (name, k)
        if "InfoNCE" in rec:
            lam = CFG[name][0]["lambda"]
            assert abs(los[2] - lam * sum(rec["InfoNCE"])) <= RTOL * abs(lam * sum(rec["InfoNCE"])), (name, k)
        np.testing.assert_allclose(eng.params.cpu().numpy(), fx[f"params_after_{k}"], rtol=RTOL, atol=1e-6, err_msg=f"{name} step {k}")
    if name != "SGL":  # SGL only snapshots from epoch 5 on (SGL.py:45-46): its golden final_* is the pre-train forward
        ue, ie = eng.forward_clean()
        np.testing.assert_allclose(ue.cpu().numpy(), fx["final_user"], rtol=RTOL, atol=1e-6)
        np.testing.assert_allclose(ie.cpu().numpy(), fx["final_item"], rtol=RTOL, atol=1e-6)


def test_op_level_dropin_runs_reference_style_train_body(torch_cuda, golden, tiny):
    """The reference's LightGCN train() body (LightGCN.py:21-29, 68-78) written against the five
    drop-in modules only -- torch.sparse.mm(handle, E), list indexing, bpr_loss, l2_reg_loss,
    torch.optim.Adam -- must reproduce the reference's parameters step for step."""
    torch = torch_cuda
    from selfrec_b200.base.torch_interface import TorchGraphInterface
    from selfrec_b200.util.loss_torch import bpr_loss, l2_reg_loss
    fx = golden("train_LightGCN.npz")
    U = tiny["U"]
    ue = torch.nn.Parameter(torch.from_numpy(fx["init_user"]).cuda())
    ie = torch.nn.Parameter(torch.from_numpy(fx["init_item"]).cuda())
    A = TorchGraphInterface.convert_sparse_mat_to_tensor(tiny["norm"]).cuda()
    opt = torch.optim.Adam([ue, ie], lr=0.001)
    for k in range(int(fx["n_steps"])):
        ego = torch.cat([ue, ie], 0)
        layers = [ego]
        for _ in range(3):
            ego = torch.sparse.mm(A, ego)
            layers.append(ego)
        out = torch.mean(torch.stack(layers, dim=1), dim=1)
        ru, ri = out[:U], out[U:]
        u, i, j = (fx[f"b{k}_{t}"].tolist() for t in ("u", "i", "j"))
        loss = bpr_loss(ru[u], ri[i], ri[j]) + l2_reg_loss(0.0001, ue[u], ie[i], ie[j]) / 128
        opt.zero_grad()
        loss.backward()
        opt.step()
        got = torch.cat([ue, ie]).detach().cpu().numpy()
        np.testing.assert_allclose(got, fx[f"params_after_{k}"], rtol=RTOL, atol=1e-6)


@pytest.mark.parametrize("name", ["XSimGCL", "SimGCL"])
def test_op_level_dropin_contrastive_train_body(torch_cuda, golden, tiny, name):
    """The reference's XSimGCL / SimGCL train() bodies (XSimGCL.py:27-37, 83-101 and :46-50; SimGCL.py:25-36, 81-93 and
    :43-50) written against the drop-in modules only -- torch.sparse.mm(handle, E), the perturbed encoder with the
    recorded rand_like draws, bpr_loss, l2_reg_loss, InfoNCE over the unique batch ids, torch.optim.Adam -- must
    reproduce the reference's parameters step for step."""
    torch = torch_cuda
    import torch.nn.functional as F
    from selfrec_b200.base.torch_interface import TorchGraphInterface
    from selfrec_b200.util.loss_torch import InfoNCE, bpr_loss, l2_reg_loss
    fx = golden(f"train_{name}.npz")
    U = tiny["U"]
    n_layers, eps, cl_rate, tau = (3, 0.2, 0.2, 0.2) if name == "XSimGCL" else (2, 0.1, 0.5, 0.2)
    ue = torch.nn.Parameter(torch.from_numpy(fx["init_user"]).cuda())
    ie = torch.nn.Parameter(torch.from_numpy(fx["init_item"]).cuda())
    A = TorchGraphInterface.convert_sparse_mat_to_tensor(tiny["norm"]).cuda()
    opt = torch.optim.Adam([ue, ie], lr=0.001)
    draws = iter(fx["noise"])  # the reference's torch.rand_like draws, in call order

    def encoder(perturbed):
        ego = torch.cat([ue, ie], 0)
        layers, cl = [], ego
        for k in range(n_layers):
            ego = torch.sparse.mm(A, ego)
            if perturbed:
                noise = torch.from_numpy(next(draws)).cuda()
                ego = ego + torch.sign(ego) * F.normalize(noise, dim=-1) * eps
            layers.append(ego)
            if k == 0:  # XSimGCL's l* = 1
                cl = ego
        out = torch.mean(torch.stack(layers, dim=1), dim=1)
        return out[:U], out[U:], cl[:U], cl[U:]

    for k in range(int(fx["n_steps"])):
        u, i, j = (fx[f"b{k}_{t}"].tolist() for t in ("u", "i", "j"))
        u_idx = torch.unique(torch.tensor(u, dtype=torch.long)).cuda()
        i_idx = torch.unique(torch.tensor(i, dtype=torch.long)).cuda()
        if name == "XSimGCL":
            ru, ri, cu, ci = encoder(True)
            cl_loss = InfoNCE(ru[u_idx], cu[u_idx], tau) + InfoNCE(ri[i_idx], ci[i_idx], tau)
        else:
            ru, ri, _, _ = encoder(False)
            v1u, v1i, _, _ = encoder(True)
            v2u, v2i, _, _ = encoder(True)
            cl_loss = InfoNCE(v1u[u_idx], v2u[u_idx], tau) + InfoNCE(v1i[i_idx], v2i[i_idx], tau)
        loss = bpr_loss(ru[u], ri[i], ri[j]) + l2_reg_loss(0.0001, ru[u], ri[i]) + cl_rate * cl_loss
        opt.zero_grad()
        loss.backward()
        opt.step()
        got = torch.cat([ue, ie]).detach().cpu().numpy()
        np.testing.assert_allclose(got, fx[f"params_after_{k}"], rtol=RTOL, atol=1e-6, err_msg=f"{name} step {k}")
    assert next(draws, None) is None, "every recorded noise draw is consumed"


# ------------------------------------------------------------------------------------------
# (iv) scoring + top-k
# ------------------------------------------------------------------------------------------
def test_rank_matches_reference_test(torch_cuda, golden, tiny):
    torch = torch_cuda
    from selfrec_b200 import ops
    r = golden("rank.npz")
    g = tiny["g"]
    uid = {n: k for k, n in enumerate(g["user_names"])}
    users = np.array([uid[u] for u in r["users"]], dtype=np.int32)
    ids, sc = ops.score_topk(torch.from_numpy(r["user_emb"]).cuda(), torch.from_numpy(r["item_emb"]).cuda(), users,
                             tiny["im"].indptr, tiny["im"].indices, 10)
    assert np.array_equal(g["item_names"][ids.cpu().numpy()], r["items"])  # bit-exact ids vs reference test()
    np.testing.assert_allclose(sc.cpu().numpy(), r["scores"], rtol=2e-5, atol=1e-7)


@pytest.mark.parametrize("d,k,n_items,n_q", [(64, 20, 1000, 70), (32, 5, 257, 33), (128, 32, 640, 40), (64, 1, 129, 3)])
def test_score_topk_bit_exact_vs_oracle(torch_cuda, orc, d, k, n_items, n_q):
    torch = torch_cuda
    from selfrec_b200 import ops
    rng = np.random.default_rng(d + k)
    n_users = 90
    ue = rng.standard_normal((n_users, d)).astype(np.float32)
    ie = rng.standard_normal((n_items, d)).astype(np.float32)
    users = rng.integers(0, n_users, n_q).astype(np.int32)
    rated = sp.random(n_users, n_items, density=0.05, random_state=7, format="csr")
    rated.sort_indices()
    oi, os_, full = orc.score_topk(ue, ie, users, rated.indptr, rated.indices, k, want_scores=True)
    ids, sc = ops.score_topk(torch.from_numpy(ue).cuda(), torch.from_numpy(ie).cuda(), users, rated.indptr, rated.indices, k)
    assert np.array_equal(ids.cpu().numpy(), oi)      # same fma chain -> identical ids
    assert np.array_equal(sc.cpu().numpy(), os_)      # and identical bits
    dense = ops.score_rows(torch.from_numpy(ue).cuda(), torch.from_numpy(ie).cuda(), users)
    assert np.array_equal(dense.cpu().numpy(), full)


def test_topk_tie_semantics_match_find_k_largest(torch_cuda, orc, golden):
    """Ties: the selected SET equals find_k_largest's; order within exactly-tied scores is the
    reference's unstable sort order and is not reproduced (DESIGN.md)."""
    torch = torch_cuda
    from selfrec_b200 import ops
    tk = golden("topk.npz")
    for tag in ("rand", "ties", "survey", "const", "masked", "asc", "desc"):
        v = tk[f"{tag}_in"]
        for K in (3, 10, 20):
            ids, sc = ops.topk_rows(torch.from_numpy(v[None]).cuda(), K)
            ref_ids, ref_sc = tk[f"{tag}_K{K}_ids"], tk[f"{tag}_K{K}_scores"]
            ids, sc = ids[0].cpu().numpy(), sc[0].cpu().numpy()
            if len(ref_ids) < K:  # fewer than K candidates: the reference returns them all, the kernel pads with id -1 / -inf
                assert (ids[len(ref_ids):] == -1).all() and np.isneginf(sc[len(ref_ids):]).all()
                ids, sc = ids[:len(ref_ids)], sc[:len(ref_ids)]
            assert sorted(ids.tolist()) == sorted(ref_ids.tolist()), (tag, K)
            assert np.array_equal(sc, ref_sc), (tag, K)  # score sequence identical
            if len(np.unique(ref_sc)) == len(ref_sc):
                assert np.array_equal(ids, ref_ids)
    # integer-valued embeddings make every dot product exact, so ties are real
    rng = np.random.default_rng(0)
    ue = rng.integers(-2, 3, (40, 64)).astype(np.float32)
    ie = rng.integers(-2, 3, (900, 64)).astype(np.float32)
    users = np.arange(40, dtype=np.int32)
    oi, os_ = orc.score_topk(ue, ie, users, None, None, 20)
    ids, sc = ops.score_topk(torch.from_numpy(ue).cuda(), torch.from_numpy(ie).cuda(), users, None, None, 20)
    assert np.array_equal(sc.cpu().numpy(), os_)
    assert all(sorted(a) == sorted(b) for a, b in zip(ids.cpu().numpy().tolist(), oi.tolist()))


def test_topk_edge_cases(torch_cuda, orc):
    torch = torch_cuda
    from selfrec_b200 import ops, _lib
    rng = np.random.default_rng(5)
    ue = rng.standard_normal((4, 64)).astype(np.float32)
    ie = rng.standard_normal((30, 64)).astype(np.float32)
    # a user who rated everything but 3 items: masked -1e9 entries surface in the top-5 like the reference
    ptr = np.array([0, 27, 27, 27, 27], dtype=np.int32)
    idx = np.arange(27, dtype=np.int32)
    oi, os_ = orc.score_topk(ue, ie, np.array([0, 1], np.int32), ptr, idx, 5)
    ids, sc = ops.score_topk(torch.from_numpy(ue).cuda(), torch.from_numpy(ie).cuda(), [0, 1], ptr, idx, 5)
    assert np.array_equal(sc.cpu().numpy(), os_) and (sc[0].cpu().numpy() == np.float32(-1e9)).sum() == 2
    assert sorted(ids[0].tolist()) == sorted(oi[0].tolist()) and np.array_equal(ids[1].cpu().numpy(), oi[1])
    with pytest.raises(_lib.SrbError):
        ops.score_topk(torch.from_numpy(ue).cuda(), torch.from_numpy(ie).cuda(), [0], None, None, 33)
    e_ids, _ = ops.score_topk(torch.from_numpy(ue).cuda(), torch.from_numpy(ie).cuda(), np.zeros(0, np.int32), None, None, 5)
    assert e_ids.shape == (0, 5)


def test_graph_recommender_test_and_fast_evaluation(torch_cuda, golden, tiny, tiny_conf, tiny_triples, in_tmp_cwd):
    """GraphRecommender.test() output format + fast_evaluation keep-best protocol (graph_recommender.py:38-104)."""
    torch = torch_cuda
    r = golden("rank.npz")
    fx = golden("train_XSimGCL.npz")
    m, eng = _make_model("XSimGCL", tiny_conf, tiny_triples, fx)
    m.user_emb, m.item_emb = torch.from_numpy(r["user_emb"]).cuda(), torch.from_numpy(r["item_emb"]).cuda()
    rec = m.test()
    assert list(rec) == list(r["users"])  # test_set dict order
    for k, u in enumerate(r["users"]):
        assert [it for it, _ in rec[u]] == list(r["items"][k])
        assert all(isinstance(s, float) for _, s in rec[u])
    measure = m.fast_evaluation(0)
    assert measure == list(r["measure"][5:])  # the 'Top 10' block of ranking_evaluation(..., [5, 10])
    assert m.bestPerformance[0] == 1 and hasattr(m, "best_user_emb")
    sc = m.predict(r["users"][0])
    assert sc.shape == (tiny["I"],) and sc.dtype == np.float32


def test_rank_hit_masks_and_fast_measure(torch_cuda, golden, tiny_triples, tiny_conf, in_tmp_cwd):
    """srb_rank_hit_masks against a numpy restatement on random lists, and the id-space fast_evaluation path
    against ranking_evaluation over the name-keyed test() output (the reference's route)."""
    torch = torch_cuda
    from selfrec_b200 import ops
    from selfrec_b200.util.evaluation import ranking_evaluation, ranking_evaluation_from_masks
    rng = np.random.default_rng(5)
    U, I, K = 300, 1000, 20
    ptr = np.zeros(U + 1, dtype=np.int32)
    rows = [np.sort(rng.choice(I, size=rng.integers(0, 30), replace=False)).astype(np.int32) for _ in range(U)]
    ptr[1:] = np.cumsum([len(x) for x in rows])
    idx = np.concatenate(rows).astype(np.int32)
    users = rng.permutation(U)[:257].astype(np.int32)
    ids = np.stack([rng.choice(I, size=K, replace=False) for _ in users]).astype(np.int32)
    got = ops.rank_hit_masks(torch.from_numpy(ids).cuda(), users, ptr, idx).cpu().numpy().view(np.uint64)
    want = np.array([sum(1 << r for r in range(K) if ids[q, r] in set(rows[u].tolist())) for q, u in enumerate(users)], dtype=np.uint64)
    assert (got == want).all()
    for k in (1, 33, 64):
        ids2 = np.stack([rng.choice(I, size=k, replace=False) for _ in users]).astype(np.int32)
        g2 = ops.rank_hit_masks(torch.from_numpy(ids2).cuda(), users, ptr, idx).cpu().numpy().view(np.uint64)
        w2 = np.array([sum(1 << r for r in range(k) if ids2[q, r] in set(rows[u].tolist())) for q, u in enumerate(users)], dtype=np.uint64)
        assert (g2 == w2).all()
    # whole fast path on the golden embeddings
    from selfrec_b200.base.graph_recommender import GraphRecommender
    train, test = tiny_triples
    r = golden("rank.npz")
    m = GraphRecommender(tiny_conf("MF"), [list(t) for t in train], [list(t) for t in test])
    m.user_emb = torch.from_numpy(r["user_emb"]).cuda()
    m.item_emb = torch.from_numpy(r["item_emb"]).cuda()
    fast = m._fast_measure()
    slow = ranking_evaluation(m.data.test_set, m.test(), [m.max_N])
    assert fast == slow


def _norm_adj(pu, pi, U, I):
    """D^-1/2 [[0, R], [R^T, 0]] D^-1/2 of the (user, item) pairs, as float32 CSR."""
    n = U + I
    half = sp.csr_matrix((np.ones(len(pu), np.float32), (pu, pi.astype(np.int64) + U)), shape=(n, n), dtype=np.float32)
    adj = half + half.T
    d = np.asarray(adj.sum(1)).ravel()
    dinv = np.power(d, -0.5, out=np.zeros_like(d), where=d > 0).astype(np.float32)  # a dropped view may isolate a node
    return sp.diags(dinv).dot(adj).dot(sp.diags(dinv)).tocsr().astype(np.float32)


class _SynthData:
    """What TrainEngine reads from an Interaction, for a random bipartite graph."""

    def __init__(self, rng, U, I, n_pairs):
        pu = rng.integers(0, U, n_pairs).astype(np.int32)
        pi = (rng.zipf(1.5, n_pairs) % I).astype(np.int32)
        pu[:U] = np.arange(U)  # every user and item appears
        pi[:I] = np.arange(I)
        self.user_num, self.item_num = U, I
        self.pair_users, self.pair_items = pu, pi
        self.norm_adj = _norm_adj(pu, pi, U, I)
        self.training_data = []


@pytest.mark.parametrize("name,d,L,lcl", [("XSimGCL", 32, 2, 1), ("XSimGCL", 128, 3, 3), ("XSimGCL", 64, 1, 1), ("XSimGCL", 64, 2, 0),
                                          ("SimGCL", 128, 2, 0), ("SimGCL", 64, 1, 0), ("SimGCL", 32, 5, 0), ("SGL", 64, 1, 0),
                                          ("SGL", 128, 3, 0), ("LightGCN", 32, 3, 0), ("MF", 128, 0, 0)])
def test_engine_steps_vs_oracle_other_widths_and_partial_batches(torch_cuda, orc, name, d, L, lcl):
    """The fused step against the float64 oracle at embedding sizes 32 / 128 (CUDA-core InfoNCE, other SpMM
    instantiations), with every position of the contrastive layer, one and five SimGCL layers, SGL on two
    edge-dropped view graphs, a short last batch and an EMPTY batch (which must leave parameters to Adam's
    zero-gradient update, exactly like the oracle)."""
    torch = torch_cuda
    from selfrec_b200.engine import TrainEngine
    rng = np.random.default_rng(d * 10 + L)
    U, I, B = 150, 220, 64
    data = _SynthData(rng, U, I, 3000)
    N = U + I
    E0 = (rng.standard_normal((N, d)) * 0.1).astype(np.float32)
    kw = dict(eps=0.2, tau=0.2, cl_rate=0.3, layer_cl=lcl) if name in ("XSimGCL", "SimGCL") else {}
    if name in ("MF", "LightGCN"):
        kw["l2_div"] = float(B)
    if name == "SGL":
        kw = dict(tau=0.2, cl_rate=0.3)
    eng = TrainEngine(name, data, d, L, B, 1e-2, 1e-3, init_user=torch.from_numpy(E0[:U]), init_item=torch.from_numpy(E0[U:]), **kw)
    view_csr = None
    if name == "SGL":  # edge dropout at rate 0.1, re-normalised (SGL.py:27-29)
        keep = [rng.random(len(data.pair_users)) >= 0.1 for _ in range(2)]
        view_csr = [_norm_adj(data.pair_users[k], data.pair_items[k], U, I) for k in keep]
        eng.set_view_graphs(*view_csr)
    views = 2 if name == "SimGCL" else 1
    p, m, v = E0.copy(), np.zeros_like(E0), np.zeros_like(E0)
    for step, b in enumerate((B, 17, 0, B), start=1):
        u = rng.integers(0, U, b).astype(np.int32)
        i = rng.integers(0, I, b).astype(np.int32)
        j = rng.integers(0, I, b).astype(np.int32)
        noise = None
        if name in ("XSimGCL", "SimGCL"):
            noise = rng.random((views, max(L, 1), N, d), dtype=np.float32)
            eng.set_noise_tensor(torch.from_numpy(noise[:, :L]).cuda())
        eng.step(_batch_words(u, i, j, B))
        torch.cuda.synchronize()
        if b == 0:
            g, ref = np.zeros((N, d)), None
        else:
            ref = orc.train_step(name, data.norm_adj if name != "MF" else None, p, U, u, i, j, n_layers=L, reg=1e-3,
                                 batch_size=B, eps=0.2, tau=0.2, cl_rate=0.3, layer_cl=lcl, noise=None if noise is None else noise[:, :L],
                                 view_csr=view_csr)
            g = ref["grad"]
        p, m, v = orc.adam_step(p, g.astype(np.float32), m, v, step, 1e-2)
        got = eng.params.cpu().numpy()
        # Adam divides by sqrt(v) + 1e-8: entries whose gradient is ~1e-8 or below are ill-conditioned in fp32
        cond = np.abs(g) > 1e-6
        np.testing.assert_allclose(got[cond], p[cond], rtol=RTOL, atol=2e-6, err_msg=f"{name} d={d} step {step} b={b}")
        assert np.abs(got - p).max() <= 2.5e-2  # lr-bounded everywhere (|update| <= lr / (1 - beta1) early on)
        if ref is not None:
            los = eng.losses.cpu().numpy()
            assert abs(los[0] - ref["rec"]) <= RTOL * abs(ref["rec"]) + 1e-7
            assert abs(los[2] - ref["cl"]) <= RTOL * abs(ref["cl"]) + 2e-7 / 0.2
        p = got.astype(np.float32).copy()  # continue from the device state: errors do not compound across steps
        m, v = eng.m.cpu().numpy().copy(), eng.v.cpu().numpy().copy()


def test_topk_lists_longer_than_the_kernel_width(torch_cuda, orc):
    """item.ranking.topN up to 100 works like the reference (find_k_largest accepts any K): lists above 32 entries are
    extracted 32 at a time with the same kernels; ids and scores equal the oracle's."""
    torch = torch_cuda
    from selfrec_b200 import ops
    rng = np.random.default_rng(9)
    U, I = 40, 700
    ue = rng.standard_normal((U, 64)).astype(np.float32)
    ie = rng.standard_normal((I, 64)).astype(np.float32)
    deg = rng.integers(0, 60, U)
    ptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int32)
    idx = np.concatenate([np.sort(rng.choice(I, k, replace=False)) for k in deg]).astype(np.int32)
    users = np.arange(U, dtype=np.int32)
    for k in (33, 50, 100):
        ids, sc = ops.score_topk(torch.from_numpy(ue).cuda(), torch.from_numpy(ie).cuda(), users, ptr, idx, k)
        oi, os_ = orc.score_topk(ue, ie, users, ptr, idx, k)
        assert np.array_equal(ids.cpu().numpy(), oi) and np.array_equal(sc.cpu().numpy(), os_), k
