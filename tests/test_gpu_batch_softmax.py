"""batch_softmax_loss on the GPU (srb_batch_softmax_fwd_bwd through ops.batch_softmax_loss) against the float64
restatement and the reference-generated fixture, on both kernel routes, and the op-level drop-in under install():
SSL4Rec- and SASRec-style train bodies on the aliased util.loss_torch / util.sampler."""
import importlib
import os
import random
import sys

import numpy as np
import pytest

import batch_softmax_oracle as bso

pytestmark = pytest.mark.gpu

RTOL = 1e-4
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
N_EDGES = [1, 2, 31, 33, 127, 129, 2049]
TC_TAU = 1 / 40  # d = 64 takes the tensor-core route up to 1/tau = 40
# absolute floor of the loss error: log p_r = S_rr - lse_r takes S_rr from two fp32 evaluations (the exact diagonal and the
# tile's), each a few ulp of |S| <= 1/tau off (n = 1 is the worst case: no averaging over rows)
LOSS_FLOOR = 6e-7


@pytest.fixture(scope="module")
def torch_cuda(built_lib):
    import torch
    assert torch.cuda.is_available()
    from selfrec_b200 import _lib
    _lib.require_device()
    return torch


def _floor(u, i, tau):
    """fp32 conditioning of the gradient near a zero loss gradient (test_infonce_batch_sizes): G_rr = c_r (P_rr - 1)
    carries an absolute error ~ eps32 / tau, through 1/(n tau), a unit-vector entry and 1/||v||."""
    n, d = u.shape
    norms = np.linalg.norm(np.concatenate([u, i]).astype(np.float64), axis=1)
    return 3 * 1.2e-7 / tau / (n * tau) / np.sqrt(d) / norms[norms > 0].min()


def _run(torch, u, i, tau):
    from selfrec_b200 import ops
    tu, ti = (torch.from_numpy(x).cuda().requires_grad_(True) for x in (u, i))
    loss = ops.batch_softmax_loss(tu, ti, tau)
    assert loss.dim() == 0
    gu, gi = torch.autograd.grad(loss, (tu, ti))
    return loss.item(), gu.cpu().numpy(), gi.cpu().numpy()


def _check(torch, u, i, tau, err=""):
    loss, gu, gi = _run(torch, u, i, tau)
    ref, ru, ri = bso.batch_softmax_loss(u, i, tau)
    # the loss is a mean of -log(p + 1e-5) with log p = S_rr - lse_r and |S| up to 1/tau
    assert abs(loss - ref) <= RTOL * abs(ref) + LOSS_FLOOR / tau, (err, loss, ref)
    cond = _floor(u, i, tau)
    for mine, want in ((gu, ru), (gi, ri)):
        np.testing.assert_allclose(mine, want, rtol=RTOL, atol=2e-5 * np.abs(want).max() + cond, err_msg=err)


def _inputs(n, d, seed, lean=0.1):
    rng = np.random.default_rng(seed)
    u = (rng.standard_normal((n, d)) * 0.1).astype(np.float32)
    i = (u + lean * rng.standard_normal((n, d)) * 0.1).astype(np.float32)
    return u, i


@pytest.mark.parametrize("n", N_EDGES)
@pytest.mark.parametrize("d", [16, 32, 64, 128, 256])
def test_batch_softmax_matches_float64(torch_cuda, d, n):
    u, i = _inputs(n, d, 1000 * d + n)
    _check(torch_cuda, u, i, 0.2, f"d={d} n={n}")


@pytest.mark.parametrize("n", N_EDGES)
@pytest.mark.parametrize("tau", [TC_TAU, 1 / 41], ids=["tensor_core", "cuda_core"])
def test_batch_softmax_both_routes_at_d64(torch_cuda, tau, n):
    """d = 64 on either side of the tensor-core limit 1/tau <= 40: the two routes compute the same loss."""
    u, i = _inputs(n, 64, 7 * n, lean=0.3)
    _check(torch_cuda, u, i, tau, f"tau={tau} n={n}")


def test_batch_softmax_zero_rows(torch_cuda):
    for d, tau in ((64, 0.2), (64, 0.02), (128, 0.07)):
        u, i = _inputs(130, d, d)
        u[[0, 64, 129]] = 0
        i[[3, 64]] = 0
        loss, gu, gi = _run(torch_cuda, u, i, tau)
        ref, ru, ri = bso.batch_softmax_loss(u, i, tau)
        assert abs(loss - ref) <= RTOL * abs(ref) + LOSS_FLOOR / tau
        cond = _floor(u, i, tau)
        for mine, want in ((gu, ru), (gi, ri)):  # a zero row's gradient is 1e12 times the others': per-row scale
            atol = 2e-5 * np.abs(want).max(1, keepdims=True) + cond
            assert (np.abs(mine - want) <= RTOL * np.abs(want) + atol).all(), (d, tau)


def test_batch_softmax_matches_reference_fixture(torch_cuda, golden):
    fx = golden("sequence.npz")
    tags = sorted({k.split("_")[1] for k in fx.files if k.startswith("bsm_")})
    assert len(tags) >= 6
    for tag in tags:
        g = lambda k: fx[f"bsm_{tag}_{k}"]
        tau = float(g("tau"))
        u, i = bso.case_inputs(int(g("n")), int(g("d")), int(g("salt")), g("zero_users"), g("zero_items"))
        loss, gu, gi = _run(torch_cuda, u, i, tau)
        ref = float(g("loss"))
        assert abs(loss - ref) <= RTOL * abs(ref) + LOSS_FLOOR / tau, (tag, loss, ref)
        rows, cond = g("rows"), _floor(u, i, tau)
        for mine, key in ((gu[rows], "gu"), (gi[rows], "gi")):
            want = g(key)
            atol = 2e-5 * np.abs(want).max(1, keepdims=True) + cond
            assert (np.abs(mine - want) <= RTOL * np.abs(want) + atol).all(), (tag, key)


@pytest.mark.parametrize("d", [64, 128])
def test_batch_softmax_stays_finite_below_tau_one_over_88(torch_cuda, d):
    """The reference's unshifted exp(S / tau) overflows fp32 once 1/tau > 88.7 and returns inf or NaN; the kernels work
    in log-sum-exp form and give the float64 value of the same formula."""
    torch = torch_cuda
    u, i = _inputs(300, d, 3, lean=0.3)  # positive cosines near 0.96: exp(S_rr / tau) overflows from 1/tau = 93 on
    for tau in (1 / 100, 1 / 300):
        loss, gu, gi = _run(torch, u, i, tau)
        assert np.isfinite(loss) and np.isfinite(gu).all() and np.isfinite(gi).all()
        _check(torch, u, i, tau, f"tau={tau}")
        tu, ti = (torch.nn.functional.normalize(torch.from_numpy(x).cuda(), dim=1) for x in (u, i))
        e = torch.exp(tu @ ti.T / tau)  # the reference's form in fp32
        assert not torch.isfinite(e.sum(1)).all()


def _torch_batch_softmax_loss(user_emb, item_emb, temperature):
    """util/loss_torch.py:25-32 in torch, for the train-body comparison."""
    import torch
    import torch.nn.functional as F
    user_emb, item_emb = F.normalize(user_emb, dim=1), F.normalize(item_emb, dim=1)
    pos_score = torch.exp((user_emb * item_emb).sum(dim=-1) / temperature)
    ttl_score = torch.exp(torch.matmul(user_emb, item_emb.transpose(0, 1)) / temperature).sum(dim=1)
    return torch.mean(-torch.log(pos_score / ttl_score + 10e-6))


@pytest.fixture()
def installed(built_lib):
    import selfrec_b200
    names = selfrec_b200.install(fused_models=False)
    yield lambda alias: importlib.import_module(alias)
    for n in names:
        sys.modules.pop(n, None)


def _ssl4rec_losses(torch, installed, tiny_conf, tiny_triples, rec_loss_fn):
    """SSL4Rec.train() (SSL4Rec.py:24-40, DNN_Encoder :52-96) written against the aliased modules: towers over the
    initial embeddings, batch_softmax_loss on the (query, item) pairs of next_batch_pairwise, InfoNCE over two dropout
    views of the item tower, l2_reg_loss, torch.optim.Adam.  Three steps; returns the per-step losses."""
    import torch.nn as nn
    sampler, losses = installed("util.sampler"), installed("util.loss_torch")
    Interaction = installed("data.ui_graph").Interaction
    train, test = tiny_triples
    data = Interaction(tiny_conf("SSL4Rec"), [list(t) for t in train], [list(t) for t in test])
    torch.manual_seed(0)
    random.seed(0)
    emb, tau, cl_rate, reg = 64, 0.07, 0.1, 1e-4

    def tower():
        return nn.Sequential(nn.Linear(emb, 1024), nn.ReLU(True), nn.Linear(1024, 128), nn.Tanh())

    user_tower, item_tower, dropout = tower().cuda(), tower().cuda(), nn.Dropout(0.1)
    user_e = nn.Parameter(nn.init.xavier_uniform_(torch.empty(data.user_num, emb)).cuda())
    item_e = nn.Parameter(nn.init.xavier_uniform_(torch.empty(data.item_num, emb)).cuda())
    params = [user_e, item_e, *user_tower.parameters(), *item_tower.parameters()]
    opt = torch.optim.Adam(params, lr=0.001)
    out = []
    for n, (query_idx, item_idx, _neg) in enumerate(sampler.next_batch_pairwise(data, 128)):
        if n == 3:
            break
        query_emb, item_emb = user_tower(user_e[query_idx]), item_tower(item_e[item_idx])
        rec_loss = rec_loss_fn(query_emb, item_emb, tau)
        i_emb = item_e[item_idx]
        cl_loss = cl_rate * losses.InfoNCE(item_tower(dropout(i_emb)), item_tower(dropout(i_emb)), tau)
        batch_loss = rec_loss + losses.l2_reg_loss(reg, query_emb, item_emb) + cl_loss
        opt.zero_grad()
        batch_loss.backward()
        opt.step()
        out.append((rec_loss.item(), batch_loss.item()))
    return out


def test_op_level_ssl4rec_style_train_body(torch_cuda, installed, tiny_conf, tiny_triples, in_tmp_cwd):
    torch = torch_cuda
    losses = installed("util.loss_torch")
    assert losses.batch_softmax_loss.__module__ == "selfrec_b200.ops"
    mine = _ssl4rec_losses(torch, installed, tiny_conf, tiny_triples, losses.batch_softmax_loss)
    ref = _ssl4rec_losses(torch, installed, tiny_conf, tiny_triples, _torch_batch_softmax_loss)
    assert len(mine) == len(ref) == 3
    for k, ((r1, t1), (r2, t2)) in enumerate(zip(mine, ref)):
        assert abs(r1 - r2) <= RTOL * abs(r2), (k, r1, r2)
        assert abs(t1 - t2) <= RTOL * abs(t2), (k, t1, t2)


def test_op_level_sasrec_style_train_body(torch_cuda, installed, golden, in_tmp_cwd):
    """SASRec.train() (SASRec.py:24-55) written against the aliased modules on the crafted sequential dataset:
    next_batch_sequence batches into an item + position embedding with one causal self-attention layer, the BCE loss
    over positives and sampled negatives at the non-padding positions, l2_reg_loss on the item table, Adam; three
    steps, then the test batches of next_batch_sequence_for_test through predict's last-position scores."""
    torch = torch_cuda
    import torch.nn as nn
    sampler, losses = installed("util.sampler"), installed("util.loss_torch")
    FileIO = installed("data.loader").FileIO
    train = FileIO.load_data_set(os.path.join(GOLDEN, "seq_crafted_train.txt"), "sequential")
    ids, original = {}, []
    for name, items in train.items():  # data/sequence.py's indexing (test_sequence_cpu checks it)
        if len(items) >= 2:
            original.append((name, [ids.setdefault(it, len(ids) + 1) for it in items]))

    class Data:
        original_seq, item_num = original, len(ids)

    torch.manual_seed(0)
    random.seed(0)
    emb, max_len = 64, 8
    item_emb = nn.Parameter(nn.init.xavier_uniform_(torch.empty(Data.item_num + 1, emb)).cuda())
    pos_emb = nn.Parameter(nn.init.xavier_uniform_(torch.empty(max_len + 1, emb)).cuda())
    attn = nn.MultiheadAttention(emb, 1, batch_first=True).cuda()
    mask = torch.triu(torch.ones(max_len, max_len, dtype=torch.bool, device="cuda"), 1)

    def forward(seq, pos):
        x = item_emb[torch.from_numpy(seq).cuda()] + pos_emb[torch.from_numpy(pos).cuda()]
        return x + attn(x, x, x, attn_mask=mask, need_weights=False)[0]

    bce = nn.BCEWithLogitsLoss()
    before = item_emb.detach().clone()
    opt = torch.optim.Adam([item_emb, pos_emb, *attn.parameters()], lr=0.001)
    steps = []
    for n, (seq, pos, y, neg, seq_len) in enumerate(sampler.next_batch_sequence(Data, 4, max_len=max_len)):
        if n == 3:
            break
        assert seq.shape == (4, max_len) and (seq_len == (pos != 0).sum(1)).all()
        assert not any(set(neg[r, :seq_len[r]]) & set(seq[r, :seq_len[r]]) for r in range(4))
        seq_out = forward(seq, pos)
        pos_logits = (seq_out * item_emb[torch.from_numpy(y).cuda()]).sum(-1)
        neg_logits = (seq_out * item_emb[torch.from_numpy(neg).cuda()]).sum(-1)
        idx = np.where(pos != 0)
        loss = bce(pos_logits[idx], torch.ones_like(pos_logits[idx])) + bce(neg_logits[idx], torch.zeros_like(neg_logits[idx]))
        batch_loss = loss + losses.l2_reg_loss(1e-4, item_emb)
        opt.zero_grad()
        batch_loss.backward()
        opt.step()
        steps.append(batch_loss.item())
    assert len(steps) == 3 and np.isfinite(steps).all()
    assert not torch.equal(before, item_emb.detach())
    with torch.no_grad():
        rows = 0
        for seq, pos, seq_len in sampler.next_batch_sequence_for_test(Data, 8, max_len=max_len):
            out = forward(seq, pos)
            last = out[torch.arange(len(seq_len), device="cuda"), torch.from_numpy(seq_len - 1).cuda()]
            score = last @ item_emb.T
            assert score.shape == (len(seq_len), Data.item_num + 1) and torch.isfinite(score).all()
            rows += len(seq_len)
    assert rows == len(original)
