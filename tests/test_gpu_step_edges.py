"""Every model's fused training step on a graph with rows at every class boundary of the SpMM and of the batch-row lists,
run from a NaN-poisoned workspace with live batch-buffer tails, against the float64 oracle.

The backward chain keeps its loss gradients in [N, d] seed tables that hold valid data only at the current batch's rows
(step_begin_kernel clears exactly those); every read of them is gated by the batch bitmap.  A read that escapes the
bitmap, or a kernel that reads past a batch count, is invisible when the stale data is finite and the buffers past the
counts hold row 0.  Here the stale data is NaN wherever an earlier step wrote it, and the batch buffers past b,
n_unique_u and n_unique_i hold valid ids of poisoned rows that are not in the batch, so such a read shows up as a
non-finite or wrong number.  The poison is float data only: every integer list the step builds comes from a valid
batch, and no trip count in the step depends on float data."""
import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu

U, I, B = 6000, 5000, 256
LR, REG, EPS, TAU, CL_RATE = 1e-2, 1e-3, 0.2, 0.2, 0.3
# special rows: user id -> degree, item id -> degree.  User 0 and item 0 are ordinary low-degree rows that the poison
# batch contains and no later batch does, so their seed rows stay NaN.
HUB_USERS = {1: 4096, 2: 4097, 3: 4095, 4: 256, 5: 255, 6: 128, 7: 127, 8: 64, 9: 63}
HUB_ITEMS = {1: 5000, 2: 4096}
# first-moment bar: per-row max error <= KAPPA * max|m_ref[row]| + 1e-6 * max|m_ref| (worst measured over all cases:
# 5.2e-5, XSimGCL d = 32, L = 3, l* = 1, on an H100 80GB HBM3)
KAPPA = 1e-4


@pytest.fixture(scope="module")
def torch_cuda(built_lib):
    import torch
    assert torch.cuda.is_available()
    from selfrec_b200 import _lib
    _lib.require_device()
    return torch


def _norm_adj(pu, pi, n_users, n_items):
    """D^-1/2 [[0, R], [R^T, 0]] D^-1/2 of the (user, item) pairs, as float32 CSR."""
    n = n_users + n_items
    half = sp.csr_matrix((np.ones(len(pu), np.float32), (pu, pi.astype(np.int64) + n_users)), shape=(n, n), dtype=np.float32)
    adj = half + half.T
    d = np.asarray(adj.sum(1)).ravel()
    dinv = np.power(d, -0.5, out=np.zeros_like(d), where=d > 0).astype(np.float32)  # a dropped view may isolate a node
    return sp.diags(dinv).dot(adj).dot(sp.diags(dinv)).tocsr().astype(np.float32)


class _HubData:
    """What the engines read from an Interaction: sizes, the (user, item) pairs and the normalised adjacency."""

    def __init__(self, pu, pi, n_users=U, n_items=I):
        self.user_num, self.item_num = n_users, n_items
        self.pair_users, self.pair_items = pu, pi
        self.norm_adj = _norm_adj(pu, pi, n_users, n_items)
        self.training_data = []


def _words(u, i, j, tail_u, tail_i):
    """Batch words whose sections are filled past b / n_unique_u / n_unique_i with the ids tail_u / tail_i (cycled)."""
    from selfrec_b200 import _lib
    H = _lib.BATCH_HEADER
    u, i, j = (np.asarray(x, dtype=np.int32) for x in (u, i, j))
    uq, iq = np.unique(u), np.unique(i)
    w = np.zeros(H + 5 * B, dtype=np.int32)
    w[0], w[1], w[2] = len(u), len(uq), len(iq)
    for k, (vals, tail) in enumerate(((u, tail_u), (i, tail_i), (j, tail_i), (uq, tail_u), (iq, tail_i))):
        sec = w[H + k * B:H + (k + 1) * B]
        sec[:len(vals)] = vals
        sec[len(vals):] = np.resize(np.asarray(tail, dtype=np.int32), B - len(vals))
    return w


def make_hub_graph(n_users, n_items, hub_users, hub_items, seed):
    """n_users x n_items bipartite graph, background user degree 3..9, with the users `hub_users` and the items
    `hub_items` ({id: degree}; the items' neighbours drawn from the other users) at the given degrees.  Users 1..9 and
    items 1, 2 must be among them: the batches below put them in the hub triples.  Returns dict(data, A, poison,
    batches, views): the graph, the poison batch, the five batches that follow it and SGL's view graphs."""
    from selfrec_b200 import ops
    U, I = n_users, n_items  # (shadow the module's sizes: everything below is sized by the graph it builds)
    rng = np.random.default_rng(seed)
    bg_items = np.setdiff1d(np.arange(I), list(hub_items))  # every item but the hubs
    pu, pi = [], []
    for u in range(U):
        k = hub_users.get(u, int(rng.integers(3, 10)))
        pu.append(np.full(k, u))
        pi.append(rng.choice(bg_items, k, replace=False))
    ordinary_users = np.setdiff1d(np.arange(U), list(hub_users))
    for it, k in hub_items.items():
        pu.append(rng.choice(ordinary_users, k, replace=False))
        pi.append(np.full(k, it))
    data = _HubData(np.concatenate(pu).astype(np.int32), np.concatenate(pi).astype(np.int32), U, I)
    A = data.norm_adj
    deg = np.diff(A.indptr)
    assert A.nnz == 2 * len(data.pair_users), "pairs are distinct"
    for u, k in hub_users.items():
        assert deg[u] == k, (u, deg[u])
    for it, k in hub_items.items():
        assert deg[U + it] == k, (it, deg[U + it])
    special = np.zeros(U + I, dtype=bool)
    special[list(hub_users)] = True
    special[[U + it for it in hub_items]] = True
    assert deg[~special].max() < ops.LONG_ROW_NNZ - 1
    assert deg[0] < ops.LONG_ROW_NNZ and deg[U] < ops.LONG_ROW_NNZ

    # disjoint pools of ordinary rows: batch 1, batch 2, tails only
    perm_u = rng.permutation(np.setdiff1d(ordinary_users, [0]))
    a_u, c_u, p_u = perm_u[:100], perm_u[100:117], perm_u[117:]
    perm_i = rng.permutation(np.setdiff1d(bg_items, [0]))
    a_i, c_i, p_i = perm_i[:150], perm_i[150:184], perm_i[184:]
    # poison batch: user 0, item 0, every hub and boundary row and every row a later batch uses, then tail-only rows
    users = np.concatenate([[0], list(hub_users), a_u, c_u])
    users = rng.permutation(np.concatenate([users, p_u[:B - len(users)]]))
    items = np.concatenate([[0], list(hub_items), a_i, c_i])
    items = rng.permutation(np.concatenate([items, p_i[:2 * B - len(items)]]))
    poison = (users, items[:B], items[B:])

    def batch(u, i, j):
        tail_u = np.setdiff1d(poison[0], u)
        tail_i = np.setdiff1d(np.concatenate(poison[1:]), np.concatenate([i, j]).astype(np.int64))
        assert 0 in tail_u and 0 in tail_i
        return _words(u, i, j, rng.permutation(tail_u), rng.permutation(tail_i)), (np.asarray(u), np.asarray(i), np.asarray(j))

    # 1. a full batch without user 0: hub users in a third of the triples, every boundary user, item 1 a positive 60
    #    times, item 2 a positive in 10 triples and a negative in 10 others, every further hub item a negative once
    more = np.array([it for it in hub_items if it not in (1, 2)], dtype=np.int64)
    u1 = np.concatenate([rng.choice([1, 2], 80), [3, 4, 5, 6, 7, 8, 9], rng.choice(a_u, B - 87)])
    i1 = np.concatenate([np.full(60, 1), np.full(10, 2), rng.choice(a_i, B - 70)])
    j1 = np.concatenate([rng.choice(a_i, 100), np.full(10, 2), more, rng.choice(a_i, B - 110 - len(more))])
    sh = rng.permutation(B)
    # 2. 17 triples on rows disjoint from batch 1; 3. one triple on a hub user; 4. empty; 5. one hub triple B times
    batches = [batch(u1[sh], i1[sh], j1[sh]), batch(c_u, c_i[:17], c_i[17:]), batch([2], [1], [a_i[0]]), batch([], [], []),
               batch(np.full(B, 1), np.full(B, 2), np.full(B, 1))]
    assert batches[0][0][1] < B and len(set(batches[0][1][0]) & set(c_u)) == 0 and batches[2][0][1] == batches[2][0][2] == 1
    poison_words = _words(*poison, poison[0], poison[1])  # b = cap: no tails

    # SGL's view graphs: edge dropout at rate 0.1, and node dropout at rate 0.1 that also removes user 1 and item 1 (in
    # the graphs here: split rows; their view rows are empty, while the batch-row lists still classify them as split rows)
    def edge_views():
        return [_norm_adj(data.pair_users[k], data.pair_items[k], U, I) for k in (rng.random(len(data.pair_users)) >= 0.1 for _ in range(2))]

    def node_views():
        out = []
        for _ in range(2):
            du = (rng.random(U) < 0.1) | (np.arange(U) == 1)
            di = (rng.random(I) < 0.1) | (np.arange(I) == 1)
            keep = ~du[data.pair_users] & ~di[data.pair_items]
            out.append(_norm_adj(data.pair_users[keep], data.pair_items[keep], U, I))
        assert np.diff(out[0].indptr)[1] == 0 and np.diff(out[0].indptr)[U + 1] == 0
        return out

    views = dict(edge=edge_views(), node=node_views())
    return dict(data=data, A=A, poison=poison_words, batches=batches, views=views)


@pytest.fixture(scope="module")
def hub():
    """U x I graph with explicit rows at every class boundary: users of degree 4096 / 4097 (split rows of 2 and 3
    chunks), 4095, 256 / 255, 128 / 127, 64 / 63 and items of degree 5000 / 4096."""
    import torch
    from selfrec_b200 import _lib, ops
    h = make_hub_graph(U, I, HUB_USERS, HUB_ITEMS, 20261016)
    A = h["A"]
    deg = np.diff(A.indptr)
    c = ops.classify_rows(torch.from_numpy(A.indptr.astype(np.int32)))
    order = c["row_order"].numpy()
    assert c["n_huge"] == 4 and set(order[:4]) == {1, 2, U + 1, U + 2}
    assert c["n_vlong"] == 2 and set(order[4:6]) == {3, 4}
    assert c["n_long"] == 4 and set(order[6:10]) == {5, 6, 7, 8}
    assert c["n_work"] == 2 + 3 + 3 + 2 and deg[order[10]] < ops.LONG_ROW_NNZ  # user 9 (63) is in the lane-group class
    assert _lib.HUB_MIN_NNZ == 4096 and _lib.HUB_CHUNK == 2048
    return h


def _has_nan(torch, buf):
    n = buf.numel() - buf.numel() % 4
    return bool(torch.isnan(buf[:n].view(torch.float32)).any())


def _poison(torch, eng, words, state, params, capture=False, workspaces=None):
    """One step with NaN parameters on `words`, then `state` put back: every float table the step writes is NaN wherever
    that step wrote it.  capture=True poisons through capture()'s warm-up steps instead of an eager step (capture()
    restores what it saved, the NaN parameters included).  `eng` needs step(words); workspaces: the buffers that must
    hold NaN afterwards (default: eng.workspace)."""
    saved = [t.clone() for t in state]
    for t in params:
        t.fill_(float("nan"))
    if capture:
        eng.batch_dev.copy_(torch.from_numpy(words))
        eng.capture()
    else:
        eng.step(words)
    torch.cuda.synchronize()
    for dst, src in zip(state, saved):
        dst.copy_(src)
    torch.cuda.synchronize()
    for k, ws in enumerate([eng.workspace] if workspaces is None else workspaces):
        assert _has_nan(torch, ws), f"the poison step left no NaN in workspace {k}"


def _unambiguous_noise(orc, A, E0, noise):
    """The perturbation sign(y) * normalize(noise) * eps (XSimGCL.py:90-91) jumps at y = 0, so a layer value within
    fp32 rounding of zero takes either sign between the kernel and the float64 oracle, and the two steps then differ by
    2 eps in that coordinate.  Zero the noise wherever the float64 layer value (before its perturbation) is within 1e-4
    of its rounding scale |A| |x|: the perturbation is then 0 there whatever the sign, and the same tensor feeds both."""
    A64 = A.astype(np.float64)
    absA = abs(A64)
    noise = noise.copy()
    for v in range(noise.shape[0]):
        x = E0.astype(np.float64)
        for k in range(noise.shape[1]):
            y = A64 @ x
            noise[v, k][np.abs(y) <= 1e-4 * (absA @ np.abs(x))] = 0
            x = orc.perturb(y, noise[v, k].astype(np.float64), EPS)
    return noise


def _run_sequence(torch, orc, hub, name, d, L, lcl, view_csr, run_step, read_state, noise_dev, tag, eps=EPS, kappa=KAPPA, reg=REG):
    """The batches after the poison step, each against the oracle, continuing from the device state every step.
    SimGCL / XSimGCL without noise_dev: the step's own noise at eps = 0, where the perturbation vanishes.  kappa: the
    first-moment bar (KAPPA); reg: the L2 weight the engine was built with (REG)."""
    KAPPA = kappa
    rng = np.random.default_rng(d * 100 + L * 10 + lcl)
    A = hub["A"]
    U, N = hub["data"].user_num, A.shape[0]
    views = 2 if name == "SimGCL" else 1
    assert noise_dev is not None or eps == 0.0 or name not in ("SimGCL", "XSimGCL")
    p, m, v, _ = read_state()
    for step, (words, (u, i, j)) in enumerate(hub["batches"], start=1):
        b = len(u)
        where = f"{tag} step {step} b={b}"
        noise = None
        if noise_dev is not None:
            noise = _unambiguous_noise(orc, A, p, rng.random((views, L, N, d), dtype=np.float32))
            noise_dev.copy_(torch.from_numpy(noise))
        elif name in ("SimGCL", "XSimGCL"):
            noise = np.zeros((views, L, 1, 1))  # (eps = 0: any noise adds nothing)
        run_step(words)
        torch.cuda.synchronize()
        gp, gm, gv, los = read_state()
        for nm, x in (("params", gp), ("m", gm), ("v", gv), ("losses", los)):
            bad = ~np.isfinite(x)
            assert not bad.any(), f"{where}: {nm} has {int(bad.sum())} non-finite entries, first rows " \
                                  f"{np.unique(np.nonzero(bad)[0])[:8].tolist()}, first values {x[bad][:4].tolist()}"
        if b == 0:
            g = np.zeros((N, d))
        else:
            ref = orc.train_step(name, A, p, U, u, i, j, n_layers=L, reg=reg, batch_size=B, eps=eps, tau=TAU, cl_rate=CL_RATE,
                                 layer_cl=lcl, noise=noise, view_csr=view_csr)
            g = ref["grad"]
            for k, key in ((0, "rec"), (1, "l2")):
                assert abs(los[k] - ref[key]) <= 1e-4 * abs(ref[key]) + 1e-7, (where, key, los[k], ref[key])
            # the InfoNCE floor (fp32 resolution of logits of size 1/tau) once per InfoNCE term: users and items
            # separately in SimGCL / XSimGCL, one over cat(users, items) in SGL
            n_nce = 1 if name == "SGL" else 2
            assert abs(los[2] - ref["cl"]) <= 1e-4 * abs(ref["cl"]) + n_nce * 2e-7 / TAU, (where, "cl", los[2], ref["cl"])
        p_ref, m_ref, v_ref = orc.adam_step(p, g.astype(np.float32), m, v, step, LR)
        # rows outside the batch's reach get exactly Adam's zero-gradient update (stale seeds must not leak into them)
        zero = ~(g != 0).any(1)
        assert np.array_equal(gv[zero], v[zero] * np.float32(0.999)), where
        m_err = np.abs(gm[zero] - m_ref[zero])
        assert (m_err <= np.spacing(np.abs(m_ref[zero]))).all(), (where, "zero-gradient m", float(m_err.max()))
        # the first moment is linear in the gradient: a check on the whole backward pass, row by row
        live = ~zero
        if live.any():
            row_err = np.abs(gm[live] - m_ref[live]).max(1)
            row_scale = np.abs(m_ref[live]).max(1)
            bound = KAPPA * row_scale + 1e-6 * np.abs(m_ref).max()
            worst = int(np.argmax(row_err - bound))
            row = int(np.nonzero(live)[0][worst])
            assert (row_err <= bound).all(), (where, "m", row, float(row_err[worst]), float(row_scale[worst]))
        # parameters: Adam divides by sqrt(v) + 1e-8, so entries whose gradient is ~1e-8 or below are ill-conditioned.  On
        # top of rtol 1e-4 / atol 2e-6, an entry may carry the first-moment error its row is allowed (above) divided by
        # its own denominator: a gradient error is relative to its row's scale, and an entry far below that scale (a
        # hub row's small coordinates) has it amplified by Adam's per-entry normalisation
        cond = np.abs(g) > 1e-6
        bc1, bc2 = 1 - 0.9 ** step, 1 - 0.999 ** step
        m_allow = KAPPA * np.abs(m_ref).max(1, keepdims=True) + 1e-6 * np.abs(m_ref).max()
        p_allow = 1e-4 * np.abs(p_ref) + 2e-6 + LR / bc1 * m_allow / (np.sqrt(v_ref) / np.sqrt(bc2) + 1e-8)
        p_err = np.abs(gp - p_ref)
        assert (p_err[cond] <= p_allow[cond]).all(), (where, "params", int((p_err > p_allow)[cond].sum()),
                                                      float((p_err - p_allow)[cond].max()))
        assert p_err.max() <= 2.5 * LR, where  # |update| <= lr / (1 - beta1) early on
        p, m, v = gp, gm, gv


CASES = [
    # name, d, L, layer_cl, SGL views, captured
    ("LightGCN", 32, 1, 0, None, False),
    ("LightGCN", 128, 3, 0, None, False),
    ("LightGCN", 64, 1, 0, None, True),
    ("XSimGCL", 64, 3, 0, None, False),
    ("XSimGCL", 32, 3, 1, None, False),
    ("XSimGCL", 128, 3, 3, None, False),
    ("XSimGCL", 64, 1, 1, None, False),
    ("XSimGCL", 128, 3, 1, None, True),
    ("SimGCL", 64, 1, 0, None, False),
    ("SimGCL", 128, 2, 0, None, False),
    ("SimGCL", 32, 3, 0, None, False),
    ("SimGCL", 32, 1, 0, None, True),
    ("SGL", 64, 1, 0, "edge", False),
    ("SGL", 32, 1, 0, "node", False),
    ("SGL", 128, 3, 0, "edge", False),
    ("SGL", 64, 3, 0, "node", False),
    ("SGL", 128, 1, 0, "node", True),
]


def _case_id(c):
    name, d, L, lcl, views, captured = c
    return f"{name}-d{d}-L{L}" + (f"-lcl{lcl}" if name == "XSimGCL" else "") + (f"-{views}" if views else "") + ("-captured" if captured else "")


@pytest.mark.parametrize("blocked", [False, True], ids=["chunked", "colblocked"])
@pytest.mark.parametrize("name,d,L,lcl,views,captured", CASES, ids=[_case_id(c) for c in CASES])
def test_step_from_poisoned_workspace_vs_oracle(torch_cuda, orc, hub, monkeypatch, name, d, L, lcl, views, captured, blocked):
    """TrainEngine: one poison step, then a full batch with hubs, 17 triples on other rows, one hub triple, an empty
    batch and one hub triple B times, eagerly or through one captured CUDA graph, with the split rows' chunk lists or
    their column-blocked lists."""
    torch = torch_cuda
    from selfrec_b200 import ops
    from selfrec_b200.engine import TrainEngine
    if blocked:
        monkeypatch.setattr(ops, "HUB_BLOCK_BYTES", 2048 * 4 * d)  # blocks of 4096 columns: three blocks at N = 11000
    data = hub["data"]
    rng = np.random.default_rng(d + L)
    E0 = (rng.standard_normal((U + I, d)) * 0.1).astype(np.float32)
    kw = dict(eps=EPS, tau=TAU, cl_rate=CL_RATE, layer_cl=lcl) if name in ("XSimGCL", "SimGCL") else {}
    if name == "LightGCN":
        kw["l2_div"] = float(B)
    if name == "SGL":
        kw = dict(tau=TAU, cl_rate=CL_RATE)
    eng = TrainEngine(name, data, d, L, B, LR, REG, init_user=torch.from_numpy(E0[:U]), init_item=torch.from_numpy(E0[U:]), **kw)
    assert bool(eng.adj.hub_struct(d).seg) == blocked
    view_csr = None
    if name == "SGL":
        view_csr = hub["views"][views]
        eng.set_view_graphs(*view_csr)
    noise_dev = None
    if name in ("XSimGCL", "SimGCL"):
        views_n = 2 if name == "SimGCL" else 1
        noise_dev = torch.from_numpy(rng.random((views_n, L, U + I, d), dtype=np.float32)).cuda()
        eng.set_noise_tensor(noise_dev)
    _poison(torch, eng, hub["poison"], (eng.params, eng.m, eng.v, eng.step_dev, eng.losses), (eng.params,), capture=captured)

    def run_step(words):
        if captured:
            eng.batch_dev.copy_(torch.from_numpy(words))
            eng.graph.replay()
        else:
            eng.step(words)

    def read_state():
        return tuple(t.cpu().numpy().copy() for t in (eng.params, eng.m, eng.v, eng.losses))

    _run_sequence(torch, orc, hub, name, d, L, lcl, view_csr, run_step, read_state, noise_dev, _case_id((name, d, L, lcl, views, captured)))


@pytest.mark.parametrize("name,d,L,views", [("LightGCN", 64, 1, None), ("LightGCN", 32, 3, None), ("SGL", 64, 1, "node"),
                                            ("SGL", 128, 3, "edge")])
def test_sharded_step_world1_from_poisoned_workspace_vs_oracle(torch_cuda, orc, hub, name, d, L, views):
    """The bipartite-sharded step at world 1 (its own seed slots, batch-row lists and launches of the SpMM) straight
    against the float64 oracle, through the same poison step and batch sequence."""
    torch = torch_cuda
    from selfrec_b200.sharded import ShardedEngine
    data = hub["data"]
    rng = np.random.default_rng(d + L + 1)
    E0 = (rng.standard_normal((U + I, d)) * 0.1).astype(np.float32)
    kw = dict(l2_div=float(B)) if name == "LightGCN" else dict(tau=TAU, cl_rate=CL_RATE)
    eng = ShardedEngine(name, data, d, L, B, LR, REG, init_user=torch.from_numpy(E0[:U]), init_item=torch.from_numpy(E0[U:]),
                        device=torch.device("cuda", torch.cuda.current_device()), **kw)
    assert eng.world == 1 and eng.Ug == U
    view_csr = None
    if name == "SGL":
        view_csr = hub["views"][views]
        eng.set_view_graphs(*view_csr)
    state = (eng.user_emb, eng.item_emb, eng.mu, eng.vu, eng.mi, eng.vi, eng.step_dev, eng.losses)
    _poison(torch, eng, hub["poison"], state, (eng.user_emb, eng.item_emb))

    def read_state():
        cat = lambda a, b: torch.cat([a, b]).cpu().numpy()
        return cat(eng.user_emb, eng.item_emb), cat(eng.mu, eng.mi), cat(eng.vu, eng.vi), eng.losses.cpu().numpy()

    _run_sequence(torch, orc, hub, name, d, L, 0, view_csr, lambda w: eng.step(words=w), read_state, None,
                  f"sharded {name}-d{d}-L{L}" + (f"-{views}" if views else ""))
