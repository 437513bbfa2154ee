"""SGL on the bipartite-sharded step, host side: a float64 model of what csrc/sharded.cu computes for one SGL step on
G ranks (against the oracle's plain restatement of SGL.py:30-41), block extraction of node-dropout views, and the
workspace plan of the other three models staying what it was."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sym_normalized(R):
    """The normalised (U+I)^2 adjacency of a users x items matrix, made exactly symmetric (see
    test_sharded_simgcl_step_algebra_model: the model is held to float64 rounding)."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import oracle
    R = sp.csr_matrix(R)
    R.eliminate_zeros()
    A = oracle.normalize_graph_mat(sp.bmat([[None, R], [R.T, None]], format="csr", dtype=np.float32))
    A = ((A.astype(np.float64) + A.astype(np.float64).T) * 0.5).astype(np.float32).tocsr()
    A.eliminate_zeros()
    A.sort_indices()
    return A


def _interactions(U, I, nnz, seed):
    rng = np.random.default_rng(seed)
    u = np.minimum((rng.pareto(1.2, nnz) * 3).astype(np.int64), U - 1)  # power-law: hubs at low ids
    i = rng.integers(0, I, nnz)
    R = sp.csr_matrix((np.ones(nnz, np.float32), (u, i)), shape=(U, I))
    R.data[:] = 1.0  # duplicates summed, then unit weights (SGL's views are rebuilt from the unit interaction matrix)
    return R


def _edge_dropout(R, rate, rng):
    V = R.copy().tocoo()
    keep = rng.random(V.nnz) >= rate
    return sp.csr_matrix((V.data[keep], (V.row[keep], V.col[keep])), shape=R.shape)


def _node_dropout(R, rate, rng):
    du = (rng.random(R.shape[0]) < rate).astype(np.float32)
    di = (rng.random(R.shape[1]) < rate).astype(np.float32)
    V = sp.diags(1 - du) @ R @ sp.diags(1 - di)
    return sp.csr_matrix(V)


def _torch_csr(A):
    import torch
    return (torch.from_numpy(A.indptr.astype(np.int32)), torch.from_numpy(A.indices.astype(np.int32)),
            torch.from_numpy(A.data.astype(np.float32)))


@pytest.mark.parametrize("G", [1, 2, 3, 4])
def test_sharded_sgl_step_algebra_model(G):
    """float64 model of one sharded SGL step: cyclic users, replicated items whose rows are rank-ordered sums of partial
    products finished by the slice owner, three encoders with the ego layer (graph, view 1, view 2) whose last layer only
    produces the batch rows, one InfoNCE over cat(unique users, unique items) whose gradient rows are routed user-to-owner
    and item-to-every-rank, three backward chains on seed tables (first product masked by the batch rows), and gd -- the
    sum of the two view chains -- kept locally (users, and items on the owner's slice only) and added at the final level of
    the next chain.  Losses and the E0 gradient must agree with the oracle to float64 rounding."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import oracle
    from selfrec_b200.sharded import extract_blocks, item_bounds, local_user_count
    U, I, d, L, B = 90, 40, 8, 3, 24
    rng = np.random.default_rng(11)
    R = _interactions(U, I, 700, 11)
    graphs = [_sym_normalized(R), _sym_normalized(_edge_dropout(R, 0.1, rng)), _sym_normalized(_node_dropout(R, 0.1, rng))]
    E0 = rng.standard_normal((U + I, d)) * 0.1
    tau, lam, reg = 0.2, 0.5, 1e-4
    u_idx, i_idx, j_idx = rng.integers(0, U, B), rng.integers(0, I, B), rng.integers(0, I, B)
    f64 = lambda A: sp.csr_matrix((A.data.astype(np.float32).astype(np.float64), A.indices, A.indptr), shape=A.shape)
    ref = oracle.train_step("SGL", f64(graphs[0]), E0, U, u_idx, i_idx, j_idx, n_layers=L, reg=reg, batch_size=B, tau=tau, cl_rate=lam,
                            view_csr=(f64(graphs[1]), f64(graphs[2])))
    ug = [local_user_count(U, g, G) for g in range(G)]
    blocks = []  # blocks[q][g] = (Ru, Rt) of graph q on rank g
    for A in graphs:
        per = []
        for g in range(G):
            (p1, c1, v1), (p2, c2, v2) = extract_blocks(*_torch_csr(A), U, I, g, G)
            per.append((sp.csr_matrix((v1.numpy().astype(np.float64), c1.numpy(), p1.numpy()), shape=(ug[g], I)),
                        sp.csr_matrix((v2.numpy().astype(np.float64), c2.numpy(), p2.numpy()), shape=(I, ug[g]))))
        blocks.append(per)
    ib = item_bounds(I, G)
    split = lambda X: ([X[:U][g::G] for g in range(G)], X[U:])

    def join(xu, xi):
        X = np.empty((U + I, d))
        for g in range(G):
            X[:U][g::G] = xu[g]
        X[U:] = xi
        return X

    def layer(q, xu, xi, seed=None, gd=None):
        """One layer on graph q: the user half per rank, the item half per owner slice (partials in rank order, then the
        owner's own seed replica and its local gd rows).  Returns (user blocks, item slices by owner)."""
        yu = [blocks[q][g][0] @ xi for g in range(G)]
        part = [blocks[q][g][1] @ xu[g] for g in range(G)]
        yi = []
        for o in range(G):
            sl = slice(ib[o], ib[o + 1])
            acc = np.zeros((ib[o + 1] - ib[o], d))
            for g in range(G):
                acc = acc + part[g][sl]
            if seed is not None:
                acc = acc + seed[1][o][sl]
            if gd is not None:
                acc = acc + gd[1][o][sl]
            yi.append(acc)
        for g in range(G):
            if seed is not None:
                yu[g] = yu[g] + seed[0][g]
            if gd is not None:
                yu[g] = yu[g] + gd[0][g]
        return yu, yi

    # ---- forward: three encoders, ego layer in the mean, last layer on the batch rows only ----
    rows = np.unique(np.concatenate([u_idx, U + i_idx, U + j_idx]))
    keep = np.zeros(U + I, bool)
    keep[rows] = True
    finals = []
    for q in range(3):
        xu, xi = split(E0)
        acc = E0.copy()
        for k in range(1, L + 1):
            yu, yi = layer(q, xu, xi)
            xu, xi = yu, np.concatenate(yi)
            y = join(xu, xi)
            if k == L:
                y[~keep] = np.nan
            acc = acc + y
        finals.append(acc / (L + 1))
    final, v1, v2 = finals
    ue, pe, ne = final[u_idx], final[U + i_idx], final[U + j_idx]
    rec, du, dp, dn = oracle.bpr_loss(ue, pe, ne)
    l2, gl = oracle.l2_reg_loss(reg, ue, pe, ne)  # SGL.py:36: (u, p, n)
    uu, ui = np.unique(u_idx), np.unique(i_idx)
    cat = np.concatenate([uu, U + ui])  # the unique users, then the unique items
    lc, d1, d2 = oracle.infonce(v1[cat], v2[cat], tau)
    assert abs(rec - ref["rec"]) < 1e-12 and abs(l2 - ref["l2"]) < 1e-12 and abs(lam * lc - ref["cl"]) < 1e-10
    # ---- seed tables: slot 0 = view 1, 1 = view 2, 2 = the graph; users on their owner, items on every rank ----
    cm = 1.0 / (L + 1)
    seeds = [([np.zeros((ug[g], d)) for g in range(G)], [np.zeros((I, d)) for g in range(G)]) for _ in range(3)]

    def route(t, ids, grads):
        for r, gr in zip(ids, grads):
            for g in range(G):
                if r >= U:  # item rows (cat's item_min = U): every rank's complete item table
                    seeds[t][1][g][r - U] += cm * gr
                elif r % G == g:
                    seeds[t][0][g][r // G] += cm * gr

    route(0, cat, lam * d1)
    route(1, cat, lam * d2)
    for ids, gg in ((u_idx, du + gl[0]), (U + i_idx, dp + gl[1]), (U + j_idx, dn + gl[2])):
        route(2, ids, gg)
    for su, si in seeds:
        assert all(np.array_equal(si[0], x) for x in si)  # the item replicas agree
        assert not np.any(join(su, si[0])[~keep])  # nothing outside the batch rows: the masked first product skips zeros

    def chain(q, t, gd=None, to_gd=False):
        xu, xi = seeds[t][0], seeds[t][1][0]
        for _k in range(L - 1, 0, -1):
            yu, yi = layer(q, xu, xi, seeds[t])
            xu, xi = yu, np.concatenate(yi)
        yu, yi = layer(q, xu, xi, seeds[t], gd)  # ego level: F again, and gd
        if not to_gd:
            return join(yu, np.concatenate(yi))
        gi = []  # gd's item rows stay on their owner: nothing else is valid (a read elsewhere would spread NaN)
        for o in range(G):
            a = np.full((I, d), np.nan)
            a[ib[o]:ib[o + 1]] = yi[o]
            gi.append(a)
        return yu, gi

    gd = chain(1, 0, to_gd=True)
    gd = chain(2, 1, gd=gd, to_gd=True)
    grad = chain(0, 2, gd=gd)
    np.testing.assert_allclose(grad, ref["grad"], rtol=1e-9, atol=1e-13)


def test_extract_blocks_tile_node_dropout_views():
    """A node-dropout view has empty rows (the dropped users and items): the blocks must still tile it."""
    from selfrec_b200.sharded import extract_blocks, local_user_count
    U, I = 403, 150
    rng = np.random.default_rng(4)
    Rv = _node_dropout(_interactions(U, I, 6000, 1), 0.3, rng)
    A = _sym_normalized(Rv)
    Rn = sp.csr_matrix(A[:U, U:])
    assert (np.diff(Rn.indptr) == 0).sum() > 50 and (np.diff(Rn.T.tocsr().indptr) == 0).sum() > 20
    for world in (1, 2, 3, 4):
        for g in range(world):
            (p1, c1, v1), (p2, c2, v2) = extract_blocks(*_torch_csr(A), U, I, g, world)
            n = local_user_count(U, g, world)
            ru = sp.csr_matrix((v1.numpy(), c1.numpy(), p1.numpy()), shape=(n, I))
            rt = sp.csr_matrix((v2.numpy(), c2.numpy(), p2.numpy()), shape=(I, n))
            assert ru.has_sorted_indices and rt.has_sorted_indices
            assert abs(ru - Rn[g::world]).max() == 0
            assert abs(rt - Rn.T.tocsr()[:, g::world]).max() == 0


# srb_shard_plan of LightGCN, SimGCL and XSimGCL before SGL joined the sharded step: (n_users, n_items, n_local_users, d,
# batch_cap, world, hub_chunks_u, hub_chunks_t) -> (sym_bytes, workspace_bytes, item_params, item_final, ctrl)
PLANS = {(1000, 400, 1000, 64, 512, 1, 0, 0): (3338496, 7710976, 256, 102656, 0),
         (3000, 4000, 1500, 64, 512, 2, 0, 0): (10813696, 11628032, 256, 1024256, 0),
         (30000, 8000, 7500, 128, 512, 4, 37, 91): (38011136, 56931328, 256, 4096256, 0),
         (138333, 98572, 17292, 64, 2048, 8, 5, 3): (212362496, 135951104, 256, 25234688, 0),
         (7, 5, 3, 32, 16, 3, 0, 1): (47360, 510208, 256, 1024, 0)}


def test_shard_plan_unchanged_for_the_other_models(built_lib):
    import ctypes as C
    from selfrec_b200 import _lib
    lib = _lib.load()
    for args, want in PLANS.items():
        for model in ("LightGCN", "SimGCL", "XSimGCL"):
            lay = _lib.ShardLayout()
            _lib.check(lib.srb_shard_plan(_lib.MODEL_IDS[model], *args, C.byref(lay)), "srb_shard_plan")
            assert (lay.sym_bytes, lay.workspace_bytes, lay.item_params, lay.item_final, lay.ctrl) == want, (model, args)
        lay = _lib.ShardLayout()
        _lib.check(lib.srb_shard_plan(_lib.MODEL_IDS["SGL"], *args, C.byref(lay)), "srb_shard_plan")
        assert (lay.sym_bytes, lay.item_params, lay.item_final, lay.ctrl) == (want[0],) + want[2:]  # same symmetric region
    assert lib.srb_shard_plan(_lib.MODEL_IDS["MF"], *next(iter(PLANS)), C.byref(_lib.ShardLayout())) != 0
