"""Bipartite-sharding host logic on CPU, incl. a real world-size-2 gloo process group: cyclic user assignment, per-rank
blocks Ru / Rt, and the layer exchange (partial item products summed over ranks) reproduce the unsharded product."""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bipartite(n_users, n_items, nnz, seed):
    rng = np.random.default_rng(seed)
    u = np.minimum((rng.pareto(1.2, nnz) * 3).astype(np.int64), n_users - 1)  # power-law: hubs at low ids
    i = rng.integers(0, n_items, nnz)
    R = sp.csr_matrix((np.ones(nnz, np.float32), (u, i)), shape=(n_users, n_items))
    R.data[:] = rng.random(R.nnz).astype(np.float32) + 0.1
    n = n_users + n_items
    A = sp.bmat([[None, R], [R.T, None]], format="csr", dtype=np.float32)
    A.sort_indices()
    assert A.shape == (n, n)
    return R.tocsr(), A


def test_cyclic_user_assignment():
    from selfrec_b200.sharded import item_bounds, local_user_count, user_ids_of
    for U in (1, 7, 64, 1001):
        for world in (1, 2, 3, 8):
            if U < world:
                continue
            ids = [user_ids_of(U, g, world) for g in range(world)]
            assert [len(x) for x in ids] == [local_user_count(U, g, world) for g in range(world)]
            allu = np.sort(np.concatenate(ids))
            assert np.array_equal(allu, np.arange(U))                      # every user exactly once
            for g, x in enumerate(ids):
                assert (x % world == g).all() and np.array_equal(x // world, np.arange(len(x)))  # local row = id // world
            ib = item_bounds(1001, world)
            assert ib[0] == 0 and ib[-1] == 1001 and (np.diff(ib) > 0).all() and np.diff(ib).max() <= -(-1001 // world)
    # hubs at the low ids (first-appearance ids of a power-law file): the cyclic split balances non-zeros AND rows
    rng = np.random.default_rng(0)
    deg = np.sort(rng.zipf(1.3, 100000) % 50000)[::-1]
    for world in (2, 4, 8):
        per = np.array([deg[g::world].sum() for g in range(world)], dtype=np.float64)
        assert per.max() / per.mean() < 1.25


def test_extract_blocks_tile_the_adjacency():
    import torch
    from selfrec_b200.sharded import extract_blocks, local_user_count
    U, I = 403, 150
    R, A = _bipartite(U, I, 6000, 1)
    rp, ci, vv = (torch.from_numpy(np.asarray(x)) for x in (A.indptr.astype(np.int32), A.indices.astype(np.int32), A.data))
    for world in (1, 2, 4):
        for g in range(world):
            (p1, c1, v1), (p2, c2, v2) = extract_blocks(rp, ci, vv, U, I, g, world)
            ug = local_user_count(U, g, world)
            ru = sp.csr_matrix((v1.numpy(), c1.numpy(), p1.numpy()), shape=(ug, I))
            rt = sp.csr_matrix((v2.numpy(), c2.numpy(), p2.numpy()), shape=(I, ug))
            assert ru.has_sorted_indices and rt.has_sorted_indices
            assert abs(ru - R[g::world]).max() == 0            # rows g, g + world, ... of R
            assert abs(rt - R.T.tocsr()[:, g::world]).max() == 0  # the matching columns of R^T, renumbered id // world


def _worker(rank, world, port, ret):
    import torch
    import torch.distributed as dist
    sys.path.insert(0, ROOT)
    from selfrec_b200.sharded import extract_blocks, item_bounds, local_user_count
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    U, I, d = 400, 150, 32
    R, A = _bipartite(U, I, 6000, 2)
    rng = np.random.default_rng(5)
    X = rng.standard_normal((U + I, d)).astype(np.float32)
    rp, ci, vv = (torch.from_numpy(np.asarray(x)) for x in (A.indptr.astype(np.int32), A.indices.astype(np.int32), A.data))
    ug = local_user_count(U, rank, world)
    (p1, c1, v1), (p2, c2, v2) = extract_blocks(rp, ci, vv, U, I, rank, world)
    Ru = sp.csr_matrix((v1.numpy(), c1.numpy(), p1.numpy()), shape=(ug, I))
    Rt = sp.csr_matrix((v2.numpy(), c2.numpy(), p2.numpy()), shape=(I, ug))
    ib = item_bounds(I, world)
    xu, xi = X[:U][rank::world], X[U:]   # this rank's users: rank, rank + world, ...
    for _ in range(2):  # two propagation layers
        part = torch.from_numpy((Rt @ xu).astype(np.float32))  # this rank's partial item product
        yu = (Ru @ xi).astype(np.float32)                      # local user half
        # reduce-scatter to the slice owners, then all-gather of the finished slices (the CPU stand-in for the
        # P2P partial pushes + owner-side reduction + multicast stores of sharded.cu)
        parts = [torch.empty_like(part) for _ in range(world)]
        dist.all_gather(parts, part)
        mine = sum(p[ib[rank]:ib[rank + 1]] for p in parts)   # fixed rank order
        sizes = [int(ib[g + 1] - ib[g]) for g in range(world)]
        pad = torch.zeros((max(sizes), d))
        pad[: sizes[rank]] = mine
        outs = [torch.empty_like(pad) for _ in range(world)]
        dist.all_gather(outs, pad)
        xi = torch.cat([o[:n] for o, n in zip(outs, sizes)]).numpy()
        xu = yu
    ref = A @ (A @ X)
    ok = np.allclose(xu, ref[:U][rank::world], rtol=1e-5, atol=1e-5) and np.allclose(xi, ref[U:], rtol=1e-5, atol=1e-5)
    out = torch.tensor([1.0 if ok else 0.0])
    dist.all_reduce(out, op=dist.ReduceOp.MIN)
    if rank == 0:
        ret.put(float(out.item()))
    dist.destroy_process_group()


def test_bipartite_sharded_propagation_world2_gloo():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, ret)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    assert ret.get(timeout=5) == 1.0


def test_sharded_simgcl_step_algebra_model():
    """float64 model of what csrc/sharded.cu computes for one SimGCL step on G ranks -- cyclic users, replicated items,
    item rows as rank-ordered sums of partial products, ONE shared first product + per-view noise (SimGCL.py:85-88), the
    last forward layer evaluated on the batch rows only, one merged backward chain on a seed table that holds the loss
    gradients at the batch rows (the first product masked by them, the seed added after every later product) -- against the oracle's plain restatement of SimGCL.py:25-36 (three full encoders, three backward chains).
    Losses and the E0 gradient must agree to float64 rounding: the rewrites are algebra, not approximations."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import oracle
    from selfrec_b200.sharded import extract_blocks, local_user_count
    import torch
    U, I, d, L, G, B = 90, 40, 8, 3, 4, 24
    R, A = _bipartite(U, I, 700, 11)
    A = oracle.normalize_graph_mat(A)  # symmetric normalisation, like the real adjacency
    # (the reference's fp32 products (d_r * a) * d_c round the two triangles differently by an ulp; the CUDA backward
    # reuses A for A^T, which the 1e-4 parity budget absorbs -- here the matrix is made exactly symmetric so that the
    # model can be held to float64 rounding)
    A = ((A.astype(np.float64) + A.astype(np.float64).T) * 0.5).astype(np.float32).tocsr()
    A.sort_indices()
    rng = np.random.default_rng(3)
    E0 = rng.standard_normal((U + I, d)) * 0.1
    noise = rng.random((2, L, U + I, d))
    eps, tau, lam, reg = 0.1, 0.2, 0.5, 1e-4
    u_idx, i_idx, j_idx = rng.integers(0, U, B), rng.integers(0, I, B), rng.integers(0, I, B)
    rp, ci, vv = (torch.from_numpy(np.asarray(x)) for x in (A.indptr.astype(np.int32), A.indices.astype(np.int32), A.data.astype(np.float32)))
    blocks = []
    for g in range(G):
        (p1, c1, v1), (p2, c2, v2) = extract_blocks(rp, ci, vv, U, I, g, G)
        ug = local_user_count(U, g, G)
        blocks.append((sp.csr_matrix((v1.numpy().astype(np.float64), c1.numpy(), p1.numpy()), shape=(ug, I)),
                       sp.csr_matrix((v2.numpy().astype(np.float64), c2.numpy(), p2.numpy()), shape=(I, ug))))
    A64 = sp.csr_matrix((A.data.astype(np.float32).astype(np.float64), A.indices, A.indptr), shape=A.shape)  # the fp32 values the blocks hold
    ref = oracle.train_step("SimGCL", A64, E0, U, u_idx, i_idx, j_idx, n_layers=L, reg=reg, batch_size=B, eps=eps, tau=tau, cl_rate=lam,
                            noise=noise)

    def layer(xu, xi):
        """xu: list of per-rank user blocks, xi: replicated item table -> (yu list, yi)."""
        yi = sum(blocks[g][1] @ xu[g] for g in range(G))  # partial products added in rank order by the slice owners
        return [blocks[g][0] @ xi for g in range(G)], yi

    split = lambda X: ([X[:U][g::G] for g in range(G)], X[U:])

    def join(xu, xi):
        X = np.empty((U + I, xi.shape[1]))
        for g in range(G):
            X[:U][g::G] = xu[g]
        X[U:] = xi
        return X

    # ---- forward: one shared first product, noise per view, last layer on the batch rows only ----
    z = join(*layer(*split(E0)))
    rows = np.unique(np.concatenate([u_idx, U + i_idx, U + j_idx]))
    finals = []
    for view in (None, 0, 1):
        x = z if view is None else oracle.perturb(z, noise[view][0], eps)
        acc = x.copy()
        for k in range(1, L):
            y = join(*layer(*split(x)))
            if k == L - 1:  # only the batch rows of the final mean are read
                keep = np.zeros(U + I, bool)
                keep[rows] = True
                y[~keep] = np.nan
            if view is not None:
                y = oracle.perturb(y, noise[view][k], eps)
            acc = acc + y
            x = y
        finals.append(acc / L)
    final, v1, v2 = finals
    ue, pe, ne = final[u_idx], final[U + i_idx], final[U + j_idx]
    rec, du, dp, dn = oracle.bpr_loss(ue, pe, ne)
    l2, gl = oracle.l2_reg_loss(reg, ue, pe)
    uu, ui = np.unique(u_idx), np.unique(i_idx)
    lu, d1u, d2u = oracle.infonce(v1[uu], v2[uu], tau)
    li, d1i, d2i = oracle.infonce(v1[U + ui], v2[U + ui], tau)
    assert abs(rec - ref["rec"]) < 1e-12 and abs(l2 - ref["l2"]) < 1e-12 and abs(lam * (lu + li) - ref["cl"]) < 1e-10
    # ---- backward: the three chains are the same linear map -> one merged Horner chain, seed = batch rows only ----
    seed = np.zeros((U + I, d))
    for idx, gg in ((u_idx, du + gl[0]), (U + i_idx, dp + gl[1]), (U + j_idx, dn), (uu, lam * (d1u + d2u)), (U + ui, lam * (d1i + d2i))):
        np.add.at(seed, idx, gg / L)
    acc = seed.copy()
    for k in range(L - 1, 0, -1):
        if k == L - 1:
            assert not np.any(acc[np.setdiff1d(np.arange(U + I), rows)])  # the masked first product skips exactly zeros
        acc = join(*layer(*split(acc))) + seed
    grad = join(*layer(*split(acc)))
    np.testing.assert_allclose(grad, ref["grad"], rtol=1e-9, atol=1e-13)
