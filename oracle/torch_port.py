"""torch_port.py -- the reference's CPU PyTorch path for the hot path, restated op for op.

TEST INFRASTRUCTURE / BASELINE ONLY (same rule as oracle.py): used by bench.py's cpu_baseline
and `--impl reference` legs and by tests; never by the product.

The reference cannot ship with this repository (and is not pip-installable: no setup.py), so the
"reference arm" is this port: the same torch ops the reference calls, in the same order, on
the host cores (torch.set_num_threads(os.cpu_count())), driven by the same Python sampler
algorithm.  tests/test_oracle_golden.py pins it against the reference-generated fixtures.
"""
import random

import numpy as np
import torch
import torch.nn.functional as F


def coo_adj(csr):
    """TorchGraphInterface.convert_sparse_mat_to_tensor  base/torch_interface.py:8-13"""
    coo = csr.tocoo()
    i = torch.from_numpy(np.vstack([coo.row, coo.col]).astype(np.int64))
    v = torch.from_numpy(coo.data.astype(np.float32))
    return torch.sparse_coo_tensor(i, v, coo.shape, check_invariants=False)


def bpr_loss(u, p, n):  # util/loss_torch.py:6-10
    return torch.mean(-torch.log(10e-6 + torch.sigmoid((u * p).sum(1) - (u * n).sum(1))))


def l2_reg_loss(reg, *embs):  # util/loss_torch.py:18-22
    return sum(torch.norm(e, p=2) / e.shape[0] for e in embs) * reg


def info_nce(v1, v2, t):  # util/loss_torch.py:35-50
    v1, v2 = F.normalize(v1, dim=1), F.normalize(v2, dim=1)
    s = (v1 @ v2.T) / t
    return -torch.diag(F.log_softmax(s, dim=1)).mean()


def xsimgcl_forward(A, ue, ie, L, eps, layer_cl, perturbed, noise=None):
    """XSimGCL_Encoder.forward  XSimGCL.py:83-101"""
    ego = torch.cat([ue, ie], 0)
    outs, cl = [], ego
    for k in range(L):
        ego = torch.sparse.mm(A, ego)
        if perturbed:
            nz = torch.rand_like(ego) if noise is None else noise[k]
            ego = ego + torch.sign(ego) * F.normalize(nz, dim=-1) * eps
        outs.append(ego)
        if k == layer_cl - 1:
            cl = ego
    final = torch.mean(torch.stack(outs, dim=1), dim=1)
    U = ue.shape[0]
    return final[:U], final[U:], cl[:U], cl[U:]


def sample_batch(pair_users, pair_items, ptr, batch_size, n_items, rated_sets):
    """next_batch_pairwise body  util/sampler.py:10-27 over id arrays (Python `random`)."""
    end = ptr + batch_size if ptr + batch_size < len(pair_users) else len(pair_users)
    u = pair_users[ptr:end].tolist()
    i = pair_items[ptr:end].tolist()
    j = []
    for user in u:
        neg = random.randrange(n_items)
        while neg in rated_sets[user]:
            neg = random.randrange(n_items)
        j.append(neg)
    return u, i, j, end


class XSimGCLCpu:
    """XSimGCL.train() batch body (XSimGCL.py:27-37) on CPU torch."""

    def __init__(self, norm_csr, n_users, n_items, d, L, eps, tau, lam, layer_cl, lr, reg, init_user=None, init_item=None):
        self.A = coo_adj(norm_csr)
        self.U, self.I, self.L = n_users, n_items, L
        self.eps, self.tau, self.lam, self.layer_cl, self.reg = eps, tau, lam, layer_cl, reg
        iu = torch.nn.init.xavier_uniform_(torch.empty(n_users, d)) if init_user is None else torch.as_tensor(init_user)
        ii = torch.nn.init.xavier_uniform_(torch.empty(n_items, d)) if init_item is None else torch.as_tensor(init_item)
        self.ue, self.ie = torch.nn.Parameter(iu.clone()), torch.nn.Parameter(ii.clone())
        self.opt = torch.optim.Adam([self.ue, self.ie], lr=lr)

    def step(self, u, i, j, noise=None):
        ru, ri, cu, ci = xsimgcl_forward(self.A, self.ue, self.ie, self.L, self.eps, self.layer_cl, True, noise)
        ue, pe, ne = ru[u], ri[i], ri[j]
        rec = bpr_loss(ue, pe, ne)
        uu = torch.unique(torch.Tensor(u).type(torch.long))
        ui = torch.unique(torch.Tensor(i).type(torch.long))
        cl = self.lam * (info_nce(ru[uu], cu[uu], self.tau) + info_nce(ri[ui], ci[ui], self.tau))
        l2 = l2_reg_loss(self.reg, ue, pe)
        loss = rec + l2 + cl
        self.opt.zero_grad()
        loss.backward()
        self.opt.step()
        return float(rec.detach()), float(l2.detach()), float(cl.detach())


def rank_users(user_emb, item_emb, users, rated_ptr, rated_idx, K, find_k_largest):
    """GraphRecommender.test() loop body  base/graph_recommender.py:46-51 on CPU torch + the
    oracle's find_k_largest (the reference uses a numba heap, util/algorithm.py:144-156)."""
    ue, ie = torch.as_tensor(user_emb), torch.as_tensor(item_emb)
    out = []
    for u in users:
        cand = torch.matmul(ue[u], ie.transpose(0, 1)).numpy().copy()
        cand[rated_idx[rated_ptr[u]:rated_ptr[u + 1]]] = -10e8
        out.append(find_k_largest(K, cand))
    return out
