"""Tensor-core scoring (impl 2: wgmma TF32 candidates + exact fp32 re-scoring) must return
exactly what the CUDA-core kernel (impl 1, bit-identical to the oracle) returns."""
import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu


def _run_both(ue, ie, users, rated, k=20):
    import torch
    from selfrec_b200 import ops
    tu, ti = torch.from_numpy(ue).cuda(), torch.from_numpy(ie).cuda()
    rp = rated.indptr if rated is not None else None
    ri = rated.indices if rated is not None else None
    i1, s1 = ops.score_topk(tu, ti, users, rp, ri, k, impl=1)
    i2, s2 = ops.score_topk(tu, ti, users, rp, ri, k, impl=2)
    torch.cuda.synchronize()
    return i1.cpu().numpy(), s1.cpu().numpy(), i2.cpu().numpy(), s2.cpu().numpy()


@pytest.mark.parametrize("n_users,n_items,n_q,k", [(900, 5000, 700, 20), (300, 1500, 300, 10), (64, 130, 40, 5), (2000, 20000, 1999, 32)])
def test_tc_matches_exact_kernel(built_lib, n_users, n_items, n_q, k):
    rng = np.random.default_rng(n_items)
    ue = (rng.standard_normal((n_users, 64)) * 0.1).astype(np.float32)
    ie = (rng.standard_normal((n_items, 64)) * 0.1).astype(np.float32)
    users = rng.choice(n_users, n_q, replace=False).astype(np.int32)
    rated = sp.random(n_users, n_items, density=0.02, random_state=3, format="csr")
    rated.sort_indices()
    i1, s1, i2, s2 = _run_both(ue, ie, users, rated, k)
    assert np.array_equal(i1, i2)
    assert np.array_equal(s1, s2)


def test_tc_handles_ties_and_saturated_users(built_lib):
    """Integer-valued embeddings (exact ties everywhere) and users with almost everything rated:
    the certificate fails and the exact fallback must take over, result still identical."""
    rng = np.random.default_rng(1)
    n_users, n_items = 200, 3000
    ue = rng.integers(-2, 3, (n_users, 64)).astype(np.float32)
    ie = rng.integers(-2, 3, (n_items, 64)).astype(np.float32)
    rows, cols = [], []
    for u in range(n_users):
        deg = n_items - 7 if u % 50 == 0 else int(rng.integers(0, 60))  # a few users with < k unrated items
        c = rng.choice(n_items, deg, replace=False)
        rows += [u] * deg
        cols += c.tolist()
    rated = sp.csr_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(n_users, n_items))
    rated.sort_indices()
    users = np.arange(n_users, dtype=np.int32)
    i1, s1, i2, s2 = _run_both(ue, ie, users, rated, 20)
    assert np.array_equal(s1, s2)
    assert np.array_equal(i1, i2)


def test_tc_full_catalog_yelp_shape(built_lib):
    from selfrec_b200 import synth
    data = synth.make_interaction("yelp2018", seed=0)
    rng = np.random.default_rng(7)
    # embeddings with popularity structure: item norm grows with degree, like a trained model
    deg_i = np.bincount(data.pair_items, minlength=data.item_num).astype(np.float32)
    ue = (rng.standard_normal((data.user_num, 64)) * 0.1).astype(np.float32)
    ie = (rng.standard_normal((data.item_num, 64)) * 0.1 * (1 + np.log1p(deg_i)[:, None] / 4)).astype(np.float32)
    rated = sp.csr_matrix(data.interaction_mat)
    rated.sort_indices()
    users = np.arange(data.user_num, dtype=np.int32)
    i1, s1, i2, s2 = _run_both(ue, ie, users, rated, 20)
    bad = np.nonzero((i1 != i2).any(1) | (s1 != s2).any(1))[0]
    assert len(bad) == 0, (len(bad), bad[:10])
