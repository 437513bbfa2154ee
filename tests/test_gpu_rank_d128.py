"""Full-catalog top-k at embedding size 128 on the tensor cores (impl 2: wgmma TF32 candidates, exact fp32
re-scoring, a per-user exactness certificate and the exact fallback) against the CUDA-core kernel (impl 1) and
the float64 oracle (oracle.score_topk).

impl 2 must return what impl 1 returns, bit for bit: the same ids in the same order (ties by id descending) and the
same fp32 scores.  Against the oracle, scores are compared bit for bit and ids as sets among equal scores (the
reference orders exact ties by an unstable sort)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

D = 128


@pytest.fixture(scope="module")
def torch_cuda(built_lib):
    import torch
    assert torch.cuda.is_available()
    from selfrec_b200 import _lib
    _lib.require_device()
    return torch


def _csr_rows(lists):
    ptr = np.zeros(len(lists) + 1, np.int32)
    ptr[1:] = np.cumsum([len(x) for x in lists])
    idx = np.concatenate([np.sort(np.asarray(x, np.int64)) for x in lists] + [np.zeros(0, np.int64)]).astype(np.int32)
    return ptr, idx


def _topk(torch, ue, ie, users, rp, ri, k, impl):
    """(ids, scores, fallback count or None) of ops.score_topk."""
    from selfrec_b200 import ops
    stats = {}
    ids, sc = ops.score_topk(torch.from_numpy(ue).cuda(), torch.from_numpy(ie).cuda(), users, rp, ri, k, impl=impl, stats=stats)
    torch.cuda.synchronize()
    fb = int(stats["fallback_count"].item()) if "fallback_count" in stats else None
    return ids.cpu().numpy(), sc.cpu().numpy(), fb


def _check(torch, orc, ue, ie, users, rp, ri, k, oracle_rows=None):
    """impl 2 == impl 1 bit for bit, both against the oracle (on oracle_rows, default all); returns the fallback count."""
    i2, s2, fb = _topk(torch, ue, ie, users, rp, ri, k, impl=2)
    i1, s1, fb1 = _topk(torch, ue, ie, users, rp, ri, k, impl=1)
    assert fb is not None and fb1 is None
    assert np.array_equal(i2, i1), np.nonzero((i2 != i1).any(1))[0][:8]
    assert np.array_equal(s2.view(np.uint32), s1.view(np.uint32))
    rows = np.arange(len(users)) if oracle_rows is None else oracle_rows
    oi, os_ = orc.score_topk(ue, ie, users[rows], rp, ri, k)
    assert np.array_equal(s2[rows].view(np.uint32), os_.view(np.uint32))
    for r, q in enumerate(rows):
        if not np.array_equal(i2[q], oi[r]):
            assert sorted(zip(s2[q].tolist(), i2[q].tolist())) == sorted(zip(os_[r].tolist(), oi[r].tolist())), q
    return fb


def _gauss(rng, n, scale=0.1):
    return (rng.standard_normal((n, D)) * scale).astype(np.float32)


@pytest.mark.parametrize("k", [1, 20, 32])
@pytest.mark.parametrize("n_q", [1, 127, 128, 129])
@pytest.mark.parametrize("n_items", [1024, 1025, 38048])
def test_rank_d128_shapes(torch_cuda, orc, n_items, n_q, k):
    rng = np.random.default_rng(n_items * 1000 + n_q * 10 + k)
    n_users = 400
    ue, ie = _gauss(rng, n_users), _gauss(rng, n_items)
    rated = [rng.choice(n_items, int(rng.integers(0, 60)), replace=False) for _ in range(n_users)]
    rated[0] = np.arange(n_items - max(k - 1, 0))               # fewer than k unrated items: k - 1
    rated[1] = rng.permutation(n_items)[k:]                      # exactly k unrated items
    rated[2] = np.concatenate([[0, n_items - 1], np.arange(128, 256)])  # first, last item and a whole tile
    rp, ri = _csr_rows(rated)
    users = np.concatenate([[0, 1, 2], rng.choice(np.arange(3, n_users), n_q, replace=False)])[:n_q].astype(np.int32)
    _check(torch_cuda, orc, ue, ie, users, rp, ri, k)


def test_rank_d128_many_ctas(torch_cuda, orc):
    """More users than one wave of 132 CTAs x 128 holds, at the yelp2018 item count: several waves of full CTAs."""
    rng = np.random.default_rng(5)
    n_users, n_items = 132 * 128 + 1000, 38048
    ue, ie = _gauss(rng, n_users), _gauss(rng, n_items)
    rated = [rng.choice(n_items, int(rng.integers(0, 40)), replace=False) for _ in range(n_users)]
    rp, ri = _csr_rows(rated)
    users = rng.permutation(n_users).astype(np.int32)
    fb = _check(torch_cuda, orc, ue, ie, users, rp, ri, 20, oracle_rows=np.r_[0:64, 16890:16960, n_users - 64:n_users])
    assert fb <= 0.05 * n_users, fb  # well-separated scores: the certificate passes for almost everyone


@pytest.mark.parametrize("k", [1, 20, 32])
def test_rank_d128_integer_ties(torch_cuda, orc, k):
    """Small-integer embeddings: many exactly equal scores, so the tie order (id descending) and the strict
    selection rule decide the lists."""
    rng = np.random.default_rng(40 + k)
    n_users, n_items = 300, 2000
    ue = rng.integers(-1, 2, (n_users, D)).astype(np.float32)
    ie = rng.integers(-1, 2, (n_items, D)).astype(np.float32)
    ie[100:400] = ie[7]  # 300 identical items
    rated = [rng.choice(n_items, int(rng.integers(0, 30)), replace=False) for _ in range(n_users)]
    rp, ri = _csr_rows(rated)
    users = rng.permutation(n_users).astype(np.int32)
    _check(torch_cuda, orc, ue, ie, users, rp, ri, k)


@pytest.mark.parametrize("k", [20, 32])
def test_rank_d128_common_component_falls_back(torch_cuda, orc, k):
    """Embeddings dominated by one common direction: every score of a user lies within the TF32 resolution of the
    others, the certificate fails, and the exact fallback still returns impl 1's lists."""
    rng = np.random.default_rng(60 + k)
    n_users, n_items = 200, 3000
    base = rng.standard_normal(D).astype(np.float32)
    ue = (base + 1e-4 * rng.standard_normal((n_users, D))).astype(np.float32)
    ie = (base + 1e-4 * rng.standard_normal((n_items, D))).astype(np.float32)
    rated = [rng.choice(n_items, int(rng.integers(0, 30)), replace=False) for _ in range(n_users)]
    rp, ri = _csr_rows(rated)
    users = rng.permutation(n_users).astype(np.int32)
    fb = _check(torch_cuda, orc, ue, ie, users, rp, ri, k)
    assert fb > 0


def test_rank_d128_auto_rule(torch_cuda):
    """impl 0 takes the tensor cores at d = 128 from 1024 items on (the fallback counter is reported), and the
    CUDA-core kernel below."""
    rng = np.random.default_rng(9)
    ue = _gauss(rng, 50)
    users = np.arange(50, dtype=np.int32)
    for n_items, tc in ((1023, False), (1024, True)):
        ie = _gauss(rng, n_items)
        ids, sc, fb = _topk(torch_cuda, ue, ie, users, None, None, 20, impl=0)
        assert (fb is not None) == tc, n_items
        i1, s1, _ = _topk(torch_cuda, ue, ie, users, None, None, 20, impl=1)
        assert np.array_equal(ids, i1) and np.array_equal(sc.view(np.uint32), s1.view(np.uint32))


def test_rank_d128_workspace_layout(built_lib):
    """The impl-2 workspace grows with d by the gathered user table only, and the fallback counter sits at the same
    offset at both widths."""
    from selfrec_b200 import _lib
    lib = _lib.load()
    n_q, n_items = 1000, 5000
    w64, w128 = lib.srb_topk_workspace_bytes(n_q, n_items, 64, 20), lib.srb_topk_workspace_bytes(n_q, n_items, 128, 20)
    n_q_pad = (n_q + 255) // 256 * 256 + 256
    assert w128 - w64 == n_q_pad * 64 * 4
    assert 0 <= lib.srb_topk_fallback_count_offset(n_q, n_items) < w64
