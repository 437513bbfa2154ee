"""Ranking on the owning rank, simulated in one process: a full user table cut into the cyclic blocks of 2, 3, 4 and 8
ranks, each block ranked against the item table with its rank-local rated / test CSRs (ShardRanker.local_topk /
local_hit_masks), the results reassembled into test order.  Ids and scores must equal ops.score_topk on the full table
bit for bit, and the measure strings must equal GraphRecommender._fast_measure() on the full table -- on the golden
tiny graph, on a yelp2018-shaped graph at d = 64 (tensor-core impl 2) and d = 32 / 128 (impl 1), and at topN 20, 50
(the 32-at-a-time wide path) and 64."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

WORLDS = (2, 3, 4, 8)


class _Data:
    """What _fast_measure and ShardRanker read: user / test_set keyed by name (here the user id itself), rated_csr,
    test_csr, user_num."""

    def __init__(self, U, I, seed, n_test_users):
        rng = np.random.default_rng(seed)
        self.user_num, self.item_num = U, I
        deg = np.minimum((rng.pareto(1.1, U) * 8).astype(np.int64) + 1, I // 4)  # power-law rated rows
        rated = [np.sort(rng.choice(I, size=int(k), replace=False)) for k in deg]
        self._rated = self._csr(rated)
        self.user = {u: u for u in range(U)}
        test_users = rng.permutation(U)[:n_test_users]  # test_set order is not id order
        self.test_set = {}
        for u in test_users.tolist():
            pool = np.setdiff1d(np.arange(I), rated[u])
            self.test_set[u] = {int(i): 1 for i in rng.choice(pool, size=int(rng.integers(1, 12)), replace=False)}
        rows = [np.array(sorted(self.test_set.get(u, {})), dtype=np.int64) for u in range(U)]
        ptr, idx = self._csr(rows)
        n_test = np.diff(ptr).astype(np.int32)
        self._test = (ptr, idx, n_test)

    @staticmethod
    def _csr(rows):
        ptr = np.zeros(len(rows) + 1, dtype=np.int32)
        ptr[1:] = np.cumsum([len(r) for r in rows])
        return ptr, (np.concatenate(rows) if rows else np.zeros(0)).astype(np.int32)

    def rated_csr(self):
        return self._rated

    def test_csr(self):
        return self._test


def _recommender(data, ue, ie, max_n):
    from selfrec_b200.base.graph_recommender import GraphRecommender
    m = object.__new__(GraphRecommender)
    m.data, m.user_emb, m.item_emb, m.max_N = data, ue, ie, max_n
    return m


def _check(data, ue, ie, k):
    import torch
    from selfrec_b200 import ops
    from selfrec_b200.shard_rank import ShardRanker, reassemble
    from selfrec_b200.util.evaluation import ranking_evaluation_from_masks
    uids = np.fromiter((data.user[u] for u in data.test_set), dtype=np.int32, count=len(data.test_set))
    want_ids, want_sc = ops.score_topk(ue, ie, uids, *data.rated_csr(), k)
    fast = _recommender(data, ue, ie, k)._fast_measure() if k <= 64 else None
    n_test = data.test_csr()[2]
    for world in WORLDS:
        ids_p, sc_p, mask_p = [], [], []
        for g in range(world):
            rk = ShardRanker(data, g, world, ue.device)
            block = ue[g::world].contiguous()  # rank g's [Ug, d] block: users g, g + world, ...
            i, s = rk.local_topk(block, ie, uids, k)
            ids_p.append(i)
            sc_p.append(s)
            if k <= 64:
                mask_p.append(rk.local_hit_masks(block, ie, uids, k))
        ids, sc = reassemble(ids_p, uids, world), reassemble(sc_p, uids, world)
        assert torch.equal(ids, want_ids), f"world {world}: ids differ"
        assert torch.equal(sc.view(torch.int32), want_sc.view(torch.int32)), f"world {world}: scores differ"
        if k <= 64:
            masks = reassemble(mask_p, uids, world).cpu().numpy().view(np.uint64)
            assert ranking_evaluation_from_masks(n_test[uids], masks, [k]) == fast, f"world {world}: measure differs"


def test_sharded_ranking_golden_tiny(torch_cuda_or_skip, golden, tiny_triples, tiny_conf, in_tmp_cwd):
    torch = torch_cuda_or_skip
    from selfrec_b200.base.graph_recommender import GraphRecommender
    train, test = tiny_triples
    r = golden("rank.npz")
    m = GraphRecommender(tiny_conf("MF"), [list(t) for t in train], [list(t) for t in test])
    _check(m.data, torch.from_numpy(r["user_emb"]).cuda(), torch.from_numpy(r["item_emb"]).cuda(), 10)


@pytest.mark.parametrize("d,k", [(64, 20), (32, 20), (128, 20), (64, 50), (64, 64), (32, 64)])
def test_sharded_ranking_yelp_shape(torch_cuda_or_skip, d, k):
    torch = torch_cuda_or_skip
    U, I = 31668, 38048
    data = _Data(U, I, seed=d + k, n_test_users=6000)
    g = torch.Generator(device="cuda").manual_seed(d * 100 + k)
    ue = torch.randn((U, d), device="cuda", generator=g) * 0.1
    ie = torch.randn((I, d), device="cuda", generator=g) * 0.1
    _check(data, ue, ie, k)


@pytest.fixture()
def torch_cuda_or_skip(built_lib):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch
