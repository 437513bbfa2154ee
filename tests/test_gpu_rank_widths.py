"""The tensor-core ranker (impl 2) at embedding sizes 16, 32 and 256 against the CUDA-core kernel (impl 1) and the
float64 oracle (oracle.score_topk).

At d = 16 a tile row is half a k-chunk: TMA zero-fills the box beyond the row and the MMA runs two k-steps.  At
d = 256 the users' k-chunks stream through the ring beside the items' (a resident user tile would not fit), so a CTA
still holds 128 users.  impl 2 must return what impl 1 returns, bit for bit: the same ids in the same order (ties by
id descending) and the same fp32 scores.  Against the oracle, scores are compared bit for bit and ids as sets among
equal scores (the reference orders exact ties by an unstable sort).  Lists of 33..256, which impl 1 cannot rank,
are held to the oracle on every row."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DS = [16, 32, 256]


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


def _gauss(rng, n, d, scale=0.1):
    return (rng.standard_normal((n, d)) * scale).astype(np.float32)


def _topk(torch, ue, ie, users, rp, ri, k, impl):
    """(ids, scores, fallback count or None) of ops.score_topk."""
    from selfrec_b200 import ops
    stats = {}
    ids, sc = ops.score_topk(torch.from_numpy(ue).cuda(), torch.from_numpy(ie).cuda(), users, rp, ri, k, impl=impl, stats=stats)
    torch.cuda.synchronize()
    fb = int(stats["fallback_count"].item()) if "fallback_count" in stats else None
    return ids.cpu().numpy(), sc.cpu().numpy(), fb


def _oracle_equal(orc, ue, ie, users, rp, ri, k, ids, sc, rows=None):
    rows = np.arange(len(users)) if rows is None else np.asarray(rows)
    oi, os_ = orc.score_topk(ue, ie, np.asarray(users)[rows], rp, ri, k)
    assert np.array_equal(sc[rows].view(np.uint32), os_.view(np.uint32))
    for r, q in enumerate(rows):
        if not np.array_equal(ids[q], oi[r]):
            assert sorted(zip(sc[q].tolist(), ids[q].tolist())) == sorted(zip(os_[r].tolist(), oi[r].tolist())), q


def _check(torch, orc, ue, ie, users, rp, ri, k, oracle_rows=None):
    """Lists of up to 32: impl 2 == impl 1 bit for bit, both equal to the oracle; longer lists: impl 2 equals the
    oracle.  Returns impl 2's fallback count."""
    i2, s2, fb = _topk(torch, ue, ie, users, rp, ri, k, impl=2)
    assert fb is not None
    if k <= 32:
        i1, s1, fb1 = _topk(torch, ue, ie, users, rp, ri, k, impl=1)
        assert fb1 is None
        assert np.array_equal(i2, i1), np.nonzero((i2 != i1).any(1))[0][:8]
        assert np.array_equal(s2.view(np.uint32), s1.view(np.uint32))
    # one order: score descending, ties by id descending
    assert ((np.diff(s2.astype(np.float64), axis=1) < 0) | ((np.diff(s2.astype(np.float64), axis=1) == 0) &
                                                             (np.diff(i2.astype(np.int64), axis=1) < 0))).all()
    _oracle_equal(orc, ue, ie, users, rp, ri, k, i2, s2, oracle_rows)
    return fb


@pytest.mark.parametrize("k", [1, 20, 32])
@pytest.mark.parametrize("n_items", [1024, 1025, 1151, 38048])
@pytest.mark.parametrize("d", DS)
def test_widths_shapes(torch_cuda, orc, d, n_items, k):
    """n_q = 1 and around the 128 users of a CTA; users with k - 1 and exactly k unrated items; a masked first,
    last item and whole tile."""
    rng = np.random.default_rng(d * 100000 + n_items * 10 + k)
    n_users = 400
    ue, ie = _gauss(rng, n_users, d), _gauss(rng, n_items, d)
    rated = [rng.choice(n_items, int(rng.integers(0, 60)), replace=False) for _ in range(n_users)]
    rated[0] = np.arange(n_items - max(k - 1, 0))
    rated[1] = rng.permutation(n_items)[k:]
    rated[2] = np.concatenate([[0, n_items - 1], np.arange(128, 256)])
    rp, ri = _csr_rows(rated)
    pool = np.concatenate([[0, 1, 2], rng.permutation(np.arange(3, n_users))]).astype(np.int32)
    for n_q in (1, 127, 128, 129):
        _check(torch_cuda, orc, ue, ie, pool[:n_q], rp, ri, k)


@pytest.mark.parametrize("d", DS)
def test_widths_many_ctas(torch_cuda, orc, d):
    """More users than one wave of 132 CTAs x 128 holds, at the yelp2018 item count."""
    rng = np.random.default_rng(5 + d)
    n_users, n_items = 132 * 128 + 1000, 38048
    ue, ie = _gauss(rng, n_users, d), _gauss(rng, n_items, d)
    rated = [rng.choice(n_items, int(rng.integers(0, 40)), replace=False) for _ in range(n_users)]
    rp, ri = _csr_rows(rated)
    users = rng.permutation(n_users).astype(np.int32)
    fb = _check(torch_cuda, orc, ue, ie, users, rp, ri, 20, oracle_rows=np.r_[0:64, 16890:16960, n_users - 64:n_users])
    assert fb <= 0.05 * n_users, fb  # well-separated scores: the certificate passes for almost everyone


@pytest.mark.parametrize("k", [33, 50, 100, 256])
@pytest.mark.parametrize("d", DS)
def test_widths_long_lists(torch_cuda, orc, d, k):
    """Lists of 33..256 through impl 2: an integer-valued table (exact ties everywhere, so find_k_largest's tie rule
    decides) and a Gaussian one whose catalogue is not a multiple of the tile."""
    rng = np.random.default_rng(40 + k + d)
    n_users, n_items = 200, 2000
    ue = rng.integers(-1, 2, (n_users, d)).astype(np.float32)
    ie = rng.integers(-1, 2, (n_items, d)).astype(np.float32)
    ie[100:400] = ie[7]
    rated = [rng.choice(n_items, int(rng.integers(0, 30)), replace=False) for _ in range(n_users)]
    rp, ri = _csr_rows(rated)
    users = rng.permutation(n_users).astype(np.int32)
    _check(torch_cuda, orc, ue, ie, users, rp, ri, k)
    n_items = 1151
    ue, ie = _gauss(rng, n_users, d), _gauss(rng, n_items, d)
    rated = [rng.choice(n_items, int(rng.integers(0, 40)), replace=False) for _ in range(n_users)]
    rated[0] = np.arange(n_items - (k - 1))  # k - 1 unrated items
    rp, ri = _csr_rows(rated)
    _check(torch_cuda, orc, ue, ie, users, rp, ri, k)


@pytest.mark.parametrize("k", [20, 100])
@pytest.mark.parametrize("d", DS)
def test_widths_zero_norm_and_few_unrated(torch_cuda, orc, d, k):
    """A zero-norm user (every score ties at 0), users with no, k - 1 and exactly k unrated items, n_q = 1."""
    rng = np.random.default_rng(7 * d + k)
    n_users, n_items = 300, 1024
    ue, ie = _gauss(rng, n_users, d), _gauss(rng, n_items, d)
    ue[5] = 0.0
    rated = [rng.choice(n_items, int(rng.integers(0, 40)), replace=False) for _ in range(n_users)]
    rated[0] = np.arange(n_items - (k - 1))
    rated[1] = rng.permutation(n_items)[k:]
    rated[2] = np.arange(n_items)
    rp, ri = _csr_rows(rated)
    users = np.concatenate([np.arange(8), rng.choice(np.arange(8, n_users), 120, replace=False)]).astype(np.int32)
    fb = _check(torch_cuda, orc, ue, ie, users, rp, ri, k)
    assert fb >= 3  # fewer than k unrated items: the exact path
    _check(torch_cuda, orc, ue, ie, users[5:6], rp, ri, k)


@pytest.mark.parametrize("k", [20, 32, 100])
@pytest.mark.parametrize("d", DS)
def test_widths_common_component_falls_back(torch_cuda, orc, d, k):
    """Tables dominated by one common direction, more users than the fallback's 256 rows: every score of a user lies
    within the TF32 resolution of the others, the certificate fails, and the exact fallback still returns the exact
    lists."""
    rng = np.random.default_rng(60 + k + d)
    n_users, n_items = 700, 2048
    base = rng.standard_normal(d).astype(np.float32)
    ue = (base + 1e-4 * rng.standard_normal((n_users, d))).astype(np.float32)
    ie = (base + 1e-4 * rng.standard_normal((n_items, d))).astype(np.float32)
    rated = [rng.choice(n_items, int(rng.integers(0, 30)), replace=False) for _ in range(n_users)]
    rp, ri = _csr_rows(rated)
    users = rng.permutation(n_users).astype(np.int32)
    fb = _check(torch_cuda, orc, ue, ie, users, rp, ri, k)
    assert fb > 256, fb


@pytest.mark.parametrize("k", [20, 100])
@pytest.mark.parametrize("d", DS)
def test_widths_nan_workspace(torch_cuda, orc, d, k):
    """A workspace filled with 0xFF bytes (NaN as floats) before the call gives the same lists."""
    torch = torch_cuda
    from selfrec_b200 import _lib, ops
    lib = _lib.load()
    rng = np.random.default_rng(k * 3 + d)
    n_users, n_items = 300, 1500
    ue, ie = _gauss(rng, n_users, d), _gauss(rng, n_items, d)
    rated = [rng.choice(n_items, int(rng.integers(0, 40)), replace=False) for _ in range(n_users)]
    rp, ri = _csr_rows(rated)
    users = rng.permutation(n_users).astype(np.int32)
    want_i, want_s, _ = _topk(torch, ue, ie, users, rp, ri, k, impl=2)
    dev = torch.device("cuda")
    ue_d, ie_d = torch.from_numpy(ue).to(dev), torch.from_numpy(ie).to(dev)
    u_d, rp_d, ri_d = (torch.from_numpy(np.asarray(x, np.int32)).to(dev) for x in (users, rp, ri))
    ids = torch.empty((len(users), k), dtype=torch.int32, device=dev)
    sc = torch.empty((len(users), k), dtype=torch.float32, device=dev)
    nb = lib.srb_topk_workspace_bytes(len(users), n_items, d, k)
    ws = torch.full((nb,), 0xFF, dtype=torch.uint8, device=dev)
    desc = _lib.TopkDesc()
    desc.user_emb, desc.item_emb, desc.n_items, desc.d = ops._p(ue_d), ops._p(ie_d), n_items, d
    desc.users, desc.n_q, desc.rated_ptr, desc.rated_idx = ops._p(u_d), len(users), ops._p(rp_d), ops._p(ri_d)
    desc.k, desc.out_ids, desc.out_scores, desc.impl = k, ops._p(ids), ops._p(sc), 2
    desc.workspace, desc.workspace_bytes = ops._p(ws), nb
    _lib.check(lib.srb_score_topk(C.byref(desc), ops._stream()), "srb_score_topk")
    torch.cuda.synchronize()
    assert np.array_equal(ids.cpu().numpy(), want_i)
    assert np.array_equal(sc.cpu().numpy().view(np.uint32), want_s.view(np.uint32))
    _oracle_equal(orc, ue, ie, users, rp, ri, k, want_i, want_s)


@pytest.mark.parametrize("d", DS)
def test_widths_auto_rule(torch_cuda, d):
    """impl 0 takes the tensor cores for lists of up to 32 from 1024 items on (the fallback counter is reported) and
    the CUDA-core kernel below; a list of 100 still comes from dense score rows."""
    torch = torch_cuda
    from selfrec_b200 import ops
    rng = np.random.default_rng(9 + d)
    ue = _gauss(rng, 50, d)
    users = np.arange(50, dtype=np.int32)
    for n_items, tc in ((1023, False), (1024, True), (38048, True)):
        ie = _gauss(rng, n_items, d)
        for k in (1, 20, 32):
            ids, sc, fb = _topk(torch, ue, ie, users, None, None, k, impl=0)
            assert (fb is not None) == tc, (n_items, k)
            i1, s1, _ = _topk(torch, ue, ie, users, None, None, k, impl=1)
            assert np.array_equal(ids, i1) and np.array_equal(sc.view(np.uint32), s1.view(np.uint32))
        stats = {}
        ops.score_topk(torch.from_numpy(ue).cuda(), torch.from_numpy(ie).cuda(), users, None, None, 100, stats=stats)
        assert "fallback_count" not in stats


def _model(tiny_conf, d, topn):
    """A GraphRecommender over a synth.make_interaction graph of 1500 items split into train and test, with random
    embedding tables."""
    import torch
    from selfrec_b200 import synth
    from selfrec_b200.base.graph_recommender import GraphRecommender
    g = synth.make_interaction((600, 1500, 12000), seed=8)
    pu, pi = g.pair_users, g.pair_items
    last = {u: j for j, u in enumerate(pu.tolist())}
    deg = np.bincount(pu, minlength=600)
    rng = np.random.default_rng(2 + d)
    train, test = [], []
    for j, (u, i) in enumerate(zip(pu.tolist(), pi.tolist())):
        held = deg[u] >= 3 and (last[u] == j or rng.random() < 0.2)
        (test if held else train).append([f"u{u}", f"i{i}", 1.0])
    m = GraphRecommender(tiny_conf("MF", **{"item.ranking.topN": topn, "embedding.size": d}), train, test)
    assert m.data.item_num >= 1024
    m.user_emb = torch.from_numpy(_gauss(rng, m.data.user_num, d)).cuda()
    m.item_emb = torch.from_numpy(_gauss(rng, m.data.item_num, d)).cuda()
    m.model_name = "MF"
    return m


@pytest.mark.parametrize("d", DS)
def test_widths_model_level(torch_cuda, orc, tiny_conf, in_tmp_cwd, tmp_path, d):
    """test() lists equal the oracle, fast_evaluation's measure equals ranking_evaluation over test(), an export
    equals rank_all, and ShardRanker ranks of loopback worlds 2 and 3 reassemble into the single-table ranking."""
    torch = torch_cuda
    from selfrec_b200 import export, ops, shard_rank
    from selfrec_b200.sharded import user_ids_of
    from selfrec_b200.util.evaluation import ranking_evaluation
    m = _model(tiny_conf, d, [10, 20])
    names = list(m.data.test_set)
    uids = np.fromiter((m.data.user[u] for u in names), dtype=np.int32, count=len(names))
    rp, ri = m.data.rated_csr()
    ue, ie = m.user_emb.cpu().numpy(), m.item_emb.cpu().numpy()
    rec = m.test()
    oi, os_ = orc.score_topk(ue, ie, uids, rp, ri, 20)
    for q, u in enumerate(names):
        got = [(float(s), m.data.item[i]) for i, s in rec[u]]
        assert sorted(got) == sorted(zip(os_[q].tolist(), oi[q].tolist())), u
    assert m._fast_measure() == ranking_evaluation(m.data.test_set, rec, [m.max_N])
    all_names = [m.data.id2user[u] for u in range(m.data.user_num)]
    _, want_ids, want_sc = m.rank_all(all_names)
    got_names, ids, sc = export.read(m.export_recommendations(str(tmp_path / "exp"), top_n=20, chunk=97))
    assert got_names == all_names
    assert np.array_equal(np.asarray(ids), want_ids) and np.array_equal(np.asarray(sc).view(np.uint32), want_sc.view(np.uint32))
    want_i, want_s = ops.score_topk(m.user_emb, m.item_emb, uids, rp, ri, 20)
    for world in (2, 3):
        ids_p, sc_p = [], []
        for g in range(world):
            rk = shard_rank.ShardRanker(m.data, g, world, m.user_emb.device)
            block = m.user_emb[torch.from_numpy(user_ids_of(m.data.user_num, g, world)).cuda().long()].contiguous()
            i, s = rk.local_topk(block, m.item_emb, uids, 20)
            ids_p.append(i)
            sc_p.append(s)
        assert torch.equal(shard_rank.reassemble(ids_p, uids, world), want_i), world
        assert torch.equal(shard_rank.reassemble(sc_p, uids, world).view(torch.int32), want_s.view(torch.int32)), world
