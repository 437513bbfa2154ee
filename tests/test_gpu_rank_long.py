"""Top-k lists of 33..256 on the tensor cores (impl 2 at d = 64 and 128: candidate buffers behind a running threshold,
exact fp32 rescoring, the certificate and the exact long-list fallback) against the float64 oracle's find_k_largest
and, where no two scores tie exactly at the cut, against the dense-row path (ops._score_topk_wide) bit for bit; the
multi-word hit masks and fast_evaluation at max_N up to 256; and a top-100 export through the new route against the
dense-row route.

On exact ties at the cut the dense-row path can keep other tied items than find_k_largest: it runs the selection
32 entries at a time, and which tied items enter the list depends on its length.  The tie cases below are therefore
held to the oracle on every row."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
for _p in (ROOT, TESTS):
    if _p not in sys.path:
        sys.path.insert(0, _p)

KS = [33, 50, 64, 65, 100, 128, 200, 256]
DS = [64, 128]


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


def _run(torch, ue, ie, users, rp, ri, k):
    """(tensor-core ids, scores, fallback count) and (dense-row ids, scores)."""
    from selfrec_b200 import ops
    ue_d, ie_d = torch.from_numpy(ue).cuda(), torch.from_numpy(ie).cuda()
    stats = {}
    ids, sc = ops.score_topk(ue_d, ie_d, users, rp, ri, k, impl=2, stats=stats)
    torch.cuda.synchronize()
    fb = int(stats["fallback_count"].item()) if "fallback_count" in stats else 0
    u_d = torch.from_numpy(np.asarray(users, np.int32)).cuda()
    wi, ws = ops._score_topk_wide(ue_d, ie_d, u_d, rp, ri, k)
    return (ids.cpu().numpy(), sc.cpu().numpy(), fb), (wi.cpu().numpy(), ws.cpu().numpy())


def _check(torch, orc, ue, ie, users, rp, ri, k, oracle_rows=(), wide=True):
    (i2, s2, fb), (iw, sw) = _run(torch, ue, ie, users, rp, ri, k)
    assert i2.shape == (len(users), k)
    if wide:
        assert np.array_equal(i2, iw), np.nonzero((i2 != iw).any(1))[0][:8]
        assert np.array_equal(s2.view(np.uint32), sw.view(np.uint32))
    else:  # the scores never depend on which tied items are kept
        assert np.array_equal(s2.view(np.uint32), sw.view(np.uint32))
    # one order: score descending, ties by id descending
    assert (np.diff(s2.astype(np.float64), axis=1) <= 0).all()
    assert ((np.diff(s2.astype(np.float64), axis=1) < 0) | (np.diff(i2.astype(np.int64), axis=1) < 0)).all()
    rows = np.asarray(oracle_rows, np.int64)
    if rows.size:
        oi, os_ = orc.score_topk(ue, ie, np.asarray(users)[rows], rp, ri, k)
        assert np.array_equal(s2[rows].view(np.uint32), os_.view(np.uint32))
        for r, q in enumerate(rows):  # the oracle orders exact ties by an unstable sort: compare them as sets
            assert sorted(zip(s2[q].tolist(), i2[q].tolist())) == sorted(zip(os_[r].tolist(), oi[r].tolist())), q
    return fb


def _gauss(rng, n, d, scale=0.1):
    return (rng.standard_normal((n, d)) * scale).astype(np.float32)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("d", DS)
def test_long_yelp_shape(torch_cuda, orc, d, k):
    """Random tables at the yelp2018 shape (31 668 x 38 048), 4096 queried users with rated lists."""
    rng = np.random.default_rng(d * 1000 + k)
    n_users, n_items = 31668, 38048
    ue, ie = _gauss(rng, n_users, d), _gauss(rng, n_items, d)
    deg = rng.integers(0, 60, n_users)
    rated = [rng.choice(n_items, int(g), replace=False) for g in deg]
    rp, ri = _csr_rows(rated)
    users = rng.choice(n_users, 4096, replace=False).astype(np.int32)
    fb = _check(torch_cuda, orc, ue, ie, users, rp, ri, k, oracle_rows=range(16))
    assert fb <= 0.05 * len(users), fb  # well-separated scores: almost every user is certified


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("d", DS)
def test_long_edges(torch_cuda, orc, d, k):
    """I = 1024 (the dispatch edge) and an I that is not a multiple of 128; users with exactly k, fewer than k and
    no unrated items; a zero-norm user (every score tied); duplicated item rows, so that ties straddle the cut and
    a 32-entry boundary; n_q = 1."""
    rng = np.random.default_rng(7 * d + k)
    for n_items in (1024, 1999):
        n_users = 300
        ue, ie = _gauss(rng, n_users, d), _gauss(rng, n_items, d)
        ie[500:800] = ie[11]                    # 300 identical items: ties across the cut at every k
        ie[40:40 + k // 2 + 3] = ie[900]         # a tied block around the middle of the list
        ue[5] = 0.0                              # zero-norm user: every score ties at 0
        rated = [rng.choice(n_items, int(rng.integers(0, 40)), replace=False) for _ in range(n_users)]
        rated[0] = np.arange(n_items - (k - 1))                 # k - 1 unrated items
        rated[1] = rng.permutation(n_items)[k:]                 # exactly k unrated items
        rated[2] = np.arange(n_items)                           # none unrated: the masked entries
        rated[3] = np.concatenate([[0, n_items - 1], np.arange(128, 256)])
        rp, ri = _csr_rows(rated)
        users = np.concatenate([np.arange(8), rng.choice(np.arange(8, n_users), 120, replace=False)]).astype(np.int32)
        _check(torch_cuda, orc, ue, ie, users, rp, ri, k, oracle_rows=range(len(users)), wide=False)
        _check(torch_cuda, orc, ue, ie, users[4:5], rp, ri, k, oracle_rows=[0], wide=False)


@pytest.mark.parametrize("k", [33, 100, 256])
@pytest.mark.parametrize("d", DS)
def test_long_integer_ties(torch_cuda, orc, d, k):
    """Small-integer embeddings: many exactly equal scores, so the selection rule and the tie order decide."""
    rng = np.random.default_rng(40 + k + d)
    n_users, n_items = 200, 2000
    ue = rng.integers(-1, 2, (n_users, d)).astype(np.float32)
    ie = rng.integers(-1, 2, (n_items, d)).astype(np.float32)
    ie[100:400] = ie[7]
    rated = [rng.choice(n_items, int(rng.integers(0, 30)), replace=False) for _ in range(n_users)]
    rp, ri = _csr_rows(rated)
    users = rng.permutation(n_users).astype(np.int32)
    _check(torch_cuda, orc, ue, ie, users, rp, ri, k, oracle_rows=range(n_users), wide=False)


@pytest.mark.parametrize("k", [50, 256])
@pytest.mark.parametrize("d", DS)
def test_long_huge_norm_item_falls_back(torch_cuda, orc, d, k):
    """One item with a huge norm widens every user's error bound past the score gaps: the certificate fails, the
    fallback counter is > 0, and the result is still exact."""
    rng = np.random.default_rng(90 + k + d)
    n_users, n_items = 300, 3000
    ue, ie = _gauss(rng, n_users, d), _gauss(rng, n_items, d)
    ie[1234] *= 1e4
    rated = [rng.choice(n_items, int(rng.integers(0, 30)), replace=False) for _ in range(n_users)]
    rp, ri = _csr_rows(rated)
    users = rng.permutation(n_users).astype(np.int32)
    fb = _check(torch_cuda, orc, ue, ie, users, rp, ri, k, oracle_rows=range(8))
    assert fb > 0


@pytest.mark.parametrize("d", DS)
def test_long_many_fallbacks(torch_cuda, orc, d):
    """More uncertified users than the fallback holds rows for at once (256 at this catalogue): every user of a
    common-direction table fails the certificate and is re-ranked in several rounds."""
    rng = np.random.default_rng(61 + d)
    n_users, n_items = 700, 2048
    base = rng.standard_normal(d).astype(np.float32)
    ue = (base + 1e-4 * rng.standard_normal((n_users, d))).astype(np.float32)
    ie = (base + 1e-4 * rng.standard_normal((n_items, d))).astype(np.float32)
    rated = [rng.choice(n_items, int(rng.integers(0, 30)), replace=False) for _ in range(n_users)]
    rp, ri = _csr_rows(rated)
    users = rng.permutation(n_users).astype(np.int32)
    fb = _check(torch_cuda, orc, ue, ie, users, rp, ri, 100, oracle_rows=range(n_users), wide=False)
    assert fb > 256, fb


def test_long_empty_and_dispatch(torch_cuda):
    """n_q = 0 returns empty lists; impl 0 takes the tensor cores for 33..256 at d = 64 / 128 from 1024 items on (the
    fallback counter is reported) and the dense rows below, at other widths and above 256."""
    torch = torch_cuda
    from selfrec_b200 import ops
    rng = np.random.default_rng(3)
    ue = torch.from_numpy(_gauss(rng, 40, 64)).cuda()
    ie = torch.from_numpy(_gauss(rng, 1024, 64)).cuda()
    ids, sc = ops.score_topk(ue, ie, np.zeros(0, np.int32), None, None, 100)
    assert ids.shape == (0, 100) and sc.shape == (0, 100)
    users = np.arange(40, dtype=np.int32)
    for n_items, k, tc in ((1023, 100, False), (1024, 100, True), (1024, 256, True), (1024, 257, False)):
        stats = {}
        ops.score_topk(ue, ie[:n_items], users, None, None, k, stats=stats)
        assert ("fallback_count" in stats) == tc, (n_items, k)


def _test_lists(rng, n_users, n_items, per_user):
    rows = [np.sort(rng.choice(n_items, size=int(rng.integers(1, per_user)), replace=False)).astype(np.int32) for _ in range(n_users)]
    ptr = np.zeros(n_users + 1, np.int32)
    ptr[1:] = np.cumsum([len(x) for x in rows])
    return rows, ptr, np.concatenate(rows).astype(np.int32)


@pytest.mark.parametrize("k", [1, 64, 65, 128, 129, 200, 256])
def test_multiword_hit_masks(torch_cuda, k):
    torch = torch_cuda
    from selfrec_b200 import ops
    rng = np.random.default_rng(k)
    U, I = 300, 2000
    rows, ptr, idx = _test_lists(rng, U, I, 200)
    users = rng.permutation(U)[:257].astype(np.int32)
    ids = np.stack([np.concatenate([rows[u][:k // 3], rng.choice(I, size=k, replace=False)])[:k] for u in users]).astype(np.int32)
    got = ops.rank_hit_masks(torch.from_numpy(ids).cuda(), users, ptr, idx).cpu().numpy().view(np.uint64)
    words = (k + 63) // 64
    assert got.shape == ((len(users),) if words == 1 else (len(users), words))
    got = got.reshape(len(users), words)
    for q, u in enumerate(users):
        want = sum(1 << r for r in range(k) if ids[q, r] in set(rows[u].tolist()))
        assert sum(int(w) << (64 * j) for j, w in enumerate(got[q])) == want


def _ranked_model(tiny_conf, d, topn):
    """A GraphRecommender over a synthetic 1500-item graph with random embedding tables."""
    import torch
    from selfrec_b200 import synth
    from selfrec_b200.base.graph_recommender import GraphRecommender
    pu, pi = synth.make_pairs(600, 1500, 12000, seed=8)
    train, test, last = [], [], {}
    for j, u in enumerate(pu.tolist()):
        last[u] = j
    deg = np.bincount(pu, minlength=600)
    rng = np.random.default_rng(2)
    for j, (u, i) in enumerate(zip(pu.tolist(), pi.tolist())):
        held = deg[u] >= 3 and (last[u] == j or rng.random() < 0.2)
        (test if held else train).append([f"u{u}", f"i{i}", 1.0])
    m = GraphRecommender(tiny_conf("MF", **{"item.ranking.topN": topn, "embedding.size": d}), train, test)
    assert m.data.item_num >= 1024
    m.user_emb = torch.from_numpy(_gauss(rng, m.data.user_num, d)).cuda()
    m.item_emb = torch.from_numpy(_gauss(rng, m.data.item_num, d)).cuda()
    return m


@pytest.mark.parametrize("max_n", [65, 100, 256])
@pytest.mark.parametrize("d", DS)
def test_fast_measure_long(torch_cuda, tiny_conf, in_tmp_cwd, d, max_n):
    """fast_evaluation's device route at max_N over 64 returns the strings of ranking_evaluation over test(), on
    the model's own tables and through ShardRanker ranks (world 1, and world 3 reassembled from loopback ranks that
    each hold only their own user rows)."""
    torch = torch_cuda
    from selfrec_b200 import ops, shard_rank
    from selfrec_b200.sharded import user_ids_of
    from selfrec_b200.util.evaluation import ranking_evaluation, ranking_evaluation_from_masks
    m = _ranked_model(tiny_conf, d, [20, max_n])
    slow = ranking_evaluation(m.data.test_set, m.test(), [max_n])
    calls = []
    orig = ops.rank_hit_masks
    try:
        ops.rank_hit_masks = lambda *a: calls.append(1) or orig(*a)
        assert m._fast_measure() == slow
        assert calls  # the device route, not test()
    finally:
        ops.rank_hit_masks = orig
    dev = m.item_emb.device
    m.shard_ranker = shard_rank.ShardRanker(m.data, 0, 1, dev)
    assert m._fast_measure() == slow
    m.shard_ranker = None
    names = list(m.data.test_set)
    uids = np.fromiter((m.data.user[u] for u in names), dtype=np.int32, count=len(names))
    world, parts = 3, []
    for g in range(world):
        r = shard_rank.ShardRanker(m.data, g, world, dev)
        block = m.user_emb[torch.from_numpy(user_ids_of(m.data.user_num, g, world)).to(dev).long()].contiguous()
        parts.append(r.local_hit_masks(block, m.item_emb, uids, max_n))
    masks = shard_rank.reassemble(parts, uids, world).cpu().numpy().view(np.uint64)
    _, _, n_test = m.data.test_csr()
    assert ranking_evaluation_from_masks(n_test[uids], masks, [max_n]) == slow


def test_export_top100_long_route(torch_cuda, tiny_conf, tmp_path, monkeypatch):
    """A top-100 export through the tensor-core route, in several chunks, writes the same part files as the
    dense-row route."""
    from selfrec_b200 import export, ops
    m = _ranked_model(tiny_conf, 128, [20])
    m.model_name = "MF"
    a = export.read(m.export_recommendations(str(tmp_path / "tc"), top_n=100, chunk=97))
    assert export.long_list_chunk(97, m.data.item_num, 128, 100) == 97
    monkeypatch.setattr(ops, "long_list_route", lambda *args, **kw: False)
    b = export.read(m.export_recommendations(str(tmp_path / "wide"), top_n=100, chunk=97))
    assert a[0] == b[0]
    assert np.array_equal(a[1], b[1]) and np.array_equal(np.asarray(a[2]).view(np.uint32), np.asarray(b[2]).view(np.uint32))
    for f in ("users.0.npy", "ids.0.npy", "scores.0.npy"):
        assert open(tmp_path / "tc" / "MF-top100" / f, "rb").read() == open(tmp_path / "wide" / "MF-top100" / f, "rb").read()
