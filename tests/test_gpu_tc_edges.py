"""The tensor-core InfoNCE and full-catalog top-k kernels at their dispatch edges, against the float64
oracle (oracle.infonce, oracle.score_topk).

InfoNCE runs on the tensor cores when d = 64, b_cos is set, a call has at most 2 problems and
1/tau <= 40; everything else runs on the CUDA cores.  Each case here runs on the paths the rule
allows, with the problem layouts the training steps use (device counts below the capacity, row offsets,
weights, scales) rather than only the single-problem layout of ops.InfoNCE.

Top-k impl 2 keeps TF32 candidates, re-scores them in fp32 and certifies the result; users that fail
the certificate are re-run exactly.  The cases here make the certificate fail on purpose (near-ties
below the TF32 resolution), read the fallback counter, and check that fast and re-run rows land in the
right output rows."""
import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu

RTOL = 1e-4
TAU_TC_MIN = 0.025  # the smallest temperature the tensor-core InfoNCE path takes (1/tau <= 40)


@pytest.fixture(scope="module")
def torch_cuda(built_lib):
    import torch
    assert torch.cuda.is_available()
    from selfrec_b200 import _lib
    _lib.require_device()
    return torch


def _on_tc(d, b_cos, n_problems, tau):
    """InfoNCE's dispatch rule (srb_infonce_fwd_bwd); test_nce_dispatch_rule checks it on the device."""
    return d == 64 and bool(b_cos) and n_problems <= 2 and np.float32(1.0) / np.float32(tau) <= 40


# ------------------------------------------------------------------------------------------
# InfoNCE
# ------------------------------------------------------------------------------------------
def _prob(table1, table2, idx, n_dev=None, row_off1=0, row_off2=0, scale1=1.0, scale2=1.0, weight=1.0):
    return dict(table1=np.ascontiguousarray(table1, np.float32), table2=np.ascontiguousarray(table2, np.float32),
                idx=np.ascontiguousarray(idx, np.int32), n_dev=n_dev, row_off1=row_off1, row_off2=row_off2,
                scale1=scale1, scale2=scale2, weight=weight)


def _rows(p):
    """The rows the kernel gathers: scale * table[idx[:n_dev] + row_off], in fp32 like the kernel."""
    m = len(p["idx"]) if p["n_dev"] is None else p["n_dev"]
    i = p["idx"][:m].astype(np.int64)
    r1 = (np.float32(p["scale1"]) * p["table1"][i + p["row_off1"]]).astype(np.float32)
    r2 = (np.float32(p["scale2"]) * p["table2"][i + p["row_off2"]]).astype(np.float32)
    return r1, r2


def _run_nce(torch, probs, d, tau, b_cos=True, workspace=None):
    """ops.infonce_raw on device copies of probs; g1 / g2 are prefilled with NaN so that rows the kernel must
    not write stay visible.  Returns (losses, [(g1, g2)]) as numpy."""
    from selfrec_b200 import ops
    tables = {}

    def dev(a):  # problems share tables, as in the training step
        if id(a) not in tables:
            tables[id(a)] = torch.from_numpy(a).cuda()
        return tables[id(a)]

    call = []
    for p in probs:
        n = len(p["idx"])
        q = dict(table1=dev(p["table1"]), table2=dev(p["table2"]), idx=torch.from_numpy(p["idx"]).cuda(), n=n,
                 row_off1=p["row_off1"], row_off2=p["row_off2"], scale1=p["scale1"], scale2=p["scale2"], weight=p["weight"],
                 g1=torch.full((n, d), float("nan"), device="cuda"), g2=torch.full((n, d), float("nan"), device="cuda"))
        if p["n_dev"] is not None:
            q["n_dev"] = torch.tensor([p["n_dev"]], dtype=torch.int32, device="cuda")
        call.append(q)
    losses, outs = ops.infonce_raw(call, d, tau, b_cos, workspace=workspace)
    torch.cuda.synchronize()
    return losses.cpu().numpy(), [(g1.cpu().numpy(), g2.cpu().numpy()) for g1, g2 in outs]


def _nce_errors(orc, probs, losses, grads, d, tau, b_cos):
    """Each problem against oracle.infonce on its gathered rows, as (what, error / bar) pairs, with
    test_infonce_batch_sizes' bars: loss within RTOL |ref| + 2e-7 / tau (unweighted), gradients (times the
    weight) within RTOL |ref| + 2e-5 max|ref| + the fp32 conditioning floor 3 eps32 / tau / (n tau) / sqrt(d).
    With b_cos every gradient row is compared times its row norm max(||v||, 1e-12): the normalisation backward
    divides row i by exactly that norm, so this measures the error of the unit-vector gradient, and zero rows
    and rows scaled by 1e-3 / 1e3 sit on one scale.  Rows [n_dev, n) must keep their NaN prefill, and a
    problem with a device count of 0 must return a loss of exactly 0."""
    out = []
    for q, p in enumerate(probs):
        g1, g2 = grads[q]
        m = len(p["idx"]) if p["n_dev"] is None else p["n_dev"]
        untouched = np.isnan(g1[m:]).all() and np.isnan(g2[m:]).all()
        out.append((f"problem {q} rows past the device count untouched", 0.0 if untouched else np.inf))
        if m == 0:
            out.append((f"problem {q} empty loss {losses[q]!r}", 0.0 if losses[q] == 0.0 else np.inf))
            continue
        r1, r2 = _rows(p)
        ref, d1, d2 = orc.infonce(r1, r2, tau, b_cos)
        err = abs(float(losses[q]) - ref)
        out.append((f"problem {q} loss {losses[q]!r} vs {ref!r}", err / (RTOL * abs(ref) + 2e-7 / tau)))
        cond = 3 * 1.2e-7 / tau / (m * tau) / np.sqrt(d)
        for got, want, rows, side in ((g1[:m], d1, r1, "g1"), (g2[:m], d2, r2, "g2")):
            want = p["weight"] * want
            got = got.astype(np.float64)
            if b_cos:
                nrm = np.maximum(np.linalg.norm(rows.astype(np.float64), axis=1, keepdims=True), 1e-12)
                got, want = got * nrm, want * nrm
            bar = RTOL * np.abs(want) + 2e-5 * np.abs(want).max() + abs(p["weight"]) * cond
            ratio = (np.abs(got - want) / bar).max() if np.isfinite(got).all() else np.inf
            out.append((f"problem {q} {side}", ratio))
    return out


def _check_nce(orc, probs, losses, grads, d, tau, b_cos):
    bad = [(what, f"{r:.3g} x the bar") for what, r in _nce_errors(orc, probs, losses, grads, d, tau, b_cos) if not r <= 1.0]
    assert not bad, bad


def _views(rng, n, d, noise=0.05):
    v1 = (rng.standard_normal((n, d)) * 0.1).astype(np.float32)
    v2 = (v1 + noise * rng.standard_normal((n, d))).astype(np.float32)
    return v1, v2


# (d, tau): two tensor-core configurations (tau = 0.2 and the threshold 0.025) and the CUDA cores at d = 64
# just past the threshold and at d = 128
TC_CONFIGS = [(64, 0.2), (64, TAU_TC_MIN), (64, 0.0249), (128, 0.2)]
CFG_IDS = ["tc-0.2", "tc-0.025", "cuda-0.0249", "cuda-d128"]


def test_nce_dispatch_rule(torch_cuda):
    """The rule _on_tc states is the one the library applies: kernel names from the profiler."""
    torch = torch_cuda
    from torch.profiler import ProfilerActivity, profile
    rng = np.random.default_rng(0)
    v1, v2 = _views(rng, 300, 64)
    cases = [(1, 0.2, True), (2, TAU_TC_MIN, True), (2, 0.0249, True), (1, 0.2, False), (3, 0.2, True)]
    for npb, tau, b_cos in cases:
        probs = [_prob(v1, v2, np.arange(300 - 7 * q)) for q in range(npb)]
        _run_nce(torch, probs, 64, tau, b_cos)  # first launch outside the profiled window
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _run_nce(torch, probs, 64, tau, b_cos)
        names = " ".join(e.name for e in prof.events())
        tc, cc = "nce_tc_kernel" in names, "nce_lse_kernel" in names
        assert tc != cc, (npb, tau, b_cos, names[:400])
        assert tc == _on_tc(64, b_cos, npb, tau), (npb, tau, b_cos)


def _engine_problems(rng, B, n_dev, d, U=2500, I=3000, weight=0.3):
    """The XSimGCL / SimGCL step's call: unique users and unique items of one batch, both gathered from the
    same [U + I, d] tables (items at row offset U), each with its own device count below the capacity B."""
    t1 = (rng.standard_normal((U + I, d)) * 0.1).astype(np.float32)
    t2 = (t1 + 0.05 * rng.standard_normal((U + I, d))).astype(np.float32)
    probs = []
    for q, (m, pool) in enumerate(zip(n_dev, (U, I))):
        idx = np.sort(rng.choice(pool, m, replace=False))
        idx = np.concatenate([idx, rng.integers(0, pool, B - m)])  # stale entries past the count: valid rows
        probs.append(_prob(t1, t2, idx, n_dev=m, row_off1=q * U, row_off2=q * U, weight=weight))
    return probs


@pytest.mark.parametrize("d,tau", TC_CONFIGS, ids=CFG_IDS)
@pytest.mark.parametrize("B,n_dev", [(2048, (1900, 37)), (512, (0, 511))])
def test_nce_engine_shape(torch_cuda, orc, B, n_dev, d, tau):
    rng = np.random.default_rng(B + n_dev[1])
    probs = _engine_problems(rng, B, n_dev, d)
    losses, grads = _run_nce(torch_cuda, probs, d, tau)
    _check_nce(orc, probs, losses, grads, d, tau, True)


@pytest.mark.parametrize("d,tau", TC_CONFIGS, ids=CFG_IDS)
def test_nce_sgl_shape(torch_cuda, orc, d, tau):
    """SGL's call: one problem over users and items, capacity 2B = 4096."""
    rng = np.random.default_rng(4096)
    U, I, nu = 2500, 3000, 1400
    t1 = (rng.standard_normal((U + I, d)) * 0.1).astype(np.float32)
    t2 = (t1 + 0.05 * rng.standard_normal((U + I, d))).astype(np.float32)
    cat = np.concatenate([np.sort(rng.choice(U, nu, replace=False)), U + np.sort(rng.choice(I, 3001 - nu, replace=False))])
    idx = np.concatenate([cat, rng.integers(0, U + I, 4096 - 3001)])
    probs = [_prob(t1, t2, idx, n_dev=3001, weight=0.1)]
    losses, grads = _run_nce(torch_cuda, probs, d, tau)
    _check_nce(orc, probs, losses, grads, d, tau, True)


@pytest.mark.parametrize("d,tau", TC_CONFIGS, ids=CFG_IDS)
@pytest.mark.parametrize("n", [1, 2, 31, 33, 63, 65, 127, 129, 255, 257, 2049])
def test_nce_size_edges(torch_cuda, orc, n, d, tau):
    """n just past the 32-row prep tile, the 64-row CUDA-core tile and the 128-row tensor-core tile / padding."""
    rng = np.random.default_rng(n)
    v1, v2 = _views(rng, n, d)
    probs = [_prob(v1, v2, rng.permutation(n))]
    losses, grads = _run_nce(torch_cuda, probs, d, tau)
    _check_nce(orc, probs, losses, grads, d, tau, True)


@pytest.mark.parametrize("tau", [0.2, TAU_TC_MIN])
def test_nce_without_cos_at_d64(torch_cuda, orc, tau):
    rng = np.random.default_rng(5)
    v1, v2 = _views(rng, 700, 64)
    probs = [_prob(v1, v2, np.arange(700), weight=0.5)]
    losses, grads = _run_nce(torch_cuda, probs, 64, tau, b_cos=False)
    _check_nce(orc, probs, losses, grads, 64, tau, False)


@pytest.mark.parametrize("tau", [0.2, TAU_TC_MIN])
@pytest.mark.parametrize("d", [32, 64, 128])
@pytest.mark.parametrize("npb", [3, 4])
def test_nce_three_and_four_problems(torch_cuda, orc, npb, d, tau):
    rng = np.random.default_rng(npb * d)
    sizes = [(300, 300), (77, 40), (1000, 999), (5, 0)][:npb]  # (capacity, device count)
    t1, t2 = _views(rng, 4000, d)
    probs = [_prob(t1, t2, rng.integers(0, 1000, n), n_dev=m, row_off1=1000 * q, row_off2=1000 * q, weight=0.2 + 0.3 * q)
             for q, (n, m) in enumerate(sizes)]
    losses, grads = _run_nce(torch_cuda, probs, d, tau)
    _check_nce(orc, probs, losses, grads, d, tau, True)


@pytest.mark.parametrize("d,tau", TC_CONFIGS, ids=CFG_IDS)
def test_nce_zero_and_scaled_rows(torch_cuda, orc, d, tau):
    """Zero rows (F.normalize's 1e-12 clamp) and rows scaled by 1e-3 and 1e3, mixed into one batch."""
    rng = np.random.default_rng(11)
    n = 600
    v1, v2 = _views(rng, n, d)
    v1 *= rng.choice(np.float32([1e-3, 1.0, 1e3]), n)[:, None]
    v2 *= rng.choice(np.float32([1e-3, 1.0, 1e3]), n)[:, None]
    v1[rng.choice(n, 9, replace=False)] = 0
    v2[rng.choice(n, 9, replace=False)] = 0
    v1[17] = v2[17] = 0
    probs = [_prob(v1, v2, np.arange(n), weight=0.7)]
    losses, grads = _run_nce(torch_cuda, probs, d, tau)
    _check_nce(orc, probs, losses, grads, d, tau, True)


@pytest.mark.parametrize("d,tau", TC_CONFIGS, ids=CFG_IDS)
def test_nce_nearly_identical_views(torch_cuda, orc, d, tau):
    """v2 = v1 + 1e-4 noise: at small tau the loss approaches 0 and the gradient is all conditioning."""
    rng = np.random.default_rng(12)
    v1, v2 = _views(rng, 1000, d, noise=1e-4)
    probs = [_prob(v1, v2, np.arange(1000))]
    losses, grads = _run_nce(torch_cuda, probs, d, tau)
    _check_nce(orc, probs, losses, grads, d, tau, True)


@pytest.mark.parametrize("tau", [TAU_TC_MIN, 0.0125])
def test_nce_opposite_views(torch_cuda, orc, tau):
    """Every cosine near -1: the tensor-core path shifts the logits by the bound 1/tau instead of a row maximum,
    so exp(S - 1/tau) ~ exp(-2/tau) must stay a normal fp32 number (the threshold 1/tau <= 40); below the
    threshold the CUDA cores shift by the running maximum."""
    rng = np.random.default_rng(18)
    a = rng.standard_normal(64) * 0.1
    v1 = (a + 0.01 * rng.standard_normal((256, 64))).astype(np.float32)
    v2 = (-a + 0.01 * rng.standard_normal((256, 64))).astype(np.float32)
    probs = [_prob(v1, v2, np.arange(256))]
    losses, grads = _run_nce(torch_cuda, probs, 64, tau)
    _check_nce(orc, probs, losses, grads, 64, tau, True)


@pytest.mark.parametrize("b_cos,tau", [(True, 0.2), (True, TAU_TC_MIN), (False, 0.2)])
def test_nce_view_scales(torch_cuda, orc, b_cos, tau):
    rng = np.random.default_rng(13)
    U, I = 900, 800
    t1, t2 = _views(rng, U + I, 64)
    probs = [_prob(t1, t2, rng.permutation(U)[:500], scale1=0.5, scale2=3.0, weight=0.4),
             _prob(t1, t2, rng.permutation(I)[:300], n_dev=250, row_off1=U, row_off2=U, scale1=1.75, scale2=0.25, weight=0.4)]
    losses, grads = _run_nce(torch_cuda, probs, 64, tau, b_cos)
    _check_nce(orc, probs, losses, grads, 64, tau, b_cos)


@pytest.mark.parametrize("tau", [0.2, 0.0249])
def test_nce_workspace_reuse(torch_cuda, orc, tau):
    """A large call and then a small one in one workspace first filled with 0xFF bytes (NaN as floats):
    nothing may depend on what the workspace held before."""
    torch = torch_cuda
    from selfrec_b200 import _lib
    rng = np.random.default_rng(14)
    big = _engine_problems(rng, 2048, (1900, 2048), 64)
    t1, t2 = _views(rng, 200, 64)
    small = [_prob(t1, t2, np.arange(100)), _prob(t1, t2, 100 + np.arange(100), n_dev=70)]
    nb = _lib.load().srb_infonce_workspace_bytes(2048, 64, 2)
    ws = torch.full((nb,), 0xFF, dtype=torch.uint8, device="cuda")
    for probs in (big, small, big):
        losses, grads = _run_nce(torch, probs, 64, tau, workspace=ws)
        _check_nce(orc, probs, losses, grads, 64, tau, True)


def test_nce_argument_checks(torch_cuda):
    torch = torch_cuda
    from selfrec_b200 import _lib
    from selfrec_b200._lib import SrbError
    rng = np.random.default_rng(15)
    v1, v2 = _views(rng, 64, 64)
    with pytest.raises(SrbError):
        _run_nce(torch, [_prob(v1, v2, np.arange(64))] * 5, 64, 0.2)
    nb = _lib.load().srb_infonce_workspace_bytes(64, 64, 1)
    with pytest.raises(SrbError):
        _run_nce(torch, [_prob(v1, v2, np.arange(64))], 64, 0.2, workspace=torch.empty(nb - 4, dtype=torch.uint8, device="cuda"))
    w1, w2 = _views(rng, 64, 48)
    with pytest.raises(SrbError):
        _run_nce(torch, [_prob(w1, w2, np.arange(64))], 48, 0.2)


# ------------------------------------------------------------------------------------------
# top-k, impl 2
# ------------------------------------------------------------------------------------------
def _csr_rows(lists, n_items):
    ptr = np.zeros(len(lists) + 1, np.int32)
    ptr[1:] = np.cumsum([len(x) for x in lists])
    idx = np.concatenate([np.sort(np.asarray(x, np.int64)) for x in lists] + [np.zeros(0, np.int64)]).astype(np.int32)
    return ptr, idx


def _topk(torch, ue, ie, users, rp, ri, k, impl=2):
    """(ids, scores, fallback count or None) of ops.score_topk."""
    from selfrec_b200 import ops
    stats = {}
    ids, sc = ops.score_topk(torch.from_numpy(ue).cuda(), torch.from_numpy(ie).cuda(), users, rp, ri, k, impl=impl, stats=stats)
    torch.cuda.synchronize()
    fb = int(stats["fallback_count"].item()) if "fallback_count" in stats else None
    return ids.cpu().numpy(), sc.cpu().numpy(), fb


def _assert_topk_exact(orc, ue, ie, users, rp, ri, k, ids, sc):
    """Scores bit for bit and ids equal to the oracle's; among exactly equal scores only the set of ids has to
    match (the reference orders those by an unstable sort, test_topk_tie_semantics_match_find_k_largest)."""
    oi, os_ = orc.score_topk(ue, ie, users, rp, ri, k)
    bad = set(np.nonzero((sc.view(np.uint32) != os_.view(np.uint32)).any(1))[0].tolist())
    for q in np.nonzero((ids != oi).any(1))[0]:
        if sorted(zip(sc[q].tolist(), ids[q].tolist())) != sorted(zip(os_[q].tolist(), oi[q].tolist())):
            bad.add(int(q))
    bad = sorted(bad)
    assert not bad, f"{len(bad)} of {len(users)} query rows differ from the oracle, first at rows {bad[:8]}"


def _tie_catalog(rng, n_items, n_ties):
    """0.1-scale Gaussian items plus n_ties copies of one TF32-exact vector b whose 13 low mantissa bits (the
    bits TF32 drops) are random: their approximate scores tie, their exact scores differ.  Returns the items,
    the tie positions and b."""
    ie = (rng.standard_normal((n_items, 64)) * 0.1).astype(np.float32)
    b = (rng.integers(1, 64, 64) * rng.choice([-1, 1], 64) / 64.0).astype(np.float32)  # 6-bit values: TF32-exact
    pos = np.sort(rng.choice(n_items, n_ties, replace=False))
    bits = (b.view(np.uint32) & np.uint32(~0x1FFF & 0xFFFFFFFF)) | rng.integers(0, 1 << 13, (n_ties, 64), dtype=np.uint32)
    ie[pos] = bits.view(np.float32)
    return ie, pos, b


def _users_for_ties(rng, n_users, tie_users, b):
    """Users of tie_users point along b (their top-k is among the tied items, more than the 48 candidate slots
    can hold); the others point away from b, so their lists are ordinary 0.1-scale Gaussian ones."""
    bh = b / np.linalg.norm(b)
    g = rng.standard_normal((n_users, 64)) * 0.1
    g -= np.outer(g @ bh, bh) + 0.5 * np.linalg.norm(g, axis=1, keepdims=True) * bh
    g[tie_users] = b + 0.01 * rng.standard_normal((len(tie_users), 64))
    return g.astype(np.float32)


@pytest.mark.parametrize("k", [20, 32])
def test_topk_near_ties_fall_back_into_their_rows(torch_cuda, orc, k):
    """Near-tied users must fail the certificate; the ordinary users in the same call must not all fail.
    The near-tied users sit at query rows at or past their count, so a fallback that wrote query row `slot`
    instead of fb_rows[slot] would leave them unwritten."""
    rng = np.random.default_rng(k)
    n_items, n_q, n_ties = 3000, 200, 100
    ie, _, b = _tie_catalog(rng, n_items, n_ties)
    users = rng.permutation(n_q).astype(np.int32)
    tie_rows = np.arange(140, 200, 2)
    ue = _users_for_ties(rng, n_q, users[tie_rows], b)
    rated = [rng.choice(n_items, int(rng.integers(0, 40)), replace=False) for _ in range(n_q)]
    rp, ri = _csr_rows(rated, n_items)
    ids, sc, fb = _topk(torch_cuda, ue, ie, users, rp, ri, k)
    assert len(tie_rows) <= fb < n_q, fb
    _assert_topk_exact(orc, ue, ie, users, rp, ri, k, ids, sc)


def test_topk_near_ties_beyond_fast_fallback_capacity(torch_cuda, orc):
    """More fallback users than the fast re-run holds (64 MB of score rows: 128 users at 131 072 items): the
    rest go through the exact kernel's query map."""
    rng = np.random.default_rng(3)
    n_items, n_q = 131072, 160
    ie, _, b = _tie_catalog(rng, n_items, 100)
    users = np.arange(n_q, dtype=np.int32)
    tie_rows = np.arange(10, 160)
    ue = _users_for_ties(rng, n_q, tie_rows, b)
    ids, sc, fb = _topk(torch_cuda, ue, ie, users, None, None, 20)
    assert 150 <= fb < n_q, fb
    _assert_topk_exact(orc, ue, ie, users, None, None, 20, ids, sc)


def test_topk_benign_fallback_rate(torch_cuda, orc):
    """0.1-scale Gaussians, 5000 items, k = 20: the certificate passes for at least 95 % of users."""
    rng = np.random.default_rng(16)
    n_users, n_items = 1000, 5000
    ue = (rng.standard_normal((n_users, 64)) * 0.1).astype(np.float32)
    ie = (rng.standard_normal((n_items, 64)) * 0.1).astype(np.float32)
    rated = sp.random(n_users, n_items, density=0.02, random_state=4, format="csr")
    rated.sort_indices()
    users = np.arange(n_users, dtype=np.int32)
    ids, sc, fb = _topk(torch_cuda, ue, ie, users, rated.indptr, rated.indices, 20)
    print(f"benign fallback count: {fb} of {n_users}")
    assert fb <= 0.05 * n_users, fb
    _assert_topk_exact(orc, ue, ie, users, rated.indptr, rated.indices, 20, ids, sc)


@pytest.mark.parametrize("k", [1, 20, 32])
def test_topk_bound_stress(torch_cuda, orc, k):
    """Item norms log-uniform over 1e-3 .. 1e3 (a large certificate margin E), an all-zero user, users with
    exactly k and k - 1 unrated items, and rated lists covering item 0, the last item and a whole tile."""
    rng = np.random.default_rng(17 + k)
    n_users, n_items = 300, 2000
    dirs = rng.standard_normal((n_items, 64))
    ie = (dirs / np.linalg.norm(dirs, axis=1, keepdims=True) * 10.0 ** rng.uniform(-3, 3, (n_items, 1))).astype(np.float32)
    ue = (rng.standard_normal((n_users, 64)) * 0.1).astype(np.float32)
    ue[3] = 0
    rated = [rng.choice(n_items, int(rng.integers(0, 50)), replace=False) for _ in range(n_users)]
    rated[5] = rng.permutation(n_items)[k:]              # exactly k unrated
    rated[6] = rng.permutation(n_items)[max(k - 1, 0):]  # k - 1 unrated
    rated[7] = np.concatenate([[0, n_items - 1], np.arange(128, 256)])
    rated[8] = np.arange(n_items - k)                    # the k unrated items are the last ones
    rp, ri = _csr_rows(rated, n_items)
    users = np.concatenate([[3, 5, 6, 7, 8], rng.permutation(n_users)]).astype(np.int32)
    ids, sc, fb = _topk(torch_cuda, ue, ie, users, rp, ri, k)
    _assert_topk_exact(orc, ue, ie, users, rp, ri, k, ids, sc)
    # alone in a call: the zero user (every score ties at 0, E = 0) and the user with k - 1 unrated items
    # cannot be certified; the user whose k unrated items are the last ones can
    for u, want in ((3, 1), (6, 1), (8, 0)):
        one = np.int32([u])
        ids, sc, fb = _topk(torch_cuda, ue, ie, one, rp, ri, k)
        assert fb == want, (u, fb)
        _assert_topk_exact(orc, ue, ie, one, rp, ri, k, ids, sc)


@pytest.mark.parametrize("k", [1, 32])
@pytest.mark.parametrize("n_q", [1, 127, 128, 129])
@pytest.mark.parametrize("n_items", [1023, 1024, 1025, 1151])
def test_topk_shape_edges(torch_cuda, orc, n_items, n_q, k):
    """Auto dispatch (impl 0) across n_items = 1024, n_q around the 128-user CTA, n_items around a 128-item tile."""
    rng = np.random.default_rng(n_items * 1000 + n_q * 10 + k)
    n_users = 300
    ue = (rng.standard_normal((n_users, 64)) * 0.1).astype(np.float32)
    ie = (rng.standard_normal((n_items, 64)) * 0.1).astype(np.float32)
    rated = [rng.choice(n_items, int(rng.integers(0, 30)), replace=False) for _ in range(n_users)]
    rp, ri = _csr_rows(rated, n_items)
    users = rng.choice(n_users, n_q, replace=False).astype(np.int32)
    ids, sc, fb = _topk(torch_cuda, ue, ie, users, rp, ri, k, impl=0)
    assert (fb is not None) == (n_items >= 1024)  # impl 0 takes the tensor cores from 1024 items on
    _assert_topk_exact(orc, ue, ie, users, rp, ri, k, ids, sc)
