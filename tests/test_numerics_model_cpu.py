"""CPU models of the two numerical arguments the tensor-core kernels rest on (numpy only, no GPU):

* 3xTF32 (csrc/infonce_tc.cuh): x = hi + lo with hi = rna_tf32(x), lo truncated to TF32; hi*hi + hi*lo + lo*hi
  reproduces an fp32 dot product to ~2^-21 relative, a single TF32 pass only to ~2^-11.
* the exactness certificate of the tensor-core ranking path (csrc/score_topk_tc.cu): with TF32-truncated operands
  every approximate score is within E = (2^-9 + 2^-16 + 2^-18) * ||u|| * max||i|| of the exact one, so if the best
  non-candidate bound max(thr_A, thr_B) + E is below the exact k-th score, the true top-k lies inside the
  2 x 24 candidates -- whatever the data; and the pruning rule of tc_rescore_kernel (drop candidates whose approximate
  score is below a_K - 2E) never removes a member of the exact top-K.
"""
import numpy as np
import pytest
from philox_model import philox4x32_10 as _philox4x32_10


def tf32_trunc(x):
    b = np.asarray(x, dtype=np.float32).view(np.uint32) & np.uint32(0xFFFFE000)
    return b.view(np.float32)


def tf32_rna(x):
    """cvt.rna.tf32.f32: round to nearest, ties away from zero, 10 explicit mantissa bits."""
    b = np.asarray(x, dtype=np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def test_3xtf32_split_error_model():
    rng = np.random.default_rng(0)
    a = rng.standard_normal((256, 64)).astype(np.float32)
    b = rng.standard_normal((256, 64)).astype(np.float32)
    exact = a.astype(np.float64) @ b.astype(np.float64).T
    scale = np.linalg.norm(a, axis=1)[:, None] * np.linalg.norm(b, axis=1)[None, :]
    one = tf32_trunc(a).astype(np.float64) @ tf32_trunc(b).astype(np.float64).T
    ah, bh = tf32_rna(a), tf32_rna(b)
    al, bl = tf32_trunc(a - ah), tf32_trunc(b - bh)  # the tensor core truncates the low parts
    f = lambda x: x.astype(np.float64)
    three = f(ah) @ f(bh).T + f(ah) @ f(bl).T + f(al) @ f(bh).T
    e1 = np.abs(one - exact).max() / scale.max()
    e3 = np.abs(three - exact).max() / scale.max()
    assert e3 < 2.0 ** -20 and e1 > 50 * e3  # the split buys ~3 decimal digits
    assert np.abs(one - exact).max() <= (2.0 ** -9) * scale.max()


def _certified_topk(U, I, k, rated):
    """numpy model of tc_score_kernel + tc_rescore_kernel for one block of users; returns (ids or None per user)."""
    n_u, n_i = U.shape[0], I.shape[0]
    approx = (tf32_trunc(U).astype(np.float64) @ tf32_trunc(I).astype(np.float64).T).astype(np.float32)
    exact = U.astype(np.float64) @ I.astype(np.float64).T
    bmax = np.linalg.norm(I.astype(np.float64), axis=1).max()
    col_half = (np.arange(n_i) // 64) % 2  # 128-item tiles, two 64-column halves
    out = []
    for q in range(n_u):
        ok = np.ones(n_i, bool)
        ok[rated[q]] = False
        cand, thr = [], -np.inf
        for h in (0, 1):
            cols = np.flatnonzero(ok & (col_half == h))
            order = cols[np.argsort(-approx[q, cols], kind="stable")]
            cand += list(order[:24])
            if len(order) > 24:
                thr = max(thr, float(approx[q, order[23]]))  # everything not kept in this half is <= its 24th best
        cand = np.array(cand, dtype=np.int64)
        if len(cand) < k:
            out.append(None)
            continue
        top = cand[np.argsort(-exact[q, cand], kind="stable")][:k]
        kth = exact[q, top[-1]]
        E = (2.0 ** -9 + 2.0 ** -16 + 2.0 ** -18) * np.linalg.norm(U[q].astype(np.float64)) * bmax
        out.append(top if thr + E < kth else None)  # None = handed to the exact fallback
    return out, exact


@pytest.mark.parametrize("spread", [1.0, 1e-2, 1e-4])
def test_ranking_certificate_is_sound(spread):
    """Whenever the certificate passes, the candidates contain the exact top-k -- also when scores are packed
    so tightly that TF32 cannot tell them apart (then users fail the certificate instead of returning wrong ids)."""
    rng = np.random.default_rng(int(1 / spread))
    n_u, n_i, d, k = 48, 1500, 64, 20
    base = rng.standard_normal(d).astype(np.float32)
    U = (base + spread * rng.standard_normal((n_u, d))).astype(np.float32)
    I = (base + spread * rng.standard_normal((n_i, d))).astype(np.float32)
    rated = [rng.choice(n_i, size=rng.integers(0, 40), replace=False) for _ in range(n_u)]
    got, exact = _certified_topk(U, I, k, rated)
    certified = 0
    for q, ids in enumerate(got):
        if ids is None:
            continue
        certified += 1
        ok = np.ones(n_i, bool)
        ok[rated[q]] = False
        cols = np.flatnonzero(ok)
        truth = cols[np.argsort(-exact[q, cols], kind="stable")][:k]
        assert set(ids.tolist()) == set(truth.tolist()), (spread, q)
    if spread == 1.0:
        assert certified == n_u  # well-separated scores: nobody needs the fallback


@pytest.mark.parametrize("spread", [1.0, 1e-2, 1e-4])
def test_rescore_pruning_never_drops_a_topk_member(spread):
    """tc_rescore_kernel prunes before the exact pass: with a_K the K-th largest APPROXIMATE score of a user's candidates,
    every candidate whose approximate score is below a_K - 2E is dropped (E bounds |approx - exact|).  numpy model of
    that rule on TF32-truncated scores: the exact top-K of the candidate set always survives, tight scores included
    (then nothing is pruned), and on separated scores roughly half of the 48 candidates go."""
    rng = np.random.default_rng(7 + int(1 / spread))
    n_u, n_i, d, k = 64, 3000, 64, 20
    base = rng.standard_normal(d).astype(np.float32)
    U = (base + spread * rng.standard_normal((n_u, d))).astype(np.float32)
    I = (base + spread * rng.standard_normal((n_i, d))).astype(np.float32)
    approx = (tf32_trunc(U).astype(np.float64) @ tf32_trunc(I).astype(np.float64).T).astype(np.float32)
    exact = U.astype(np.float64) @ I.astype(np.float64).T
    bmax = np.linalg.norm(I.astype(np.float64), axis=1).max()
    col_half = (np.arange(n_i) // 64) % 2
    kept_total = cand_total = 0
    for q in range(n_u):
        cand = []
        for h in (0, 1):
            cols = np.flatnonzero(col_half == h)
            cand += list(cols[np.argsort(-approx[q, cols], kind="stable")][:24])
        cand = np.array(cand)
        E = np.float32((2.0 ** -9 + 2.0 ** -16 + 2.0 ** -18) * np.linalg.norm(U[q].astype(np.float64)) * bmax)
        assert np.abs(approx[q, cand] - exact[q, cand]).max() <= E  # the premise of the rule
        a_sorted = np.sort(approx[q, cand])[::-1]
        cut = a_sorted[k - 1] - np.float32(2.0) * E                  # the kernel's fp32 arithmetic
        keep = cand[approx[q, cand] >= cut]
        truth = cand[np.argsort(-exact[q, cand], kind="stable")][:k]
        assert set(truth.tolist()) <= set(keep.tolist()), (spread, q)
        kept_total += len(keep)
        cand_total += len(cand)
    if spread == 1.0:
        assert kept_total < 0.75 * cand_total  # separated scores: the rule removes a good part of the exact work


@pytest.mark.parametrize("tau", [0.5, 0.2, 0.05, 0.025])
def test_fixed_shift_logsumexp_model(tau):
    """InfoNCE pass A (csrc/infonce_tc.cuh) shifts every logit by the bound 1/tau of a cosine logit instead of a
    running maximum, which makes column-split partial sums plainly additive.  fp32 model: the result equals the
    max-shifted log-sum-exp to fp32 rounding for every temperature the tensor-core path accepts (tau >= 0.025)."""
    rng = np.random.default_rng(7)
    n, d = 512, 64
    v1 = rng.standard_normal((n, d))
    v2 = v1 + 0.3 * rng.standard_normal((n, d))
    v1 /= np.linalg.norm(v1, axis=1, keepdims=True)
    v2 /= np.linalg.norm(v2, axis=1, keepdims=True)
    S = (v1 @ v2.T / tau)
    ref = np.log(np.exp(S - S.max(1, keepdims=True)).sum(1)) + S.max(1)
    S32 = S.astype(np.float32)
    shift = np.float32(1.0 / tau)
    parts = [np.exp(S32[:, c::4] - shift, dtype=np.float32).sum(1, dtype=np.float32) for c in range(4)]  # 4 column splits
    l = parts[0] + parts[1] + parts[2] + parts[3]
    got = shift + np.log(l, dtype=np.float32)
    assert np.isfinite(got).all() and (l > 0).all()
    assert np.abs(got - ref).max() <= 4e-7 / tau + 1e-6


def test_philox_counter_layout_keeps_view_and_step_streams_apart():
    """Perf-mode noise of the SpMM epilogue (csrc/spmm.cu): counter = (row, column block | view << 16, layer tag, step),
    key = seed.  Every (view, step) pair must be its own stream (the reference draws fresh noise on every perturbed
    forward, SimGCL.py:87-88).  The round-1 layout put view ^ step into ONE counter word, which made (view 1, step s)
    equal (view 0, step s ^ 1): the model shows that collision and that the current layout has none."""
    rows = np.arange(64, dtype=np.uint32)
    colblk, layer_tag, key = np.uint32(3), np.uint32(0x10), (0x5EED, 0x1234)

    def current(view, step):
        z = np.zeros_like(rows)
        return _philox4x32_10((rows, z + (colblk | np.uint32(view << 16)), z + layer_tag, z + np.uint32(step)), key)

    def round1(view, step):  # counter word 3 = view ^ step
        z = np.zeros_like(rows)
        return _philox4x32_10((rows, z + colblk, z + layer_tag, z + np.uint32(view ^ step)), key)

    streams = {(v, s): current(v, s) for v in (0, 1) for s in range(6)}
    keys = list(streams)
    for a in range(len(keys)):
        for b in range(a + 1, len(keys)):
            assert not np.array_equal(streams[keys[a]], streams[keys[b]]), (keys[a], keys[b])
    assert np.array_equal(round1(1, 2), round1(0, 3))  # what the advisor found
    # known-answer vector of Philox4x32-10 (Random123 kat_vectors: counter 0, key 0)
    z = np.zeros(1, dtype=np.uint32)
    assert _philox4x32_10((z, z, z, z), (0, 0))[0].tolist() == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
