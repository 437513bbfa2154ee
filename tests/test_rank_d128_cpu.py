"""numpy model of the tensor-core ranking path (csrc/score_topk_tc.cu) at embedding size 128, no GPU.

At d = 128 a 128-item tile is 16 chained wgmma k-steps instead of 8.  The operand term of the error bound (TF32
truncation, 2^-9 * ||u|| * max||i||) does not depend on d; the accumulation term does: every k-step adds its block of 8
products into the fp32 accumulator, so it doubles with the chain, E(d) = 2^-9 + (d / 64) * 2^-16 + 2^-18.  The model
below runs the k-step chain with the block sums and the running sum truncated toward zero at every step (the
pessimistic choice: errors of one sign add up), and shows that
* every approximate score lies within E(128) * ||u|| * max||i|| of the exact one, and
* the certificate max(thr_A, thr_B) + E < exact k-th score implies that the 2 x 24 candidates contain the exact top-k,
  also when scores are packed too tightly for TF32 (then users fail the certificate instead).
"""
import numpy as np
import pytest

from test_numerics_model_cpu import tf32_trunc


def E_const(d):
    """TcShape<D>::E, in the kernel's fp32 arithmetic."""
    return np.float32(np.float32(1.0 / 512.0) + np.float32(d // 64) * np.float32(1.0 / 65536.0)) + np.float32(1.0 / 262144.0)


def _to_f32_rz(x):
    """float64 -> float32 rounded toward zero."""
    f = x.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(x)
    f[over] = np.nextafter(f[over], np.float32(0))
    return f


def tc_scores(U, I):
    """Scores as the k-step chain forms them: 8 TF32 products per k-step, block sum and accumulation each
    truncated to fp32."""
    Ut, It = tf32_trunc(U).astype(np.float64), tf32_trunc(I).astype(np.float64)
    acc = np.zeros((U.shape[0], I.shape[0]), np.float32)
    for k0 in range(0, U.shape[1], 8):
        blk = _to_f32_rz(Ut[:, k0:k0 + 8] @ It[:, k0:k0 + 8].T)
        acc = _to_f32_rz(acc.astype(np.float64) + blk.astype(np.float64))
    return acc


def test_kernel_constant_is_unchanged_at_64():
    assert E_const(64) == np.float32(1.0 / 512.0 + 1.0 / 65536.0 + 1.0 / 262144.0)
    assert E_const(128) == np.float32(1.0 / 512.0 + 1.0 / 32768.0 + 1.0 / 262144.0)


@pytest.mark.parametrize("spread", [1.0, 1e-2, 1e-4])
def test_sixteen_k_steps_stay_inside_the_bound(spread):
    rng = np.random.default_rng(3 + int(1 / spread))
    base = rng.standard_normal(128)
    U = (base + spread * rng.standard_normal((64, 128))).astype(np.float32)
    I = (base + spread * rng.standard_normal((700, 128))).astype(np.float32)
    approx = tc_scores(U, I)
    exact = U.astype(np.float64) @ I.astype(np.float64).T
    scale = np.linalg.norm(U.astype(np.float64), axis=1)[:, None] * np.linalg.norm(I.astype(np.float64), axis=1).max()
    assert (np.abs(approx - exact) <= float(E_const(128)) * scale).all()


def _certified_topk(U, I, k, rated):
    """tc_score_kernel + tc_rescore_kernel on one block of users at d = 128; (ids or None per user), exact scores."""
    n_u, n_i = U.shape[0], I.shape[0]
    approx = tc_scores(U, I)
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
                thr = max(thr, float(approx[q, order[23]]))
        cand = np.array(cand, dtype=np.int64)
        if len(cand) < k:
            out.append(None)
            continue
        top = cand[np.argsort(-exact[q, cand], kind="stable")][:k]
        E = float(E_const(128)) * np.linalg.norm(U[q].astype(np.float64)) * bmax
        out.append(top if thr + E < exact[q, top[-1]] else None)
    return out, exact


@pytest.mark.parametrize("spread", [1.0, 1e-2, 1e-4])
def test_d128_certificate_is_sound(spread):
    rng = np.random.default_rng(11 + int(1 / spread))
    n_u, n_i, k = 48, 1500, 20
    base = rng.standard_normal(128).astype(np.float32)
    U = (base + spread * rng.standard_normal((n_u, 128))).astype(np.float32)
    I = (base + spread * rng.standard_normal((n_i, 128))).astype(np.float32)
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
    if spread == 1e-4:
        assert certified < n_u  # scores within the TF32 resolution: the fallback takes over
