"""The tensor-core ranker (csrc/score_topk_tc.cu) at every width it ranks, without a GPU: a numpy model of its
error bound and certificate, the bound's constant in the library, the dispatch predicates and the workspace layout.

A 128-item tile is d / 8 chained wgmma k-steps: 2 at d = 16, 4 at d = 32, 32 at d = 256.  The operand term of the
bound (TF32 truncation, 2^-9 * ||u|| * max||i||) does not depend on d; the accumulation term does, 2^-19 per k-step:
E(d) = 2^-9 + (d / 8) * 2^-19 + 2^-18 (the last term covers the slot tags and the final roundings).  The model runs
the chain with the block sums and the running sum truncated toward zero at every step (the pessimistic choice:
errors of one sign add up), and shows that
* every approximate score lies within E(d) * ||u|| * max||i|| of the exact one, and
* the certificate max(thr_A, thr_B) + E < exact k-th score implies that the 2 x 24 candidates hold the exact top k.
"""
import numpy as np
import pytest

from test_numerics_model_cpu import tf32_trunc

WIDTHS = (16, 32, 64, 128, 256)


def E(d):
    """TcShape<D>::E in the kernel's fp32 arithmetic."""
    return np.float32(np.float32(np.float32(1.0 / 512.0) + np.float32(d // 8) * np.float32(1.0 / 524288.0)) + np.float32(1.0 / 262144.0))


def _to_f32_rz(x):
    """float64 -> float32 rounded toward zero."""
    f = x.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(x)
    f[over] = np.nextafter(f[over], np.float32(0))
    return f


def tc_scores(U, I):
    """Scores as the k-step chain forms them: 8 TF32 products per k-step, block sum and accumulation each truncated
    to fp32."""
    Ut, It = tf32_trunc(U).astype(np.float64), tf32_trunc(I).astype(np.float64)
    acc = np.zeros((U.shape[0], I.shape[0]), np.float32)
    for k0 in range(0, U.shape[1], 8):
        blk = _to_f32_rz(Ut[:, k0:k0 + 8] @ It[:, k0:k0 + 8].T)
        acc = _to_f32_rz(acc.astype(np.float64) + blk.astype(np.float64))
    return acc


def test_bound_constant_matches_the_library(built_lib):
    """The library's E(d) is the formula's float at every width, and today's values at d = 64 and 128."""
    for d in WIDTHS:
        assert np.float32(built_lib.srb_topk_tc_error_bound(d)) == E(d), d
    assert E(64) == np.float32(1.0 / 512.0 + 1.0 / 65536.0 + 1.0 / 262144.0)
    assert E(128) == np.float32(1.0 / 512.0 + 1.0 / 32768.0 + 1.0 / 262144.0)
    assert [E(d) - np.float32(1.0 / 512.0 + 1.0 / 262144.0) for d in WIDTHS] == pytest.approx([2.0 ** -s for s in (18, 17, 16, 15, 14)])
    for d in (0, 8, 48, 96, 512):
        assert built_lib.srb_topk_tc_error_bound(d) == -1.0


@pytest.mark.parametrize("spread", [1.0, 1e-2, 1e-4])
@pytest.mark.parametrize("d", [16, 32, 256])
def test_k_step_chain_stays_inside_the_bound(d, spread):
    rng = np.random.default_rng(d + int(1 / spread))
    base = rng.standard_normal(d)
    U = (base + spread * rng.standard_normal((64, d))).astype(np.float32)
    I = (base + spread * rng.standard_normal((700, d))).astype(np.float32)
    approx = tc_scores(U, I)
    exact = U.astype(np.float64) @ I.astype(np.float64).T
    scale = np.linalg.norm(U.astype(np.float64), axis=1)[:, None] * np.linalg.norm(I.astype(np.float64), axis=1).max()
    assert (np.abs(approx - exact) <= float(E(d)) * scale).all()


def _certified_topk(U, I, k, rated, d):
    """tc_score_kernel + tc_rescore_kernel on one block of users: (ids or None per user), exact scores."""
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
        e = float(E(d)) * np.linalg.norm(U[q].astype(np.float64)) * bmax
        out.append(top if thr + e < exact[q, top[-1]] else None)
    return out, exact


@pytest.mark.parametrize("spread", [1.0, 1e-2, 1e-4])
@pytest.mark.parametrize("d", [16, 32, 256])
def test_certificate_is_sound(d, spread):
    rng = np.random.default_rng(11 * d + int(1 / spread))
    n_u, n_i, k = 48, 1500, 20
    base = rng.standard_normal(d).astype(np.float32)
    U = (base + spread * rng.standard_normal((n_u, d))).astype(np.float32)
    I = (base + spread * rng.standard_normal((n_i, d))).astype(np.float32)
    rated = [rng.choice(n_i, size=rng.integers(0, 40), replace=False) for _ in range(n_u)]
    got, exact = _certified_topk(U, I, k, rated, d)
    certified = 0
    for q, ids in enumerate(got):
        if ids is None:
            continue
        certified += 1
        ok = np.ones(n_i, bool)
        ok[rated[q]] = False
        cols = np.flatnonzero(ok)
        truth = cols[np.argsort(-exact[q, cols], kind="stable")][:k]
        assert set(ids.tolist()) == set(truth.tolist()), (d, spread, q)
    if spread == 1.0:
        assert certified == n_u  # well-separated scores: nobody needs the fallback
    if spread == 1e-4:
        assert certified < n_u  # scores within the TF32 resolution: the fallback takes over


def test_dispatch_predicates():
    """impl 2 ranks every width when asked for; auto takes it for lists of up to 32 at every width from 1024 items on,
    and for lists of 33..256 at d = 64 / 128 only; impl 1 never takes it."""
    from selfrec_b200 import ops
    for d in WIDTHS:
        for n in (1, 1023, 1024, 38048):
            assert ops._tc_route(d, n, 2)
            assert ops._tc_route(d, n, 0) == (n >= 1024)
            assert not ops._tc_route(d, n, 1)
            for k in (33, 100, 256):
                assert ops.long_list_route(d, n, k, impl=2)
                assert ops.long_list_route(d, n, k) == (d in (64, 128) and n >= 1024)
                assert not ops.long_list_route(d, n, k, impl=1)
            for k in (1, 32, 257):
                assert not ops.long_list_route(d, n, k, impl=2)
    for d in (8, 48, 512):
        assert not ops._tc_route(d, 38048, 0) and not ops._tc_route(d, 38048, 2)


def _align(x):
    return (x + 255) // 256 * 256


def _cap(k):
    return (2 * k + 256 + 31) // 32 * 32


def test_workspace_arithmetic_at_every_width(built_lib):
    """The workspace differs between widths by the gathered [n_q_pad, d] user table only, the long-list buffers do
    not depend on d, and the fallback counter sits at one offset for every width and list length."""
    lib = built_lib
    for n_q, n_items in ((1, 1024), (129, 1151), (31668, 38048)):
        n_q_pad = (n_q + 255) // 256 * 256 + 256
        off = lib.srb_topk_fallback_count_offset(n_q, n_items)
        for k in (1, 20, 32, 33, 100, 256):
            w64 = lib.srb_topk_workspace_bytes(n_q, n_items, 64, k)
            for d in WIDTHS:
                w = lib.srb_topk_workspace_bytes(n_q, n_items, d, k)
                assert w - w64 == n_q_pad * (d - 64) * 4, (n_q, n_items, d, k)
                assert 0 <= off < w - _align(n_q_pad * d * 4) - 2 * _align(n_q * 2 * (_cap(k) if k > 32 else 0) * 4)
                if k > 32:
                    assert w - lib.srb_topk_workspace_bytes(n_q, n_items, d, 20) == 2 * _align(n_q * 2 * _cap(k) * 4)
