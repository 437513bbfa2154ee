"""CPU checks of tests/loss_stage_ref.py: its float64 references against the oracle pinned to the golden fixtures, and
the step-level L2 share on test_gpu_step_edges' hub fixture that tests/test_gpu_loss_stage.py relies on."""
import numpy as np
import pytest

import loss_stage_ref as R


@pytest.mark.parametrize("seed", range(4))
def test_references_match_oracle(orc, seed):
    rng = np.random.default_rng(seed)
    b, d = int(rng.integers(1, 40)), int(rng.choice([16, 64, 256]))
    u, p, n = (rng.standard_normal((b, d)) * 0.3 for _ in range(3))
    loss, c, dcdx, _, x = R.bpr_ref(u, p, n)
    ol, du, dp, dn = orc.bpr_loss(u, p, n)
    assert np.isclose(loss, ol, rtol=1e-13)
    for got, want in ((c[:, None] * (p - n), du), (c[:, None] * u, dp), (-c[:, None] * u, dn)):
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-300)
    # dc/dx against a central difference of c(x)
    h = 1e-6
    cp = R.bpr_ref(np.ones((b, 1)), (x + h)[:, None], np.zeros((b, 1)))[1]
    cm = R.bpr_ref(np.ones((b, 1)), (x - h)[:, None], np.zeros((b, 1)))[1]
    np.testing.assert_allclose(dcdx, (cp - cm) / (2 * h), rtol=1e-5, atol=1e-12)
    terms = [rng.standard_normal((int(rng.integers(1, 30)), d)) for _ in range(int(rng.integers(1, 5)))]
    reg = float(rng.random())
    loss, grads = R.l2_ref(reg, terms)
    ol, og = orc.l2_reg_loss(reg, *terms)
    assert np.isclose(loss, ol, rtol=1e-13)
    for g, o in zip(grads, og):
        np.testing.assert_allclose(g, o, rtol=1e-13)
    loss, grads = R.l2_ref(reg, [terms[0], np.zeros((3, d))], 8.0)
    assert np.isclose(loss, orc.l2_reg_loss(reg, terms[0])[0] / 8.0, rtol=1e-13) and not grads[1].any()


@pytest.fixture(scope="module")
def hub():
    import test_gpu_step_edges as edges
    return edges.make_hub_graph(edges.U, edges.I, edges.HUB_USERS, edges.HUB_ITEMS, 20261016)


def _parts(orc, h, name, d, L, lcl, views, seed):
    import test_gpu_step_edges as edges
    U, I = h["data"].user_num, h["data"].item_num
    E0 = (np.random.default_rng(seed).standard_normal((U + I, d)) * 0.1).astype(np.float32)
    _, (u, i, j) = h["batches"][0]
    vc = h["views"][views] if views else None
    return R.step_l2_parts(orc, h["A"], E0, U, u, i, j, name, L, edges.B, lcl, vc, edges.TAU, edges.CL_RATE)


def test_step_l2_share_at_chosen_regs(orc, hub):
    """The regs tests/test_gpu_loss_stage.py's step cases pick (same fixture, E0 seeds and batch) pass the share
    precondition: 90 % of the reached rows in 5-50 %, none below SHARE_FLOOR."""
    import test_gpu_loss_stage as T
    cases = [(c[0], c[1], c[2], c[3], c[4], c[1] + c[2]) for c in T.STEP_CASES]
    cases += [("LightGCN", 32, 1, 0, None, 33), ("SGL", 32, 1, 0, "node", 33)]
    for name, d, L, lcl, views, seed in cases:
        g0, g1 = _parts(orc, hub, name, d, L, lcl, views, seed)
        reg = R.choose_reg(g0, g1)
        R.check_share(g0, g1, reg, T.SHARE_FLOOR)
    import shard_loopback as lb
    h = lb.loopback_graph()
    for world, d, L in (2, 64, 3), (3, 32, 1):  # run_oracle_case's E0 seed
        g0, g1 = _parts(orc, h, "LightGCN", d, L, 0, None, d + L + world)
        R.check_share(g0, g1, R.choose_reg(g0, g1), T.SHARE_FLOOR)


@pytest.mark.parametrize("name,d,L", [("LightGCN", 32, 1), ("LightGCN", 128, 3), ("LightGCN", 64, 1), ("MF", 32, 0)])
def test_step_l2_below_kappa_at_fixture_reg(orc, hub, name, d, L):
    """Why the step cases above exist: at test_gpu_step_edges.REG the L2 gradient of LightGCN (and MF) on the full
    batch 1 is below the first-moment bar KAPPA on every row it reaches, so that batch cannot see it.  (Only the
    one-triple batch, where the L2 term is divided by b = 1, shows a missing L2 gradient to test_gpu_step_edges.)"""
    import test_gpu_step_edges as edges
    g0, g1 = _parts(orc, hub, name, d, L, 0, None, d + L)
    _, share = R.l2_share(g0, g1, edges.REG)
    assert share.max() < edges.KAPPA, share.max()
