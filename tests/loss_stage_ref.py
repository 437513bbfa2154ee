"""Float64 references of the training step's loss stage, and the L2 share of the step's gradient.

The loss stage (srb_bpr_l2_fwd_bwd) computes, for b triples (u, i, j) gathered from the rows e_u, e_p, e_n:
  bpr = mean_t -log(10e-6 + sigmoid(<e_u, e_p> - <e_u, e_n>))                 util/loss_torch.py:6-10
  l2  = reg * sum_terms ||E_term||_F / b / l2_div    (not squared)            util/loss_torch.py:18-22
with the terms (u, p) or (u, p, n).  The references below are plain numpy in float64 and return the per-triple
quantities the fp32 rounding bars of tests/test_gpu_loss_stage.py are built from.

At the step level the L2 gradient is a small addend of the rows' gradients: at the hub fixture's REG = 1e-3 it is below
the first-moment bar KAPPA for LightGCN, so a step that dropped it would pass.  step_l2_parts() splits the float64
step gradient into its reg-free part and its part per unit reg (the gradient is affine in reg), choose_reg() picks a reg
at which the L2 part is a visible share of the rows it reaches, and check_share() asserts that it is."""
import numpy as np

SHARE_LO, SHARE_HI = 0.05, 0.5


def bpr_ref(u, p, n):
    """(loss, c, dc/dx, sigmoid(x), x) of mean_t -log(10e-6 + sigmoid(x_t)), x_t = <u_t, p_t> - <u_t, n_t>, in float64.
    c_t is d loss / d x_t: the gradients are c (p - n), c u and -c u."""
    u, p, n = (np.asarray(a, dtype=np.float64) for a in (u, p, n))
    b = len(u)
    x = (u * p).sum(1) - (u * n).sum(1)
    with np.errstate(over="ignore"):
        sig = 1.0 / (1.0 + np.exp(-x))
    k = 10e-6
    loss = float(np.mean(-np.log(k + sig))) if b else 0.0
    c = -(sig * (1 - sig)) / (k + sig) / max(b, 1)
    # d/ds of s (1 - s) / (k + s), times ds/dx = s (1 - s)
    dfds = ((1 - 2 * sig) * (k + sig) - sig * (1 - sig)) / (k + sig) ** 2
    dcdx = -dfds * sig * (1 - sig) / max(b, 1)
    return loss, c, dcdx, sig, x


def l2_ref(reg, terms, div=1.0):
    """(loss, grads) of reg * sum_t ||E_t||_F / rows_t / div in float64; the gradient of an all-zero term is 0."""
    loss, grads = 0.0, []
    for e in terms:
        e = np.asarray(e, dtype=np.float64)
        nrm = np.sqrt((e ** 2).sum())
        loss += nrm / e.shape[0]
        grads.append(reg * e / (nrm * e.shape[0] * div) if nrm > 0 else np.zeros_like(e))
    return reg * loss / div, grads


def step_l2_parts(orc, A, E0, U, u, i, j, name, L, batch_size, lcl=0, view_csr=None, tau=0.2, cl_rate=0.3):
    """The float64 step gradient of batch (u, i, j) as g0 + reg * g1: (g0, g1).  SimGCL / XSimGCL at eps = 0."""
    kw = dict(n_layers=L, batch_size=batch_size, eps=0.0, tau=tau, cl_rate=cl_rate, layer_cl=lcl, view_csr=view_csr,
              noise=np.zeros((2, max(L, 1), 1, 1)) if name in ("SimGCL", "XSimGCL") else None)
    g0 = orc.train_step(name, A, E0, U, u, i, j, reg=0.0, **kw)["grad"]
    g1 = orc.train_step(name, A, E0, U, u, i, j, reg=1.0, **kw)["grad"] - g0
    return g0, g1


def l2_share(g0, g1, reg):
    """Per row the L2 gradient reaches (g1 != 0): x / (1 + x), x = max |reg g1| / max |g0|, the L2 part's share of the
    row's gradient scale.  Returns (rows, shares)."""
    rows = np.nonzero((g1 != 0).any(1))[0]
    a, r = np.abs(reg * g1[rows]).max(1), np.abs(g0[rows]).max(1)
    return rows, a / (a + r)


def choose_reg(g0, g1):
    """The reg (two significant digits) that centres the 5th to 95th percentile of the reached rows' L2-to-rest ratios
    geometrically in the share band [SHARE_LO, SHARE_HI]."""
    rows = np.nonzero((g1 != 0).any(1))[0]
    r = np.abs(g1[rows]).max(1) / np.abs(g0[rows]).max(1)
    q5, q95 = np.quantile(r, [0.05, 0.95])
    lo, hi = SHARE_LO / (1 - SHARE_LO), SHARE_HI / (1 - SHARE_HI)
    return float(f"{np.sqrt(lo * hi / (q5 * q95)):.2g}")


def check_share(g0, g1, reg, floor):
    """The step-level precondition: 90 % of the rows the L2 gradient reaches have their L2 share in [SHARE_LO,
    SHARE_HI], and none less than `floor`, so that an L2 gradient off by a fraction f of itself moves every reached row
    by at least floor * f of its scale.  Returns the shares' 0th, 5th, 95th and 100th percentiles."""
    _, s = l2_share(g0, g1, reg)
    q = np.quantile(s, [0.0, 0.05, 0.95, 1.0])
    assert q[1] >= SHARE_LO and q[2] <= SHARE_HI and q[0] >= floor, (reg, q.tolist())
    return q
