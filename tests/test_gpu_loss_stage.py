"""The training step's loss stage at the C ABI and in the step, against float64, each gradient term at its own scale.

  * srb_bpr_l2_fwd_bwd (fused BPR + L2 gather, loss and gradient) at every width in the step's layout: one [U + I, d]
    table with the item rows at U + i, b = capacity with a device count b_dev below it, and index tails past b_dev
    holding the ids of NaN rows.  The BPR planes and the L2 planes are compared with float64 separately (g_l2 given),
    and merged (g_l2 = NULL) at a reg where the L2 part is 5-50 % of every row.  Bars come from fp32 rounding scales.
  * srb_scatter_add_segments / srb_scatter_add_rows (the seed scatters) with 1, 3 and 8 segments, device counts,
    row offsets, scales and rows listed up to 2048 times.
  * srb_l2_reg_fwd / srb_l2_reg_bwd through ops.l2_reg_loss with 1 to 4 terms.
  * Every model's training step on test_gpu_step_edges' hub fixture at a reg where the L2 gradient is a visible share
    of the rows it reaches: at that fixture's REG = 1e-3 the L2 gradient of a full batch sits below the first-moment
    bar KAPPA, and only the one-triple batch shows it.
Every output and scratch buffer the tests hand to a kernel starts as NaN."""
import ctypes as C

import numpy as np
import pytest

import loss_stage_ref as R
import test_gpu_step_edges as edges

pytestmark = pytest.mark.gpu

WIDTHS = [16, 32, 64, 128, 256]
EPS32 = float(np.finfo(np.float32).eps)
F32 = np.float32


@pytest.fixture(scope="module")
def torch_cuda(built_lib):
    import torch
    assert torch.cuda.is_available()
    from selfrec_b200 import _lib
    _lib.require_device()
    return torch


def _nan(torch, shape):
    return torch.full(shape, float("nan"), device="cuda")


def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


# ---------------------------------------------------------------------------------------------------------------------
# srb_bpr_l2_fwd_bwd
# ---------------------------------------------------------------------------------------------------------------------
def run_bpr(torch, emb, u, i, j, n_users, b_dev=None, l2_emb=None, g_l2=False, reg=0.0, l2_terms=3, l2_div=1.0,
            emb_scale=1.0, grad_scale=1.0):
    """srb_bpr_l2_fwd_bwd through a raw descriptor on the numpy table emb ([U + I, d]) and index lists of length b (the
    capacity).  l2_emb: a separate table (None: emb); g_l2: pass a g_l2 buffer.  Returns (losses [2], g_emb [3, b, d],
    g_l2 [3, b, d] or None) as numpy."""
    from selfrec_b200 import _lib, ops
    lib = _lib.load()
    b, d = len(u), emb.shape[1]
    E = _dev(torch, emb.astype(F32))
    L2 = None if l2_emb is None else _dev(torch, l2_emb.astype(F32))
    idx = [_dev(torch, np.asarray(x, dtype=np.int32) if b else np.zeros(1, np.int32)) for x in (u, i, j)]
    bd = None if b_dev is None else _dev(torch, np.array([b_dev], dtype=np.int32))
    losses, scratch = _nan(torch, (2,)), _nan(torch, (8,))
    g = _nan(torch, (3, max(b, 1), d))
    gl = _nan(torch, (3, max(b, 1), d)) if g_l2 else None
    desc = _lib.BprDesc()
    desc.emb, desc.l2_emb, desc.n_users, desc.d = ops._p(E), ops._p(L2), n_users, d
    desc.u_idx, desc.i_idx, desc.j_idx, desc.b_dev, desc.b = ops._p(idx[0]), ops._p(idx[1]), ops._p(idx[2]), ops._p(bd), b
    desc.emb_scale, desc.reg, desc.l2_terms, desc.l2_div, desc.grad_scale = emb_scale, reg, l2_terms, l2_div, grad_scale
    desc.losses, desc.g_emb, desc.g_l2, desc.scratch = ops._p(losses), ops._p(g), ops._p(gl), ops._p(scratch)
    _lib.check(lib.srb_bpr_l2_fwd_bwd(C.byref(desc), ops._stream()), "srb_bpr_l2_fwd_bwd")
    torch.cuda.synchronize()
    return losses.cpu().numpy(), g.cpu().numpy()[:, :b], (gl.cpu().numpy()[:, :b] if g_l2 else None)


def bpr_case(rng, d, U=40, I=60, cap=300):
    """A [U + I, d] table and cap triples in the step's layout.  Users [0, U - 8) and items [0, I - 8) are live; the
    last 8 of each are NaN rows that only the index tails (past any b_dev) name.  User 0 is in a third of the triples,
    item 0 is the positive of a fifth, item 1 a positive in some triples and the negative in others, and every 10th
    triple has i == j.  Item rows are half the users' scale, so the L2 norms of the three terms differ."""
    sig = 0.3 * d ** -0.25  # |x| = |<u, p - n>| ~ 0.13: sigmoid(x) near 1/2, c near -1 / (2 b) in every triple
    emb = np.concatenate([rng.standard_normal((U, d)) * sig, rng.standard_normal((I, d)) * (sig / 2)]).astype(F32)
    emb[U - 8:U] = np.nan
    emb[U + I - 8:] = np.nan
    u = np.where(rng.random(cap) < 1 / 3, 0, rng.integers(1, U - 8, cap))
    i = np.where(rng.random(cap) < 0.2, 0, rng.integers(1, I - 8, cap))
    j = rng.integers(2, I - 8, cap)
    j[::7] = 1
    i[3::7] = 1
    j[5::10] = i[5::10]
    return emb, u.astype(np.int32), i.astype(np.int32), j.astype(np.int32)


def with_tails(rng, u, i, j, b, U, I):
    """The lists with entries [b, cap) replaced by ids of the NaN rows (what a batch buffer holds past its count)."""
    u, i, j = u.copy(), i.copy(), j.copy()
    n = len(u) - b
    u[b:] = rng.integers(U - 8, U, n)
    i[b:] = rng.integers(I - 8, I, n)
    j[b:] = rng.integers(I - 8, I, n)
    return u, i, j


def bpr_reference(emb, l2_tab, u, i, j, U, reg, l2_terms, l2_div, emb_scale, grad_scale):
    """float64: (bpr loss, l2 loss, BPR planes [3, b, d], L2 planes [3, b, d], BPR bars [3, b, d], L2 bars [3, b, d],
    BPR loss bar, L2 loss bar).  l2_tab None: the L2 term reads the scaled rows of emb."""
    b, d = len(u), emb.shape[1]
    s = float(F32(emb_scale))
    rows = [emb[u].astype(np.float64) * s, emb[U + i].astype(np.float64) * s, emb[U + j].astype(np.float64) * s]
    loss, c, dcdx, sg, x = R.bpr_ref(*rows)
    ru, rp, rn = rows
    gs = float(F32(grad_scale))
    bpr = np.stack([c[:, None] * (rp - rn), c[:, None] * ru, -c[:, None] * ru]) * gs
    # fp32 dot products: <= 4 Q + 5 roundings deep (fma chain per lane, q loop, 5 shuffle levels), one more for pos - neg
    dx = 8 * EPS32 * (np.abs(ru) * (np.abs(rp) + np.abs(rn))).sum(1)
    # c = -(s (1 - s)) / (1e-5 + s) / b: relative error of s (expf, add, divide) ~3 eps turns into an absolute error of
    # ~3 eps s / b through the cancellation in 1 - s; a few more roundings of c itself
    dc = np.abs(dcdx) * dx + 4 * EPS32 * sg / max(b, 1) + 6 * EPS32 * np.abs(c)
    k = (dc + 3 * EPS32 * np.abs(c))[:, None] * abs(gs)
    bpr_bar = np.stack([k * (np.abs(rp) + np.abs(rn)), k * np.abs(ru), k * np.abs(ru)])
    lt = -np.log(10e-6 + sg)
    Q = (d + 127) // 128
    depth = 4 * Q + 5 + 8 + (b + 7) // 8  # sum of squares: lane fma chain, shuffles, 8 warps, one atomic per block
    bpr_loss_bar = float(np.mean(np.abs(c) * max(b, 1) * dx)) + (depth + 8) * EPS32 * float(np.mean(np.abs(lt) + 1)) if b else 0.0
    l2rows = rows if l2_tab is None else [l2_tab[u].astype(np.float64), l2_tab[U + i].astype(np.float64), l2_tab[U + j].astype(np.float64)]
    l2_loss, gl = R.l2_ref(reg, l2rows[:l2_terms], l2_div)
    l2 = np.stack(gl + [np.zeros((b, d))] * (3 - l2_terms)) * gs
    rel = (depth / 4 + 6) * EPS32
    return loss, l2_loss, bpr, l2, bpr_bar, rel * np.abs(l2), bpr_loss_bar, rel * abs(l2_loss)


def _check_planes(where, got, ref, bar):
    err = np.abs(got.astype(np.float64) - ref)
    bad = err > bar
    assert not bad.any(), (where, int(bad.sum()), np.argwhere(bad)[:4].tolist(), float((err - bar).max()))


def _merged_reg(bpr, l2u, live):
    """reg at which the L2 planes (computed at reg = 1) are centred in the 5-50 % share band over the triples' rows."""
    a = np.abs(l2u[:, live]).max(2)
    r = np.abs(bpr[:, live]).max(2)
    ok = r > 0
    ratio = a[ok] / r[ok]
    lo, hi = R.SHARE_LO / (1 - R.SHARE_LO), R.SHARE_HI / (1 - R.SHARE_HI)
    return float(np.sqrt(lo * hi / (ratio.min() * ratio.max())))


CONFIGS = [
    # l2_terms, emb_scale, grad_scale, l2_div
    (3, 1.0, 1.0, 1.0),
    (2, 0.25, 2.0, 64.0),
]


@pytest.mark.parametrize("d", WIDTHS)
def test_bpr_l2_planes_vs_float64(torch_cuda, d):
    """Separate route (l2_emb, g_l2: LightGCN), the same table with g_l2 given, and the merged route (g_l2 = NULL) at
    b_dev = 1, 17 and cap, l2_terms 3 and 2, emb_scale / grad_scale / l2_div = 1 and not.  A separate l2_emb is read
    unscaled; with l2_emb == emb the L2 term regularises the gathered (scaled) rows.  Rows past b_dev stay NaN."""
    torch = torch_cuda
    rng = np.random.default_rng(1000 + d)
    U, I, cap = 40, 60, 300
    emb, u0, i0, j0 = bpr_case(rng, d, U, I, cap)
    l2_tab = (rng.standard_normal(emb.shape) * 0.2).astype(F32)
    l2_tab[U - 8:U] = np.nan
    l2_tab[U + I - 8:] = np.nan
    for l2_terms, es, gs, div in CONFIGS:
        for b in (1, 17, cap):
            u, i, j = with_tails(rng, u0, i0, j0, b, U, I)
            lu, li, lj = u[:b], i[:b], j[:b]
            tag = f"d={d} b_dev={b} terms={l2_terms} scale={es} gs={gs} div={div}"
            # separate table: BPR planes and L2 planes each against float64
            reg = 0.7
            ref = bpr_reference(emb, l2_tab, lu, li, lj, U, reg, l2_terms, div, es, gs)
            los, g, gl = run_bpr(torch, emb, u, i, j, U, b_dev=b, l2_emb=l2_tab, g_l2=True, reg=reg, l2_terms=l2_terms,
                                 l2_div=div, emb_scale=es, grad_scale=gs)
            _check_planes(tag + " separate bpr", g[:, :b], ref[2], ref[4])
            _check_planes(tag + " separate l2", gl[:, :b], ref[3], ref[5])
            assert np.isnan(g[:, b:]).all() and np.isnan(gl[:, b:]).all(), tag
            assert abs(los[0] - ref[0]) <= ref[6] and abs(los[1] - ref[1]) <= ref[7], (tag, los.tolist(), ref[:2])
            if l2_terms == 2:  # (0 times the row: a signed zero)
                assert (gl[2, :b] == 0).all(), (tag, "third L2 plane is not 0")
            # the same table with g_l2 given, and merged at a reg where L2 is 5-50 % of every row
            unit = bpr_reference(emb, None, lu, li, lj, U, 1.0, l2_terms, div, es, gs)
            live = np.nonzero(li != lj)[0]  # (i == j: the user row has no BPR part at all)
            reg = _merged_reg(unit[2][:l2_terms], unit[3][:l2_terms], live)
            ref = bpr_reference(emb, None, lu, li, lj, U, reg, l2_terms, div, es, gs)
            tot = ref[2] + ref[3]
            a = np.abs(ref[3][:, live]).max(2)
            share = a / (a + np.abs(ref[2][:, live]).max(2))
            if l2_terms == 2:
                share = share[:2]
            assert share.min() >= R.SHARE_LO and share.max() <= R.SHARE_HI, (tag, reg, share.min(), share.max())
            los_s, g_s, gl_s = run_bpr(torch, emb, u, i, j, U, b_dev=b, g_l2=True, reg=reg, l2_terms=l2_terms, l2_div=div,
                                       emb_scale=es, grad_scale=gs)
            _check_planes(tag + " same-table bpr", g_s[:, :b], ref[2], ref[4])
            _check_planes(tag + " same-table l2", gl_s[:, :b], ref[3], ref[5])
            los_m, g_m, _ = run_bpr(torch, emb, u, i, j, U, b_dev=b, reg=reg, l2_terms=l2_terms, l2_div=div, emb_scale=es,
                                    grad_scale=gs)
            _check_planes(tag + " merged", g_m[:, :b], tot, ref[4] + ref[5] + EPS32 * np.abs(tot))
            assert np.isnan(g_m[:, b:]).all(), tag
            assert abs(los_m[0] - ref[0]) <= ref[6] and abs(los_m[1] - ref[1]) <= ref[7], (tag, los_m.tolist(), ref[:2])
            if b <= 8:  # one block: the norms are summed in one fixed order, so merged = BPR plane + L2 plane in fp32
                assert np.array_equal(_bits(g_m[:, :b]), _bits(g_s[:, :b] + gl_s[:, :b])), tag
                assert np.array_equal(_bits(los_m), _bits(los_s)), tag


@pytest.mark.parametrize("d", WIDTHS)
def test_bpr_l2_empty_batch_and_zero_table(torch_cuda, d):
    """b_dev = 0: both losses exactly 0 and every gradient row untouched.  An all-zero L2 table: finite losses, an L2
    loss of 0 and a g_l2 of exactly 0 (the gradient of ||E||_F at the origin)."""
    torch = torch_cuda
    rng = np.random.default_rng(2000 + d)
    U, I, cap = 40, 60, 300
    emb, u, i, j = bpr_case(rng, d, U, I, cap)
    u, i, j = with_tails(rng, u, i, j, 0, U, I)
    for sep in (False, True):
        los, g, gl = run_bpr(torch, emb, u, i, j, U, b_dev=0, l2_emb=emb + 1 if sep else None, g_l2=sep, reg=0.5)
        assert los[0] == 0 and los[1] == 0, los.tolist()
        assert np.isnan(g).all() and (gl is None or np.isnan(gl).all())
    emb, u, i, j = bpr_case(rng, d, U, I, cap)
    u, i, j = with_tails(rng, u, i, j, 100, U, I)
    zero = np.zeros_like(emb)
    for terms in (2, 3):
        los, g, gl = run_bpr(torch, emb, u, i, j, U, b_dev=100, l2_emb=zero, g_l2=True, reg=0.5, l2_terms=terms)
        assert np.isfinite(los).all() and los[1] == 0, los.tolist()
        assert (_bits(gl[:, :100]) == 0).all() and np.isnan(gl[:, 100:]).all()
        assert np.isfinite(g[:, :100]).all()


SAT_X = [-100.0, -89.0, -30.0, -11.5, 0.0, 11.5, 30.0, 100.0]


@pytest.mark.parametrize("d", WIDTHS)
def test_bpr_saturation(torch_cuda, d):
    """One triple with x = <u, p> - <u, n> exact in fp32 (u = e_0, p_0 = x / 2, n_0 = -x / 2).  Below -88.7 expf(-x)
    overflows: sigmoid is 0, the loss exactly -logf(1e-5f) and the gradient 0.  Elsewhere loss and c = d loss / dx
    against float64 at the fp32 scale of sigmoid."""
    torch = torch_cuda
    rng = np.random.default_rng(3000 + d)
    floor = None
    for x in SAT_X:
        emb = np.zeros((3, d), dtype=F32)
        emb[0, 0] = 1
        emb[1] = rng.standard_normal(d) * 0.1
        emb[2] = rng.standard_normal(d) * 0.1
        emb[1, 0], emb[2, 0] = x / 2, -x / 2
        z = np.zeros(1, np.int32)
        los, g, _ = run_bpr(torch, emb, z, z, z + 1, 1, reg=0.0)
        loss, c, _, sg, xr = R.bpr_ref(emb[0:1], emb[1:2], emb[2:3])
        assert xr[0] == x
        if x < -88.7:
            want = F32(-np.log(np.float64(F32(1e-5))))
            assert abs(float(los[0]) - float(want)) <= np.spacing(want), (x, los[0], want)
            floor = los[0] if floor is None else floor
            assert los[0] == floor, (x, los[0], floor)  # one value for every overflowing x
            assert (g == 0).all(), x
            continue
        assert abs(los[0] - loss) <= 4 * EPS32 * (abs(loss) + 1), (x, los[0], loss)
        # c from the kernel's u-plane: g_u = c (p - n), and p_0 - n_0 = x exactly
        got_c = g[0, 0, 0] / x if x != 0 else g[1, 0, 0]  # (x = 0: g_p = c u, u_0 = 1)
        assert abs(got_c - c[0]) <= 4 * EPS32 * float(sg[0]) + 8 * EPS32 * abs(c[0]), (x, got_c, c[0])


# ---------------------------------------------------------------------------------------------------------------------
# seed scatters
# ---------------------------------------------------------------------------------------------------------------------
SCALES = [1.0, -0.5, 1.0 / 3.0]  # 1 / (L + 1) at L = 2
REPEATS = [2048, 256, 17, 3, 2]


def scatter_case(rng, d, nseg, R_rows=3000):
    """nseg segments into one [R_rows, d] table.  Live destination rows lie in [50, 2000), rows [2000, R_rows) are named
    only past a segment's device count (with NaN source rows).  Segment q lists a row of its own 2048 / 256 / 17 / 3 / 2
    times (segment 0) or one row 64 times, 40 rows of its own once, and 10 rows every segment lists once.  The last of
    3 or more segments has n = 0, the one before it *n_dev = 0."""
    dst = rng.standard_normal((R_rows, d)).astype(F32)
    pool = rng.permutation(np.arange(50, 2000))
    shared, pool = pool[:10], pool[10:]
    segs = []
    for q in range(nseg):
        off = 7 + 3 * q
        scale = SCALES[q % len(SCALES)]
        if q == 0:
            mine, pool = pool[:len(REPEATS)], pool[len(REPEATS):]
            rep = np.concatenate([np.full(k, r) for k, r in zip(REPEATS, mine)])
        else:
            rep, pool = np.full(64, pool[0]), pool[1:]
        once, pool = pool[:40], pool[40:]
        live = rng.permutation(np.concatenate([rep, once, shared]))
        n_dev = len(live)
        if nseg >= 3 and q == nseg - 2:
            n_dev = 0
        tail = rng.integers(2000, R_rows, 37)
        rows = np.concatenate([live, tail]) if n_dev else np.concatenate([tail, tail])
        n = len(rows)
        if nseg >= 3 and q == nseg - 1:
            rows, n = rows[:1], 0
        src = rng.standard_normal((max(n, 1), d)).astype(F32)
        src[n_dev:] = np.nan
        segs.append(dict(src=src, dst_rows=rows, rows=(rows - off).astype(np.int32), n=n, n_dev=n_dev, off=off, scale=scale))
    return dst, segs


def scatter_reference(dst, segs):
    """float64 sum, per row: contribution count, sum of |terms| (dst included), and which rows a scale-1 segment alone
    touches once."""
    ref, mag = dst.astype(np.float64), np.abs(dst.astype(np.float64))
    cnt, cnt1 = np.zeros(len(dst), np.int64), np.zeros(len(dst), np.int64)
    for s in segs:
        k = min(s["n"], s["n_dev"])
        rows = s["dst_rows"][:k]
        term = s["src"][:k].astype(np.float64) * float(F32(s["scale"]))
        np.add.at(ref, rows, term)
        np.add.at(mag, rows, np.abs(term))
        np.add.at(cnt, rows, 1)
        if s["scale"] == 1.0:
            np.add.at(cnt1, rows, 1)
    return ref, mag, cnt, (cnt == 1) & (cnt1 == 1)


def _seg_array(torch, segs, keep):
    from selfrec_b200 import _lib, ops
    arr = (_lib.ScatterSeg * len(segs))()
    for q, s in enumerate(segs):
        t = dict(src=_dev(torch, s["src"]), rows=_dev(torch, s["rows"]), n_dev=_dev(torch, np.array([s["n_dev"]], np.int32)))
        keep.append(t)
        arr[q].src, arr[q].rows, arr[q].n_dev = ops._p(t["src"]), ops._p(t["rows"]), ops._p(t["n_dev"])
        arr[q].n, arr[q].row_off, arr[q].scale = s["n"], s["off"], s["scale"]
    return arr


@pytest.mark.parametrize("nseg", [1, 3, 8])
@pytest.mark.parametrize("d", WIDTHS)
def test_scatter_segments_vs_float64(torch_cuda, d, nseg):
    """One launch of nseg segments (one segment: srb_scatter_add_rows).  Untouched rows bit-identical (the NaN sources
    past every device count included), a row with one scale-1 contribution exactly dst + src in fp32, every other row
    the float64 sum within count * eps32 * sum |terms| (the atomics' order varies)."""
    torch = torch_cuda
    from selfrec_b200 import _lib, ops
    lib = _lib.load()
    rng = np.random.default_rng(4000 + 10 * d + nseg)
    dst, segs = scatter_case(rng, d, nseg)
    D = _dev(torch, dst)
    keep = []
    if nseg == 1:
        s = segs[0]
        src, rows, nd = _dev(torch, s["src"]), _dev(torch, s["rows"]), _dev(torch, np.array([s["n_dev"]], np.int32))
        rc = lib.srb_scatter_add_rows(ops._p(D), d, ops._p(src), ops._p(rows), s["n"], ops._p(nd), s["off"], s["scale"], ops._stream())
    else:
        rc = lib.srb_scatter_add_segments(ops._p(D), d, nseg, _seg_array(torch, segs, keep), ops._stream())
    _lib.check(rc, "scatter")
    torch.cuda.synchronize()
    got = D.cpu().numpy()
    ref, mag, cnt, single = scatter_reference(dst, segs)
    assert cnt.max() >= 2048 and single.any()
    untouched = cnt == 0
    assert np.array_equal(_bits(got[untouched]), _bits(dst[untouched])), "an untouched row changed"
    want1 = np.zeros_like(dst)
    for s in segs:  # the single scale-1 contributions in fp32
        k = min(s["n"], s["n_dev"])
        if s["scale"] == 1.0:
            for r, row in enumerate(s["dst_rows"][:k]):
                if single[row]:
                    want1[row] = dst[row] + s["src"][r]
    assert np.array_equal(_bits(got[single]), _bits(want1[single])), "dst + src differs in fp32"
    rep = cnt >= 1
    err = np.abs(got[rep].astype(np.float64) - ref[rep])
    bar = cnt[rep, None] * EPS32 * mag[rep]
    assert (err <= bar).all(), (int((err > bar).sum()), float((err - bar).max()))


def test_scatter_refusals_leave_dst_alone(torch_cuda):
    """9 segments, d = 48, a negative n and a null src are refused before anything runs: dst is unchanged."""
    torch = torch_cuda
    from selfrec_b200 import _lib, ops
    lib = _lib.load()
    rng = np.random.default_rng(5000)
    dst, segs = scatter_case(rng, 64, 8)
    segs.append(dict(segs[0]))
    D = _dev(torch, dst)
    keep = []
    arr = _seg_array(torch, segs, keep)
    st = ops._stream()
    assert lib.srb_scatter_add_segments(ops._p(D), 64, 9, arr, st) != 0
    arr8 = _seg_array(torch, segs[:8], keep)
    D48 = _dev(torch, rng.standard_normal((3000, 48)).astype(F32))
    before48 = D48.cpu().numpy()
    assert lib.srb_scatter_add_segments(ops._p(D48), 48, 8, arr8, st) != 0
    assert "unsupported d" in _lib.last_error()
    arr8[1].n = -1
    assert lib.srb_scatter_add_segments(ops._p(D), 64, 8, arr8, st) != 0
    arr8[1].n, arr8[2].src = segs[1]["n"], None
    assert lib.srb_scatter_add_segments(ops._p(D), 64, 8, arr8, st) != 0
    s = keep[0]
    assert lib.srb_scatter_add_rows(ops._p(D), 64, None, ops._p(s["rows"]), 10, None, 0, 1.0, st) != 0
    assert lib.srb_scatter_add_rows(ops._p(D), 64, ops._p(s["src"]), ops._p(s["rows"]), -1, None, 0, 1.0, st) != 0
    assert lib.srb_scatter_add_rows(ops._p(D48), 48, ops._p(s["src"]), ops._p(s["rows"]), 10, None, 0, 1.0, st) != 0
    torch.cuda.synchronize()
    assert np.array_equal(_bits(D.cpu().numpy()), _bits(dst))
    assert np.array_equal(_bits(D48.cpu().numpy()), _bits(before48))


# ---------------------------------------------------------------------------------------------------------------------
# standalone l2_reg_loss
# ---------------------------------------------------------------------------------------------------------------------
L2_TERMS = [
    [(300, 64)],
    [(4100, 128), (7, 33)],
    [(7, 33), (300, 64), (5, 16)],
    [(256, 64), (4100, 128), (7, 33), (19, 16)],
]


@pytest.mark.parametrize("shapes", L2_TERMS, ids=[f"{len(s)}terms" for s in L2_TERMS])
def test_l2_reg_loss_vs_float64(torch_cuda, shapes):
    """ops.l2_reg_loss with 1 to 4 terms of different row counts: one of 4100 x 128 elements (more than the 1024 blocks
    x 256 threads of one grid-stride pass), [7, 33] (not a multiple of 4), and in the 4-term call an all-zero term
    (gradient exactly 0).  Upstream gradient 2.5.  Loss and every gradient against float64."""
    torch = torch_cuda
    from selfrec_b200 import ops
    rng = np.random.default_rng(6000 + len(shapes))
    xs = [(rng.standard_normal(s) * (0.5 + k)).astype(F32) for k, s in enumerate(shapes)]
    if len(xs) == 4:
        xs[2][:] = 0
    reg, go = 0.37, 2.5
    ts = [_dev(torch, x).requires_grad_(True) for x in xs]
    loss = ops.l2_reg_loss(reg, *ts)
    (loss * go).backward()
    torch.cuda.synchronize()
    ref, grads = R.l2_ref(reg, xs)
    # sum of squares: a thread's grid-stride fma chain, 5 shuffles, 8 warps, <= 1024 atomics; the norm halves that
    n_max = max(x.size for x in xs)
    bx = min((n_max + 255) // 256, 1024)
    depth = -(-n_max // (bx * 256)) + 5 + 8 + bx
    rel = (depth / 4 + 6) * EPS32
    assert abs(float(loss.detach()) - ref) <= rel * ref, (float(loss.detach()), ref)
    for k, (t, g) in enumerate(zip(ts, grads)):
        got = t.grad.cpu().numpy()
        if not xs[k].any():
            assert (_bits(got) == 0).all(), k
            continue
        err = np.abs(got - go * g)
        assert (err <= rel * np.abs(go * g) + 1e-30).all(), (k, float(err.max()))


# ---------------------------------------------------------------------------------------------------------------------
# the step, with the L2 gradient visible
# ---------------------------------------------------------------------------------------------------------------------
SHARE_FLOOR = 20 * edges.KAPPA  # every reached row: an L2 gradient off by 5 % moves it by >= KAPPA of its scale

STEP_CASES = [
    # name, d, L, layer_cl, SGL views
    ("MF", 32, 0, 0, None),
    ("LightGCN", 64, 1, 0, None),
    ("SimGCL", 64, 2, 0, None),
    ("XSimGCL", 64, 3, 1, None),
    ("SGL", 64, 1, 0, "edge"),
]


def chosen_reg(orc, h, name, d, L, lcl, views, E0):
    """The reg of test_gpu_step_edges' batch 1 at which the L2 gradient is visible (loss_stage_ref.choose_reg), with
    the precondition asserted."""
    words, (u, i, j) = h["batches"][0]
    vc = h["views"][views] if views else None
    g0, g1 = R.step_l2_parts(orc, h["A"], E0, h["data"].user_num, u, i, j, name, L, edges.B, lcl, vc, edges.TAU, edges.CL_RATE)
    reg = R.choose_reg(g0, g1)
    R.check_share(g0, g1, reg, SHARE_FLOOR)
    return reg


def _step_kw(name, lcl):
    if name in ("MF", "LightGCN"):
        return dict(l2_div=float(edges.B))
    if name == "SGL":
        return dict(tau=edges.TAU, cl_rate=edges.CL_RATE)
    return dict(eps=0.0, tau=edges.TAU, cl_rate=edges.CL_RATE, layer_cl=lcl)


@pytest.fixture(scope="module")
def hub(torch_cuda):
    return edges.make_hub_graph(edges.U, edges.I, edges.HUB_USERS, edges.HUB_ITEMS, 20261016)


@pytest.mark.parametrize("name,d,L,lcl,views", STEP_CASES, ids=[f"{c[0]}-d{c[1]}-L{c[2]}" for c in STEP_CASES])
def test_step_l2_visible_vs_oracle(torch_cuda, orc, hub, name, d, L, lcl, views):
    """TrainEngine from the poisoned workspace through test_gpu_step_edges' batch sequence and bars, at the reg where
    the L2 gradient is 5-50 % of most rows it reaches (SimGCL / XSimGCL at eps = 0)."""
    torch = torch_cuda
    from selfrec_b200.engine import TrainEngine
    U, I = edges.U, edges.I
    E0 = (np.random.default_rng(d + L).standard_normal((U + I, d)) * 0.1).astype(F32)
    reg = chosen_reg(orc, hub, name, d, L, lcl, views, E0)
    eng = TrainEngine(name, hub["data"], d, L, edges.B, edges.LR, reg, init_user=torch.from_numpy(E0[:U]),
                      init_item=torch.from_numpy(E0[U:]), **_step_kw(name, lcl))
    view_csr = hub["views"][views] if views else None
    if view_csr is not None:
        eng.set_view_graphs(*view_csr)
    edges._poison(torch, eng, hub["poison"], (eng.params, eng.m, eng.v, eng.step_dev, eng.losses), (eng.params,))

    def read_state():
        return tuple(t.cpu().numpy().copy() for t in (eng.params, eng.m, eng.v, eng.losses))

    edges._run_sequence(torch, orc, hub, name, d, L, lcl, view_csr, eng.step, read_state, None, f"{name} reg={reg:g}",
                        eps=0.0, reg=reg)


@pytest.mark.parametrize("name,d,L,views", [("LightGCN", 32, 1, None), ("SGL", 32, 1, "node")])
def test_sharded_step_world1_l2_visible_vs_oracle(torch_cuda, orc, hub, name, d, L, views):
    """ShardedEngine at world 1, same sequence, at the reg where the L2 gradient is visible."""
    torch = torch_cuda
    from selfrec_b200.sharded import ShardedEngine
    U, I = edges.U, edges.I
    E0 = (np.random.default_rng(d + L).standard_normal((U + I, d)) * 0.1).astype(F32)
    reg = chosen_reg(orc, hub, name, d, L, 0, views, E0)
    eng = ShardedEngine(name, hub["data"], d, L, edges.B, edges.LR, reg, init_user=torch.from_numpy(E0[:U]),
                        init_item=torch.from_numpy(E0[U:]), device=torch.device("cuda", torch.cuda.current_device()),
                        **_step_kw(name, 0))
    assert eng.world == 1
    view_csr = hub["views"][views] if views else None
    if view_csr is not None:
        eng.set_view_graphs(*view_csr)
    state = (eng.user_emb, eng.item_emb, eng.mu, eng.vu, eng.mi, eng.vi, eng.step_dev, eng.losses)
    edges._poison(torch, eng, hub["poison"], state, (eng.user_emb, eng.item_emb))

    def read_state():
        cat = lambda a, b: torch.cat([a, b]).cpu().numpy()
        return cat(eng.user_emb, eng.item_emb), cat(eng.mu, eng.mi), cat(eng.vu, eng.vi), eng.losses.cpu().numpy()

    edges._run_sequence(torch, orc, hub, name, d, L, 0, view_csr, lambda w: eng.step(words=w), read_state, None,
                        f"sharded {name} reg={reg:g}", reg=reg)


@pytest.mark.parametrize("world,d,L", [(2, 64, 3), (3, 32, 1)])
def test_loopback_lightgcn_l2_visible_vs_oracle(built_lib, orc, world, d, L):
    """LightGCN on loopback worlds 2 and 3 (its g_l2 seeds reach the cyclic-owned user rows through their own scatter
    segment), at the reg where the L2 gradient is visible, in a subprocess as test_gpu_shard_loopback runs it."""
    import shard_loopback as lb
    import test_gpu_shard_loopback as tl
    h = lb.loopback_graph()
    U, I = h["data"].user_num, h["data"].item_num
    E0 = (np.random.default_rng(d + L + world).standard_normal((U + I, d)) * 0.1).astype(F32)  # run_oracle_case's
    reg = chosen_reg(orc, h, "LightGCN", d, L, 0, None, E0)
    tl._run(dict(kind="oracle", name="LightGCN", world=world, d=d, L=L, lcl=0, views=None, reg=reg))
