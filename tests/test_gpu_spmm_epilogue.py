"""The SpMM's epilogue and the encoder's batch-row last layer at the C ABI, at every supported width, against exact twins.

A training step's forward pass ends in srb_encoder_forward with last_rows: the last layer runs on the batch rows only,
from a device-classified row list, and rebuilds the layer mean from the earlier layers' buffers (SpmmArgs.sum_add).
Its backward pass ends in the SpMM's fused Adam epilogue.  Each of these is compared here with a twin built from
separate calls whose arithmetic is the same operation by operation, so the comparison is bit for bit:
  * fused Adam (Y = NULL) against the same product into Y followed by srb_adam_step, and both against
    torch.optim.Adam on CUDA;
  * the dense addend at scale 1 against a torch fp32 add, at other scales against the correctly rounded float64 value;
  * a device-classified list against the same rows in other slot and chunk-slot orders;
  * the encoder's listed-row mean against per-layer products and the fp32 sum in the documented order
    ((E0 + y1) + y2) + ... + yL, times 1 / (L + ego).
Tolerances remain where nothing exact exists: listed products against the float64 oracle (_check_product), the noise
epilogue against a float64 model that starts from the kernel's own plain product, and one encoder case per width
against oracle.encoder_forward.  Every output and work buffer starts as NaN, so a result that reads one shows up."""
import ctypes as C

import numpy as np
import pytest

import test_gpu_d256 as w256
import test_gpu_step_edges as edges
from philox_model import noise_offset

pytestmark = pytest.mark.gpu

WIDTHS = [16, 32, 64, 128, 256]
LR = 1e-2
EPS = edges.EPS  # (the noise of the oracle anchor is made unambiguous at this eps)
SEED = 0x0123456789ABCDEF
EPS32 = float(np.finfo(np.float32).eps)
ADAM = dict(beta1=0.9, beta2=0.999, adam_eps=1e-8)


@pytest.fixture(scope="module")
def torch_cuda(built_lib):
    import torch
    assert torch.cuda.is_available()
    from selfrec_b200 import _lib
    _lib.require_device()
    return torch


@pytest.fixture(scope="module")
def graphs(torch_cuda):
    """test_gpu_d256's every-class graph (split rows of 3 chunks, CTA, warp, short and empty rows; 900 x 9000) with
    its split rows in chunk lists and in column-blocked lists (blocks of 4096 columns) at every width, and
    test_gpu_step_edges' hub graph (split rows of 2 and 3 chunks, CTA, warp and lane-group rows) in chunk lists."""
    from selfrec_b200 import ops
    every = w256._every_class_graph(np.random.default_rng(900))
    h = edges.make_hub_graph(edges.U, edges.I, edges.HUB_USERS, edges.HUB_ITEMS, 20261016)
    chunked, blocked, hub = ops.SparseAdj(every).cuda(), ops.SparseAdj(every).cuda(), ops.SparseAdj(h["A"]).cuda()
    saved = ops.HUB_BLOCK_BYTES
    try:
        for d in WIDTHS:
            assert not chunked.hub_struct(d).seg and not hub.hub_struct(d).seg
            ops.HUB_BLOCK_BYTES = 2048 * 4 * d
            assert blocked.hub_struct(d).seg
            ops.HUB_BLOCK_BYTES = saved
    finally:
        ops.HUB_BLOCK_BYTES = saved
    assert chunked.n_huge == 2 and chunked.n_vlong == 3 and chunked.n_long == 2
    assert hub.n_huge == 4 and hub.n_vlong == 2 and hub.n_long == 4
    return dict(every=every, chunked=chunked, colblocked=blocked, hub_A=h["A"], hub=hub)


def _nan(torch, shape):
    return torch.full(shape, float("nan"), device="cuda")


def _rand(torch, rng, shape, scale=1.0):
    return w256._rand(torch, rng, shape, scale)


# ---------------------------------------------------------------------------------------------------------------------
# row lists
# ---------------------------------------------------------------------------------------------------------------------
def device_list(torch, rowptr, rows, d, rng, shuffle=False, slack=0, fill_short=False, spare=0):
    """A device-classified row list of `rows` (duplicates allowed) in the format list_batch_row writes
    (srb_spmm_desc.n_vlong_dev): row_order holds four segments of capacity cap = len(rows) + slack -- split rows
    (>= HUB_MIN_NNZ non-zeros, with their chunks in hub.work), CTA rows (>= 128), warp rows, lane-group rows --, counts =
    (rows per class, chunks), hub.first[slot] = first chunk slot of the split row in that slot, hub.work[w] = (row,
    chunk index), hub.n_work = the chunk capacity (chunks + slack).
    shuffle: slot order within each class and the order in which the split rows' chunk blocks are allocated are
    random, as device atomics leave them; fill_short: rows below LONG_ROW_NNZ go to the lane-group class, which the
    engine leaves empty; spare: an unlisted row id written into every unused entry, so a read past a count shows up."""
    from selfrec_b200 import _lib, ops
    rows = np.asarray(rows, dtype=np.int64)
    deg = np.diff(rowptr)[rows]
    cls = np.where(deg >= _lib.HUB_MIN_NNZ, 0, np.where(deg >= 128, 1, 2))
    if fill_short:
        cls[deg < ops.LONG_ROW_NNZ] = 3
    segs = [rows[cls == c] for c in range(4)]
    if shuffle:
        segs = [rng.permutation(s) for s in segs]
    cap = len(rows) + slack
    order = np.full(4 * cap, spare, dtype=np.int32)
    for c, s in enumerate(segs):
        order[c * cap:c * cap + len(s)] = s
    nch = (np.diff(rowptr)[segs[0]] + _lib.HUB_CHUNK - 1) // _lib.HUB_CHUNK
    n_chunks = int(nch.sum())
    hub_cap = n_chunks + slack
    first = np.zeros(cap, dtype=np.int32)
    work = np.zeros((max(hub_cap, 1), 2), dtype=np.int32)
    work[:, 0] = spare
    pos = 0
    for slot in (rng.permutation(len(segs[0])) if shuffle else range(len(segs[0]))):
        first[slot] = pos
        work[pos:pos + nch[slot], 0] = segs[0][slot]
        work[pos:pos + nch[slot], 1] = np.arange(nch[slot])
        pos += nch[slot]
    counts = np.array([len(s) for s in segs] + [n_chunks], dtype=np.int32)
    dev = lambda a: torch.from_numpy(a).cuda()
    lst = dict(kind="device", rows=rows, cap=cap, order=dev(order), counts=dev(counts), first=dev(first), work=dev(work),
               part=_nan(torch, (max(hub_cap, 1), d)), hub_cap=hub_cap, n_class=counts[:4])
    return lst


def static_list(torch, rows):
    """The listed rows as srb_encoder_forward hands a static last_rows list to the SpMM: a CTA per listed row."""
    rows = np.asarray(rows, dtype=np.int64)
    return dict(kind="static", rows=rows, cap=len(rows), order=torch.from_numpy(rows.astype(np.int32)).cuda())


def _hub_split(lst):
    from selfrec_b200 import _lib, ops
    h = _lib.HubSplit()
    h.n_rows, h.n_work = 0, lst["hub_cap"]
    h.first, h.work, h.part = ops._p(lst["first"]), ops._p(lst["work"]), ops._p(lst["part"])
    return h


def list_fields(lst):
    """srb_spmm_desc fields of a row list, as srb_encoder_forward fills them for its last layer."""
    from selfrec_b200 import _lib
    if lst["kind"] == "static":
        return dict(row_order=lst["order"], n_rows=lst["cap"], n_vlong_rows=lst["cap"], n_long_rows=0, hub=_lib.HubSplit())
    return dict(row_order=lst["order"], n_rows=lst["cap"], n_vlong_rows=0, n_long_rows=0, hub=_hub_split(lst),
                n_vlong_dev=lst["counts"])


def _class_fields(kind):
    """srb_spmm_desc overrides of a row-class layout: natural order, or the handle's own static classes."""
    from selfrec_b200 import _lib
    return dict(row_order=None, n_long_rows=0, n_vlong_rows=0, hub=_lib.HubSplit()) if kind == "natural" else {}


def _listed_every_rows(rng, n_rows, dup=False):
    """Rows 0..11 of the every-class graph (split, CTA, warp, short, empty) and 200 others, in random order."""
    rows = np.concatenate([np.arange(12), rng.choice(np.arange(12, n_rows), 200, replace=False)])
    if dup:
        rows = np.concatenate([rows, rows[rng.integers(0, len(rows), 40)], [0, 1]])
    return rng.permutation(rows)


# ---------------------------------------------------------------------------------------------------------------------
# 1. fused Adam
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", WIDTHS)
def test_fused_adam_equals_adam_after_product(torch_cuda, graphs, d):
    """One srb_spmm_csr with Y = NULL and the Adam epilogue gives the bits of the same product into Y followed by
    srb_adam_step, over five steps (srb_adam_prepare each step), in natural order, on the static classes with chunk
    lists and with column-blocked lists, and on a device-classified list; srb_spmm_epilogue_rows with Adam gives the bits
    of srb_adam_step on X.  Empty rows have g = 0: their moments still decay."""
    torch = torch_cuda
    from selfrec_b200 import ops
    A = graphs["every"]
    n_rows, n_cols = A.shape
    deg = np.diff(A.indptr)
    rng = np.random.default_rng(d)
    listed = _listed_every_rows(rng, n_rows)
    unlisted = np.setdiff1d(np.arange(n_rows), listed)
    kinds = [("natural", graphs["chunked"]), ("chunked", graphs["chunked"]), ("colblocked", graphs["colblocked"]),
             ("device", graphs["chunked"]), ("epilogue_rows", None)]
    for kind, adj in kinds:
        if kind == "epilogue_rows":
            import scipy.sparse as sp
            adj = ops.SparseAdj(sp.identity(n_rows, dtype=np.float32, format="csr")).cuda()
        fields = _class_fields(kind)
        if kind == "device":
            lst = device_list(torch, A.indptr, listed, d, rng, shuffle=True, slack=7, spare=int(unlisted[0]))
            fields = list_fields(lst)
        p0 = rng.standard_normal((n_rows, d)).astype(np.float32)
        m0 = (rng.standard_normal((n_rows, d)) * 0.1).astype(np.float32)
        v0 = (rng.random((n_rows, d)) * 0.01).astype(np.float32)
        fused = [torch.from_numpy(a.copy()).cuda() for a in (p0, m0, v0)]
        twin = [torch.from_numpy(a.copy()).cuda() for a in (p0, m0, v0)]
        step = torch.zeros(1, dtype=torch.int32, device="cuda")
        scal = torch.zeros(16, device="cuda")
        entry = "srb_spmm_epilogue_rows" if kind == "epilogue_rows" else "srb_spmm_csr"
        for k in range(1, 6):
            X = _rand(torch, rng, (adj.shape[1], d))
            ops.adam_prepare(step, scal, LR)
            v_before = fused[2].clone()
            ops._spmm_raw(adj, X, None, _entry=entry, adam_p=fused[0], adam_m=fused[1], adam_v=fused[2], adam_scalars=scal,
                          **ADAM, **fields)
            Y = _nan(torch, (n_rows, d))
            ops._spmm_raw(adj, X, Y, _entry=entry, **fields)
            ops.adam_step(twin[0], twin[1], twin[2], Y, scal)
            torch.cuda.synchronize()
            where = (kind, d, "step", k)
            rows = torch.from_numpy(listed).cuda() if kind == "device" else slice(None)
            for name, f, t in zip("pmv", fused, twin):
                same = (f[rows] == t[rows]).all(1)
                assert bool(same.all()), (where, name, "rows differ", int((~same).sum()))
            if kind == "device":  # unlisted rows: no Adam update at all
                un = torch.from_numpy(unlisted).cuda()
                for name, f, a0 in zip("pmv", fused, (p0, m0, v0)):
                    assert np.array_equal(f[un].cpu().numpy(), a0[unlisted]), (where, name, "unlisted row updated")
            # empty rows: g = 0, and the moments still decay (v exactly by beta2)
            empty = np.nonzero(deg == 0)[0] if kind != "epilogue_rows" else np.zeros(0, dtype=np.int64)
            if kind == "device":
                empty = np.intersect1d(empty, listed)
            if len(empty):
                e = torch.from_numpy(empty).cuda()
                assert torch.equal(fused[2][e], v_before[e] * np.float32(0.999)), where
        assert int(step.item()) == 5


def test_adam_kernels_round_like_torch_cuda_adam(torch_cuda):
    """srb_adam_step (vector body and scalar tail) and the SpMM's Adam epilogue give the bits of torch.optim.Adam on
    CUDA tensors -- its foreach kernels, the default there -- over five steps of gradients from 1e-6 to 1 in size."""
    torch = torch_cuda
    import scipy.sparse as sp
    from selfrec_b200 import ops
    rng = np.random.default_rng(7)
    n, d = 1000, 64
    eye = ops.SparseAdj(sp.identity(n, dtype=np.float32, format="csr")).cuda()
    p_tab = _rand(torch, rng, (n, d))
    p_flat = _rand(torch, rng, (10007,))  # (not a multiple of 4: the scalar tail)
    params = [torch.nn.Parameter(p_tab.clone()), torch.nn.Parameter(p_flat.clone())]
    opt = torch.optim.Adam(params, lr=LR, foreach=True)
    fused = [p_tab.clone(), torch.zeros_like(p_tab), torch.zeros_like(p_tab)]
    plain = [[p.clone(), torch.zeros_like(p), torch.zeros_like(p)] for p in (p_tab, p_flat)]
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    scal = torch.zeros(16, device="cuda")
    for k in range(1, 6):
        grads = [_rand(torch, rng, tuple(p.shape), 10.0 ** -int(rng.integers(0, 7))) for p in params]
        for p, g in zip(params, grads):
            p.grad = g.clone()
        opt.step()
        ops.adam_prepare(step, scal, LR)
        for (p, m, v), g in zip(plain, grads):
            ops.adam_step(p, m, v, g, scal)
        ops._spmm_raw(eye, grads[0], None, _entry="srb_spmm_epilogue_rows", adam_p=fused[0], adam_m=fused[1], adam_v=fused[2],
                      adam_scalars=scal, **ADAM)
        torch.cuda.synchronize()
        for q, p in enumerate(params):
            st = opt.state[p]
            ref = (p.detach(), st["exp_avg"], st["exp_avg_sq"])
            for name, mine, want in zip("pmv", plain[q], ref):
                assert torch.equal(mine, want), ("srb_adam_step", q, k, name, int((mine != want).sum()))
        for name, mine, want in zip("pmv", fused, (params[0].detach(), opt.state[params[0]]["exp_avg"], opt.state[params[0]]["exp_avg_sq"])):
            assert torch.equal(mine, want), ("epilogue", k, name, int((mine != want).sum()))


# ---------------------------------------------------------------------------------------------------------------------
# 2. the dense addend
# ---------------------------------------------------------------------------------------------------------------------
def _correctly_rounded(got, ref64):
    """got (fp32) is ref64 rounded to fp32: within half an fp32 ulp, plus ref64's own float64 rounding."""
    ulp = np.spacing(np.abs(ref64).astype(np.float32)).astype(np.float64)
    return np.abs(got.astype(np.float64) - ref64) <= 0.5 * ulp + 2.0 ** -52 * np.abs(ref64)


@pytest.mark.parametrize("d", WIDTHS)
def test_dense_addend_and_its_place_in_the_epilogue(torch_cuda, graphs, d):
    """Y += extra_scale * extra: at scale 1 the bits of the plain Y plus extra (one rounding, a torch fp32 add); at
    -0.5 and 3 the float64 value of the kernel's own plain Y plus the scaled addend, correctly rounded.  Then one launch
    with the addend, noise, the running sum and Adam: Y against a float64 model of addend-then-noise that starts from
    the plain Y (the noise's sign(y) taken from the same fp32 value), and the running sum and Adam against the bits of
    an fp32 sum and srb_adam_step on that Y -- the addend comes before all three."""
    torch = torch_cuda
    from selfrec_b200 import ops
    A = graphs["every"]
    adj = graphs["chunked"]
    n_rows, n_cols = A.shape
    rng = np.random.default_rng(d + 1)
    X = _rand(torch, rng, (n_cols, d))
    extra = _rand(torch, rng, (n_rows, d), 3.0)
    Y0 = _nan(torch, (n_rows, d))
    ops._spmm_raw(adj, X, Y0)
    Y1 = _nan(torch, (n_rows, d))
    ops._spmm_raw(adj, X, Y1, extra=extra, extra_scale=1.0)
    assert torch.equal(Y1, Y0 + extra), d
    y0, e = Y0.double().cpu().numpy(), extra.double().cpu().numpy()
    for s in (-0.5, 3.0):
        Ys = _nan(torch, (n_rows, d))
        ops._spmm_raw(adj, X, Ys, extra=extra, extra_scale=s)
        ok = _correctly_rounded(Ys.cpu().numpy(), y0 + s * e)
        assert ok.all(), (d, s, int((~ok).sum()))
    # all four epilogue stages in one launch
    s, sum_scale = -0.5, 0.5
    noise = torch.from_numpy(rng.random((n_rows, d), dtype=np.float32)).cuda()
    sum_in = _rand(torch, rng, (n_rows, d))
    p = _rand(torch, rng, (n_rows, d))
    m = _rand(torch, rng, (n_rows, d), 0.1)
    v = torch.from_numpy((rng.random((n_rows, d)) * 0.01).astype(np.float32)).cuda()
    tp, tm, tv = p.clone(), m.clone(), v.clone()
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    scal = torch.zeros(16, device="cuda")
    ops.adam_prepare(step, scal, LR)
    Y, S = _nan(torch, (n_rows, d)), _nan(torch, (n_rows, d))
    ops._spmm_raw(adj, X, Y, extra=extra, extra_scale=s, noise_mode=1, noise=noise, eps=EPS, sum_in=sum_in, sum_out=S,
                  sum_scale=sum_scale, adam_p=p, adam_m=m, adam_v=v, adam_scalars=scal, **ADAM)
    ops.adam_step(tp, tm, tv, Y, scal)
    torch.cuda.synchronize()
    # float64 model of addend, then noise, from the kernel's plain product
    y = (y0 + s * e).astype(np.float32).astype(np.float64)
    n64 = noise.double().cpu().numpy()
    pert = np.sign(y) * (n64 / np.maximum(np.sqrt((n64 ** 2).sum(1, keepdims=True)), 1e-12)) * np.float32(EPS)
    ref = y + pert
    # bound: a few roundings of y, and the fp32 sum of d squares behind the norm (relative (d + 8) eps32 of pert)
    tol = 8 * EPS32 * np.abs(y) + (d + 8) * EPS32 * np.abs(pert) + 1e-30
    err = np.abs(Y.double().cpu().numpy() - ref)
    assert (err <= tol).all(), (d, "Y", float((err / tol).max()))
    assert torch.equal(S, (Y + sum_in) * sum_scale), (d, "running sum")
    for name, f, t in zip("pmv", (p, m, v), (tp, tm, tv)):
        assert torch.equal(f, t), (d, name)


# ---------------------------------------------------------------------------------------------------------------------
# 3. device-classified lists in srb_spmm_csr
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", WIDTHS)
def test_device_classified_list_product(torch_cuda, orc, graphs, d):
    """A device-classified list over split, CTA, warp, short and empty rows (with and without the lane-group class,
    with and without duplicates, with capacity slack): the listed rows against the float64 oracle, the running sum of
    the listed rows equal to an fp32 add of Y, every other row of Y and sum_out still NaN, and the bits of every
    listed row unchanged when the slots and the split rows' chunk slots are permuted."""
    torch = torch_cuda
    from selfrec_b200 import ops
    A = graphs["every"]
    adj = graphs["chunked"]
    n_rows, n_cols = A.shape
    rng = np.random.default_rng(d + 2)
    X = _rand(torch, rng, (n_cols, d))
    Xh = X.cpu().numpy()
    sum_in = _rand(torch, rng, (n_rows, d))
    for fill_short in (False, True):
        for dup in (False, True):
            listed = _listed_every_rows(rng, n_rows, dup)
            uniq = np.unique(listed)
            unlisted = np.setdiff1d(np.arange(n_rows), uniq)
            where = (d, "fill_short", fill_short, "dup", dup)
            outs = []
            for shuffle, slack in ((False, 0), (True, 5), (True, 13)):
                lst = device_list(torch, A.indptr, listed, d, rng, shuffle=shuffle, slack=slack, fill_short=fill_short,
                                  spare=int(unlisted[0]))
                assert lst["n_class"][0] >= 2 and (lst["n_class"][3] > 0) == fill_short
                Y, S = _nan(torch, (n_rows, d)), _nan(torch, (n_rows, d))
                ops._spmm_raw(adj, X, Y, sum_in=sum_in, sum_out=S, **list_fields(lst))
                torch.cuda.synchronize()
                outs.append((Y.cpu().numpy(), S.cpu().numpy()))
            Yh, Sh = outs[0]
            As = A[uniq]
            w256._check_product(Yh[uniq], As, Xh, orc.spmm(As, Xh))
            empty = uniq[np.diff(A.indptr)[uniq] == 0]
            assert len(empty) >= 4 and (Yh[empty] == 0).all(), where
            assert np.array_equal(Sh[uniq], Yh[uniq] + sum_in.cpu().numpy()[uniq]), where
            assert np.isnan(Yh[unlisted]).all() and np.isnan(Sh[unlisted]).all(), where
            for k, (Yk, Sk) in enumerate(outs[1:], start=1):
                assert np.array_equal(Yk[uniq], Yh[uniq]) and np.array_equal(Sk[uniq], Sh[uniq]), (where, "permutation", k)
                assert np.isnan(Yk[unlisted]).all() and np.isnan(Sk[unlisted]).all(), (where, "permutation", k)


# ---------------------------------------------------------------------------------------------------------------------
# 4. the encoder's listed-row mean
# ---------------------------------------------------------------------------------------------------------------------
def _noise_spec(torch, mode, N, d, rng):
    if mode == 0:
        return dict(mode=0)
    if mode == 1:
        return dict(mode=1, t=torch.from_numpy(rng.random((4, N, d), dtype=np.float32)).cuda())
    return dict(mode=2, seed=SEED, off=noise_offset(1, 0), step=torch.tensor([3], dtype=torch.int32, device="cuda"))


def _layer_noise(nz, k):
    """srb_spmm_desc noise fields of encoder layer k (0-based), as srb_encoder_forward sets them."""
    if nz["mode"] == 1:
        return dict(noise_mode=1, noise=nz["t"][k], eps=EPS)
    if nz["mode"] == 2:
        return dict(noise_mode=2, philox_seed=nz["seed"], philox_offset=nz["off"] + k, philox_step_dev=nz["step"], eps=EPS)
    return {}


def _encoder_desc(adj, d, E0, L, ego, lcl, nz, bufs, lst=None, x1=None):
    from selfrec_b200 import _lib, ops
    p = ops._p
    e = _lib.EncoderDesc()
    e.rowptr, e.colidx, e.vals, e.row_order = p(adj.rowptr), p(adj.colidx), p(adj.vals), p(adj.row_order)
    e.n_long_rows, e.n_vlong_rows = adj.n_long, adj.n_vlong
    e.hub = adj.hub_struct(d)
    e.n, e.d, e.n_layers, e.include_ego, e.layer_cl = E0.shape[0], d, L, int(ego), lcl
    e.noise_mode, e.eps = nz["mode"], EPS
    if nz["mode"] == 1:
        e.noise = p(nz["t"])
    elif nz["mode"] == 2:
        e.philox_seed, e.philox_offset, e.philox_step_dev = nz["seed"], nz["off"], p(nz["step"])
    e.E0, e.final_out, e.cl_out, e.work0, e.work1, e.x1 = p(E0), p(bufs["final"]), p(bufs.get("cl")), p(bufs["w0"]), p(bufs["w1"]), p(x1)
    if lst is not None:
        e.last_rows, e.n_last_rows, e.last_rows_out = p(lst["order"]), lst["cap"], p(bufs["out"])
        if lst["kind"] == "device":
            e.last_rows_nv_dev, e.last_rows_hub = p(lst["counts"]), _hub_split(lst)
    return e


def _run_encoder(torch, adj, d, E0, L, ego, lcl, nz, lst, x1=None):
    from selfrec_b200 import _lib, ops
    lib = _lib.require_device()
    shape = tuple(E0.shape)
    bufs = {k: _nan(torch, shape) for k in ("final", "cl", "w0", "w1", "out")}
    e = _encoder_desc(adj, d, E0, L, ego, lcl, nz, bufs, lst, x1)
    _lib.check(lib.srb_encoder_forward(C.byref(e), ops._stream()), "srb_encoder_forward")
    return bufs


def _twin(torch, adj, d, E0, L, ego, nz, lst, x1=None):
    """The encoder's last_rows call rebuilt from separate srb_spmm_csr calls: full layers 1..L-1 on the static classes,
    layer L on the row list described as srb_encoder_forward describes it, then the fp32 mean of the listed rows in the
    documented order.  Returns (mean of the listed rows [n_listed, d], {layer: full output of layers 0..L-1})."""
    from selfrec_b200 import ops
    shape = tuple(E0.shape)
    layers = {0: E0}
    x, k0 = E0, 0
    if x1 is not None:
        layers[1], x, k0 = x1, x1, 1
    for k in range(k0, L - 1):
        y = _nan(torch, shape)
        ops._spmm_raw(adj, x, y, **_layer_noise(nz, k))
        layers[k + 1] = x = y
    yL = _nan(torch, shape)
    ops._spmm_raw(adj, x, yL, **_layer_noise(nz, L - 1), **list_fields(lst))
    rows = torch.from_numpy(lst["rows"]).cuda()
    terms = [layers[k][rows].cpu().numpy() for k in range(0 if ego else 1, L)] + [yL[rows].cpu().numpy()]
    acc = terms[0]
    for t in terms[1:]:
        acc = acc + t
    return acc * (np.float32(1) / np.float32(L + ego)), layers


def _hub_rows(rng, N, dup):
    """Rows of the hub graph for last_rows: the split rows (users 1, 2, items 1, 2), users 3..9 at the class
    boundaries, 300 others; with dup, 60 repeats (split rows among them); in random order."""
    U = edges.U
    special = np.array([1, 2, U + 1, U + 2, 3, 4, 5, 6, 7, 8, 9])
    others = rng.choice(np.setdiff1d(np.arange(N), special), 300, replace=False)
    rows = np.concatenate([special, others])
    if dup:
        rows = np.concatenate([rows, rows[rng.integers(0, len(rows), 56)], [1, 2, U + 1, U + 2]])
    return rng.permutation(rows)


ENCODER_CASES = [(L, ego, lcl, False) for L in (1, 2, 3, 4) for ego in (0, 1) for lcl in range(L)] + \
                [(L, 0, lcl, True) for L in (2, 3, 4) for lcl in range(L) if lcl != 1]


@pytest.mark.parametrize("kind", ["static", "device"])
@pytest.mark.parametrize("d", WIDTHS)
def test_encoder_listed_row_mean_equals_twin(torch_cuda, graphs, d, kind):
    """srb_encoder_forward with last_rows, for L in 1..4, with and without the ego layer, every CL layer below L, x1
    where it is allowed, noise modes 0, 1 and 2, on static and device-classified lists with duplicates and rows in any
    order: the listed rows of last_rows_out equal the twin bit for bit (L = 4 without x1 reuses work0, so the last
    layer falls back to the running sum), the other rows stay NaN, and cl_out equals the twin's layer layer_cl."""
    torch = torch_cuda
    from selfrec_b200 import ops
    adj, A = graphs["hub"], graphs["hub_A"]
    N = A.shape[0]
    rng = np.random.default_rng(d + 3)
    E0 = _rand(torch, rng, (N, d), 0.1)
    x1 = _nan(torch, (N, d))
    ops._spmm_raw(adj, E0, x1, noise_mode=1, noise=torch.from_numpy(rng.random((N, d), dtype=np.float32)).cuda(), eps=EPS)
    specs = [_noise_spec(torch, mode, N, d, rng) for mode in (0, 1, 2)]
    n_cases = 0
    for dup in (False, True):
        rows = _hub_rows(rng, N, dup)
        unlisted = np.setdiff1d(np.arange(N), rows)
        if kind == "static":
            lst = static_list(torch, rows)
        else:
            lst = device_list(torch, A.indptr, rows, d, rng, shuffle=True, slack=9, spare=int(unlisted[0]))
            assert lst["n_class"][0] >= 8 if dup else lst["n_class"][0] == 4
        un = torch.from_numpy(unlisted).cuda()
        for L, ego, lcl, with_x1 in ENCODER_CASES:
            for nz in specs:
                where = (d, kind, "dup", dup, "L", L, "ego", ego, "layer_cl", lcl, "x1", with_x1, "noise", nz["mode"])
                xx = x1 if with_x1 else None
                bufs = _run_encoder(torch, adj, d, E0, L, ego, lcl, nz, lst, xx)
                mean, layers = _twin(torch, adj, d, E0, L, ego, nz, lst, xx)
                got = bufs["out"][torch.from_numpy(lst["rows"]).cuda()].cpu().numpy()
                assert np.array_equal(got, mean), (where, int((got != mean).any(1).sum()))
                assert bool(torch.isnan(bufs["out"][un]).all()), (where, "unlisted rows written")
                assert torch.equal(bufs["cl"], layers[lcl]), (where, "cl_out")
                n_cases += 1
    assert n_cases == 2 * len(ENCODER_CASES) * 3


@pytest.mark.parametrize("d", WIDTHS)
def test_encoder_listed_row_mean_vs_oracle(torch_cuda, orc, graphs, d):
    """One encoder call per width (L = 3 with the ego layer, noise tensor, a device-classified list) against
    oracle.encoder_forward within 1e-4, where the noise is zero at layer values within rounding of zero (their sign is
    ambiguous)."""
    torch = torch_cuda
    adj, A = graphs["hub"], graphs["hub_A"]
    N = A.shape[0]
    rng = np.random.default_rng(d + 4)
    E0 = (rng.standard_normal((N, d)) * 0.1).astype(np.float32)
    noise = edges._unambiguous_noise(orc, A, E0, rng.random((1, 3, N, d), dtype=np.float32))[0]
    rows = _hub_rows(rng, N, True)
    lst = device_list(torch, A.indptr, rows, d, rng, shuffle=True, slack=3, spare=int(np.setdiff1d(np.arange(N), rows)[0]))
    nz = dict(mode=1, t=torch.from_numpy(noise).cuda())
    bufs = _run_encoder(torch, adj, d, torch.from_numpy(E0).cuda(), 3, 1, 0, nz, lst)
    ref = orc.encoder_forward(A, E0, 3, True, noise, EPS)[0][rows]
    got = bufs["out"][torch.from_numpy(rows).cuda()].cpu().numpy()
    np.testing.assert_allclose(got, ref, rtol=1e-4, atol=1e-6 * np.abs(ref).max())


# ---------------------------------------------------------------------------------------------------------------------
# 5. last_rows where the last layer is not computed on the listed rows
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["static", "device"])
def test_encoder_refuses_last_rows_it_cannot_honour(torch_cuda, graphs, kind):
    """last_rows_out receives the listed rows of the mean whenever last_rows is given, so srb_encoder_forward refuses
    the two calls where the last layer is not run on the list: the CL view at the last layer (that layer is needed in
    full) and no layer at all.  Nothing is written."""
    torch = torch_cuda
    from selfrec_b200 import _lib, ops
    lib = _lib.require_device()
    adj, A = graphs["hub"], graphs["hub_A"]
    N, d = A.shape[0], 32
    rng = np.random.default_rng(5)
    E0 = _rand(torch, rng, (N, d), 0.1)
    rows = _hub_rows(rng, N, True)
    lst = static_list(torch, rows) if kind == "static" else device_list(torch, A.indptr, rows, d, rng, shuffle=True)
    for L, ego, lcl in ((1, 0, 1), (2, 1, 2), (3, 0, 3), (0, 1, 0)):
        shape = (N, d)
        bufs = {k: _nan(torch, shape) for k in ("final", "cl", "w0", "w1", "out")}
        e = _encoder_desc(adj, d, E0, L, ego, lcl, dict(mode=0), bufs, lst)
        rc = lib.srb_encoder_forward(C.byref(e), ops._stream())
        torch.cuda.synchronize()
        assert rc != 0, (kind, L, lcl, "accepted")
        assert "no CL view at the last layer" in _lib.last_error(), _lib.last_error()
        for k, b in bufs.items():
            assert bool(torch.isnan(b).all()), (kind, L, lcl, k, "written")
        # the same call without last_rows runs the last layer in full
        e = _encoder_desc(adj, d, E0, L, ego, lcl, dict(mode=0), bufs)
        _lib.check(lib.srb_encoder_forward(C.byref(e), ops._stream()), "srb_encoder_forward")
        assert not bool(torch.isnan(bufs["final"]).any()), (kind, L, lcl)
