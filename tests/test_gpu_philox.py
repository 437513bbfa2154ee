"""The in-kernel Philox noise of SimGCL and XSimGCL (noise mode 2) pinned bit for bit to its host model,
tests/philox_model.py.

Mode 2 draws the noise in the SpMM epilogue; mode 1 reads the same values from a tensor.  Everything after the noise
values is shared code, and the forward products are deterministic (split rows are summed in chunk order), so mode 2
must give exactly the bits mode 1 gives when it is fed philox_noise(): the SpMM-level comparisons use torch.equal.
Negative controls key the host noise wrongly in one field at a time and must change the outputs, which shows that the
comparison sees every counter field.

The training steps are compared with a twin: engine P draws Philox noise, engine T has the same tables and batches and
is fed step_noise() of the step counter the step will read.  Their forward passes are identical; only the order of the
float atomics differs (InfoNCE dV, the BPR scratch, the seed scatter), so the two are compared against bars set from
two mode-1 twins fed the same noise."""
import functools

import numpy as np
import pytest
import test_gpu_step_edges as edges
from philox_model import noise_offset, philox_noise, step_noise

pytestmark = pytest.mark.gpu

SEED = 0x0123456789ABCDEF
SEEDS = [SEED, 0xFEDC0000_89ABCDEF]  # the second differs from the first in the high word only
OFFSETS = [noise_offset(v, t - 0x10) for v in (0, 1) for t in range(0x10, 0x15)] + [0]
STEPS = [None, 1, 2, 0x7FFFFFFF, -1]  # None: no step pointer; -1 is read as 0xFFFFFFFF
EPS = 0.2


@pytest.fixture(scope="module")
def torch_cuda(built_lib):
    import torch
    assert torch.cuda.is_available()
    from selfrec_b200 import _lib
    _lib.require_device()
    return torch


@pytest.fixture(scope="module")
def hub(torch_cuda):
    """The hub graph of test_gpu_step_edges (split rows of 2 and 3 chunks, CTA, warp and lane-group rows) and two
    device handles of it: split rows in chunk lists, and in column-blocked lists (blocks of 4096 columns)."""
    from selfrec_b200 import ops
    h = edges.make_hub_graph(edges.U, edges.I, edges.HUB_USERS, edges.HUB_ITEMS, 20261016)
    chunked = ops.SparseAdj(h["A"]).cuda()
    blocked = ops.SparseAdj(h["A"]).cuda()
    for d in (32, 64, 128):  # the split-row lists are built (and cached per d) on first use
        assert not chunked.hub_struct(d).seg
    saved = ops.HUB_BLOCK_BYTES
    try:
        for d in (32, 64, 128):
            ops.HUB_BLOCK_BYTES = 2048 * 4 * d  # blocks of 4096 columns: three blocks at N = 11000
            assert blocked.hub_struct(d).seg
    finally:
        ops.HUB_BLOCK_BYTES = saved
    assert chunked.n_huge == 4 and chunked.n_vlong == 2 and chunked.n_long == 4
    h["adj"] = dict(chunked=chunked, colblocked=blocked)
    return h


def _spmm(torch, adj, x, base, entry, **epi):
    from selfrec_b200 import ops
    y, s = torch.empty_like(x), torch.empty_like(x)
    ops._spmm_raw(adj, x, y, _entry=entry, sum_in=base, sum_out=s, sum_scale=0.5, eps=EPS, **epi)
    return y, s


def _step_ptr(torch, step):
    return None if step is None else torch.tensor([step], dtype=torch.int32, device="cuda")


@pytest.mark.parametrize("d", [32, 64, 128])
def test_spmm_philox_noise_equals_host_model(torch_cuda, hub, d):
    """srb_spmm_csr and srb_spmm_epilogue_rows on the hub graph, chunked and column-blocked split rows: Philox noise
    (mode 2) gives the bits of the noise-tensor path (mode 1) fed the host model's noise, over two seeds that differ in
    the high word, views 0 and 1 x tags 0x10..0x14 and offset 0, and step pointers null, 1, 2, 2^31 - 1 and -1."""
    torch = torch_cuda
    N = hub["A"].shape[0]
    rng = np.random.default_rng(d)
    x = torch.from_numpy((rng.standard_normal((N, d)) * 0.1).astype(np.float32)).cuda()
    base = torch.from_numpy((rng.standard_normal((N, d)) * 0.1).astype(np.float32)).cuda()
    n_cmp = 0
    for seed in SEEDS:
        for off in OFFSETS:
            for step in STEPS:
                noise = torch.from_numpy(philox_noise(seed, off, step, N, d)).cuda()
                sp = _step_ptr(torch, step)
                for kind, adj in hub["adj"].items():
                    for entry in ("srb_spmm_csr", "srb_spmm_epilogue_rows"):
                        y2, s2 = _spmm(torch, adj, x, base, entry, noise_mode=2, philox_seed=seed, philox_offset=off, philox_step_dev=sp)
                        y1, s1 = _spmm(torch, adj, x, base, entry, noise_mode=1, noise=noise)
                        where = (kind, entry, hex(seed), hex(off), step)
                        assert torch.equal(y2, y1), (where, int((y2 != y1).any(1).sum()))
                        assert torch.equal(s2, s1), where
                        n_cmp += 1
    assert n_cmp == len(SEEDS) * len(OFFSETS) * len(STEPS) * 4


@pytest.mark.parametrize("d", [32, 64, 128])
def test_spmm_philox_noise_wrong_keys_differ(torch_cuda, hub, d):
    """Negative controls: host noise keyed with step - 1, the views swapped, tag + 1, the seed's high word zeroed or row
    stride 0 changes every noisy row of the output but row 0 (stride 0 keeps row 0's key)."""
    torch = torch_cuda
    N = hub["A"].shape[0]
    rng = np.random.default_rng(d + 1)
    x = torch.from_numpy((rng.standard_normal((N, d)) * 0.1).astype(np.float32)).cuda()
    base = torch.zeros_like(x)
    off, step = noise_offset(1, 2), 2
    wrong = dict(step_minus_1=(SEED, off, step - 1, 1), views_swapped=(SEED, noise_offset(0, 2), step, 1),
                 tag_plus_1=(SEED, off + 1, step, 1), seed_high_zero=(SEED & 0xFFFFFFFF, off, step, 1), row_stride_0=(SEED, off, step, 0))
    sp = _step_ptr(torch, step)
    for kind, adj in hub["adj"].items():
        for entry in ("srb_spmm_csr", "srb_spmm_epilogue_rows"):
            clean, _ = _spmm(torch, adj, x, base, entry)
            y2, _ = _spmm(torch, adj, x, base, entry, noise_mode=2, philox_seed=SEED, philox_offset=off, philox_step_dev=sp)
            noisy = (y2 != clean).any(1)
            assert int(noisy.sum()) > 0.9 * N, (kind, entry)  # rows with a zero value are not perturbed there
            right, _ = _spmm(torch, adj, x, base, entry, noise_mode=1, noise=torch.from_numpy(philox_noise(SEED, off, step, N, d)).cuda())
            assert torch.equal(right, y2), (kind, entry)
            for name, (s, o, t, stride) in wrong.items():
                noise = torch.from_numpy(philox_noise(s, o, t, N, d, row_stride=stride)).cuda()
                y1, _ = _spmm(torch, adj, x, base, entry, noise_mode=1, noise=noise)
                same = ((y1 == y2).all(1) & noisy).nonzero().flatten().tolist()
                assert same == ([0] if stride == 0 and bool(noisy[0]) else []), (kind, entry, name, same[:8])


@pytest.mark.parametrize("d", [32, 64, 128])
def test_encoder_forward_philox_equals_host_model(torch_cuda, hub, d):
    """ops.encoder_forward(philox_seed=...) (offset 0 + layer, no step pointer) against noise= fed the host model's
    noise, at L = 1..3: the final mean and the CL view, bit for bit."""
    torch = torch_cuda
    from selfrec_b200 import ops
    N = hub["A"].shape[0]
    rng = np.random.default_rng(d + 2)
    e0 = torch.from_numpy((rng.standard_normal((N, d)) * 0.1).astype(np.float32)).cuda()
    for kind, adj in hub["adj"].items():
        for L in (1, 2, 3):
            noise = torch.from_numpy(np.stack([philox_noise(SEED, k, None, N, d) for k in range(L)])).cuda()
            for ego, lcl in ((False, 1), (False, L), (True, L)):
                f2, c2 = ops.encoder_forward(adj, e0, L, ego, philox_seed=SEED, eps=EPS, layer_cl=lcl, want_cl=True)
                f1, c1 = ops.encoder_forward(adj, e0, L, ego, noise=noise, eps=EPS, layer_cl=lcl, want_cl=True)
                assert torch.equal(f2, f1), (kind, L, ego, lcl)
                assert torch.equal(c2, c1), (kind, L, ego, lcl)
            # the layers are keyed apart: layer k's noise moved to layer k + 1 gives another mean
            if L >= 2:
                f3, _ = ops.encoder_forward(adj, e0, L, False, noise=noise.roll(1, 0).contiguous(), eps=EPS)
                assert not torch.equal(f3, f2), (kind, L)


# ---------------------------------------------------------------------------------------------------------------------
# training steps against a mode-1 twin
# ---------------------------------------------------------------------------------------------------------------------
LR, REG, TAU, CL_RATE = 1e-2, 1e-3, 0.2, 0.3
# Bars between P and T after every step: max|a - b| / max|b| per tensor (BAR) and ||m_P - m_T|| / ||m_T|| (M_FRO_BAR),
# at about 10x the worst spread of two mode-1 twins fed the same noise, over every case below, eager and captured, in two
# runs on an H100 80GB HBM3 (700 W): losses 3.6e-5, m 2.4e-5, v 2.9e-5, params 6.6e-5, m Frobenius 3.4e-6 (P against T:
# 1.8e-5, 2.5e-5, 2.9e-5, 7.5e-5, 3.2e-6).  The max-norm spread comes from the hub rows, whose gradients sum the most
# atomics; the Frobenius norm weighs every row, so the wrong-keyed control (nearest seen: 1.2e-2, SimGCL d128 L3 with the
# views swapped) must be CONTROL_MARGIN Frobenius bars away from P.
BAR = dict(losses=4e-4, m=2.5e-4, v=3e-4, params=7e-4)
M_FRO_BAR = 3.5e-5
CONTROL_MARGIN = 100

TWIN_CASES = [
    # name, d, L, layer_cl
    ("XSimGCL", 64, 3, 1),   # the bench configuration
    ("XSimGCL", 32, 2, 2),   # the CL view is the full last layer
    ("XSimGCL", 128, 1, 1),
    ("SimGCL", 64, 1, 0),    # no shared first product
    ("SimGCL", 32, 2, 0),    # perturb_rows on the shared first product
    ("SimGCL", 128, 3, 0),
    ("SimGCL", 64, 5, 0),    # the running-sum path
]


def _twin_id(c):
    name, d, L, lcl = c
    return f"{name}-d{d}-L{L}" + (f"-lcl{lcl}" if name == "XSimGCL" else "")


def _rel(a, b):
    return float(np.abs(a - b).max() / max(float(np.abs(b).max()), 1e-30))


def _fro(a, b):
    a, b = a.astype(np.float64), b.astype(np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def make_engine(torch, hub, name, d, L, lcl, E0, noise_fn):
    """A TrainEngine on the hub graph.  noise_fn None: Philox noise (seed SEED); else noise_fn(k) is the
    [views, L, N, d] noise fed before the step that reads step counter k.  Returns (engine, feed), feed(k) copies it."""
    from selfrec_b200.engine import TrainEngine
    U = hub["data"].user_num
    eng = TrainEngine(name, hub["data"], d, L, edges.B, LR, REG, eps=EPS, tau=TAU, cl_rate=CL_RATE, layer_cl=lcl,
                      init_user=torch.from_numpy(E0[:U]), init_item=torch.from_numpy(E0[U:]), philox_seed=SEED)
    if noise_fn is None:
        return eng, lambda k: None
    views = 2 if name == "SimGCL" else 1
    buf = torch.zeros((views, L, E0.shape[0], d), device="cuda", dtype=torch.float32)
    eng.set_noise_tensor(buf)
    return eng, lambda k: buf.copy_(torch.from_numpy(noise_fn(k)))


def run_twins(torch, hub, captured, engines):
    """Steps every engine in `engines` ({key: (engine, feed)}) through a full batch with every hub row (the poison
    batch of test_gpu_step_edges, on finite tables) and the hub graph's five batches (a full batch, 17 triples, one hub
    triple, empty, one hub triple B times); engine "P" steps eagerly or through capture() + replay, like
    FusedGraphModel.train.  Checks every engine's step counter and returns, per step, dict(step, b, dist) with
    dist[key][tensor] = _rel(engine key's tensor, P's tensor) and dist[key]["m_fro"] = _fro of their m, for every
    other engine."""
    P = engines["P"][0]
    seq = [(hub["poison"], edges.B)] + [(w, len(u)) for w, (u, _, _) in hub["batches"]]
    if captured:
        P.batch_dev.copy_(torch.from_numpy(seq[0][0]))
        P.capture()
        torch.cuda.synchronize()
        assert int(P.step_dev.item()) == 0, "capture() must put the step counter back"
    out = []
    for k, (words, b) in enumerate(seq, start=1):
        for key, (eng, feed) in engines.items():
            feed(k)
            eng.step(words)
        torch.cuda.synchronize()
        state = {key: dict(step=int(eng.step_dev.item()), losses=eng.losses.cpu().numpy(), m=eng.m.cpu().numpy(),
                           v=eng.v.cpu().numpy(), params=eng.params.cpu().numpy()) for key, (eng, _) in engines.items()}
        for key, st in state.items():
            assert st["step"] == k, (key, k, st["step"])
            for t in ("losses", "m", "v", "params"):
                assert np.isfinite(st[t]).all() or (t == "losses" and b == 0), (key, k, t)
        dist = {}
        for key, st in state.items():
            if key != "P":
                dist[key] = {t: _rel(st[t], state["P"][t]) for t in ("m", "v", "params")}
                dist[key]["losses"] = _rel(st["losses"], state["P"]["losses"]) if b > 0 else 0.0
                dist[key]["m_fro"] = _fro(st["m"], state["P"]["m"])
        out.append(dict(step=k, b=b, dist=dist))
    return out


def _E0(N, d, L):
    return (np.random.default_rng(d * 10 + L).standard_normal((N, d)) * 0.1).astype(np.float32)


def twin_noise(name, L, N, d):
    """(noise(k), wrong(k)): step_noise of step counter k, and the control's wrong keying of it (XSimGCL: the previous
    step's noise; SimGCL: the two views swapped)."""
    noise = functools.lru_cache(4)(lambda k: step_noise(name, SEED, L, N, d, k))
    if name == "SimGCL":
        return noise, lambda k: noise(k)[::-1].copy()
    return noise, lambda k: noise(k - 1)


@pytest.mark.parametrize("captured", [False, True], ids=["eager", "captured"])
@pytest.mark.parametrize("name,d,L,lcl", TWIN_CASES, ids=[_twin_id(c) for c in TWIN_CASES])
def test_train_step_philox_equals_noise_tensor_twin(torch_cuda, hub, name, d, L, lcl, captured):
    """TrainEngine in Philox mode (P) against a twin fed step_noise() before every step (T): step counters, losses, m, v
    and parameters after every step within the atomics-order bars; a third engine keyed wrongly (XSimGCL: the previous
    step's noise, SimGCL: the two views swapped) lands at least CONTROL_MARGIN Frobenius bars away in m.  The step
    counter reads 0 after capture() and k after the k-th step."""
    torch = torch_cuda
    N = hub["A"].shape[0]
    E0 = _E0(N, d, L)
    noise, wrong = twin_noise(name, L, N, d)
    engines = dict(P=make_engine(torch, hub, name, d, L, lcl, E0, None), T=make_engine(torch, hub, name, d, L, lcl, E0, noise),
                   W=make_engine(torch, hub, name, d, L, lcl, E0, wrong))
    for r in run_twins(torch, hub, captured, engines):
        where = (_twin_id((name, d, L, lcl)), "step", r["step"], "b", r["b"])
        for t, bar in BAR.items():
            assert r["dist"]["T"][t] <= bar, (where, t, r["dist"]["T"][t])
        assert r["dist"]["T"]["m_fro"] <= M_FRO_BAR, (where, "m_fro", r["dist"]["T"]["m_fro"])
        assert r["dist"]["W"]["m_fro"] >= CONTROL_MARGIN * M_FRO_BAR, (where, "control", r["dist"]["W"]["m_fro"])
