"""Torch-facing wrappers over the C ABI (selfrec_b200/_lib.py).

PyTorch is plumbing here: it owns device memory, streams and autograd bookkeeping; every
computation is a hand-written sm_90a kernel reached through ctypes with raw pointers.
All ops are stream-ordered on torch's current stream and raise SrbError without a GPU.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import SrbError

_SUPPORTED_D = (16, 32, 64, 128, 256)
LONG_ROW_NNZ = 64    # rows at least this long are processed by a whole warp (srb_spmm_desc.n_long_rows)
VLONG_ROW_NNZ = 256  # rows at least this long are processed by a whole CTA (srb_spmm_desc.n_vlong_rows)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _f32c(t, name):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name}: expected a torch.Tensor")
    if not t.is_cuda:
        raise SrbError(f"{name}: selfrec_b200 ops need CUDA tensors (no CPU fallback)")
    if t.dtype != torch.float32:
        raise TypeError(f"{name}: expected float32, got {t.dtype}")
    return t.contiguous()


def _i32(x, device):
    """Index list / array / tensor -> int32 device tensor (the reference passes Python lists)."""
    if isinstance(x, torch.Tensor):
        return x.to(device=device, dtype=torch.int32).contiguous()
    arr = np.ascontiguousarray(np.asarray(x, dtype=np.int32))
    return torch.from_numpy(arr).to(device, non_blocking=False)


# ----------------------------------------------------------------------------------------
# adjacency handle + SpMM
# ----------------------------------------------------------------------------------------
def classify_rows(rowptr):
    """Row classes of the SpMM for a CSR row-pointer tensor (int32, any device): processing order (degree-descending,
    stable), class sizes, and the chunk lists of the split rows (srb_hub_split in include/selfrec_b200.h).
    Returns dict(row_order, n_huge, n_vlong, n_long, hub_first, hub_work, n_work)."""
    rp = rowptr.to(torch.int64)
    deg = rp[1:] - rp[:-1]
    order = torch.sort(deg, descending=True, stable=True).indices
    n_huge = int((deg >= _lib.HUB_MIN_NNZ).sum())
    n_vlong = int((deg >= VLONG_ROW_NNZ).sum()) - n_huge
    n_long = int((deg >= LONG_ROW_NNZ).sum()) - n_huge - n_vlong
    out = dict(row_order=order.to(torch.int32), n_huge=n_huge, n_vlong=n_vlong, n_long=n_long, hub_first=None, hub_work=None, n_work=0)
    if n_huge:
        rows = order[:n_huge]
        nch = (deg[rows] + _lib.HUB_CHUNK - 1) // _lib.HUB_CHUNK
        first = torch.cumsum(nch, 0) - nch
        n_work = int(nch.sum())
        wrow = torch.repeat_interleave(rows, nch)
        wci = torch.arange(n_work, device=rp.device) - torch.repeat_interleave(first, nch)
        out.update(hub_first=first.to(torch.int32).contiguous(), hub_work=torch.stack([wrow, wci], 1).to(torch.int32).contiguous(),
                   n_work=n_work)
    return out


HUB_BLOCK_BYTES = None  # X rows of one column block of the column-blocked split-row lists; None: a quarter of the L2


def hub_block_bytes(device):
    """Column-block size of the split-row lists: a quarter of the device's L2 (12.5 MB on an H100), so that one block
    of X stays resident next to the CSR and output streams.  HUB_BLOCK_BYTES overrides it."""
    if HUB_BLOCK_BYTES is not None:
        return HUB_BLOCK_BYTES
    device = torch.device(device)
    if device.type != "cuda":  # lists built from host tensors: the current GPU's L2, else the H100's 50 MB
        if not torch.cuda.is_available():
            return (50 << 20) // 4
        device = torch.device("cuda", torch.cuda.current_device())
    return torch.cuda.get_device_properties(device).L2_cache_size // 4


def column_blocked_segments(rowptr, colidx, rows, n_cols, d):
    """Column-blocked work lists of the split rows `rows` (device tensors; srb_hub_split.seg in the header): every
    split row is cut at column-block boundaries (block = hub_block_bytes() of X rows) and at most HUB_CHUNK non-zeros,
    and the segments are ordered by (column block, row) so that one block of X stays L2-resident while ALL rows'
    segments of that block are processed.  Returns dict(seg, first, cnt, order_cta, order_warp) or None when the
    matrix has a single column block."""
    W = max(4096, hub_block_bytes(rowptr.device) // (4 * d))
    if n_cols <= 2 * W or rows.numel() == 0:
        return None
    dev = rowptr.device
    rp = rowptr.to(torch.int64)
    beg, end = rp[rows], rp[rows + 1]
    deg = end - beg
    n_rows = rows.numel()
    total = int(deg.sum())
    slot = torch.repeat_interleave(torch.arange(n_rows, device=dev), deg, output_size=total)      # split-row index of every non-zero
    pos = torch.arange(total, device=dev) - torch.repeat_interleave(torch.cumsum(deg, 0) - deg, deg, output_size=total) + beg[slot]
    blk = colidx[pos].to(torch.int64) // W
    nblk = (n_cols + W - 1) // W
    key = slot * nblk + blk                                          # non-decreasing: rows ascending, columns ascending within a row
    ukey, cnt = torch.unique_consecutive(key, return_counts=True)
    sbeg = pos[torch.cumsum(cnt, 0) - cnt]                           # CSR position of each (row, block) segment
    # cut segments longer than a chunk
    pieces = (cnt + _lib.HUB_CHUNK - 1) // _lib.HUB_CHUNK
    n_seg = int(pieces.sum())
    src = torch.repeat_interleave(torch.arange(ukey.numel(), device=dev), pieces, output_size=n_seg)
    sub = torch.arange(n_seg, device=dev) - torch.repeat_interleave(torch.cumsum(pieces, 0) - pieces, pieces, output_size=n_seg)
    b = sbeg[src] + sub * _lib.HUB_CHUNK
    e = torch.minimum(b + _lib.HUB_CHUNK, sbeg[src] + cnt[src])
    srow = ukey[src] // nblk
    sblk = ukey[src] % nblk
    per_row = torch.bincount(srow, minlength=n_rows)
    first = torch.cumsum(per_row, 0) - per_row                       # slots are row-major: a row's segments are consecutive
    order = torch.sort(sblk * n_rows + srow, stable=True).indices    # processing order: column block, then row
    long_seg = (e - b)[order] > _lib.HUB_WARP_SEG
    i32 = lambda t: t.to(torch.int32).contiguous()
    return dict(seg=i32(torch.stack([b, e], 1)), first=i32(first), cnt=i32(per_row), order_cta=i32(order[long_seg]),
                order_warp=i32(order[~long_seg]), n_seg=n_seg, block_cols=W)


class SparseAdj:
    """Device CSR handle returned by TorchGraphInterface.convert_sparse_mat_to_tensor.

    Stands in for the torch COO tensor of base/torch_interface.py:8-13: `.cuda()` uploads
    (identity afterwards) and `torch.sparse.mm(handle, X)` routes to the CUDA SpMM through
    __torch_function__, differentiable w.r.t. X.  from_device() wraps a CSR that was assembled
    on the GPU (srb_graph_assemble: config-5 graphs, SGL's per-epoch views) without a host copy.
    """

    def __init__(self, mat):
        import scipy.sparse as sp

        csr = sp.csr_matrix(mat, dtype=np.float32)
        csr.sort_indices()
        if csr.nnz >= 2**31:
            raise SrbError("SparseAdj: nnz must fit in int32")
        self._csr = csr
        self.shape = tuple(csr.shape)
        self.nnz = int(csr.nnz)
        self.device = torch.device("cpu")
        self.rowptr = self.colidx = self.vals = self.row_order = None
        self.n_long = self.n_vlong = self.n_huge = self.n_work = 0
        self.hub_first = self.hub_work = None
        self._hub_part = {}
        self._t = None  # transposed handle (backward), built lazily
        self._symmetric = None

    @classmethod
    def from_device(cls, rowptr, colidx, vals, shape, symmetric=None, classes=None):
        """Wrap device CSR arrays (int32 rowptr [n+1], int32 colidx [nnz], fp32 vals [nnz], columns ascending)."""
        self = cls.__new__(cls)
        self._csr = None
        self.shape = tuple(int(x) for x in shape)
        self.nnz = int(colidx.numel())
        self.device = rowptr.device
        self.rowptr, self.colidx, self.vals = rowptr, colidx, vals
        self._hub_part = {}
        self._t = None
        self._symmetric = symmetric
        self._set_classes(classify_rows(rowptr) if classes is None else classes)
        return self

    def _set_classes(self, c):
        self.row_order = c["row_order"]
        self.n_huge, self.n_vlong, self.n_long = c["n_huge"], c["n_vlong"], c["n_long"]
        self.hub_first, self.hub_work, self.n_work = c["hub_first"], c["hub_work"], c["n_work"]

    # -- reference-compatible surface -------------------------------------------------
    def cuda(self, device=None):
        _lib.require_device()
        dev = torch.device("cuda", torch.cuda.current_device() if device is None else device) if not isinstance(device, torch.device) else device
        if self.rowptr is not None and self.device == dev:
            return self
        if self._csr is None:
            raise SrbError("SparseAdj.from_device handles stay on the device they were built on")
        csr = self._csr
        self.rowptr = torch.from_numpy(csr.indptr.astype(np.int32)).to(dev)
        self.colidx = torch.from_numpy(csr.indices.astype(np.int32)).to(dev)
        self.vals = torch.from_numpy(csr.data.astype(np.float32)).to(dev)
        # long rows first: evens out the tail of the warp-per-row kernel on power-law graphs
        self._set_classes(classify_rows(self.rowptr))
        self._hub_part = {}
        self.device = dev
        return self

    def to(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise SrbError("SparseAdj lives on a CUDA device (no CPU fallback)")
        return self.cuda(device)

    def size(self, dim=None):
        return self.shape if dim is None else self.shape[dim]

    def _nnz(self):
        return self.nnz

    def _host_csr(self):
        if self._csr is None:
            import scipy.sparse as sp
            self._csr = sp.csr_matrix((self.vals.cpu().numpy(), self.colidx.cpu().numpy(), self.rowptr.cpu().numpy()), shape=self.shape)
        return self._csr

    def _indices(self):
        coo = self._host_csr().tocoo()
        return torch.from_numpy(np.vstack([coo.row, coo.col]).astype(np.int64)).to(self.device)

    def _values(self):
        return torch.from_numpy(self._host_csr().tocoo().data.astype(np.float32)).to(self.device)

    def is_symmetric(self):
        if self._symmetric is None:
            a = self._host_csr()
            self._symmetric = a.shape[0] == a.shape[1] and (abs(a - a.T) > 0).nnz == 0
        return self._symmetric

    def transposed(self):
        if self.is_symmetric():
            return self
        if self._t is None:
            self._t = SparseAdj(self._host_csr().T.tocsr())
            self._t._t = self
        if self.rowptr is not None:
            self._t.cuda(self.device)
        return self._t

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        if func is torch.sparse.mm or func is torch.mm or func is torch.matmul:
            return spmm(args[0], args[1])
        return NotImplemented

    def hub_struct(self, d):
        """srb_hub_split of this graph for embedding size d (lists and partial-sum scratch are made on first use).
        Matrices wider than two column blocks get the column-blocked lists (see column_blocked_segments)."""
        h = _lib.HubSplit()
        if self.n_huge:
            ent = self._hub_part.get(d)
            if ent is None:
                segs = column_blocked_segments(self.rowptr, self.colidx, self.row_order[: self.n_huge].to(torch.int64), self.shape[1], d)
                n_part = segs["n_seg"] if segs else self.n_work
                ent = self._hub_part[d] = (torch.empty((n_part, d), device=self.device, dtype=torch.float32), segs)
            part, segs = ent
            h.n_rows, h.part = self.n_huge, _p(part)
            if segs:
                h.n_work, h.first = segs["n_seg"], _p(segs["first"])
                h.seg, h.seg_cnt = _p(segs["seg"]), _p(segs["cnt"])
                h.order_cta, h.order_warp = _p(segs["order_cta"]), _p(segs["order_warp"])
                h.n_cta, h.n_warp = int(segs["order_cta"].numel()), int(segs["order_warp"].numel())
                h.work = _p(self.hub_work)
            else:
                h.n_work, h.first, h.work = self.n_work, _p(self.hub_first), _p(self.hub_work)
        return h

    def graph_struct(self, d):
        g = _lib.GraphCsr()
        g.rowptr, g.colidx, g.vals, g.row_order = _p(self.rowptr), _p(self.colidx), _p(self.vals), _p(self.row_order)
        g.n_long_rows = self.n_long
        g.n_vlong_rows = self.n_vlong
        g.hub = self.hub_struct(d)
        return g


def _spmm_raw(adj, x, y=None, _entry="srb_spmm_csr", **epi):
    """Y = epilogue(A @ X) (srb_spmm_csr); _entry="srb_spmm_epilogue_rows": the epilogue alone on the rows of X."""
    lib = _lib.require_device()
    if adj.rowptr is None:
        adj.cuda(x.device)
    n_rows, n_cols = adj.shape
    d = x.shape[1]
    if x.shape[0] != n_cols:
        raise ValueError(f"spmm: A is {adj.shape} but X has {x.shape[0]} rows")
    if d not in _SUPPORTED_D:
        raise SrbError(f"spmm: embedding size {d} unsupported (16, 32, 64, 128, 256)")
    desc = _lib.SpmmDesc()
    desc.rowptr, desc.colidx, desc.vals = _p(adj.rowptr), _p(adj.colidx), _p(adj.vals)
    desc.row_order = _p(adj.row_order)
    desc.n_long_rows, desc.n_vlong_rows = adj.n_long, adj.n_vlong
    desc.hub = adj.hub_struct(d)
    desc.n_rows, desc.n_cols, desc.d = n_rows, n_cols, d
    desc.X = _p(x)
    desc.Y = _p(y)
    desc.extra_scale = 1.0
    desc.sum_scale = 1.0
    keep = []
    for k, v in epi.items():
        if isinstance(v, torch.Tensor):
            keep.append(v)
            setattr(desc, k, _p(v))
        else:
            setattr(desc, k, v)
    _lib.check(getattr(lib, _entry)(C.byref(desc), _stream()), _entry)


class _SpmmFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, adj):
        x = _f32c(x, "spmm X")
        y = torch.empty((adj.shape[0], x.shape[1]), device=x.device, dtype=torch.float32)
        _spmm_raw(adj, x, y)
        ctx.adj = adj
        return y

    @staticmethod
    def backward(ctx, gy):
        gy = _f32c(gy, "spmm grad")
        at = ctx.adj.transposed()
        gx = torch.empty((at.shape[0], gy.shape[1]), device=gy.device, dtype=torch.float32)
        _spmm_raw(at, gy, gx)
        return gx, None


def spmm(adj, x):
    """Y = A @ X on the CUDA CSR kernel; differentiable w.r.t. X (torch.sparse.mm drop-in)."""
    if not isinstance(adj, SparseAdj):
        raise TypeError("spmm: first argument must be a SparseAdj handle")
    return _SpmmFn.apply(x, adj)


def encoder_forward(adj, e0, n_layers, include_ego, noise=None, eps=0.0, layer_cl=0, philox_seed=None, want_cl=False):
    """Fused encoder forward (no autograd): returns (final, cl_view or None).

    noise: [n_layers, N, d] uniform[0,1) tensor (parity mode) or None; philox_seed: int for
    in-kernel noise.  See srb_encoder_forward in include/selfrec_b200.h.
    """
    lib = _lib.require_device()
    e0 = _f32c(e0, "encoder E0")
    if adj.rowptr is None:
        adj.cuda(e0.device)
    n, d = e0.shape
    final = torch.empty_like(e0)
    cl = torch.empty_like(e0) if want_cl else None
    w0 = torch.empty_like(e0)
    w1 = torch.empty_like(e0)
    desc = _lib.EncoderDesc()
    desc.rowptr, desc.colidx, desc.vals, desc.row_order = _p(adj.rowptr), _p(adj.colidx), _p(adj.vals), _p(adj.row_order)
    desc.n_long_rows, desc.n_vlong_rows = adj.n_long, adj.n_vlong
    desc.hub = adj.hub_struct(d)
    desc.n, desc.d, desc.n_layers, desc.include_ego, desc.layer_cl = n, d, n_layers, int(include_ego), int(layer_cl)
    if noise is not None:
        noise = _f32c(noise, "encoder noise")
        if tuple(noise.shape) != (n_layers, n, d):
            raise ValueError("encoder noise must be [n_layers, N, d]")
        desc.noise_mode, desc.noise = 1, _p(noise)
    elif philox_seed is not None:
        desc.noise_mode, desc.philox_seed = 2, int(philox_seed)
    desc.eps = float(eps)
    desc.E0, desc.final_out, desc.cl_out, desc.work0, desc.work1 = _p(e0), _p(final), _p(cl), _p(w0), _p(w1)
    _lib.check(lib.srb_encoder_forward(C.byref(desc), _stream()), "srb_encoder_forward")
    return final, cl


# ----------------------------------------------------------------------------------------
# losses (op-level drop-in: inputs are already-gathered [b, d] rows)
# ----------------------------------------------------------------------------------------
class _BprFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, u, p, n):
        lib = _lib.require_device()
        u, p, n = _f32c(u, "bpr user_emb"), _f32c(p, "bpr pos_item_emb"), _f32c(n, "bpr neg_item_emb")
        b, d = u.shape
        table = torch.cat([u, p, n], 0)
        ar = torch.arange(b, device=u.device, dtype=torch.int32)
        j = ar + b
        losses = torch.empty(2, device=u.device, dtype=torch.float32)
        g = torch.empty((3, b, d), device=u.device, dtype=torch.float32)
        scratch = torch.empty(8, device=u.device, dtype=torch.float32)
        desc = _lib.BprDesc()
        desc.emb, desc.l2_emb, desc.n_users, desc.d = _p(table), _p(table), b, d
        desc.u_idx, desc.i_idx, desc.j_idx, desc.b = _p(ar), _p(ar), _p(j), b
        desc.emb_scale, desc.reg, desc.l2_terms, desc.l2_div, desc.grad_scale = 1.0, 0.0, 2, 1.0, 1.0
        desc.losses, desc.g_emb, desc.scratch = _p(losses), _p(g), _p(scratch)
        _lib.check(lib.srb_bpr_l2_fwd_bwd(C.byref(desc), _stream()), "srb_bpr_l2_fwd_bwd")
        ctx.save_for_backward(g)
        return losses[0]

    @staticmethod
    def backward(ctx, go):
        (g,) = ctx.saved_tensors
        g = g * go
        return g[0], g[1], g[2]


def bpr_loss(user_emb, pos_item_emb, neg_item_emb):
    return _BprFn.apply(user_emb, pos_item_emb, neg_item_emb)


class _L2Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, reg, *embs):
        lib = _lib.require_device()
        embs = [_f32c(e, "l2_reg_loss emb") for e in embs]
        if not 1 <= len(embs) <= 4:
            raise SrbError("l2_reg_loss: 1..4 embeddings per call")
        dev = embs[0].device
        n = len(embs)
        ptrs = (C.c_void_p * n)(*[e.data_ptr() for e in embs])
        nel = (C.c_int64 * n)(*[e.numel() for e in embs])
        rows = (C.c_int32 * n)(*[e.shape[0] for e in embs])
        sumsq = torch.empty(4, device=dev, dtype=torch.float32)
        loss = torch.empty((), device=dev, dtype=torch.float32)
        _lib.check(lib.srb_l2_reg_fwd(n, ptrs, nel, rows, float(reg), _p(sumsq), _p(loss), _stream()), "srb_l2_reg_fwd")
        ctx.reg = float(reg)
        ctx.save_for_backward(sumsq, *embs)
        return loss

    @staticmethod
    def backward(ctx, go):
        lib = _lib.require_device()
        sumsq, *embs = ctx.saved_tensors
        n = len(embs)
        go = go.to(torch.float32).contiguous()
        grads = [torch.empty_like(e) for e in embs]
        ptrs = (C.c_void_p * n)(*[e.data_ptr() for e in embs])
        gptrs = (C.c_void_p * n)(*[g.data_ptr() for g in grads])
        nel = (C.c_int64 * n)(*[e.numel() for e in embs])
        rows = (C.c_int32 * n)(*[e.shape[0] for e in embs])
        _lib.check(lib.srb_l2_reg_bwd(n, ptrs, gptrs, nel, rows, ctx.reg, _p(sumsq), _p(go), _stream()), "srb_l2_reg_bwd")
        return (None, *grads)


def l2_reg_loss(reg, *args):
    return _L2Fn.apply(reg, *args)


def infonce_raw(problems, d, temperature, b_cos=True, max_n=None, workspace=None, batch_softmax=False):
    """Run srb_infonce_fwd_bwd (srb_batch_softmax_fwd_bwd with batch_softmax=True, which needs b_cos).
    problems: list of dicts(table1, table2, idx, n, and optionally n_dev,
    weight, row_off1, row_off2, scale1, scale2, and g1 / g2 output tensors to write into).
    workspace: optional uint8 device tensor to use instead of a fresh one (its whole size is offered).
    Returns (losses [P], [(g1, g2)])."""
    lib = _lib.require_device()
    dev = problems[0]["table1"].device
    npb = len(problems)
    if not 1 <= npb <= 4:  # srb_infonce_desc.prob[4]
        raise SrbError(f"infonce: n_problems must be 1..4 (got {npb})")
    if workspace is None:
        mx = max(p["n"] for p in problems) if max_n is None else max_n
        ws_bytes = lib.srb_infonce_workspace_bytes(mx, d, npb)
        ws = torch.empty(max(ws_bytes, 16), device=dev, dtype=torch.uint8)
    else:
        ws = workspace
        ws_bytes = ws.numel() * ws.element_size()
    losses = torch.empty(npb, device=dev, dtype=torch.float32)
    desc = _lib.InfoNceDesc()
    desc.n_problems, desc.d, desc.b_cos, desc.temperature = npb, d, int(bool(b_cos)), float(temperature)
    outs = []
    for q, p in enumerate(problems):
        g1 = p["g1"] if "g1" in p else torch.empty((p["n"], d), device=dev, dtype=torch.float32)
        g2 = p["g2"] if "g2" in p else torch.empty((p["n"], d), device=dev, dtype=torch.float32)
        for g in (g1, g2):
            if g.shape != (p["n"], d) or g.dtype != torch.float32 or not g.is_contiguous():
                raise SrbError(f"infonce: g1 / g2 of problem {q} must be contiguous float32 [{p['n']}, {d}]")
        pr = desc.prob[q]
        pr.table1, pr.table2 = _p(p["table1"]), _p(p["table2"])
        pr.row_off1, pr.row_off2 = p.get("row_off1", 0), p.get("row_off2", 0)
        pr.scale1, pr.scale2 = float(p.get("scale1", 1.0)), float(p.get("scale2", 1.0))
        pr.idx, pr.n_dev, pr.n, pr.weight = _p(p["idx"]), _p(p.get("n_dev")), p["n"], float(p.get("weight", 1.0))
        pr.g1, pr.g2 = _p(g1), _p(g2)
        pr.loss = C.c_void_p(losses.data_ptr() + 4 * q)
        outs.append((g1, g2))
    desc.workspace, desc.workspace_bytes = _p(ws), ws_bytes
    entry = "srb_batch_softmax_fwd_bwd" if batch_softmax else "srb_infonce_fwd_bwd"
    _lib.check(getattr(lib, entry)(C.byref(desc), _stream()), entry)
    return losses, outs


class _InfoNceFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, v1, v2, temperature, b_cos):
        v1, v2 = _f32c(v1, "InfoNCE view1"), _f32c(v2, "InfoNCE view2")
        if v1.shape != v2.shape:
            raise ValueError("InfoNCE: views must have the same shape")
        n, d = v1.shape
        if d not in _SUPPORTED_D:
            raise SrbError(f"InfoNCE: embedding size {d} unsupported (16, 32, 64, 128, 256)")
        idx = torch.arange(n, device=v1.device, dtype=torch.int32)
        losses, outs = infonce_raw([dict(table1=v1, table2=v2, idx=idx, n=n, weight=1.0)], d, temperature, b_cos)
        ctx.save_for_backward(*outs[0])
        return losses[0]

    @staticmethod
    def backward(ctx, go):
        g1, g2 = ctx.saved_tensors
        return g1 * go, g2 * go, None, None


def InfoNCE(view1, view2, temperature, b_cos=True):
    return _InfoNceFn.apply(view1, view2, float(temperature), bool(b_cos))


class _BatchSoftmaxFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, user_emb, item_emb, temperature):
        u, i = _f32c(user_emb, "batch_softmax_loss user_emb"), _f32c(item_emb, "batch_softmax_loss item_emb")
        if u.dim() != 2 or u.shape != i.shape:
            raise ValueError("batch_softmax_loss: user_emb and item_emb must both be [n, d]")
        n, d = u.shape
        if d not in _SUPPORTED_D:
            raise SrbError(f"batch_softmax_loss: embedding size {d} unsupported (16, 32, 64, 128, 256)")
        idx = torch.arange(n, device=u.device, dtype=torch.int32)
        losses, outs = infonce_raw([dict(table1=u, table2=i, idx=idx, n=n, weight=1.0)], d, temperature, True,
                                   batch_softmax=True)
        ctx.save_for_backward(*outs[0])
        return losses[0]

    @staticmethod
    def backward(ctx, go):
        g1, g2 = ctx.saved_tensors
        return g1 * go, g2 * go, None


def batch_softmax_loss(user_emb, item_emb, temperature):
    """util/loss_torch.py:25-32: mean_r -log(softmax(S)_rr + 1e-5), S = normalize(user) normalize(item)^T / temperature.
    Computed in log-sum-exp form, so it stays finite below temperature 1/88.7, where the reference overflows."""
    return _BatchSoftmaxFn.apply(user_emb, item_emb, float(temperature))


# ----------------------------------------------------------------------------------------
# scoring + top-k
# ----------------------------------------------------------------------------------------
def score_topk(user_emb, item_emb, users, rated_ptr, rated_idx, k, impl=0, stats=None):
    """ids [n_q, k] int32, scores [n_q, k] fp32 for the listed users (masked, score-descending).
    stats: optional dict; impl 2 stores the fallback-counter tensor view under "fallback_count"."""
    lib = _lib.require_device()
    user_emb, item_emb = _f32c(user_emb, "score user_emb"), _f32c(item_emb, "score item_emb")
    dev = user_emb.device
    users = _i32(users, dev)
    n_q = users.numel()
    d = user_emb.shape[1]
    if not 1 <= int(k) <= item_emb.shape[0]:
        raise SrbError(f"score_topk: k={k} must be in 1..n_items={item_emb.shape[0]} (find_k_largest seeds its heap with the first K candidates)")
    if k > TOPK_KERNEL_MAX and not (impl in (0, 2) and long_list_route(d, item_emb.shape[0], k, impl)):
        return _score_topk_wide(user_emb, item_emb, users, rated_ptr, rated_idx, int(k))
    out_ids = torch.empty((n_q, k), device=dev, dtype=torch.int32)
    out_sc = torch.empty((n_q, k), device=dev, dtype=torch.float32)
    desc = _lib.TopkDesc()
    desc.user_emb, desc.item_emb, desc.n_items, desc.d = _p(user_emb), _p(item_emb), item_emb.shape[0], d
    desc.users, desc.n_q = _p(users), n_q
    if rated_ptr is not None:
        rated_ptr, rated_idx = _i32(rated_ptr, dev), _i32(rated_idx, dev)
        desc.rated_ptr, desc.rated_idx = _p(rated_ptr), _p(rated_idx)
    if impl == 0:  # auto: tensor-core path where it is measured faster, else the CUDA-core kernel
        impl = 2 if _tc_route(d, item_emb.shape[0], 0) else 1
    desc.k, desc.out_ids, desc.out_scores, desc.impl = k, _p(out_ids), _p(out_sc), impl
    ws = None
    if impl == 2:
        nb = lib.srb_topk_workspace_bytes(n_q, item_emb.shape[0], d, k)
        ws = torch.empty(max(nb, 16), device=dev, dtype=torch.uint8)
        desc.workspace, desc.workspace_bytes = _p(ws), nb
    _lib.check(lib.srb_score_topk(C.byref(desc), _stream()), "srb_score_topk")
    if stats is not None and impl == 2 and n_q > 0:
        off = lib.srb_topk_fallback_count_offset(n_q, item_emb.shape[0])
        stats["fallback_count"] = ws[off:off + 4].view(torch.int32)
    return out_ids, out_sc


TOPK_KERNEL_MAX = 32  # list length of the selection kernels (one entry per lane)
TOPK_TC_MAX = 256     # longest list of the tensor-core route (impl 2)
TOPK_TC_WIDTHS = (16, 32, 64, 128, 256)       # embedding sizes impl 2 is built for
TOPK_TC_AUTO_WIDTHS = (16, 32, 64, 128, 256)  # auto (impl 0) takes impl 2 for lists of up to 32 (DESIGN 9.4)
TOPK_TC_LONG_AUTO_WIDTHS = (64, 128)          # ... and for lists of 33..256


def long_list_route(d, n_items, k, impl=0):
    """True when score_topk ranks a list of k > 32 on the tensor cores (impl 2, candidate buffers behind a running
    threshold) rather than from dense score rows (_score_topk_wide): k <= 256, and either impl 2 asked for explicitly
    (every width) or, under impl 0, d in {64, 128} from 1024 items on."""
    return TOPK_KERNEL_MAX < int(k) <= TOPK_TC_MAX and _tc_route(d, n_items, impl, TOPK_TC_LONG_AUTO_WIDTHS)


def _tc_route(d, n_items, impl, auto_widths=TOPK_TC_AUTO_WIDTHS):
    """True when impl 2 (tensor cores) ranks at this width: asked for explicitly, or under impl 0 (auto) at one of
    auto_widths from 1024 items on."""
    d, impl = int(d), int(impl)
    return d in TOPK_TC_WIDTHS and (impl == 2 or (impl == 0 and d in auto_widths and int(n_items) >= 1024))


def _score_topk_wide(user_emb, item_emb, users, rated_ptr, rated_idx, k):
    """Lists above 32 off the tensor-core route (other widths, small catalogues, k > 256; long_list_route): the
    selection kernels keep 32 entries per user, so the list is
    extracted 32 at a time from dense score rows -- srb_score_rows (the exact fp32 fma chains of predict()), the rated
    items masked with -10e8 like graph_recommender.py:48-50, srb_topk_rows, the winners struck out, repeat -- in
    user blocks of 2048.  Same selection rule (strictly greater replaces the minimum: earliest ids win ties at the
    cut) and the same order (score descending, ties by id descending) as the single-pass kernels."""
    dev = user_emb.device
    n_q, n_items = users.numel(), item_emb.shape[0]
    out_ids = torch.empty((n_q, k), device=dev, dtype=torch.int32)
    out_sc = torch.empty((n_q, k), device=dev, dtype=torch.float32)
    rp = None
    if rated_ptr is not None:
        rp, ri = _i32(rated_ptr, dev).long(), _i32(rated_idx, dev).long()
    for lo in range(0, n_q, 2048):
        blk = users[lo:lo + 2048]
        rows = score_rows(user_emb, item_emb, blk)
        if rp is not None:
            cnt = rp[blk.long() + 1] - rp[blk.long()]
            r = torch.repeat_interleave(torch.arange(blk.numel(), device=dev), cnt)
            c = ri[torch.repeat_interleave(rp[blk.long()], cnt) + (torch.arange(int(cnt.sum()), device=dev) - torch.repeat_interleave(torch.cumsum(cnt, 0) - cnt, cnt))]
            rows[r, c] = -10e8
        ids_parts, sc_parts = [], []
        left = k
        while left > 0:
            kk = min(left, TOPK_KERNEL_MAX)
            ids, sc = topk_rows(rows, kk)
            ids_parts.append(ids)
            sc_parts.append(sc)
            rows.scatter_(1, ids.long(), float("-inf"))
            left -= kk
        ids, sc = torch.cat(ids_parts, 1), torch.cat(sc_parts, 1)
        # one order for the whole list: score descending, ties by id descending (ties may straddle a 32-entry pass)
        o = torch.sort(ids, dim=1, descending=True, stable=True).indices
        ids, sc = torch.gather(ids, 1, o), torch.gather(sc, 1, o)
        o = torch.sort(sc, dim=1, descending=True, stable=True).indices
        out_ids[lo:lo + 2048], out_sc[lo:lo + 2048] = torch.gather(ids, 1, o), torch.gather(sc, 1, o)
    return out_ids, out_sc


def score_rows(user_emb, item_emb, users):
    """Dense fp32 scores [n_q, n_items] for the listed user ids."""
    lib = _lib.require_device()
    user_emb, item_emb = _f32c(user_emb, "score user_emb"), _f32c(item_emb, "score item_emb")
    users = _i32(users, user_emb.device)
    out = torch.empty((users.numel(), item_emb.shape[0]), device=user_emb.device, dtype=torch.float32)
    _lib.check(lib.srb_score_rows(_p(user_emb), _p(item_emb), user_emb.shape[1], _p(users), users.numel(), item_emb.shape[0],
                                  _p(out), _stream()), "srb_score_rows")
    return out


def topk_rows(scores, k):
    lib = _lib.require_device()
    scores = _f32c(scores, "topk scores")
    n_q, n_items = scores.shape
    if not 1 <= int(k) <= TOPK_KERNEL_MAX:
        raise SrbError(f"topk_rows: k={k} outside 1..{TOPK_KERNEL_MAX} (score_topk extracts longer lists 32 at a time)")
    out_ids = torch.empty((n_q, k), device=scores.device, dtype=torch.int32)
    out_sc = torch.empty((n_q, k), device=scores.device, dtype=torch.float32)
    _lib.check(lib.srb_topk_rows(_p(scores), n_q, n_items, k, _p(out_ids), _p(out_sc), _stream()), "srb_topk_rows")
    return out_ids, out_sc


# ----------------------------------------------------------------------------------------
# neighbourhood baselines (ItemKNN / UserKNN)
# ----------------------------------------------------------------------------------------
def _i32c(t, name):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name}: expected a torch.Tensor")
    if not t.is_cuda:
        raise SrbError(f"{name}: selfrec_b200 ops need CUDA tensors (no CPU fallback)")
    if t.dtype != torch.int32:
        raise TypeError(f"{name}: expected int32, got {t.dtype}")
    t = t.contiguous()
    return t if t.numel() else torch.zeros(1, dtype=torch.int32, device=t.device)  # an empty list still needs an address


def knn_neighbors(row_ptr, row_idx, t_ptr, t_idx, rank, topk, shrinkage):
    """Neighbour table of the rows of a binary CSR (row_ptr, row_idx) against each other through its transpose (t_ptr,
    t_idx): the topk rows b != a of largest (sim, rank[b]), sim as in ItemKNN.py:14-30.  Device int32 inputs.
    Returns (ids int32 [n_rows, topk], sims float64 [n_rows, topk], counts int32 [n_rows]); entries past counts[a]
    are -1 / 0."""
    lib = _lib.require_device()
    topk, shrinkage = int(topk), int(shrinkage)
    if not 1 <= topk <= _lib.KNN_MAX_TOPK:
        raise SrbError(f"knn_neighbors: topK={topk} outside 1..{_lib.KNN_MAX_TOPK}")
    if shrinkage < 0:
        raise SrbError(f"knn_neighbors: shrinkage={shrinkage} must be >= 0")
    row_ptr, row_idx = _i32c(row_ptr, "knn row_ptr"), _i32c(row_idx, "knn row_idx")
    t_ptr, t_idx, rank = _i32c(t_ptr, "knn t_ptr"), _i32c(t_idx, "knn t_idx"), _i32c(rank, "knn rank")
    n = row_ptr.numel() - 1
    if n < 1 or rank.numel() != n:
        raise SrbError(f"knn_neighbors: {n} rows and {rank.numel()} name ranks")
    dev = row_ptr.device
    rows = _lib.KnnRows(_p(row_ptr), _p(row_idx), _p(t_ptr), _p(t_idx), _p(rank), n)
    ws_bytes = int(lib.srb_knn_neighbors_workspace_bytes(n))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    ids = torch.empty((n, topk), dtype=torch.int32, device=dev)
    sims = torch.empty((n, topk), dtype=torch.float64, device=dev)
    cnt = torch.empty(n, dtype=torch.int32, device=dev)
    _lib.check(lib.srb_knn_neighbors(C.byref(rows), topk, shrinkage, _p(ids), _p(sims), _p(cnt), _p(ws), ws_bytes, _stream()),
               "srb_knn_neighbors")
    return ids, sims, cnt


KNN_ITEM, KNN_USER = 0, 1  # srb_knn_score_rows modes


def knn_score_rows(mode, users, n_items, table, seq_ptr, seq_idx, rated_ptr=None, rated_idx=None):
    """Float64 predict() rows [len(users), n_items] of ItemKNN (mode KNN_ITEM: seq = each user's items in training_set_u
    order, table = the items' neighbours) or UserKNN (KNN_USER: seq = each user's items, table = the users' neighbours);
    table = knn_neighbors(...).  With rated_ptr / rated_idx the rated items are set to -10e8."""
    lib = _lib.require_device()
    ids, sims, cnt = table
    if mode not in (KNN_ITEM, KNN_USER):
        raise SrbError(f"knn_score_rows: mode={mode} (KNN_ITEM or KNN_USER)")
    if sims.dtype != torch.float64 or not sims.is_cuda or sims.shape != ids.shape:
        raise SrbError("knn_score_rows: the table's sims must be a CUDA float64 tensor shaped like its ids")
    dev = ids.device
    users = _i32(users, dev)
    n_q = users.numel()
    users = _i32c(users, "knn users")
    if (rated_ptr is None) != (rated_idx is None):
        raise SrbError("knn_score_rows: rated_ptr and rated_idx go together")
    rp = None if rated_ptr is None else _i32c(_i32(rated_ptr, dev), "knn rated_ptr")
    ri = None if rated_idx is None else _i32c(_i32(rated_idx, dev), "knn rated_idx")
    seq_ptr, seq_idx = _i32c(_i32(seq_ptr, dev), "knn seq_ptr"), _i32c(_i32(seq_idx, dev), "knn seq_idx")
    out = torch.empty((n_q, int(n_items)), dtype=torch.float64, device=dev)
    _lib.check(lib.srb_knn_score_rows(mode, _p(users), n_q, int(n_items), _p(ids.contiguous()), _p(sims.contiguous()), _p(_i32c(cnt, "knn counts")),
                                      ids.shape[1], _p(seq_ptr), _p(seq_idx), _p(rp), _p(ri), _p(out), _stream()), "srb_knn_score_rows")
    return out


def topk_rows_f64(rows, k):
    """find_k_largest(k, row) of util/algorithm.py:144-156 for every float64 row of rows [n_q, n_items], ties in the
    reference's heap-and-quicksort order; k in 1..n_items.  Returns (ids int32 [n_q, k], scores float64 [n_q, k])."""
    lib = _lib.require_device()
    if not isinstance(rows, torch.Tensor) or not rows.is_cuda or rows.dtype != torch.float64 or rows.dim() != 2:
        raise SrbError("topk_rows_f64: expected a CUDA float64 [n_q, n_items] tensor")
    rows = rows.contiguous()
    n_q, n_items = rows.shape
    k = int(k)
    if not 1 <= k <= n_items:
        raise SrbError(f"topk_rows_f64: k={k} outside 1..n_items={n_items}")
    ws_bytes = int(lib.srb_topk_f64_workspace_bytes(n_q, k))
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=rows.device)
    out_ids = torch.empty((n_q, k), dtype=torch.int32, device=rows.device)
    out_sc = torch.empty((n_q, k), dtype=torch.float64, device=rows.device)
    _lib.check(lib.srb_topk_rows_f64(_p(rows), n_q, n_items, k, _p(out_ids), _p(out_sc), _p(ws), ws_bytes, _stream()), "srb_topk_rows_f64")
    return out_ids, out_sc


# ----------------------------------------------------------------------------------------
# Adam
# ----------------------------------------------------------------------------------------
def adam_prepare(step_dev, scalars, lr, beta1=0.9, beta2=0.999):
    lib = _lib.require_device()
    _lib.check(lib.srb_adam_prepare(_p(step_dev), _p(scalars), lr, beta1, beta2, _stream()), "srb_adam_prepare")


def adam_step(p, m, v, g, scalars, beta1=0.9, beta2=0.999, eps=1e-8):
    lib = _lib.require_device()
    _lib.check(lib.srb_adam_step(_p(p), _p(m), _p(v), _p(g), p.numel(), _p(scalars), beta1, beta2, eps, _stream()), "srb_adam_step")


def rank_hit_masks(topk_ids, users, test_ptr, test_idx):
    """Hit masks of the ranked lists: bit r set iff topk_ids[q, r] is a test item of users[q].  k <= 64: one
    uint64 per query row, int64 [n_q]; 64 < k <= 256: ceil(k / 64) words per row, int64 [n_q, W], bit r % 64 of
    word r // 64.  topk_ids: device int32 [n_q, k]; users / test_ptr / test_idx: int32 arrays or tensors."""
    lib = _lib.require_device()
    dev = topk_ids.device
    ids = topk_ids.contiguous()
    if ids.dtype != torch.int32 or ids.dim() != 2:
        raise TypeError("topk_ids must be an int32 [n_q, k] tensor")
    to = lambda a: a.to(dev) if isinstance(a, torch.Tensor) else torch.as_tensor(np.ascontiguousarray(a, dtype=np.int32)).to(dev)
    users, test_ptr, test_idx = to(users), to(test_ptr), to(test_idx)
    if test_idx.numel() == 0:
        test_idx = torch.zeros(1, dtype=torch.int32, device=dev)
    words = (ids.shape[1] + 63) // 64
    out = torch.zeros((ids.shape[0],) if words == 1 else (ids.shape[0], words), dtype=torch.int64, device=dev)
    _lib.check(lib.srb_rank_hit_masks(_p(ids), ids.shape[0], ids.shape[1], _p(users), _p(test_ptr), _p(test_idx), _p(out), _stream()),
               "srb_rank_hit_masks")
    return out


def scatter_add_segments(dst, segs):
    """dst[rows + off] += scale * src for up to 8 (src, rows, n_dev, n, off, scale) segments, one launch."""
    lib = _lib.require_device()
    arr = (_lib.ScatterSeg * len(segs))()
    for q, (src, rows, n_dev, n, off, scale) in enumerate(segs):
        arr[q].src, arr[q].rows, arr[q].n_dev = _p(src), _p(rows), _p(n_dev)
        arr[q].n, arr[q].row_off, arr[q].scale = int(n), int(off), float(scale)
    _lib.check(lib.srb_scatter_add_segments(_p(dst), dst.shape[1], len(segs), arr, _stream()), "srb_scatter_add_segments")


def scatter_add_rows(dst, src, rows, row_off=0, scale=1.0):
    lib = _lib.require_device()
    rows = _i32(rows, dst.device)
    _lib.check(lib.srb_scatter_add_rows(_p(dst), dst.shape[1], _p(src), _p(rows), rows.numel(), None, row_off, scale, _stream()),
               "srb_scatter_add_rows")
