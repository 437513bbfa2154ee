"""Bipartite-sharded multi-GPU path (SURVEY 8e): one process per GPU.

The normalised adjacency is A = [[0, R], [R^T, 0]].  Rank g owns the USERS u with u % world == g (local row
u // world; their rows of every [U, d] table never leave the GPU); the ITEM tables are replicated.  Per propagation
layer only the item half crosses NVLink: every rank's partial product R_g^T X_u is stored by the SpMM epilogue into the
staging area of the rank owning that item slice, the owner adds the partials, applies the epilogue and stores the
finished rows into every rank's copy (selfrec_b200/csrc/sharded.cu).  torch.distributed is plumbing only: rendezvous
of the symmetric-memory region (peer pointers, multicast mapping); no NCCL collective touches the data path.

Why cyclic and not contiguous nnz-balanced blocks: ids follow first appearance in the training file
(ui_graph.py:29-40), so on a power-law graph the hubs have the low ids -- at config-5 size an nnz-balanced 2-way split
is 142 k users against 9.86 M, and the second rank's products (cold gathers, 70x the rows to write) take 1.5x longer.
Every rank taking each world-th user gets the same mix of degrees, rows and non-zeros.

Host logic here (user assignment, block extraction) is plain tensor code that also runs on CPU tensors and is
exercised with a world-size-2 gloo group in tests/test_sharding_cpu.py.
"""
import ctypes as C
import os

import numpy as np

from . import _lib
from .engine import HostFeed


def local_user_count(n_users, rank, world):
    """Users rank, rank + world, rank + 2 world, ... below n_users."""
    return (int(n_users) - int(rank) + int(world) - 1) // int(world)


def user_ids_of(n_users, rank, world):
    """Global ids of rank's users in local-row order (numpy int64)."""
    return np.arange(int(rank), int(n_users), int(world), dtype=np.int64)


def owner_of(users, world):
    """Rank owning each global user id (numpy int64)."""
    return np.asarray(users, dtype=np.int64) % int(world)


def local_row_of(users, world):
    """Local row of each global user id on its owning rank (numpy int64)."""
    return np.asarray(users, dtype=np.int64) // int(world)


def item_bounds(n_items, world):
    """Item slice whose reduction rank g owns: [g * I / world, (g + 1) * I / world) (sharded.cu)."""
    return np.array([g * n_items // world for g in range(world + 1)], dtype=np.int64)


def extract_blocks(rowptr, colidx, vals, n_users, n_items, rank, world):
    """Rank-local blocks of the normalised (U+I)^2 adjacency given as CSR tensors (any device), for the cyclic user
    assignment: Ru [Ug x I] = rows rank, rank + world, ... of A[:U, U:] (columns: item ids) and Rt [I x Ug] = the
    columns of A[U:, :U] with col % world == rank, renumbered col // world (monotone: the rows stay sorted).
    Returns two (rowptr, colidx, vals) triples of int32 / int32 / fp32 tensors."""
    import torch
    U, I, G, g = int(n_users), int(n_items), int(world), int(rank)
    rp = rowptr.to(torch.int64)
    dev = rp.device
    if G == 1:
        lo, hi = 0, int(rp[U])
        ru = (rp[:U + 1].to(torch.int32), (colidx[lo:hi] - U).to(torch.int32).contiguous(), vals[lo:hi].contiguous())
    else:
        rows = torch.arange(g, U, G, device=dev)
        beg = rp[rows]
        deg = rp[rows + 1] - beg
        ru_ptr = torch.zeros(rows.numel() + 1, dtype=torch.int64, device=dev)
        torch.cumsum(deg, 0, out=ru_ptr[1:])
        total = int(ru_ptr[-1])
        pos = torch.arange(total, device=dev) + torch.repeat_interleave(beg - ru_ptr[:-1], deg, output_size=total)
        ru = (ru_ptr.to(torch.int32), (colidx[pos] - U).to(torch.int32).contiguous(), vals[pos].contiguous())
        del pos, beg, deg, rows
    ilo, ihi = int(rp[U]), int(rp[U + I])
    cols = colidx[ilo:ihi]
    if G == 1:
        rt = ((rp[U:U + I + 1] - ilo).to(torch.int32), cols.to(torch.int32).contiguous(), vals[ilo:ihi].contiguous())
        return ru, rt
    keep = (cols % G) == g
    pref = torch.zeros(ihi - ilo + 1, dtype=torch.int64, device=dev)
    torch.cumsum(keep, 0, out=pref[1:])
    rt_ptr = pref[rp[U:U + I + 1] - ilo].to(torch.int32)
    rt = (rt_ptr, torch.div(cols[keep], G, rounding_mode="floor").to(torch.int32).contiguous(), vals[ilo:ihi][keep].contiguous())
    return ru, rt


class ShardedEngine(HostFeed):
    """LightGCN / SimGCL / XSimGCL / SGL training on bipartite-sharded tables; world == 1 works without torch.distributed.

    Same constructor surface as TrainEngine, and the same batches() / step(words, fetch_loss=...) host feed.  Every rank
    must feed the SAME batch buffer to step(): draw batches() from the same Python `random` state on every rank.
    Parameters: `user_emb` = this rank's users [Ug, d] (global ids `user_ids`: rank, rank + world, ...), `item_emb` = the full
    replicated [I, d] item table.  The in-kernel Philox noise is keyed by global row ids, so a sharded run with the same
    philox_seed draws the noise the single-GPU TrainEngine draws.  SGL needs set_view_graphs() once per epoch."""

    def __init__(self, model, data, emb_size, n_layers, batch_size, lr, reg, *, eps=0.0, tau=0.2, cl_rate=0.0, layer_cl=0,
                 l2_div=1.0, init_user=None, init_item=None, group=None, philox_seed=0x5EED, device=None, multicast=None, nvls=None):
        import torch
        from . import ops
        from .engine import fill_step_fields, fork_resources
        lib = _lib.require_device()
        if model not in ("LightGCN", "SimGCL", "XSimGCL", "SGL"):
            raise _lib.SrbError("the sharded engine covers LightGCN, SimGCL, XSimGCL and SGL")
        if int(emb_size) not in ops._SUPPORTED_D:
            raise _lib.SrbError(f"embedding.size {emb_size} is not supported by the CUDA path {ops._SUPPORTED_D}")
        self.torch, self.ops, self.lib = torch, ops, lib
        self.model_name = model
        self.data = data
        self.dist = None
        self.group = None
        self.rank, self.world = 0, 1
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            self.dist = dist
            self.group = dist.group.WORLD if group is None else group
            self.rank, self.world = dist.get_rank(self.group), dist.get_world_size(self.group)
        if self.world > 8:
            raise _lib.SrbError("the sharded engine supports up to 8 ranks (one NVSwitch domain)")
        self.dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        dev = self.dev
        self.U, self.I, self.d = int(data.user_num), int(data.item_num), int(emb_size)
        self.N, self.L, self.B = self.U + self.I, int(n_layers), int(batch_size)
        # ---- graph blocks of this rank ----
        na = data.norm_adj
        adj = na if isinstance(na, ops.SparseAdj) else ops.SparseAdj(na)
        had = adj.rowptr is not None
        adj.cuda(dev)
        if self.U < self.world:
            raise _lib.SrbError(f"{self.U} users cannot be spread over {self.world} ranks")
        self.Ug = local_user_count(self.U, self.rank, self.world)
        self.user_ids = torch.arange(self.rank, self.U, self.world, device=dev)  # global id of every local row
        ru, rt = extract_blocks(adj.rowptr, adj.colidx, adj.vals, self.U, self.I, self.rank, self.world)
        self.Ru = ops.SparseAdj.from_device(*ru, (self.Ug, self.I), symmetric=False)
        self.Rt = ops.SparseAdj.from_device(*rt, (self.I, self.Ug), symmetric=False)
        self.nnzA = adj.nnz
        if not had and self.world > 1:
            adj.rowptr = adj.colidx = adj.vals = adj.row_order = None  # the full matrix is not needed on the device any more
        self.ib = item_bounds(self.I, self.world)
        # ---- memory ----
        lay = _lib.ShardLayout()
        gu, gt = self.Ru.graph_struct(self.d), self.Rt.graph_struct(self.d)
        self.hub_cap = (int(gu.hub.n_work), int(gt.hub.n_work))  # split-row chunk capacity of the batch-row lists (SGL: views too)
        _lib.check(lib.srb_shard_plan(_lib.MODEL_IDS[model], self.U, self.I, self.Ug, self.d, self.B, self.world, *self.hub_cap,
                                      C.byref(lay)), "srb_shard_plan")
        self.layout = lay
        self.sym_handle = None
        mc_ptr = 0
        if self.world > 1:
            import torch.distributed._symmetric_memory as symm
            self.sym = symm.empty(int(lay.sym_bytes), dtype=torch.uint8, device=dev)
            self.sym_handle = symm.rendezvous(self.sym, self.group)
            peers = [int(p) for p in self.sym_handle.buffer_ptrs]
            want = os.environ.get("SRB_MULTICAST", "auto") if multicast is None else ("1" if multicast else "0")
            mc = int(getattr(self.sym_handle, "multicast_ptr", 0) or 0)
            if mc and (want == "1" or (want == "auto" and self.world >= 4)):
                mc_ptr = mc
        else:
            self.sym = torch.empty(int(lay.sym_bytes), dtype=torch.uint8, device=dev)
            peers = [self.sym.data_ptr()]
        self.sym.zero_()
        self.use_multicast = bool(mc_ptr)
        self.workspace = torch.zeros(int(lay.workspace_bytes) + 256, dtype=torch.uint8, device=dev)
        ws_ptr = (self.workspace.data_ptr() + 255) // 256 * 256
        self._ctrl = self.workspace[ws_ptr - self.workspace.data_ptr() + int(lay.ctrl):][:8].view(torch.int32)
        nd_i = self.I * self.d
        self.item_emb = self.sym[int(lay.item_params): int(lay.item_params) + 4 * nd_i].view(torch.float32).view(self.I, self.d)
        self._item_final = self.sym[int(lay.item_final): int(lay.item_final) + 4 * nd_i].view(torch.float32).view(self.I, self.d)
        self.user_emb = torch.empty((self.Ug, self.d), device=dev, dtype=torch.float32)
        if init_user is None:
            if self.N * self.d > (1 << 27):  # config-5 sized tables: drawn on the device, identically on every rank
                g = torch.Generator(device=dev).manual_seed(int(philox_seed) & 0x7FFFFFFF)
                bound_u, bound_i = (6.0 / (self.U + self.d)) ** 0.5, (6.0 / (self.I + self.d)) ** 0.5
                chunk = 1 << 20
                for lo in range(0, self.U, chunk):  # the same stream on every rank; keep the owned rows
                    hi = min(self.U, lo + chunk)
                    blk = torch.empty((hi - lo, self.d), device=dev).uniform_(-bound_u, bound_u, generator=g)
                    first = lo + (self.rank - lo) % self.world  # first owned id >= lo
                    if first < hi:
                        mine = blk[first - lo:: self.world]
                        self.user_emb[first // self.world: first // self.world + mine.shape[0]].copy_(mine)
                self.item_emb.uniform_(-bound_i, bound_i, generator=g)
            else:
                g = torch.Generator().manual_seed(int(philox_seed) & 0x7FFFFFFF)  # every rank starts from the same tables
                init_user = torch.nn.init.xavier_uniform_(torch.empty(self.U, self.d), generator=g)
                init_item = torch.nn.init.xavier_uniform_(torch.empty(self.I, self.d), generator=g)
        if init_user is not None:
            self.user_emb.copy_(torch.as_tensor(init_user)[self.rank:: self.world])
            self.item_emb.copy_(torch.as_tensor(init_item))
        self.mu, self.vu = torch.zeros_like(self.user_emb), torch.zeros_like(self.user_emb)
        self.mi = torch.zeros((self.I, self.d), device=dev)
        self.vi = torch.zeros((self.I, self.d), device=dev)
        self.step_dev = torch.zeros(1, dtype=torch.int32, device=dev)
        self.scalars = torch.zeros(16, device=dev)
        self.losses = torch.zeros(4, device=dev)
        self.words = _lib.BATCH_HEADER + 5 * self.B
        self.batch_dev = torch.zeros(self.words, dtype=torch.int32, device=dev)
        self._init_feed()
        s = _lib.ShardDesc()
        fill_step_fields(s, model, self.U, self.I, self.d, self.L, self.B, lr=lr, reg=reg, eps=eps, tau=tau, cl_rate=cl_rate,
                         layer_cl=layer_cl, l2_div=l2_div, philox_seed=philox_seed)
        s.world, s.rank = self.world, self.rank
        s.Ru, s.Rt = gu, gt
        p = ops._p
        s.batch, s.pu, s.mu, s.vu, s.mi, s.vi = p(self.batch_dev), p(self.user_emb), p(self.mu), p(self.vu), p(self.mi), p(self.vi)
        s.step_dev, s.scalars, s.losses = p(self.step_dev), p(self.scalars), p(self.losses)
        for g in range(self.world):
            s.sym[g] = peers[g]
        s.sym_mc = mc_ptr or None
        s.sym_bytes = int(lay.sym_bytes)
        s.workspace, s.workspace_bytes = C.c_void_p(ws_ptr), int(lay.workspace_bytes)
        if self.world > 1 and os.environ.get("SRB_SHARD_OVERLAP", "1") != "0":
            # the owner-side reduction of a layer runs on this stream beside the user-side product
            self._fork_stream, self._fork_events = fork_resources(s, dev)
        want_nvls = (os.environ.get("SRB_SHARD_NVLS", "0") == "1") if nvls is None else bool(nvls)
        s.nvls = 1 if (want_nvls and mc_ptr) else 0
        self.use_nvls = bool(s.nvls)
        self.desc = s
        self.hyper = dict(lr=float(lr), reg=float(reg), eps=float(eps), tau=float(tau), cl_rate=float(cl_rate), layer_cl=int(layer_cl),
                          l2_div=float(l2_div), philox_seed=int(philox_seed))
        self.view_blocks = None
        self.graph = None
        self._warm = False
        torch.cuda.synchronize()
        self._host_barrier()

    # ---- configuration -------------------------------------------------------------------
    def set_view_graphs(self, adj1, adj2):
        """SGL: the epoch's two dropped, re-normalised (U+I)^2 graphs (SGL.py:27-29; e.g. DeviceBipartite.assemble output),
        drawn identically on every rank.  Keeps this rank's Ru / Rt blocks of each; the full views are not kept.  Drops a
        captured graph (capture() again, on every rank)."""
        torch, ops = self.torch, self.ops
        if self.model_name != "SGL":
            raise _lib.SrbError(f"set_view_graphs: {self.model_name} has no view graphs")
        views = []
        for k, a in enumerate((adj1, adj2)):
            a = a if isinstance(a, ops.SparseAdj) else ops.SparseAdj(a)
            if tuple(a.shape) != (self.N, self.N):
                raise ValueError(f"set_view_graphs: view {k + 1} is {tuple(a.shape)}, the graph is {(self.N, self.N)}")
            a.cuda(self.dev)
            ru, rt = extract_blocks(a.rowptr, a.colidx, a.vals, self.U, self.I, self.rank, self.world)
            bru = ops.SparseAdj.from_device(*ru, (self.Ug, self.I), symmetric=False)
            brt = ops.SparseAdj.from_device(*rt, (self.I, self.Ug), symmetric=False)
            gu, gt = bru.graph_struct(self.d), brt.graph_struct(self.d)
            if gu.hub.n_work > self.hub_cap[0] or gt.hub.n_work > self.hub_cap[1]:
                raise _lib.SrbError(f"set_view_graphs: view {k + 1} has more split-row chunks ({gu.hub.n_work}, {gt.hub.n_work}) than "
                                    f"the graph the workspace was planned for ({self.hub_cap[0]}, {self.hub_cap[1]})")
            views.append((a, bru, brt, gu, gt))
        if self.dist is not None and self.world > 1:
            # every rank must have drawn the same views: their nnz and a position-weighted sum of their column indices
            sig = []
            for a, *_ in views:
                w = torch.arange(a.nnz, device=self.dev, dtype=torch.int64) % 65521 + 1
                sig += [a.nnz, int((a.colidx.to(torch.int64) * w).sum().item())]
            t = torch.tensor(sig + [-x for x in sig], dtype=torch.int64,
                             device=self.dev if self.dist.get_backend(self.group) == "nccl" else "cpu")
            self.dist.all_reduce(t, op=self.dist.ReduceOp.MAX, group=self.group)
            hi, lo = t[: len(sig)].tolist(), [-x for x in t[len(sig):].tolist()]
            if hi != lo:
                raise _lib.SrbError("set_view_graphs: the ranks drew different view graphs (seed every rank's `random` alike)")
        self.view_blocks = [(bru, brt) for _a, bru, brt, _gu, _gt in views]
        for k, (_a, _bru, _brt, gu, gt) in enumerate(views):
            self.desc.Ru_view[k], self.desc.Rt_view[k] = gu, gt
        self.graph = None  # pointers changed: a captured graph is stale

    # ---- plumbing ------------------------------------------------------------------------
    def _host_barrier(self):
        if self.dist is not None and self.world > 1:
            self.dist.barrier(self.group)

    def _quiesce(self):
        """Every rank's enqueued work finished, peer stores included: drain this device, then a host barrier (each rank
        passes it only after its own device is drained, so every store a peer made into this rank's memory has landed)."""
        self.torch.cuda.synchronize(self.dev)
        self._host_barrier()

    def all_ok(self, ok):
        """True when `ok` is true on every rank (one all-reduce; a rank that failed tells the others instead of leaving
        them in a barrier).  Collective."""
        if self.dist is None or self.world == 1:
            return bool(ok)
        torch = self.torch
        dev = self.dev if self.dist.get_backend(self.group) == "nccl" else "cpu"
        t = torch.tensor([0 if ok else 1], dtype=torch.int32, device=dev)
        self.dist.all_reduce(t, op=self.dist.ReduceOp.MAX, group=self.group)
        return int(t.item()) == 0

    def check_peers(self):
        """Raise if a device-side barrier ever timed out (a peer died or fell out of step)."""
        if int(self._ctrl[1].item()) != 0:
            raise _lib.SrbError("sharded step: a peer rank did not reach a device-side barrier in time")

    def nvlink_bytes_per_layer(self):
        """Bytes this rank sends per propagation layer: the partial rows it hands to the other slices' owners plus
        the finished rows of its own slice (one multicast store, or one store per peer)."""
        if self.world == 1:
            return 0
        own = int(self.ib[self.rank + 1] - self.ib[self.rank]) * self.d * 4
        part = self.I * self.d * 4 - own
        return part + own * (1 if self.use_multicast else self.world - 1)

    # ---- stepping ------------------------------------------------------------------------
    def _enqueue(self):
        _lib.check(self.lib.srb_shard_step(C.byref(self.desc), self.ops._stream()), "srb_shard_step")

    def step(self, words=None, words_dev=None, fetch_loss=False):
        """One step on host batch words (copied through a pinned slot), on a device batch buffer, or on whatever
        batch_dev holds.  fetch_loss=True returns a LossHandle, as TrainEngine.step does."""
        if words_dev is not None:
            self.batch_dev.copy_(words_dev, non_blocking=True)
        elif words is not None:
            self._feed(words)
        self.step_resident()
        return self._fetch_loss() if fetch_loss else None

    def step_resident(self):
        if self.graph is not None:
            self.graph.replay()
        else:
            self._enqueue()

    def capture(self):
        """CUDA graph of one step (device-side barriers included).  Collective: every rank must call it."""
        from .engine import capture_step
        state = (self.user_emb, self.item_emb, self.mu, self.vu, self.mi, self.vi, self.step_dev, self.losses)
        self.graph = capture_step(self._enqueue, state, self._warm, 1, self._host_barrier)
        self._warm = True
        return self.graph

    # ---- checkpoints -----------------------------------------------------------------------
    def state_dict(self):
        """This rank's training state on the host, in TrainEngine.state_dict()'s layout: its users' rows (global ids
        `user_ids`) of the parameters and moments, the replicated item table, and the item moments of the slice
        [ib[rank], ib[rank + 1]) whose reduction it owns (only the owner updates those rows of mi / vi).

        Collective.  A step returns without waiting for its peers: the owners' last item stores into this rank's copy of
        the item table (the Adam epilogue of the owner-side reduction) may still be in flight when this rank's own stream
        is done.  Every rank therefore drains its device and meets the others at a barrier before anything is read."""
        self._quiesce()
        lo, hi = int(self.ib[self.rank]), int(self.ib[self.rank + 1])
        return {"step": int(self.step_dev.item()), "user_ids": self.user_ids.cpu().numpy().astype(np.int64),
                "user": {"params": self.user_emb.cpu().numpy(), "m": self.mu.cpu().numpy(), "v": self.vu.cpu().numpy()},
                "item_params": self.item_emb.cpu().numpy(), "item_rows": (lo, hi),
                "item": {"m": self.mi[lo:hi].cpu().numpy(), "v": self.vi[lo:hi].cpu().numpy()}}

    def load_state_dict(self, state):
        """Copy a saved state into this rank's existing tensors (no address moves).  state: step, user {params, m, v}
        [Ug, d] of this rank's users in local-row order, item_params [I, d] and item {m, v} [I, d] (every rank reads the
        same item arrays, so the replicas stay bit-identical).  Collective: no peer's step may still be storing into
        this rank's item table while it is overwritten (see state_dict())."""
        from .engine import copy_rows_in
        self._quiesce()
        for name, dst in (("params", self.user_emb), ("m", self.mu), ("v", self.vu)):
            copy_rows_in(dst, state["user"][name], "user " + name)
        copy_rows_in(self.item_emb, state["item_params"], "item params")
        for name, dst in (("m", self.mi), ("v", self.vi)):
            copy_rows_in(dst, state["item"][name], "item " + name)
        self.step_dev.fill_(int(state["step"]))
        self.torch.cuda.synchronize(self.dev)
        self._host_barrier()

    # ---- inference -------------------------------------------------------------------------
    def forward_clean(self):
        """Clean forward -> (final embeddings of this rank's users [Ug, d], final item embeddings [I, d])."""
        torch = self.torch
        out_u = torch.empty_like(self.user_emb)
        _lib.check(self.lib.srb_shard_forward(C.byref(self.desc), self.ops._p(out_u), self.ops._stream()), "srb_shard_forward")
        return out_u, self._item_final.clone()

    def all_user_rows(self, local):
        """[U, d] table from every rank's [Ug, d] block (test / evaluation plumbing: one NCCL all_gather)."""
        torch = self.torch
        if self.world == 1:
            return local.clone()
        sizes = [local_user_count(self.U, g, self.world) for g in range(self.world)]
        pad = torch.zeros((max(sizes), self.d), device=self.dev)
        pad[: self.Ug].copy_(local)
        outs = [torch.empty_like(pad) for _ in range(self.world)]
        self.dist.all_gather(outs, pad, group=self.group)
        full = torch.empty((self.U, self.d), device=self.dev)
        for g, (o, n) in enumerate(zip(outs, sizes)):
            full[g:: self.world].copy_(o[:n])
        return full
