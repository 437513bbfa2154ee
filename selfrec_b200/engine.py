"""TrainEngine: device state + one fused training step per call (srb_train_step).

Owns (as torch tensors, i.e. PyTorch's allocator) the single contiguous [U+I, d] parameter
table -- users first, items after, so the reference's torch.cat (LightGCN.py:69) disappears
-- the Adam moments, the step counter, the workspace and the device batch buffer.  step()
enqueues one H2D copy of the batch words plus the whole forward/backward/Adam sequence on
the current stream; nothing synchronises.  capture() wraps the same sequence in a CUDA graph.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib, ops
from .util.sampler import NativePairSampler, permute_training_data, stream_epoch


class LossHandle:
    """Pinned-memory copy of a step's [rec, l2, cl, total] losses; get() waits for the D2H copy."""

    __slots__ = ("_buf", "_ev")

    def __init__(self, buf, ev):
        self._buf, self._ev = buf, ev

    def get(self):
        self._ev.synchronize()
        return self._buf.numpy().copy()


def fill_step_fields(desc, model, n_users, n_items, d, n_layers, batch_cap, *, lr, reg, eps, tau, cl_rate, layer_cl, l2_div,
                     philox_seed):
    """The model, shape and hyperparameter fields that srb_step_desc and srb_shard_desc share."""
    desc.model, desc.n_users, desc.n_items, desc.d, desc.n_layers = _lib.MODEL_IDS[model], n_users, n_items, d, n_layers
    desc.batch_cap, desc.layer_cl = batch_cap, int(layer_cl)
    desc.eps, desc.tau, desc.cl_rate, desc.reg = float(eps), float(tau), float(cl_rate), float(reg)
    desc.lr, desc.beta1, desc.beta2, desc.adam_eps = float(lr), 0.9, 0.999, 1e-8
    desc.l2_div = float(l2_div)
    desc.noise_mode = 2 if model in ("SimGCL", "XSimGCL") else 0  # in-kernel Philox noise (MF, LightGCN, SGL: none)
    desc.philox_seed = int(philox_seed)


def fork_resources(desc, device):
    """A side stream and two events of the engine's own, set as desc.fork_stream / fork_event / join_event, so that two
    engines on one device never share events.  Returns (stream, events): the caller keeps them alive."""
    stream = torch.cuda.Stream(device=device)
    events = (torch.cuda.Event(), torch.cuda.Event())
    for ev in events:
        ev.record(stream)  # torch creates the CUDA event lazily, on first record
    desc.fork_stream = C.c_void_p(stream.cuda_stream)
    desc.fork_event, desc.join_event = (C.c_void_p(ev.cuda_event) for ev in events)
    return stream, events


def capture_step(enqueue, state, warm, warmups, barrier=lambda: None):
    """CUDA graph of one enqueue().  Unless `warm`, first runs `warmups` eager steps outside the capture (lazy module
    load, smem attributes).  A warm-up IS a training step on whatever the batch buffer holds: the tensors in `state`
    (parameters, moments, the step counter that keys Adam's bias correction and the Philox stream) are put back
    afterwards, so capturing never changes the training trajectory.  `barrier` keeps the ranks of a multi-process
    engine together around the warm-up, the restore and the capture."""
    torch.cuda.synchronize()
    if not warm:
        saved = [t.clone() for t in state]
        barrier()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmups):
                enqueue()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        barrier()
        for dst, src in zip(state, saved):
            dst.copy_(src)
        del saved
        torch.cuda.synchronize()
        barrier()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        enqueue()
    barrier()
    return g


def copy_rows_in(dst, src, what, chunk=1 << 20):
    """dst [n, d] (device tensor, written in place) <- src [n, d] (numpy array or memmap), `chunk` rows at a time so a
    memory-mapped source is never read into host memory whole."""
    if tuple(src.shape) != tuple(dst.shape):
        raise _lib.SrbError(f"load_state_dict: {what} is {tuple(src.shape)}, the engine's is {tuple(dst.shape)}")
    for lo in range(0, dst.shape[0], chunk):
        hi = min(dst.shape[0], lo + chunk)
        dst[lo:hi].copy_(torch.from_numpy(np.require(src[lo:hi], np.float32, ["C", "W"])))  # a read-only map is copied


def initial_tables(n_users, n_items, out):
    """The reference's initial tables, drawn into `out` [U+I, d] (any device) from torch's global state: CPU
    xavier_uniform_ users then items, the same initialiser calls in the same order as LightGCN.py:60-66; above 2^27
    elements (config-5 sized tables, where a 6 GB host tensor is not worth its copy) xavier-uniform drawn on out's
    device from a generator keyed by torch.initial_seed().  Returns (out[:U], out[U:])."""
    U, N, d = int(n_users), int(n_users) + int(n_items), out.shape[1]
    if N * d > (1 << 27):
        g = torch.Generator(device=out.device).manual_seed(torch.initial_seed() & 0x7FFFFFFF)
        for lo, hi in ((0, U), (U, N)):
            bound = (6.0 / ((hi - lo) + d)) ** 0.5
            out[lo:hi].uniform_(-bound, bound, generator=g)
    else:
        out[:U].copy_(torch.nn.init.xavier_uniform_(torch.empty(U, d)))
        out[U:].copy_(torch.nn.init.xavier_uniform_(torch.empty(N - U, d)))
    return out[:U], out[U:]


class HostFeed:
    """Host side of a training engine, shared by TrainEngine and the sharded engine: the epoch's batch words from the
    native sampler, their copy through a ring of pinned slots into `batch_dev`, and the pinned D2H copy of `losses`.
    The engine sets data, B, words, batch_dev and losses, then calls _init_feed()."""

    def _init_feed(self):
        self.ring = [torch.zeros(self.words, dtype=torch.int32).pin_memory() for _ in range(8)]
        self.ring_ev = [None] * len(self.ring)
        self.ring_pos = 0
        self.loss_ring = [torch.zeros(4, dtype=torch.float32).pin_memory() for _ in range(8)]
        self.loss_pos = 0
        self.sampler = None

    def _feed(self, batch_words):
        """Enqueue the H2D copy of one batch through the next pinned slot."""
        slot = self.ring_pos
        self.ring_pos = (slot + 1) % len(self.ring)
        ev = self.ring_ev[slot]
        if ev is not None:
            ev.synchronize()  # the copy that last used this pinned slot has finished
        pin = self.ring[slot]
        if isinstance(batch_words, torch.Tensor):
            pin.copy_(batch_words)
        else:
            pin.numpy()[:] = batch_words
        self.batch_dev.copy_(pin, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self.ring_ev[slot] = ev

    def _fetch_loss(self):
        """Enqueue the D2H copy of the four loss values; returns a LossHandle."""
        ls = self.loss_pos
        self.loss_pos = (ls + 1) % len(self.loss_ring)
        self.loss_ring[ls].copy_(self.losses, non_blocking=True)
        lev = torch.cuda.Event()
        lev.record()
        return LossHandle(self.loss_ring[ls], lev)

    def _sampler(self):
        if self.sampler is None:
            self.sampler = NativePairSampler(self.data, track_order=getattr(self, "_track_order", False))
        return self.sampler

    def track_pair_order(self):
        """Have the sampler keep the pair order as file positions, which feed_state() records (one n_pairs gather per
        epoch; off by default).  Call it before the first epoch: an order shuffled untracked cannot be recovered."""
        self._track_order = True
        if self.sampler is not None:
            self.sampler.track_order()

    def feed_state(self):
        """The sampler's position between two batches: {"order": int64 file positions of the pairs, "cursor": pairs
        consumed in the open epoch (-1 between epochs), "random": Python's `random` state at that point}."""
        order, cursor, st = self._sampler().position()
        return {"order": order, "cursor": cursor, "random": st}

    def load_feed_state(self, state):
        """Restore feed_state(): the next batches() continues the saved epoch (or starts the next one)."""
        self._sampler().restore(self.data, state["order"], state["cursor"], state["random"])

    def batches(self, exact_lazy=False):
        """One epoch of batch words from the native sampler (advances Python's `random`).  The yielded buffer is
        reused: consume it (step() copies it into a pinned slot) before asking for the next one.  exact_lazy=True
        hands Python's `random` state back after every batch, like the reference's generator would.  After
        load_feed_state() of a mid-epoch position, the first call continues that epoch."""
        s = self._sampler()
        if not exact_lazy:
            yield from stream_epoch(s, self.data, self.B, self.B)
            return
        resume, s._resume = s._resume, False
        if not resume:
            s.pull_state()
            perm = s.begin_epoch(want_perm=True)
            permute_training_data(self.data, perm)
            s.push_state()
        buf = np.empty(self.words, dtype=np.int32)
        while True:
            s.pull_state()
            b = s.next_batch(self.B, self.B, buf)
            s.push_state()
            if b == 0:
                return
            yield buf


class TrainEngine(HostFeed):
    def __init__(self, model, data, emb_size, n_layers, batch_size, lr, reg, *, eps=0.0, tau=0.2, cl_rate=0.0,
                 layer_cl=0, l2_div=1.0, device=None, init_user=None, init_item=None, philox_seed=0x5EED):
        lib = _lib.require_device()
        self.lib = lib
        if model not in _lib.MODEL_IDS:
            raise ValueError(f"TrainEngine: unknown model {model!r} (one of {sorted(_lib.MODEL_IDS)})")
        if int(emb_size) not in ops._SUPPORTED_D:
            raise _lib.SrbError(f"TrainEngine: embedding.size {emb_size} is not supported by the CUDA path "
                                f"(supported: {ops._SUPPORTED_D}); there is no fallback")
        if int(batch_size) <= 0:
            raise ValueError("TrainEngine: batch.size must be positive")
        self.model_name = model
        self.model_id = _lib.MODEL_IDS[model]
        self.data = data
        self.U, self.I, self.d = int(data.user_num), int(data.item_num), int(emb_size)
        self.N = self.U + self.I
        self.L = int(n_layers) if model != "MF" else 0
        self.B = int(batch_size)
        self.dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        dev = self.dev
        self.params = torch.empty((self.N, self.d), device=dev, dtype=torch.float32)
        if init_user is None:
            initial_tables(self.U, self.I, self.params)
        else:
            self.params[: self.U].copy_(init_user)
            self.params[self.U:].copy_(init_item)
        self.m = torch.zeros_like(self.params)
        self.v = torch.zeros_like(self.params)
        self.step_dev = torch.zeros(1, device=dev, dtype=torch.int32)
        self.scalars = torch.zeros(16, device=dev, dtype=torch.float32)
        self.losses = torch.zeros(4, device=dev, dtype=torch.float32)
        self.words = _lib.BATCH_HEADER + 5 * self.B
        self.batch_dev = torch.zeros(self.words, device=dev, dtype=torch.int32)
        self._init_feed()
        self.adj = None
        if model != "MF":
            na = data.norm_adj
            self.adj = na if isinstance(na, ops.SparseAdj) else ops.SparseAdj(na)
            self.adj.cuda(dev)
        ws_bytes = lib.srb_step_workspace_bytes(self.model_id, self.N, self.d, self.B, self.adj.hub_struct(self.d).n_work if self.adj is not None else 0)
        self.workspace = torch.empty(ws_bytes + 256, device=dev, dtype=torch.uint8)
        ws_ptr = (self.workspace.data_ptr() + 255) // 256 * 256
        self.view_adj = [None, None]
        self.noise = None
        s = _lib.StepDesc()
        fill_step_fields(s, model, self.U, self.I, self.d, self.L, self.B, lr=lr, reg=reg, eps=eps, tau=tau, cl_rate=cl_rate,
                         layer_cl=layer_cl, l2_div=l2_div, philox_seed=philox_seed)
        if self.adj is not None:
            s.adj = self.adj.graph_struct(self.d)
        s.batch, s.params, s.adam_m, s.adam_v = ops._p(self.batch_dev), ops._p(self.params), ops._p(self.m), ops._p(self.v)
        s.step_dev, s.scalars, s.losses = ops._p(self.step_dev), ops._p(self.scalars), ops._p(self.losses)
        s.workspace, s.workspace_bytes = C.c_void_p(ws_ptr), ws_bytes
        self._fork_stream, self._fork_events = fork_resources(s, self.dev)  # BPR beside InfoNCE
        self.desc = s
        self.eps, self.layer_cl = float(eps), int(layer_cl)
        self.hyper = dict(lr=float(lr), reg=float(reg), eps=float(eps), tau=float(tau), cl_rate=float(cl_rate), layer_cl=int(layer_cl),
                          l2_div=float(l2_div), philox_seed=int(philox_seed))
        self.graph = None
        self._warm = False

    # ---- parameters as the reference exposes them ------------------------------------
    @property
    def user_emb(self):
        return self.params[: self.U]

    @property
    def item_emb(self):
        return self.params[self.U:]

    # ---- configuration -----------------------------------------------------------------
    def set_noise_tensor(self, noise):
        """Parity mode: noise is an INPUT, uniform[0,1) of shape [views, L, N, d]."""
        noise = ops._f32c(noise, "noise")
        views = 2 if self.model_name == "SimGCL" else 1
        if tuple(noise.shape) != (views, self.L, self.N, self.d):
            raise ValueError(f"noise must be [{views}, {self.L}, {self.N}, {self.d}]")
        self.noise = noise
        self.desc.noise_mode, self.desc.noise = 1, ops._p(noise)
        self.graph = None  # the step sequence changed: a captured graph is stale

    def set_view_graphs(self, adj1, adj2):
        """SGL: the two dropped, re-normalised graphs of this epoch (SGL.py:27-29)."""
        self.view_adj = [a if isinstance(a, ops.SparseAdj) else ops.SparseAdj(a) for a in (adj1, adj2)]
        for k, a in enumerate(self.view_adj):
            a.cuda(self.dev)
            self.desc.adj_view[k] = a.graph_struct(self.d)
        self.graph = None  # pointers changed: a captured graph is stale

    # ---- stepping ------------------------------------------------------------------------
    def _enqueue(self):
        _lib.check(self.lib.srb_train_step(C.byref(self.desc), ops._stream()), "srb_train_step")

    def step(self, batch_words, fetch_loss=False):
        """batch_words: int32 array/tensor of `words` entries laid out by srb_sampler_next_batch.
        Enqueues the H2D copy and the step (the captured CUDA graph when capture() was called) and
        returns without synchronising.  fetch_loss=True also enqueues a D2H copy of the four loss
        values into pinned memory and returns a LossHandle; .get() waits for that copy only, so the
        caller can sample the next batch while this step runs."""
        self._feed(batch_words)
        if self.graph is not None:
            self.graph.replay()
        else:
            self._enqueue()
        return self._fetch_loss() if fetch_loss else None

    def step_resident(self):
        """Step on whatever batch_dev currently holds (inputs already in HBM)."""
        self._enqueue()

    def capture(self):
        """CUDA graph of one step on the resident batch buffer; replay with graph.replay()."""
        self.graph = capture_step(self._enqueue, (self.params, self.m, self.v, self.step_dev, self.losses), self._warm, 2)
        self._warm = True
        return self.graph

    # ---- checkpoints ---------------------------------------------------------------------
    def state_dict(self):
        """The training state on the host, in the layout both engines share (checkpoint.py writes it):
        step (the counter keying Adam's bias correction and the Philox stream), user_ids (global ids of the user rows,
        here 0..U-1), user {params, m, v} [U, d], item_params [I, d], item_rows (the item rows whose moments this
        engine owns: all of them) and item {m, v} of those rows.  Nothing else carries over from one step to the next:
        the workspace, scalars and losses are rewritten by every step.  SGL's view graphs are the caller's (set_view_graphs)."""
        U = self.U
        return {"step": int(self.step_dev.item()), "user_ids": np.arange(U, dtype=np.int64),
                "user": {"params": self.params[:U].cpu().numpy(), "m": self.m[:U].cpu().numpy(), "v": self.v[:U].cpu().numpy()},
                "item_params": self.params[U:].cpu().numpy(), "item_rows": (0, self.I),
                "item": {"m": self.m[U:].cpu().numpy(), "v": self.v[U:].cpu().numpy()}}

    def load_state_dict(self, state):
        """Copy a saved state into the engine's existing tensors (a captured CUDA graph stays valid: no address moves).
        state: step, user {params, m, v} [U, d] in user id order, item_params [I, d], item {m, v} [I, d]; the arrays may
        be memory maps (read in row chunks) and `user` / `item` any mapping that yields them on access."""
        U = self.U
        for name, dst in (("params", self.params), ("m", self.m), ("v", self.v)):
            copy_rows_in(dst[:U], state["user"][name], "user " + name)
        copy_rows_in(self.params[U:], state["item_params"], "item params")
        for name, dst in (("m", self.m), ("v", self.v)):
            copy_rows_in(dst[U:], state["item"][name], "item " + name)
        self.step_dev.fill_(int(state["step"]))
        torch.cuda.synchronize(self.dev)

    # ---- inference ---------------------------------------------------------------------
    def forward_clean(self):
        """no_grad clean forward -> (user_emb, item_emb), e.g. XSimGCL.py:40-41."""
        if self.model_name == "MF":
            out = self.params.clone()
        else:
            include_ego = self.model_name in ("LightGCN", "SGL")
            out, _ = ops.encoder_forward(self.adj, self.params, self.L, include_ego)
        return out[: self.U], out[self.U:]
