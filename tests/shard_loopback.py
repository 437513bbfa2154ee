"""Loopback ranks: the W ranks of one bipartite-sharded world as W ShardedEngines in one process on one GPU.

The sharded step sees its peers only through the pointers srb_shard_desc.sym[g], and the pointers of peers on the same
device are plain device pointers.  So one GPU can run the whole exchange of a W-rank world: the item-side partial
products stored into the owners' staging areas, the owners' reductions and their stores to every rank, the gathers into
every rank's compact tables, the cyclic user blocks of the seed scatter and the Philox keys of the user rows.  What it
cannot run are the multicast / NVLS stores and the in-kernel wait / signal protocol; those need >= 2 GPUs.

The fake process group covers the surface ShardedEngine reads: torch.distributed's is_available, is_initialized,
get_rank, get_world_size (keyed by the FakeGroup passed as group=), barrier and get_backend (no-ops), all_reduce (identity:
every rank passes the same view graphs), and torch.distributed._symmetric_memory's empty (rank r gets buffer r of W
same-sized device buffers) and rendezvous (all W buffers, no multicast mapping, so the stores take the unicast route).

Safety guards.  The GPU may be shared with other work, and a loopback that could stall it must not run:
  * Barrier mode only (SRB_SHARD_SYNC=barrier).  In the default mode the waits are folded into the SpMM and reduction
    kernels, and a waiting grid can fill the GPU and starve the peer it waits for; one GPU cannot guarantee that the
    ranks' grids are co-resident.  In barrier mode the only cross-rank wait is the 32-thread shard_barrier_kernel, and
    every other kernel finishes without its peers.
  * Separate hardware queues (CUDA_DEVICE_MAX_CONNECTIONS at least the number of streams in use, set before CUDA
    starts).  Otherwise a spinning barrier can serialise a peer's kernels behind it in one queue.
  * Every kernel loaded before the first step (CUDA_MODULE_LOADING=EAGER).  With lazy loading the first launch of a
    kernel loads it, and the load can wait for the kernels running in the context -- a peer's spinning barrier among
    them -- so the launching rank stalls until that barrier times out.
  * No capture() at world > 1: its warm-up runs and synchronises one rank alone, which would sit in the barrier until
    its ~30 s timeout.  LoopbackWorld steps eagerly only.
  * The ranks are never launched serially from one thread: every rank enqueues from its own host thread on its own
    stream (ctypes releases the GIL, so the enqueues overlap).
  * A tripped error flag is a finding.  After every step the threads are joined, the device synchronised and every
    rank's check_peers() called; a timed-out barrier is an error to explain, not a flake to re-run.
LoopbackWorld refuses to start unless the environment is LOOPBACK_ENV (SRB_SHARD_OVERLAP=0 and SRB_PDL=0 besides the
three above), so it only runs in a process started for it: tests/test_gpu_shard_loopback.py launches this file as a
script, one case per subprocess, with a timeout.
"""
import json
import os
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

LOOPBACK_ENV = {"SRB_SHARD_SYNC": "barrier", "SRB_SHARD_OVERLAP": "0", "SRB_PDL": "0", "CUDA_DEVICE_MAX_CONNECTIONS": "32",
                "CUDA_MODULE_LOADING": "EAGER"}

# The loopback graph: users 1..9 at every class boundary of the SpMM (test_gpu_step_edges.HUB_USERS), items 1 and 2 of
# degree >= 4096 * 8, so that at every world up to 8 they stay split rows of >= 2 chunks in every rank's [I x Ug] block,
# and items of degree 3000 / 1400 / 700 / 300, so that every rank's block also has CTA rows (256..4095) and warp rows
# (64..255) at every tested world.  7 divides neither LB_USERS nor LB_ITEMS: uneven user blocks and item slices.
LB_USERS, LB_ITEMS = 34000, 6500
LB_HUB_ITEMS = {1: 33900, 2: 33000, 3: 3000, 4: 1400, 5: 700, 6: 300}
LB_SEED = 20261017
# first-moment bar of the oracle sequence (test_gpu_step_edges.KAPPA there): the item rows are sums of W partial sums,
# and a hub item's gradient sums ~33000 terms that largely cancel.  Worst measured: 1.3e-4 of the row's scale, item 2
# (degree 33000) in the last batch of SimGCL d = 128, L = 2 at W = 3, on an H100 80GB HBM3 (700 W)
LB_KAPPA = 2.5e-4


# ---------------------------------------------------------------------------------------
# fake process group
# ---------------------------------------------------------------------------------------
class _Pool:
    """The W symmetric buffers of one loopback world, allocated on the first request."""

    def __init__(self, world, device):
        self.world, self.device, self.bufs = int(world), device, None

    def buffer(self, rank, nbytes):
        import torch
        if self.bufs is None:
            self.bufs = [torch.empty(nbytes, dtype=torch.uint8, device=self.device) for _ in range(self.world)]
        if self.bufs[rank].numel() != nbytes:
            raise RuntimeError(f"loopback: rank {rank} asked for {nbytes} symmetric bytes, the world has {self.bufs[rank].numel()}")
        return self.bufs[rank]


class FakeGroup:
    """Rank `rank` of a loopback world (what the engine of that rank is given as group=)."""

    def __init__(self, pool, rank):
        self.pool, self.rank = pool, int(rank)


class _Handle:
    def __init__(self, pool):
        self.buffer_ptrs = [b.data_ptr() for b in pool.bufs]
        self.multicast_ptr = 0


_building = [None]  # the group whose engine is being constructed (symmetric_memory.empty takes no group)


def _group(group):
    if not isinstance(group, FakeGroup):
        raise RuntimeError(f"loopback: a collective without a loopback group ({group!r})")
    return group


def install(patch=setattr):
    """Replace the torch.distributed surface ShardedEngine reads by the loopback fakes (patch: setattr, or
    pytest's monkeypatch.setattr)."""
    import torch
    import torch.distributed as dist
    import torch.distributed._symmetric_memory as symm

    def empty(*size, dtype=None, device=None):
        g = _building[0]
        if g is None or dtype != torch.uint8:
            raise RuntimeError("loopback: symmetric memory is only handed out while a rank's engine is built")
        return g.pool.buffer(g.rank, int(np.prod(size)))

    def barrier(group=None, **kw):
        _group(group)  # every rank runs in this process: nothing to wait for

    def get_backend(group=None):
        _group(group)
        return "gloo"  # (the view signature of set_view_graphs then lives on the host)

    def all_reduce(tensor, op=None, group=None, async_op=False):
        _group(group)  # identity: every rank passes the same tensor

    patch(dist, "is_available", lambda: True)
    patch(dist, "is_initialized", lambda: True)
    patch(dist, "get_rank", lambda group=None: _group(group).rank)
    patch(dist, "get_world_size", lambda group=None: _group(group).pool.world)
    patch(dist, "barrier", barrier)
    patch(dist, "get_backend", get_backend)
    patch(dist, "all_reduce", all_reduce)
    patch(symm, "empty", empty)
    patch(symm, "rendezvous", lambda tensor, group=None: _Handle(_group(group).pool))


def make_ranks(world, make_engine, device):
    """make_engine(group) for the ranks 0..world-1 of one loopback world, in rank order (construction launches nothing
    that waits for a peer)."""
    pool = _Pool(world, device)
    engines = []
    try:
        for r in range(world):
            _building[0] = FakeGroup(pool, r)
            engines.append(make_engine(_building[0]))
    finally:
        _building[0] = None
    return engines


# ---------------------------------------------------------------------------------------
# the world
# ---------------------------------------------------------------------------------------
class LoopbackWorld:
    """W ShardedEngines of one world on one GPU, stepped together.  No capture(): eager steps only (module docstring)."""

    def __init__(self, world, make_engine, device):
        import torch
        for k, v in LOOPBACK_ENV.items():
            if k == "CUDA_DEVICE_MAX_CONNECTIONS":
                if int(os.environ.get(k, "8")) < world + 2:
                    raise RuntimeError(f"loopback: {k} must be set to >= {world + 2} before CUDA starts (every rank's stream its own queue)")
            elif os.environ.get(k) != v:
                raise RuntimeError(f"loopback: needs {k}={v} in the environment of the process")
        self.torch = torch
        self.engines = make_ranks(world, make_engine, device)
        e0 = self.engines[0]
        assert all(e.world == world and e.rank == r for r, e in enumerate(self.engines))
        assert not any(e.use_multicast or e.use_nvls for e in self.engines)
        self.world, self.U, self.I, self.d = world, e0.U, e0.I, e0.d
        self.ib = e0.ib
        self.streams = [torch.cuda.Stream(device=device) for _ in range(world)]
        assert len({s.cuda_stream for s in self.streams}) == world, "two ranks on one stream would serialise a barrier"
        self.device = device
        torch.cuda.synchronize()

    @property
    def workspaces(self):
        return [e.workspace for e in self.engines]

    def _run(self, fn):
        """fn(engine) of every rank from its own thread, on its own stream; then join, synchronise, check_peers()."""
        torch = self.torch
        out, err = [None] * self.world, [None] * self.world

        def body(r):
            try:
                with torch.cuda.device(self.device), torch.cuda.stream(self.streams[r]):
                    out[r] = fn(self.engines[r])
            except BaseException as e:  # noqa: BLE001 -- re-raised below, after every thread is joined
                err[r] = e

        threads = [threading.Thread(target=body, args=(r,)) for r in range(self.world)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        torch.cuda.synchronize()
        for e in self.engines:
            e.check_peers()
        for e in err:
            if e is not None:
                raise e
        return out

    def step(self, words):
        """One eager training step of every rank on the batch words (uploaded to every rank's batch_dev first)."""
        torch = self.torch
        w = torch.from_numpy(np.ascontiguousarray(words, dtype=np.int32))
        for e in self.engines:
            e.batch_dev.copy_(w)
        torch.cuda.synchronize()
        self._run(lambda e: e.step_resident())
        self.check_replicas(final=False)

    def forward_clean(self):
        """Clean forward of every rank -> ([U, d] users reassembled from the ranks, [I, d] items), as numpy."""
        outs = self._run(lambda e: e.forward_clean())
        self.check_replicas(final=True)
        items = [o[1] for o in outs]
        for r in range(1, self.world):
            self._same("forward_clean items", r, items[r], items[0])
        return self.users([o[0] for o in outs]), items[0].cpu().numpy()

    # ---- reassembly and the replica invariant ----
    def users(self, tabs):
        """[U, d] numpy table from every rank's [Ug, d] block (user u is row u // W of rank u % W)."""
        full = np.empty((self.U, tabs[0].shape[1]), dtype=np.float32)
        for r, t in enumerate(tabs):
            full[r::self.world] = t.cpu().numpy()
        return full

    def owned_items(self, tabs):
        """[I, d] numpy table whose slice [ib[r], ib[r + 1]) comes from rank r (the only rank that updates it)."""
        full = np.empty((self.I, tabs[0].shape[1]), dtype=np.float32)
        for r, t in enumerate(tabs):
            lo, hi = int(self.ib[r]), int(self.ib[r + 1])
            full[lo:hi] = t[lo:hi].cpu().numpy()
        return full

    def state(self):
        """(params, m, v, losses) of the world as the single-GPU [U + I, d] tables."""
        es = self.engines
        for r in range(1, self.world):  # every rank computes them on the same rows (sums of atomics: not bit-identical)
            a, b = es[r].losses.cpu().numpy(), es[0].losses.cpu().numpy()
            assert (np.abs(a - b) <= 1e-5 * np.abs(b) + 1e-8).all(), ("losses of rank", r, a.tolist(), b.tolist())
        p = np.concatenate([self.users([e.user_emb for e in es]), es[0].item_emb.cpu().numpy()])
        m = np.concatenate([self.users([e.mu for e in es]), self.owned_items([e.mi for e in es])])
        v = np.concatenate([self.users([e.vu for e in es]), self.owned_items([e.vi for e in es])])
        return p, m, v, es[0].losses.cpu().numpy()

    def _same(self, name, r, a, b):
        """Bit-identical (NaN included): every replicated row has exactly one writer, whose stores reach every rank."""
        ai, bi = a.contiguous().view(self.torch.int32), b.contiguous().view(self.torch.int32)
        diff = ai != bi
        if diff.any():
            rows = self.torch.nonzero(diff.reshape(diff.shape[0], -1).any(1)).flatten().tolist() if diff.dim() > 1 else []
            raise AssertionError(f"{name}: rank {r}'s replica differs from rank 0's in {int(diff.sum())} entries, first rows {rows[:8]}")

    def check_replicas(self, final):
        """item_emb after every step; with final, also the final item mean, which only the clean forward pushes to every
        rank (a training step keeps each owner's slice of it local: the gathers read it there)."""
        es = self.engines
        for r in range(1, self.world):
            self._same("item_emb", r, es[r].item_emb, es[0].item_emb)
            if final:
                self._same("_item_final", r, es[r]._item_final, es[0]._item_final)

    def assert_split_rows(self):
        """Every rank's [I x Ug] block has a split row of >= 2 chunks, a CTA row and a warp row."""
        from selfrec_b200 import _lib, ops
        for r, e in enumerate(self.engines):
            rp = e.Rt.rowptr.to(self.torch.int64)
            deg = (rp[1:] - rp[:-1]).cpu().numpy()
            c = ops.classify_rows(e.Rt.rowptr)
            assert c["n_huge"] >= 1 and deg.max() >= 2 * _lib.HUB_CHUNK, (r, c["n_huge"], int(deg.max()))
            assert c["n_vlong"] >= 1 and c["n_long"] >= 1, (r, c["n_vlong"], c["n_long"])


# ---------------------------------------------------------------------------------------
# cases (tests/test_gpu_shard_loopback.py)
# ---------------------------------------------------------------------------------------
def loopback_graph():
    import test_gpu_step_edges as edges
    return edges.make_hub_graph(LB_USERS, LB_ITEMS, edges.HUB_USERS, LB_HUB_ITEMS, LB_SEED)


def _model_kw(edges, name, lcl, eps):
    if name == "LightGCN":
        return dict(l2_div=float(edges.B))
    if name == "SGL":
        return dict(tau=edges.TAU, cl_rate=edges.CL_RATE)
    return dict(eps=eps, tau=edges.TAU, cl_rate=edges.CL_RATE, layer_cl=lcl)


def run_oracle_case(name, world, d, L, lcl=0, views=None, reg=None):
    """Poison step, then test_gpu_step_edges' batch sequence against the float64 oracle (SimGCL / XSimGCL at eps = 0),
    then the clean forward against the oracle's.  reg: the L2 weight (test_gpu_step_edges.REG by default)."""
    import torch
    import oracle as orc
    import test_gpu_step_edges as edges
    from selfrec_b200.sharded import ShardedEngine
    orc.build()
    dev = torch.device("cuda", torch.cuda.current_device())
    h = loopback_graph()
    data, A = h["data"], h["A"]
    U, I, B = data.user_num, data.item_num, edges.B
    rng = np.random.default_rng(d + L + world)
    E0 = (rng.standard_normal((U + I, d)) * 0.1).astype(np.float32)
    kw = _model_kw(edges, name, lcl, 0.0)
    reg = edges.REG if reg is None else float(reg)
    w = LoopbackWorld(world, lambda g: ShardedEngine(name, data, d, L, B, edges.LR, reg, init_user=torch.from_numpy(E0[:U]),
                                                     init_item=torch.from_numpy(E0[U:]), group=g, device=dev, **kw), dev)
    w.assert_split_rows()
    view_csr = None
    if name == "SGL":
        view_csr = h["views"][views]
        for e in w.engines:
            e.set_view_graphs(*view_csr)
    es = w.engines
    state = [t for e in es for t in (e.user_emb, e.item_emb, e.mu, e.vu, e.mi, e.vi, e.step_dev, e.losses)]
    tag = f"loopback W={world} {name}-d{d}-L{L}" + (f"-lcl{lcl}" if name == "XSimGCL" else "") + (f"-{views}" if views else "") + \
        (f" reg={reg:g}" if reg != edges.REG else "")
    t0 = time.time()
    edges._poison(torch, w, h["poison"], state, [t for e in es for t in (e.user_emb, e.item_emb)], workspaces=w.workspaces)
    print(f"{tag}: poison step done in {time.time() - t0:.1f} s", flush=True)
    edges._run_sequence(torch, orc, h, name, d, L, lcl, view_csr, w.step, w.state, None, tag, eps=0.0, kappa=LB_KAPPA, reg=reg)
    print(f"{tag}: sequence done in {time.time() - t0:.1f} s", flush=True)
    # the clean forward against the oracle's, from the trained tables
    p = w.state()[0]
    fu, fi = w.forward_clean()
    ref, _, _ = orc.encoder_forward(A, p, L, name in ("LightGCN", "SGL"))
    got = np.concatenate([fu, fi])
    err = np.abs(got - ref).max(1)
    bound = edges.KAPPA * np.abs(ref).max(1) + 1e-6 * np.abs(ref).max()
    worst = int(np.argmax(err - bound))
    assert (err <= bound).all(), (tag, "clean forward", int((err > bound).sum()), worst, float(err[worst]), float(bound[worst]))
    print(f"{tag}: 5 steps and the clean forward match the oracle", flush=True)


def run_philox_case(name, world, d, L, lcl=0):
    """SimGCL / XSimGCL at the configured eps: the loopback world against TrainEngine on the same tables, batches and
    philox_seed.  The in-kernel noise is keyed by global row id, so only the y ~ 0 elements whose sign differs under
    the two summation orders (and their neighbours) may differ."""
    import torch
    import test_gpu_step_edges as edges
    from selfrec_b200.engine import TrainEngine
    from selfrec_b200.sharded import ShardedEngine
    dev = torch.device("cuda", torch.cuda.current_device())
    h = loopback_graph()
    data = h["data"]
    U, I, B = data.user_num, data.item_num, edges.B
    rng = np.random.default_rng(d + L + world + 1)
    E0 = (rng.standard_normal((U + I, d)) * 0.1).astype(np.float32)
    kw = _model_kw(edges, name, lcl, edges.EPS)
    seed = 0x5EED + world
    iu, ii = torch.from_numpy(E0[:U]), torch.from_numpy(E0[U:])
    w = LoopbackWorld(world, lambda g: ShardedEngine(name, data, d, L, B, edges.LR, edges.REG, init_user=iu, init_item=ii, group=g,
                                                     device=dev, philox_seed=seed, **kw), dev)
    ref = TrainEngine(name, data, d, L, B, edges.LR, edges.REG, init_user=iu, init_item=ii, device=dev, philox_seed=seed, **kw)
    tag = f"loopback W={world} {name}-d{d}-L{L} eps={edges.EPS}"
    N = U + I
    for step, (words, (u, _i, _j)) in enumerate(h["batches"], start=1):
        ref.step(words)
        torch.cuda.synchronize()
        w.step(words)
        _p, gm, _v, los = w.state()
        rl, rm = ref.losses.cpu().numpy(), ref.m.cpu().numpy()
        # rec, l2, cl, total; cl and total also get test_gpu_step_edges' InfoNCE floor (fp32 resolution of logits of
        # size 1 / tau, once for the users and once for the items)
        floor = np.array([1e-7, 1e-7, 4e-7 / edges.TAU, 4e-7 / edges.TAU])
        assert (np.abs(los - rl) <= 1e-4 * np.abs(rl) + floor).all(), (tag, step, los.tolist(), rl.tolist())
        off = int((np.abs(gm - rm).max(1) > 1e-4 * np.abs(rm).max()).sum())
        print(f"{tag} step {step} b={len(u)}: {off} of {N} rows of m off", flush=True)
        assert off <= 1e-3 * N, (tag, step, off)


def main():
    case = json.loads(sys.argv[1])
    import torch
    torch.cuda.set_device(0)
    install()
    kind = case.pop("kind")
    if kind == "oracle":
        run_oracle_case(**case)
    elif kind == "philox":
        run_philox_case(**case)
    else:
        raise ValueError(kind)
    print("LOOPBACK_CASE PASS", flush=True)


if __name__ == "__main__":
    main()
