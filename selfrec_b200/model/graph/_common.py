"""Shared scaffolding of the fused in-scope models (MF, LightGCN, SimGCL, XSimGCL, SGL).

Each model keeps the reference class name, constructor signature, YAML keys, attributes
(`model.embedding_dict`, `user_emb`, `item_emb`, `best_user_emb`, ...) and train()/save()/
predict() contract; the batch loop body is one engine step().

Inside a process group (install() starts one under torchrun) the propagating models train on the bipartite-sharded
engine, at any world size including 1: each rank holds its own users' rows, `best_user_emb` is that [Ug, d] block,
and ranking goes through shard_rank.ShardRanker.  MF has no propagation to shard and keeps TrainEngine at world 1."""
import os

import numpy as np
import torch
import torch.nn as nn

from ... import shard_rank
from ..._lib import SrbError
from ...base.graph_recommender import GraphRecommender
from ...engine import TrainEngine, initial_tables


class _EncoderView(nn.Module):
    """Exposes the engine's single [U+I, d] table as the reference's embedding_dict."""

    def __init__(self, engine):
        super().__init__()
        self.engine = engine
        self.embedding_dict = nn.ParameterDict({
            "user_emb": nn.Parameter(engine.user_emb, requires_grad=False),
            "item_emb": nn.Parameter(engine.item_emb, requires_grad=False),
        })

    def forward(self, *args, **kwargs):
        with torch.no_grad():
            return self.engine.forward_clean()

    def cuda(self, device=None):
        return self


class FusedGraphModel(GraphRecommender):
    MODEL = None
    EVAL_EVERY = 1      # fast_evaluation cadence (epochs)
    EVAL_FROM = 0

    def _engine_kwargs(self):
        return {}

    def _make_engine(self, n_layers, **kw):
        args = (self.MODEL, self.data, self.emb_size, n_layers, self.batch_size, self.lRate, self.reg)
        pg = shard_rank.process_group()
        if pg is not None:
            rank, world = pg
            if self.MODEL == "MF" and world > 1:
                raise SrbError(f"MF has no propagation to shard: run it in one process, not on {world} ranks")
            shard_rank.broadcast_start_state()  # one trajectory: rank 0's sampler stream, view draws and tables
        if pg is None or self.MODEL == "MF":
            self.engine = TrainEngine(*args, **kw)
        else:
            from ...sharded import ShardedEngine
            dev = torch.device("cuda", torch.cuda.current_device())
            n, d = int(self.data.user_num) + int(self.data.item_num), int(self.emb_size)
            # the tables a single-process TrainEngine would draw; the engine keeps this rank's rows of them
            init_user, init_item = initial_tables(self.data.user_num, self.data.item_num, torch.empty((n, d), device=dev))
            self.engine = ShardedEngine(*args, init_user=init_user, init_item=init_item, device=dev, **kw)
            del init_user, init_item
            self.shard_ranker = shard_rank.ShardRanker(self.data, rank, world, dev)
        self.model = _EncoderView(self.engine)

    def _epoch_prologue(self, epoch):
        pass

    def _log_line(self, epoch, n, losses):
        print("training:", epoch + 1, "batch", n, "rec_loss:", losses[0], "cl_loss", losses[2])

    # ---- checkpoints (optional YAML keys checkpoint.dir / checkpoint.every / checkpoint.resume) ------------------
    def _checkpoint_conf(self):
        if getattr(self, "_ckpt", None) is None:
            conf = self.config
            get = lambda key: conf[key] if conf.contain(key) else None
            every = get("checkpoint.every")
            self._ckpt = {"dir": get("checkpoint.dir"), "every": int(every) if every else 0, "resume": get("checkpoint.resume")}
            if self._ckpt["every"] < 0:
                raise SrbError(f"checkpoint.every must be a positive number of batches, not {every}")
        return self._ckpt

    def _fingerprint(self):
        from ... import checkpoint
        if getattr(self, "_pairs_fp", None) is None:
            self._pairs_fp = checkpoint.pairs_fingerprint(self.data.pair_users, self.data.pair_items)
        return self._pairs_fp

    def _checkpoint_extra(self):
        """{file name: array} of the model's own state inside an epoch (SGL: the draws of the epoch's views)."""
        return {}

    def _restore_extra(self, path):
        pass

    def _rank_world(self):
        eng = self.engine
        return (int(eng.rank), int(eng.world)) if hasattr(eng, "world") else (0, 1)

    def save_checkpoint(self, epoch, batch):
        """Write the run's state under checkpoint.dir: the engine, the sampler's position, the RNG states and the
        keep-best tables, to continue at batch `batch` of epoch `epoch` (0-based).  Collective under a process group."""
        from ... import checkpoint
        eng = self.engine
        rank, world = self._rank_world()
        pos = eng.feed_state()  # first: the stream position, before anything else could draw
        state = eng.state_dict()
        man = checkpoint.identity(self.MODEL, eng, self.data, self._fingerprint())
        bounds = [int(x) for x in eng.ib] if hasattr(eng, "ib") else [0, int(eng.I)]
        man.update(epoch=int(epoch), batch=int(batch), step=state["step"], cursor=int(pos["cursor"]), item_bounds=bounds,
                   bestPerformance=self.bestPerformance, rng=checkpoint.rng_states(pos["random"]))
        common = {"item_params.npy": state["item_params"], "pair_order.npy": pos["order"]}
        best_user = None
        if getattr(self, "best_item_emb", None) is not None:
            common["best_item.npy"] = self.best_item_emb.cpu().numpy()
            best_user = self.best_user_emb.cpu().numpy()
        if pos["cursor"] >= 0:
            common.update(self._checkpoint_extra())
        agree = eng.all_ok if world > 1 else (lambda ok: ok)
        return checkpoint.save(self._checkpoint_conf()["dir"], man, {rank: (state, best_user)}, common, rank=rank, world=world,
                               agree=agree)

    def load(self, path=None):
        """Restore a checkpoint (default: checkpoint.resume) into this model: the engine's tables, moments and step
        counter, the sampler's order and position, the RNG states, the keep-best tables and bestPerformance.  train()
        then continues at the saved epoch and batch.  A checkpoint of another model, shape, hyperparameter set or
        training set is refused (SrbError) before anything is loaded."""
        from ... import checkpoint
        ck = self._checkpoint_conf()
        path = checkpoint.resolve(ck["resume"] if path is None else path, ck["dir"])
        man = checkpoint.read_manifest(path)
        eng = self.engine
        checkpoint.verify(man, checkpoint.identity(self.MODEL, eng, self.data, self._fingerprint()), path)
        ids = checkpoint.engine_user_ids(eng)
        eng.load_state_dict(checkpoint.engine_state(path, man, ids))
        checkpoint.set_rng_states(man["rng"], python=False)
        eng.load_feed_state({"order": np.load(os.path.join(path, "pair_order.npy")), "cursor": int(man["cursor"]),
                             "random": checkpoint.python_random_state(man["rng"])})
        self.bestPerformance = man["bestPerformance"]
        if os.path.exists(os.path.join(path, "best_item.npy")):
            dev = eng.dev
            self.best_item_emb = torch.from_numpy(np.load(os.path.join(path, "best_item.npy"))).to(dev)
            self.best_user_emb = torch.from_numpy(checkpoint.read_user_rows(path, man, "best", ids)).to(dev)
        self._resume_at = (int(man["epoch"]), int(man["batch"]), int(man["cursor"]) >= 0)
        if self._resume_at[2]:
            self._restore_extra(path)
        return path

    def build(self):
        if self._checkpoint_conf()["resume"] is not None:
            self.load()

    def train(self):
        eng = self.engine
        ck = self._checkpoint_conf()
        every = ck["every"] if ck["dir"] is not None else 0
        start_epoch, start_batch, mid_epoch = getattr(self, "_resume_at", (0, 0, False))
        if ck["dir"] is not None:
            eng.track_pair_order()  # the sampler keeps the pair order a checkpoint records (one gather per epoch)
        for epoch in range(start_epoch, self.maxEpoch):
            resumed = mid_epoch and epoch == start_epoch  # this epoch's prologue (SGL: its views) came with the checkpoint
            if not resumed:
                self._epoch_prologue(epoch)
            if eng.graph is None:
                eng.capture()  # one CUDA graph launch per batch from here on
            for n, words in enumerate(eng.batches(), start_batch if resumed else 0):
                if n % 100 == 0 and n > 0:
                    losses = eng.step(words, fetch_loss=True).get().tolist()
                    if shard_rank.is_main_process():  # the losses are replicated over the ranks
                        self._log_line(epoch, n, losses)
                else:
                    eng.step(words)
                if every and (n + 1) % every == 0:
                    self.save_checkpoint(epoch, n + 1)
            with torch.no_grad():
                self.user_emb, self.item_emb = eng.forward_clean()
            if epoch >= self.EVAL_FROM and epoch % self.EVAL_EVERY == 0:
                self.fast_evaluation(epoch)
            if ck["dir"] is not None:
                self.save_checkpoint(epoch + 1, 0)
        self.user_emb, self.item_emb = self.best_user_emb, self.best_item_emb

    def save(self):
        with torch.no_grad():
            ue, ie = self.engine.forward_clean()
            self.best_user_emb, self.best_item_emb = ue.clone(), ie.clone()

    def predict(self, u):
        name, u = u, self.data.get_user_id(u)
        if self.shard_ranker is not None:  # this rank holds the rows of the users it owns only
            r = self.shard_ranker
            if r.owner(u) != r.rank:
                raise SrbError(f"predict: user {name!r} is owned by rank {r.owner(u)}, this is rank {r.rank}")
            u = r.local_row(u)
        # one user's full-catalog scores (reference predict(), e.g. XSimGCL.py:57-60); test()
        # never calls this -- it uses the fused scoring + top-k kernel.
        from ... import ops
        return ops.score_rows(self.user_emb, self.item_emb, [u])[0].cpu().numpy()


class OpLevelEncoder(nn.Module):
    """Autograd-visible encoder on the drop-in ops, for the reference models that import another model's encoder
    class (`from model.graph.LightGCN import LGCN_Encoder`: DirectAU.py:7, SelfCF.py:6; `from model.graph.MF import
    Matrix_Factorization`: DirectAU.py:6).  Same attributes the callers touch (data, latent_size, layers, norm_adj,
    embedding_dict, sparse_norm_adj) and the same forward() contract: (user embeddings, item embeddings), the mean of
    the ego layer and `layers` propagated ones (LightGCN.py:68-78); zero layers is matrix factorisation (MF.py:52-53).
    Propagation is torch.sparse.mm on the SparseAdj handle, i.e. the CUDA SpMM, differentiable w.r.t. the table."""

    def __init__(self, data, emb_size, n_layers=0):
        super().__init__()
        from ...base.torch_interface import TorchGraphInterface
        self.data = data
        self.latent_size = emb_size
        self.layers = n_layers
        init = nn.init.xavier_uniform_  # users first, then items: the reference's draw order (LightGCN.py:60-66)
        self.embedding_dict = nn.ParameterDict({
            "user_emb": nn.Parameter(init(torch.empty(data.user_num, emb_size))),
            "item_emb": nn.Parameter(init(torch.empty(data.item_num, emb_size))),
        })
        if n_layers > 0:
            self.norm_adj = data.norm_adj
            self.sparse_norm_adj = TorchGraphInterface.convert_sparse_mat_to_tensor(self.norm_adj).cuda()

    def forward(self):
        pd = self.embedding_dict
        if self.layers == 0:
            return pd["user_emb"], pd["item_emb"]
        x = torch.cat([pd["user_emb"], pd["item_emb"]], 0)
        total = x
        for _ in range(self.layers):
            x = torch.sparse.mm(self.sparse_norm_adj, x)
            total = total + x
        out = total / float(self.layers + 1)
        n_u = self.data.user_num
        return out[:n_u], out[n_u:]
