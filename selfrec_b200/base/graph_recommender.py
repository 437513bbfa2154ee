"""Drop-in for base/graph_recommender.py:10-104.

test() replaces the per-user predict -> mask -> find_k_largest loop (:38-58) with ONE
full-catalog scoring + mask + top-k launch whenever the model exposes `user_emb` /
`item_emb` (MF, LightGCN, SimGCL, XSimGCL, SGL, ...).  Models whose predict() is not a
single dot product keep their own predict(); their score rows still go through the CUDA
top-k kernel in batches.  Output format is unchanged:
    {user_name: [(item_name, score), ...]}  length max_N, score-descending.
"""
from os.path import abspath
from time import localtime, strftime, time

import numpy as np
import torch

from .. import ops
from ..shard_rank import is_main_process
from ..data.loader import FileIO
from ..data.ui_graph import Interaction
from ..util.evaluation import ranking_evaluation, ranking_evaluation_from_masks
from .recommender import Recommender


class GraphRecommender(Recommender):
    shard_ranker = None  # shard_rank.ShardRanker of a model whose user_emb is this rank's block of a sharded table

    def __init__(self, conf, training_set, test_set, **kwargs):
        super(GraphRecommender, self).__init__(conf, training_set, test_set, **kwargs)
        self.data = Interaction(conf, training_set, test_set)
        self.bestPerformance = []
        self.topN = [int(num) for num in self.ranking]
        self.max_N = max(self.topN)
        if self.max_N < 1 or self.max_N > self.data.item_num:
            raise ValueError(f"item.ranking.topN {self.topN}: the longest list must be in 1..item_num={self.data.item_num}")

    def print_model_info(self):
        super(GraphRecommender, self).print_model_info()
        tr, te = self.data.training_size(), self.data.test_size()
        print(f"Training Set Size: (user number: {tr[0]}, item number: {tr[1]}, interaction number: {tr[2]})")
        print(f"Test Set Size: (user number: {te[0]}, item number: {te[1]}, interaction number: {te[2]})")
        print("=" * 80)

    def build(self):
        pass

    def train(self):
        pass

    def predict(self, u):
        pass

    def save(self):
        pass

    # ---- (iv) ranking ----------------------------------------------------------------
    def _has_embedding_tables(self):
        ue, ie = getattr(self, "user_emb", None), getattr(self, "item_emb", None)
        return (isinstance(ue, torch.Tensor) and isinstance(ie, torch.Tensor) and ue.dim() == 2 and ie.dim() == 2
                and ue.shape[0] == self.data.user_num and ie.shape[0] == self.data.item_num)

    def rank_all(self, users=None):
        """(user_names, ids [n, max_N] np.int32, scores [n, max_N] np.float32) on the GPU path."""
        data = self.data
        names = list(data.test_set) if users is None else list(users)
        uids = np.fromiter((data.user[u] for u in names), dtype=np.int32, count=len(names))
        if self.shard_ranker is not None:
            ids, scores = self.shard_ranker.topk(self.user_emb.detach(), self.item_emb.detach(), uids, self.max_N)
            return names, ids.cpu().numpy(), scores.cpu().numpy()
        rated_ptr, rated_idx = data.rated_csr()
        if self._has_embedding_tables():
            ids, scores = ops.score_topk(self.user_emb.detach(), self.item_emb.detach(), uids, rated_ptr, rated_idx, self.max_N)
            return names, ids.cpu().numpy(), scores.cpu().numpy()
        ids, sc = self._predict_topk(names, uids, self.max_N)
        return names, ids.cpu().numpy(), sc.cpu().numpy()

    def _predict_topk(self, names, uids, n):
        """Generic models: their own predict() rows, rated items masked, batched through the CUDA row top-k.
        (ids int32 [len(names), n], scores fp32) on the device."""
        rated_ptr, rated_idx = self.data.rated_csr()
        ids_out = torch.empty((len(names), n), dtype=torch.int32, device="cuda")
        sc_out = torch.empty((len(names), n), dtype=torch.float32, device="cuda")
        step = 512
        for s in range(0, len(names), step):
            rows = np.stack([np.asarray(self.predict(u), dtype=np.float32) for u in names[s:s + step]])
            for r, uid in enumerate(uids[s:s + step]):
                rows[r, rated_idx[rated_ptr[uid]:rated_ptr[uid + 1]]] = -10e8
            dev_rows = torch.from_numpy(rows).cuda()
            parts = []
            for lo in range(0, n, ops.TOPK_KERNEL_MAX):  # 32 per pass, winners struck out (ops._score_topk_wide)
                ids, sc = ops.topk_rows(dev_rows, min(ops.TOPK_KERNEL_MAX, n - lo))
                parts.append((ids, sc))
                dev_rows.scatter_(1, ids.long(), float("-inf"))
            ids_out[s:s + step], sc_out[s:s + step] = torch.cat([p[0] for p in parts], 1), torch.cat([p[1] for p in parts], 1)
        return ids_out, sc_out

    def export_recommendations(self, out_dir, top_n=None, users=None, chunk=None):
        """Write the top-N lists (default N = max_N) of `users` (names; default every training user) under out_dir,
        rated items masked as in test(); returns the export directory (export.py describes the format)."""
        from .. import export
        return export.export_recommendations(self, out_dir, top_n=top_n, users=users, chunk=chunk)

    def test(self):
        names, ids, scores = self.rank_all()
        id2item = self.data.id2item
        rec_list = {}
        for r, user in enumerate(names):
            rec_list[user] = list(zip([id2item[i] for i in ids[r].tolist()], scores[r].tolist()))
        return rec_list

    def evaluate(self, rec_list):
        self.recOutput.append("userId: recommendations in (itemId, ranking score) pairs, * means the item is hit.\n")
        for user in self.data.test_set:
            line = user + ":" + "".join(
                f" ({it[0]},{it[1]}){'*' if it[0] in self.data.test_set[user] else ''}" for it in rec_list[user])
            self.recOutput.append(line + "\n")
        stamp = strftime("%Y-%m-%d %H-%M-%S", localtime(time()))
        out_dir = self.output
        name = self.config["model"]["name"]
        main = is_main_process()  # every rank holds the same rec_list: one set of result files
        if main:
            FileIO.write_file(out_dir, f"{name}@{stamp}-top-{self.max_N}items.txt", self.recOutput)
            print("The result has been output to ", abspath(out_dir), ".")
        self.result = ranking_evaluation(self.data.test_set, rec_list, self.topN)
        self.model_log.add("###Evaluation Results###")
        self.model_log.add(self.result)
        if main:
            FileIO.write_file(out_dir, f"{name}@{stamp}-performance.txt", self.result)
            print(f"The result of {self.model_name}:\n{''.join(self.result)}")
        conf = self.config
        if conf.contain("export.dir"):  # optional: every training user's top-N lists (export.topN, default max_N)
            top_n = int(conf["export.topN"]) if conf.contain("export.topN") else None
            path = self.export_recommendations(conf["export.dir"], top_n=top_n)
            if main:
                print("The recommendation lists have been exported to ", abspath(path), ".")

    def _fast_measure(self):
        """fast_evaluation's metrics without leaving id space: full-catalog top-k on the device, hit masks on
        the device (srb_rank_hit_masks, ceil(max_N / 64) words per user), the reference's float expressions on the
        masks, for max_N <= 256.  Same strings as
        ranking_evaluation(self.data.test_set, self.test(), [self.max_N])."""
        data = self.data
        names = list(data.test_set)
        ranker = self.shard_ranker
        if not ((ranker is not None or self._has_embedding_tables()) and self.max_N <= ops.TOPK_TC_MAX and all(u in data.user for u in names)):
            return ranking_evaluation(data.test_set, self.test(), [self.max_N])
        uids = np.fromiter((data.user[u] for u in names), dtype=np.int32, count=len(names))
        test_ptr, test_idx, n_test = data.test_csr()
        if ranker is not None:
            masks = ranker.hit_masks(self.user_emb.detach(), self.item_emb.detach(), uids, self.max_N).cpu().numpy()
        else:
            rated_ptr, rated_idx = data.rated_csr()
            ids, _ = ops.score_topk(self.user_emb.detach(), self.item_emb.detach(), uids, rated_ptr, rated_idx, self.max_N)
            masks = ops.rank_hit_masks(ids, uids, test_ptr, test_idx).cpu().numpy()
        return ranking_evaluation_from_masks(n_test[uids], masks.view(np.uint64), [self.max_N])

    def fast_evaluation(self, epoch):
        print("Evaluating the model...")
        measure = self._fast_measure()
        performance = {k: float(v) for m in measure[1:] for k, v in [m.strip().split(":")]}
        if self.bestPerformance:
            # strictly more metrics improved than worsened (graph_recommender.py:88-92)
            count = sum(1 if self.bestPerformance[1][k] > performance[k] else -1 for k in performance)
            if count < 0:
                self.bestPerformance = [epoch + 1, performance]
                self.save()
        else:
            self.bestPerformance = [epoch + 1, performance]
            self.save()
        if is_main_process():
            print("-" * 80)
            print(f"Real-Time Ranking Performance (Top-{self.max_N} Item Recommendation)")
            print(f"*Current Performance*\nEpoch: {epoch + 1}, " + ", ".join(f"{k}: {v}" for k, v in performance.items()))
            print(f"*Best Performance*\nEpoch: {self.bestPerformance[0]}, " + ", ".join(f"{k}: {v}" for k, v in self.bestPerformance[1].items()))
            print("-" * 80)
        return measure
