"""Shared body of ItemKNN and UserKNN (reference model/graph/ItemKNN.py, model/graph/UserKNN.py).

Same class names, constructor, YAML keys (`topK`, `shrinkage`) and train() / predict(u) / test() contract as the
reference.  train() builds the neighbour table on the device (knn.NeighbourTable), predict(u) returns the reference's
float64 [item_num] row computed on the device, and test() ranks every test user on the device with float64 scores in
the reference's exact list order.  Neither model is sharded: under a process group of more than one rank they refuse
to start."""
import time

import numpy as np
import torch

from ... import shard_rank
from ..._lib import SrbError
from ...base.graph_recommender import GraphRecommender
from ...knn import NeighbourTable


class KNNRecommender(GraphRecommender):
    BY = None  # "item" (ItemKNN) or "user" (UserKNN)

    def __init__(self, conf, training_set, test_set):
        super(KNNRecommender, self).__init__(conf, training_set, test_set)
        self.topk = int(self.config["topK"])
        self.shrinkage = int(self.config["shrinkage"])
        if self.topk < 1:
            raise SrbError(f"{self.model_name}: topK={self.topk} must be >= 1")
        if self.shrinkage < 0:
            raise SrbError(f"{self.model_name}: shrinkage={self.shrinkage} must be >= 0")
        pg = shard_rank.process_group()
        if pg is not None and pg[1] > 1:
            raise SrbError(f"{self.model_name} is not sharded: run it in one process, not on {pg[1]} ranks")
        self.neighbour_table = None
        self._sim_dict = None

    def _sims(self):
        """{name: [(sim, name), ...]} of the trained table, built from the device table on first access."""
        if self._sim_dict is None:
            self._sim_dict = {} if self.neighbour_table is None else self.neighbour_table.as_dict()
        return self._sim_dict

    def train(self):
        kind = self.BY
        print(f"[{self.model_name}] Computing {kind}-{kind} similarity with top-{self.topk}...")
        start = time.time()
        self.neighbour_table = NeighbourTable(self.data, self.BY, self.topk, self.shrinkage)
        self._sim_dict = None
        torch.cuda.current_stream().synchronize()
        print(f"[{self.model_name}] Similarity computation done in {time.time() - start:.2f}s.")

    def _table(self):
        if self.neighbour_table is None:
            raise SrbError(f"{self.model_name}: call train() before predict() or test()")
        return self.neighbour_table

    def predict(self, u):
        """Float64 scores [item_num] for the user named u (rated items not masked), as the reference's predict()."""
        return self._table().score_rows([self.data.user[u]])[0].cpu().numpy()

    def rank_all(self, users=None):
        """(user_names, ids [n, max_N] int32, scores [n, max_N] float64): find_k_largest of every masked predict row."""
        data = self.data
        names = list(data.test_set) if users is None else list(users)
        uids = np.fromiter((data.user[u] for u in names), dtype=np.int32, count=len(names))
        ids, scores = self._table().rank(uids, self.max_N)
        return names, ids, scores
