"""ItemKNN (reference model/graph/ItemKNN.py) on the GPU: item-item cosine neighbours with shrinkage, item-neighbour
weighted scores.  See _knn.py."""
from ._knn import KNNRecommender


class ItemKNN(KNNRecommender):
    BY = "item"

    @property
    def item_sim(self):
        """item name -> [(sim, similar item name), ...], the reference's form (ItemKNN.py:12, 51)."""
        return self._sims()
