"""UserKNN (reference model/graph/UserKNN.py) on the GPU: user-user cosine neighbours with shrinkage, scores from the
neighbours' items.  See _knn.py."""
from ._knn import KNNRecommender


class UserKNN(KNNRecommender):
    BY = "user"

    @property
    def user_sim(self):
        """user name -> [(sim, neighbour user name), ...], the reference's form (UserKNN.py:12, 53)."""
        return self._sims()
