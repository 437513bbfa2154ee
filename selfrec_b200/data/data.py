"""Base of Interaction (data/data.py): the run's configuration plus the raw training / test triples.

`training_data` is the list the reference's sampler shuffles in place every epoch (util/sampler.py:7).  The native
sampler shuffles ids, not Python lists, so the list order is kept as a pending permutation and applied (to the
same list object) when somebody reads `training_data` -- 0.3 s of list copying per epoch at yelp2018 otherwise."""
import numpy as np


class _PendingShuffles(object):
    """Epoch shuffles not yet applied to the list: new[k] = old[perm[k]], composed on demand."""

    def __init__(self, fold=8):
        self.perms = []
        self.fold = int(fold)

    def add(self, perm):
        self.perms.append(np.asarray(perm, dtype=np.int64))
        if len(self.perms) >= self.fold:  # bound the memory: fold them into one permutation
            self.perms = [self.take()]

    def take(self):
        """The composition of everything recorded (None if nothing is pending); clears the record."""
        total = None
        for p in self.perms:
            total = p if total is None else total[p]
        self.perms = []
        return total


class Data(object):
    def __init__(self, conf, training, test):
        self.config, self.test_data = conf, test
        self._td, self._td_pending = training, _PendingShuffles()

    @property
    def training_data(self):
        order = self._td_pending.take()
        if order is not None:
            src = self._td
            src[:] = [src[k] for k in order.tolist()]
        return self._td

    @training_data.setter
    def training_data(self, rows):
        self._td, self._td_pending = rows, _PendingShuffles()

    def shuffle_training_data(self, perm):
        """Record an in-place shuffle: new[k] = old[perm[k]] (applied when training_data is next read)."""
        self._td_pending.add(perm)
