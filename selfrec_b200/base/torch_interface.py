"""Drop-in for base/torch_interface.py:3-13.

convert_sparse_mat_to_tensor returns a SparseAdj handle instead of a torch COO tensor: the
callers' `.cuda()` uploads the CSR once and `torch.sparse.mm(handle, dense)` dispatches to
the sm_90a SpMM kernel (differentiable w.r.t. the dense operand)."""
from ..ops import SparseAdj


class TorchGraphInterface(object):
    def __init__(self):
        pass

    @staticmethod
    def convert_sparse_mat_to_tensor(X):
        return SparseAdj(X)
