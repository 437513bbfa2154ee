"""Drop-in for util/loss_torch.py: bpr_loss (:6-10), l2_reg_loss (:18-22), batch_softmax_loss (:25-32),
InfoNCE (:35-50).

Same signatures, autograd-differentiable, composable with + and *; each one runs the
hand-written CUDA kernels through the C ABI (selfrec_b200.ops).  batch_softmax_loss works in
log-sum-exp form and stays finite at temperatures below 1/88.7, where the reference's exp overflows
(INTEGRATION §4).  The remaining helpers of the reference file (triplet_loss, info_nce,
kl_divergence) are not imported by any reference model and are intentionally absent (SURVEY 2).
"""
from ..ops import InfoNCE, batch_softmax_loss, bpr_loss, l2_reg_loss

__all__ = ["bpr_loss", "l2_reg_loss", "batch_softmax_loss", "InfoNCE"]
