"""selfrec_b200: the H100-native hot path behind SELFRec's plugin surface.

    import selfrec_b200
    selfrec_b200.install()          # alias base.*, util.*, data.*, model.graph.* in sys.modules

after which the reference launcher (`SELFRec(conf).execute()`) and the reference's own
model files import this package's drop-in modules.  See INTEGRATION.md.

Under torchrun (`torchrun --nproc-per-node N main.py`) install() also starts the NCCL process group, one
GPU per process, and LightGCN / SimGCL / XSimGCL / SGL then train, evaluate and rank on the
bipartite-sharded engine.
"""
import importlib
import os
import sys

__version__ = "0.1.0"

_DROPIN = {
    # the five boundary modules (BASELINE.json north_star / SURVEY 8b)
    "base.graph_recommender": "selfrec_b200.base.graph_recommender",
    "base.torch_interface": "selfrec_b200.base.torch_interface",
    "util.loss_torch": "selfrec_b200.util.loss_torch",
    "util.sampler": "selfrec_b200.util.sampler",
    "data.ui_graph": "selfrec_b200.data.ui_graph",
    # SURVEY 8(f) rows: file -> CSR through the native builder, ranking metrics from device hit masks
    "data.loader": "selfrec_b200.data.loader",
    "util.evaluation": "selfrec_b200.util.evaluation",
}
_FUSED_MODELS = {f"model.graph.{m}": f"selfrec_b200.model.graph.{m}" for m in ("MF", "LightGCN", "SimGCL", "XSimGCL", "SGL", "ItemKNN", "UserKNN")}


def install(fused_models=True):
    """Register the drop-in modules under the reference's import names.

    With fused_models=True the five in-scope model classes resolve to the fused-engine
    versions too, and ItemKNN / UserKNN to their GPU versions; with False the reference's own model files run on top of the five
    boundary modules (op-level drop-in)."""
    if "WORLD_SIZE" in os.environ:  # started by torchrun: one process per GPU
        _init_process_group()
    table = dict(_DROPIN)
    if fused_models:
        table.update(_FUSED_MODELS)
    for alias, target in table.items():
        sys.modules[alias] = importlib.import_module(target)
    return sorted(table)


def _init_process_group():
    """NCCL default group on the GPU LOCAL_RANK names, unless the caller already made a group."""
    import atexit

    import torch
    import torch.distributed as dist
    if not dist.is_available() or dist.is_initialized():
        return
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    atexit.register(lambda: dist.destroy_process_group() if dist.is_initialized() else None)
