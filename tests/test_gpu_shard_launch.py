"""`torchrun --nproc-per-node N` of the launcher flow (install() + execute()) for LightGCN, XSimGCL, SimGCL and SGL
on the sharded engine, against the same flow in one plain process (tests/shard_launch_gpu_check.py).  World 1 runs
on any box with a GPU; worlds 2, 4 and 8 when the box has the GPUs."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHECK = os.path.join(ROOT, "tests", "shard_launch_gpu_check.py")


@pytest.fixture(scope="module")
def reference_run(built_lib, tmp_path_factory):
    """The plain single-process run every world is compared with."""
    out = str(tmp_path_factory.mktemp("shard_launch"))
    env = {k: v for k, v in os.environ.items() if k not in ("WORLD_SIZE", "RANK", "LOCAL_RANK")}
    r = subprocess.run([sys.executable, CHECK, "--ref", "--out", out], capture_output=True, text=True, timeout=900, env=env)
    assert "SHARD_LAUNCH REF" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    return out


@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_launcher_flow_on_the_sharded_engine(reference_run, world):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs at least {world} GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(29711 + world), CHECK, "--out", reference_run]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1200)
    print(r.stdout[-4000:])
    assert "SHARD_LAUNCH PASS" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
