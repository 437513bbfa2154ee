"""The bipartite-sharded step's multi-rank exchange on one GPU: W loopback ranks in one process (tests/shard_loopback.py,
whose docstring states the safety guards), one subprocess per case, against the float64 oracle and the single-GPU engine.

Worlds 2, 3, 8 and 7 (7 divides neither the users nor the items: uneven user blocks and item slices) on a graph whose
item hubs stay split rows in every rank's item block.  Every case checks after every step that each rank's item table is
bit-identical to rank 0's and that no device-side barrier timed out."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HARNESS = os.path.join(ROOT, "tests", "shard_loopback.py")
if os.path.dirname(HARNESS) not in sys.path:
    sys.path.insert(0, os.path.dirname(HARNESS))

ORACLE_CASES = [
    # name, world, d, L, layer_cl, SGL views
    ("LightGCN", 2, 64, 3, 0, None),
    ("LightGCN", 7, 32, 1, 0, None),
    ("SimGCL", 3, 128, 2, 0, None),
    ("SimGCL", 8, 32, 1, 0, None),
    ("XSimGCL", 8, 64, 3, 1, None),
    ("XSimGCL", 7, 128, 2, 2, None),
    ("SGL", 2, 128, 1, 0, "edge"),
    ("SGL", 3, 64, 3, 0, "edge"),
    ("SGL", 8, 64, 2, 0, "node"),
    ("SGL", 7, 32, 3, 0, "node"),
]
PHILOX_CASES = [
    # name, world, d, L, layer_cl
    ("SimGCL", 8, 64, 2, 0),
    ("SimGCL", 7, 32, 3, 0),
    ("XSimGCL", 3, 32, 3, 1),
]


def _run(case):
    from shard_loopback import LOOPBACK_ENV
    env = dict(os.environ, **LOOPBACK_ENV)
    r = subprocess.run([sys.executable, HARNESS, json.dumps(case)], capture_output=True, text=True, timeout=300, env=env, cwd=ROOT)
    assert r.returncode == 0 and "LOOPBACK_CASE PASS" in r.stdout, r.stdout[-3000:] + r.stderr[-5000:]
    print(r.stdout)


def _oracle_id(c):
    name, world, d, L, lcl, views = c
    return f"W{world}-{name}-d{d}-L{L}" + (f"-lcl{lcl}" if name == "XSimGCL" else "") + (f"-{views}" if views else "")


@pytest.mark.parametrize("name,world,d,L,lcl,views", ORACLE_CASES, ids=[_oracle_id(c) for c in ORACLE_CASES])
def test_loopback_step_from_poisoned_workspace_vs_oracle(built_lib, orc, name, world, d, L, lcl, views):
    """A poison step, then a full batch with hubs, 17 triples, one hub triple, an empty batch and one hub triple B times,
    each step against the float64 oracle (SimGCL / XSimGCL at eps = 0), then the clean forward against the oracle's."""
    _run(dict(kind="oracle", name=name, world=world, d=d, L=L, lcl=lcl, views=views))


@pytest.mark.parametrize("name,world,d,L,lcl", PHILOX_CASES, ids=[f"W{c[1]}-{c[0]}-d{c[2]}-L{c[3]}" for c in PHILOX_CASES])
def test_loopback_philox_noise_matches_single_gpu(built_lib, name, world, d, L, lcl):
    """At eps > 0 the user rows' noise is keyed by global id (rank + row * world): the loopback world follows TrainEngine
    with the same philox_seed, up to the few rows a sign flip at y ~ 0 moves (at most 1e-3 of the rows)."""
    _run(dict(kind="philox", name=name, world=world, d=d, L=L, lcl=lcl))


@pytest.mark.parametrize("world,n_users,match", [(9, 40, "up to 8 ranks"), (3, 2, "cannot be spread")])
def test_loopback_world_refused_like_sharded_engine(built_lib, monkeypatch, world, n_users, match):
    """More than 8 ranks, or fewer users than ranks: every rank's engine refuses before it allocates or launches anything."""
    import torch
    import shard_loopback as lb
    from test_gpu_step_edges import _HubData
    from selfrec_b200 import _lib
    from selfrec_b200.sharded import ShardedEngine
    lb.install(monkeypatch.setattr)
    pu = np.arange(n_users, dtype=np.int32)
    data = _HubData(pu, pu % 3, n_users, 3)
    dev = torch.device("cuda", torch.cuda.current_device())
    for r in range(world):
        group = lb.FakeGroup(lb._Pool(world, dev), r)
        with pytest.raises(_lib.SrbError, match=match):
            ShardedEngine("LightGCN", data, 32, 1, 8, 1e-3, 1e-4, group=group, device=dev)
