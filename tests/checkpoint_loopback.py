"""Checkpoints across world sizes on one GPU: a run saved by W loopback ranks (tests/shard_loopback.py, whose docstring
states the safety guards) or by TrainEngine, resumed by another world or by TrainEngine.  One case per process, started by
tests/test_gpu_checkpoint.py with shard_loopback.LOOPBACK_ENV.

World 0 stands for the single-process TrainEngine.  The source trains K steps and saves; a destination built from other
initial tables loads the checkpoint; its global state must equal the source's bit for bit (every rank's item table
too); then both take the same M steps and must agree within 1e-4 of each table's scale."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

K, M, TOL = 6, 6, 1e-4
D, L, B = 64, 2, 256
KW = dict(eps=0.0, tau=0.2, cl_rate=0.2, layer_cl=1)


class _Single:
    """TrainEngine behind the LoopbackWorld surface the case uses."""

    def __init__(self, eng):
        self.engines, self.world = [eng], 0

    def step(self, words):
        import torch
        self.engines[0].step(words)
        torch.cuda.synchronize()

    def state(self):
        e = self.engines[0]
        return e.params.cpu().numpy(), e.m.cpu().numpy(), e.v.cpu().numpy(), e.losses.cpu().numpy()

    def check_replicas(self, final=False):
        pass


def _make(world, data, seed, dev):
    import torch
    import shard_loopback as lb
    from selfrec_b200.engine import TrainEngine
    from selfrec_b200.sharded import ShardedEngine
    U, I = data.user_num, data.item_num
    E0 = (np.random.default_rng(seed).standard_normal((U + I, D)) * 0.1).astype(np.float32)
    iu, ii = torch.from_numpy(E0[:U]), torch.from_numpy(E0[U:])
    if world == 0:
        return _Single(TrainEngine("XSimGCL", data, D, L, B, 1e-3, 1e-4, init_user=iu, init_item=ii, device=dev, **KW))
    return lb.LoopbackWorld(world, lambda g: ShardedEngine("XSimGCL", data, D, L, B, 1e-3, 1e-4, init_user=iu, init_item=ii, group=g,
                                                            device=dev, **KW), dev)


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def run(src, dst, root):
    import random
    import torch
    from selfrec_b200 import checkpoint, synth
    from selfrec_b200.util.sampler import NativePairSampler, stream_epoch
    dev = torch.device("cuda", 0)
    data = synth.make_interaction((2000, 1500, 30000), seed=5)
    random.seed(4)
    batches = [w.copy() for _, w in zip(range(K + M), stream_epoch(NativePairSampler(data), data, B, B))]
    a = _make(src, data, 1, dev)
    for w in batches[:K]:
        a.step(w)
    man = {"format": checkpoint.FORMAT_VERSION, "epoch": 0, "batch": K, "cursor": -1}
    path = checkpoint.save_engines(root, man, a.engines)
    man = checkpoint.read_manifest(path)
    assert man["world"] == max(src, 1) and man["step"] == K, man
    b = _make(dst, data, 2, dev)
    for e in b.engines:
        e.load_state_dict(checkpoint.engine_state(path, man, checkpoint.engine_user_ids(e)))
    b.check_replicas(final=False)  # every rank's item table bit-identical to rank 0's
    sa, sb = a.state(), b.state()
    for name, x, y in zip(("params", "m", "v"), sa[:3], sb[:3]):
        assert np.array_equal(x.view(np.int32), y.view(np.int32)), f"{name} differs after the load"
    assert all(int(e.step_dev.item()) == K for e in b.engines)
    worst = 0.0
    for k, w in enumerate(batches[K:]):
        a.step(w)
        b.step(w)
        sa, sb = a.state(), b.state()
        rels = [_rel(x, y) for x, y in zip(sb, sa)]
        worst = max(worst, max(rels))
        assert max(rels) <= TOL, (k, rels)
    print(f"checkpoint W{src} -> W{dst}: state bit-identical after the load, {M} more steps within {worst:.2e}", flush=True)


def main():
    case = json.loads(sys.argv[1])
    import torch
    import shard_loopback as lb
    torch.cuda.set_device(0)
    lb.install()
    run(case["src"], case["dst"], case["root"])
    print("CHECKPOINT_CASE PASS", flush=True)


if __name__ == "__main__":
    main()
