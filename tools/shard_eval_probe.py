#!/usr/bin/env python
"""Times evaluation on the sharded engine on one GPU; prints the card and one JSON line.

    tools/shard_eval_probe.py [--d 64] [--topn 20] [--reps 7]

On a yelp2018-shaped synthetic graph (31 668 x 38 048 x 1 237 259; 30 % of the users hold out 1-10 unrated items):
  * one fast_evaluation (top-k + hit masks + measure strings + the keep-best save()) of LightGCN through both routes:
    TrainEngine with the full tables, and the world-1 ShardedEngine ranking through ShardRanker;
  * the ranking of one rank of an N-GPU run (N = 2, 4, 8): local top-k + hit masks of its 1/N cyclic slice of the test
    users, i.e. what each rank spends before the all-gather of the masks.  The slowest of the N slices is reported.
Median of --reps host-clock timings, each ending in a device synchronise, after two warm-up calls."""
import argparse
import contextlib
import io
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


class _EvalData:
    """A synthetic interaction graph plus the name-keyed test set fast_evaluation reads (names are the ids)."""

    def __init__(self, base, seed):
        rng = np.random.default_rng(seed)
        self.base, self.user_num, self.item_num = base, base.user_num, base.item_num
        self.user = {u: u for u in range(self.user_num)}
        rp, ri = base.rated_csr()
        self.test_set = {}
        for u in rng.permutation(self.user_num)[: int(0.3 * self.user_num)].tolist():
            cand = rng.integers(0, self.item_num, 12)
            cand = np.setdiff1d(cand, ri[rp[u]:rp[u + 1]])[: int(rng.integers(1, 11))]
            if cand.size:
                self.test_set[u] = {int(i): 1 for i in cand}
        rows = [sorted(self.test_set.get(u, {})) for u in range(self.user_num)]
        ptr = np.zeros(self.user_num + 1, dtype=np.int32)
        ptr[1:] = np.cumsum([len(r) for r in rows])
        self._test = (ptr, np.fromiter((i for r in rows for i in r), dtype=np.int32, count=int(ptr[-1])), np.diff(ptr).astype(np.int32))

    def __getattr__(self, name):  # norm_adj, pair_users, ... for the engines
        return getattr(self.base, name)

    def rated_csr(self):
        return self.base.rated_csr()

    def test_csr(self):
        return self._test


def _timed(fn, reps):
    import torch
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--d", type=int, default=64)
    ap.add_argument("--topn", type=int, default=20)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    import torch
    from selfrec_b200 import build, synth
    build.build()
    from selfrec_b200.engine import TrainEngine
    from selfrec_b200.model.graph._common import FusedGraphModel
    from selfrec_b200.shard_rank import ShardRanker
    from selfrec_b200.sharded import ShardedEngine
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("card:", card.splitlines()[0] if card else "unknown", flush=True)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    data = _EvalData(synth.make_interaction("yelp2018", seed=3), seed=5)
    uids = np.fromiter(data.test_set, dtype=np.int32, count=len(data.test_set))
    torch.manual_seed(0)
    rec = {"card": card.splitlines()[0] if card else "unknown", "shape": [data.user_num, data.item_num], "d": args.d, "topN": args.topn,
           "test_users": int(uids.size)}

    def model(engine, ranker):
        m = object.__new__(FusedGraphModel)
        m.data, m.engine, m.max_N, m.shard_ranker = data, engine, args.topn, ranker
        m.user_emb, m.item_emb = engine.forward_clean()
        return m

    def fast_eval(m):
        m.bestPerformance = []  # every call takes the keep-best branch: save() included
        with contextlib.redirect_stdout(io.StringIO()):
            return m.fast_evaluation(0)

    eng = TrainEngine("LightGCN", data, args.d, 2, 2048, 1e-3, 1e-4, device=dev)
    init_u, init_i = eng.user_emb.clone(), eng.item_emb.clone()
    single = model(eng, None)
    sh = ShardedEngine("LightGCN", data, args.d, 2, 2048, 1e-3, 1e-4, init_user=init_u, init_item=init_i, device=dev)
    sharded = model(sh, ShardRanker(data, 0, 1, dev))
    same = fast_eval(single) == fast_eval(sharded)
    t_single, t_sharded = [], []
    for _ in range(3):  # alternate the two routes
        t_single.append(_timed(lambda: fast_eval(single), args.reps))
        t_sharded.append(_timed(lambda: fast_eval(sharded), args.reps))
    rec["fast_evaluation_ms"] = {"TrainEngine": min(t_single), "ShardedEngine_world1": min(t_sharded), "same_measure": same}
    ue, ie = single.user_emb, single.item_emb
    per_rank = {}
    for world in (1, 2, 4, 8):
        worst = 0.0
        for g in range(world):
            rk = ShardRanker(data, g, world, dev)
            block = ue[g::world].contiguous()
            worst = max(worst, _timed(lambda: rk.local_hit_masks(block, ie, uids, args.topn), args.reps))
        per_rank[str(world)] = worst
    rec["per_rank_ranking_ms"] = per_rank
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
