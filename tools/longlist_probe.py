"""Time top-k lists of 33..256 on the tensor-core route (impl 2: candidate buffers behind a running threshold) against
the dense-row route (ops._score_topk_wide), fast_evaluation at topN [20, 100], and a top-100 export.

1. Rank every user of the yelp2018 shape (synth.make_interaction, random N(0, 0.1) tables) at k in {20, 50, 100, 256} and
   d in {64, 128}: CUDA events over --reps calls after a warm-up call, the users the exact fallback re-ran, and for
   k > 32 the dense-row route on the same tables (which must return the same lists, bit for bit).
2. One fast_evaluation measure at topN [20, 100] on a yelp2018-sized synthetic split (a random held-out fifth of each
   user's pairs): the device route (_fast_measure) against ranking_evaluation over test() on the dense-row route, the
   route max_N = 100 took before.  Both must return the same strings.
3. Export the top-100 lists of every user of the --export-shape model (default synthetic-5M: 5 M users x 1 M items) at
   d = 128: wall time, GB written, peak device memory above the tables.  The dense-row route is timed on
   --wide-users users only (one of its chunks is 268 users at 1 M items); its full-size time is not measured.
Prints the card's name and power limit, then one JSON line per measurement.

    python tools/longlist_probe.py [--reps 3] [--skip-export] [--export-shape synthetic-5M] [--wide-users 2144]"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from export_probe import _Model, _Names, card  # noqa: E402


def _time(fn, reps):
    import torch
    out = fn()  # warm-up
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1) / reps


def rank_times(reps):
    import numpy as np
    import torch
    from selfrec_b200 import ops, synth
    data = synth.make_interaction("yelp2018", seed=0)
    U, I = data.user_num, data.item_num
    rp, ri = (torch.from_numpy(a).cuda() for a in data.rated_csr())
    users = torch.arange(U, dtype=torch.int32, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    for d in (64, 128):
        ue = torch.randn((U, d), device="cuda", generator=g) * 0.1
        ie = torch.randn((I, d), device="cuda", generator=g) * 0.1
        for k in (20, 50, 100, 256):
            st = {}
            (ids, sc), ms = _time(lambda: ops.score_topk(ue, ie, users, rp, ri, k, stats=st), reps)
            row = dict(what="rank_all_users", shape="yelp2018", users=U, items=I, d=d, k=k, route="tensor_cores", ms=ms, reps=reps,
                       fallback_users=int(st["fallback_count"].item()))
            if k > 32:
                (wi, ws), wms = _time(lambda: ops._score_topk_wide(ue, ie, users, rp, ri, k), reps)
                row.update(wide_ms=wms, equal_to_wide=bool(torch.equal(ids, wi) and torch.equal(sc.view(torch.int32), ws.view(torch.int32))))
            print(json.dumps(row), flush=True)
        del ue, ie


class _Conf:
    def __init__(self, **over):
        self.config = {"model": {"name": "MF", "type": "graph"}, "item.ranking.topN": [20, 100], "embedding.size": 64,
                       "max.epoch": 1, "batch.size": 2048, "learning.rate": 0.001, "reg.lambda": 0.0001, "output": "./results/"}
        self.config.update(over)

    def __getitem__(self, k):
        return self.config[k]

    def contain(self, k):
        return k in self.config


def fast_eval_times():
    import numpy as np
    import torch
    from selfrec_b200 import ops, synth
    from selfrec_b200.base.graph_recommender import GraphRecommender
    from selfrec_b200.util.evaluation import ranking_evaluation
    pu, pi = synth.make_pairs(31668, 38048, 1561406, seed=0)
    rng = np.random.default_rng(0)
    held = rng.random(pu.size) < 0.2
    train = [[f"u{u}", f"i{i}", 1.0] for u, i in zip(pu[~held].tolist(), pi[~held].tolist())]
    test = [[f"u{u}", f"i{i}", 1.0] for u, i in zip(pu[held].tolist(), pi[held].tolist())]
    m = GraphRecommender(_Conf(), train, test)
    g = torch.Generator(device="cuda").manual_seed(2)
    m.user_emb = torch.randn((m.data.user_num, 64), device="cuda", generator=g) * 0.1
    m.item_emb = torch.randn((m.data.item_num, 64), device="cuda", generator=g) * 0.1
    m._fast_measure()  # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fast = m._fast_measure()
    fast_s = time.perf_counter() - t0
    route = ops.long_list_route
    ops.long_list_route = lambda *a, **kw: False  # the route max_N = 100 took before: dense rows, then test()'s dicts
    try:
        ranking_evaluation(m.data.test_set, m.test(), [m.max_N])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        slow = ranking_evaluation(m.data.test_set, m.test(), [m.max_N])
        slow_s = time.perf_counter() - t0
    finally:
        ops.long_list_route = route
    print(json.dumps(dict(what="fast_evaluation", topN=[20, 100], users=m.data.user_num, items=m.data.item_num,
                          test_users=len(m.data.test_set), d=64, device_route_s=fast_s, test_dict_route_s=slow_s,
                          same_strings=fast == slow)), flush=True)


def export_time(shape, top_n, out_dir, wide_users):
    import numpy as np
    import torch
    from selfrec_b200 import export, ops, synth
    data = synth.make_device_interaction(shape, seed=0)
    data.id2user, data.id2item = _Names(), _Names()
    data.rated_csr(), data.pair_users
    U, I = data.user_num, data.item_num
    g = torch.Generator(device="cuda").manual_seed(1)
    ue = torch.randn((U, 128), device="cuda", generator=g) * 0.1
    ie = torch.randn((I, 128), device="cuda", generator=g) * 0.1
    data.bip = data.norm_adj = None
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    m = _Model(data, ue, ie, top_n)
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    path = export.export_recommendations(m, out_dir, top_n=top_n)
    export_s = time.perf_counter() - t0
    nbytes = sum(os.path.getsize(os.path.join(path, f)) for f in os.listdir(path))
    print(json.dumps(dict(what="export", route="tensor_cores", shape=shape, users=U, items=I, d=128, N=top_n, seconds=export_s,
                          gb_written=nbytes / 1e9, peak_device_gb_above_tables=(torch.cuda.max_memory_allocated() - base) / 1e9,
                          chunk=export.long_list_chunk(export.EXPORT_CHUNK, I, 128, top_n))), flush=True)
    _, ids_all, sc_all = export.read(path)
    # the dense-row route on the first wide_users users only
    rp, ri = (torch.from_numpy(a).cuda() for a in data.rated_csr())
    users = torch.arange(wide_users, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    wi, ws = ops._score_topk_wide(ue, ie, users, rp, ri, top_n)
    torch.cuda.synchronize()
    wide_s = time.perf_counter() - t0
    same = np.array_equal(wi.cpu().numpy(), np.asarray(ids_all[:wide_users])) and \
        np.array_equal(ws.cpu().numpy().view(np.uint32), np.asarray(sc_all[:wide_users]).view(np.uint32))
    print(json.dumps(dict(what="export_slice_dense_rows", shape=shape, users=wide_users, items=I, d=128, N=top_n, seconds=wide_s,
                          equal_to_export=bool(same))), flush=True)
    shutil.rmtree(path, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--export-shape", default="synthetic-5M")
    ap.add_argument("--wide-users", type=int, default=2144)
    ap.add_argument("--skip-export", action="store_true")
    ap.add_argument("--skip-fast-eval", action="store_true")
    args = ap.parse_args()
    from selfrec_b200 import _lib
    _lib.require_device()
    print(json.dumps(dict(card=card())), flush=True)
    rank_times(args.reps)
    if not args.skip_fast_eval:
        fast_eval_times()
    if not args.skip_export:
        out = tempfile.mkdtemp(prefix="longlist_probe_")
        try:
            export_time(args.export_shape, 100, out, args.wide_users)
        finally:
            shutil.rmtree(out, ignore_errors=True)


if __name__ == "__main__":
    main()
