"""Golden vectors of the neighbourhood baselines: runs the UNMODIFIED reference ItemKNN and UserKNN (train(), test(),
ranking_evaluation) and writes tests/golden/knn.npz, plus the crafted dataset it uses.  Needs a checkout of the
reference and numba; run on a CPU machine:

    python tools/gen_golden_knn.py --ref <reference checkout> [--out tests/golden]

Datasets: the golden tiny set (tiny_train.txt / tiny_test.txt) and a crafted one (knn_crafted_*.txt) with items of
identical user sets (exactly equal sims), names whose string order differs from id order, users with one rated item
(zero-score ties reach the top-N), an item and a user with no candidates, duplicate lines, and rated items among the
first ids (masked entries seed the heap and get replaced).  Settings: the shipped topK 50 / shrinkage 100, and
topK 5 / shrinkage 2, where the cut falls inside tie groups.
"""
import argparse
import os
import sys
import tempfile

import numpy as np

SETTINGS = ((50, 100), (5, 2))
TOP_N = [10, 20]


def crafted_lines():
    rng = np.random.default_rng(20261017)
    users = [f"u{n}" for n in (9, 10, 2, 100, 11, 1, 27, 3, 30, 5, 50, 7, 70, 12, 120, 8, 80, 4, 40, 6, 60, 13, 21, 999)]
    items = [f"i{n}" for n in (9, 10, 1, 100, 11, 2, 20, 3, 30, 4, 40, 5, 50, 6, 60, 7, 70, 8, 80, 12, 21, 13, 31, 14, 41, 999)]
    train = []
    # u9 rates the first ids: its mask covers ids < max_N, so masked entries seed the heap
    for it in ("i9", "i10", "i1", "i100", "i11", "i2"):
        train.append(f"u9 {it} 1")
    # i3 and i30 have the same user set {u10, u2}: their sims to every other item are equal
    train += ["u10 i3 1", "u10 i30 1", "u2 i3 4", "u2 i30 2", "u10 i9 1", "u2 i10 1"]
    pool = [it for it in items[:-1]]
    for u in users[3:-1]:
        if u in ("u7", "u70"):
            continue
        for it in rng.choice(pool, size=int(rng.integers(2, 7)), replace=False):
            train.append(f"{u} {it} {int(rng.integers(1, 6))}")
    train += ["u7 i1 1", "u70 i20 3"]  # one rated item each
    train += ["u999 i999 1"]            # a user and an item with no candidates
    train += [train[3], train[8], "u2 i3 5"]  # duplicate lines keep their first position
    test = []
    for u in users:
        rated = {ln.split()[1] for ln in train if ln.split()[0] == u}
        cand = [it for it in items if it not in rated]
        for it in rng.choice(cand, size=2, replace=False):
            test.append(f"{u} {it} 1")
    test.append("ghost i9 1")  # a user unknown to training is filtered
    return [ln + "\n" for ln in train], [ln + "\n" for ln in test]


class Conf:
    def __init__(self, model, topk, shrinkage):
        self.config = {"training.set": "train.txt", "test.set": "test.txt", "model": {"name": model, "type": "graph"},
                       "item.ranking.topN": TOP_N, "topK": topk, "shrinkage": shrinkage, "embedding.size": 64,
                       "max.epoch": 1, "batch.size": 2048, "learning.rate": 0.001, "reg.lambda": 0.0001, "output": "./results/"}

    def __getitem__(self, k):
        return self.config[k]

    def contain(self, k):
        return k in self.config


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", required=True, help="root of a Coder-Yu/SELFRec checkout")
    ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden"))
    args = ap.parse_args()
    out = os.path.abspath(args.out)
    train_lines, test_lines = crafted_lines()
    for name, lines in (("knn_crafted_train.txt", train_lines), ("knn_crafted_test.txt", test_lines)):
        with open(os.path.join(out, name), "w") as f:
            f.writelines(lines)
    os.chdir(tempfile.mkdtemp(prefix="srb_golden_knn_"))  # the reference's logger writes under ./log
    sys.path.insert(0, os.path.abspath(args.ref))
    import numba
    from data.loader import FileIO
    from model.graph.ItemKNN import ItemKNN
    from model.graph.UserKNN import UserKNN
    from util.evaluation import ranking_evaluation

    fx = dict(meta=np.array(str(dict(python=sys.version.split()[0], numpy=np.__version__, numba=numba.__version__))),
              top_n=np.array(TOP_N), settings=np.array(SETTINGS))
    for ds, (tr, te) in (("tiny", ("tiny_train.txt", "tiny_test.txt")), ("crafted", ("knn_crafted_train.txt", "knn_crafted_test.txt"))):
        train = FileIO.load_data_set(os.path.join(out, tr), "graph")
        test = FileIO.load_data_set(os.path.join(out, te), "graph")
        for cls, kind in ((ItemKNN, "item"), (UserKNN, "user")):
            for topk, shrink in SETTINGS:
                tag = f"{ds}_{cls.__name__}_{topk}_{shrink}"
                m = cls(Conf(cls.__name__, topk, shrink), [list(t) for t in train], [list(t) for t in test])
                m.train()
                d = m.data
                sim = m.item_sim if kind == "item" else m.user_sim
                names = [d.id2item[k] for k in range(d.item_num)] if kind == "item" else [d.id2user[k] for k in range(d.user_num)]
                index = d.item if kind == "item" else d.user
                ids = np.full((len(names), topk), -1, dtype=np.int32)
                sims = np.zeros((len(names), topk), dtype=np.float64)
                cnt = np.zeros(len(names), dtype=np.int32)
                for a, nm in enumerate(names):
                    lst = sim[nm]
                    cnt[a] = len(lst)
                    for t, (s, other) in enumerate(lst):
                        ids[a, t], sims[a, t] = index[other], s
                unames = [d.id2user[k] for k in range(d.user_num)]
                rows = np.stack([m.predict(u) for u in unames]).astype(np.float64)
                rec = m.test()
                test_users = list(d.test_set)
                rec_ids = np.array([[d.item[it] for it, _ in rec[u]] for u in test_users], dtype=np.int32)
                rec_sc = np.array([[s for _, s in rec[u]] for u in test_users], dtype=np.float64)
                result = ranking_evaluation(d.test_set, rec, m.topN)
                fx.update({tag + "_nbr_ids": ids, tag + "_nbr_sims": sims, tag + "_nbr_cnt": cnt, tag + "_predict": rows,
                           tag + "_test_users": np.array([d.user[u] for u in test_users], dtype=np.int32),
                           tag + "_rec_ids": rec_ids, tag + "_rec_scores": rec_sc, tag + "_metrics": np.array(result)})
                print(tag, "done")
    np.savez_compressed(os.path.join(out, "knn.npz"), **fx)
    print("wrote", os.path.join(out, "knn.npz"))


if __name__ == "__main__":
    main()
