"""Golden vectors for R11 (data/augmentor.py): runs the UNMODIFIED reference GraphAugmentor on a fixed matrix with
fixed `random` seeds and records what it drops.  Test infrastructure; run in the build container only
(needs a checkout of the reference):

    python oracle/gen_golden_augment.py --ref <reference checkout> [--out tests/golden]
"""
import argparse
import os
import random
import sys

import numpy as np
import scipy.sparse as sp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", required=True, help="root of a Coder-Yu/SELFRec checkout")
    ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden"))
    args = ap.parse_args()
    sys.path.insert(0, args.ref)
    from data.augmentor import GraphAugmentor  # the reference's own

    mat = sp.random(150, 220, density=0.03, random_state=7, format="csr", dtype=np.float32)
    mat.data[:] = 1.0
    mat.sort_indices()
    fx = dict(meta=str(dict(python=sys.version.split()[0], numpy=np.__version__, scipy=sp.__name__)),
              in_indptr=mat.indptr, in_indices=mat.indices, in_shape=np.array(mat.shape))
    cases = []
    for kind in ("node_dropout", "edge_dropout"):
        for rate, seed in ((0.1, 11), (0.5, 12), (0.0, 13)):
            random.seed(seed)
            out = sp.csr_matrix(getattr(GraphAugmentor, kind)(mat, rate))
            out.sum_duplicates()
            out.eliminate_zeros()
            out.sort_indices()
            tag = f"{kind}_{len(cases)}"
            cases.append(f"{kind}:{rate}:{seed}:{tag}")
            fx[tag + "_indptr"], fx[tag + "_indices"], fx[tag + "_data"] = out.indptr, out.indices, out.data.astype(np.float32)
            fx[tag + "_next_random"] = np.array([random.random()])  # where the generator stands afterwards
    fx["cases"] = np.array(cases)
    np.savez_compressed(os.path.join(args.out, "augment.npz"), **fx)
    print("wrote", os.path.join(args.out, "augment.npz"), cases)


if __name__ == "__main__":
    main()
