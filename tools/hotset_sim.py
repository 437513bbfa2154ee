#!/usr/bin/env python
"""CPU simulation behind DESIGN 4.1.1 / 6 (no GPU): on the config-5 recipe graph (SURVEY 8d: Zipf(1.1) on both sides,
de-duplicated, first-appearance ids; here the 1/5-size shape synthetic-2M so that it runs in a minute on the host),
  * which share of the SpMM's row gathers a STATIC hot set of K rows (what an L2 of that size could pin at best) covers,
    per phase (user rows gather item rows, item rows gather user rows) and mixed -- the floor of the DRAM traffic of the
    product on a graph whose only locality is column popularity;
  * how contiguous nnz-balanced user blocks compare with the cyclic assignment (rows per rank), and how many
    (rank, item) partial rows of the item-side product are empty.

    python tools/hotset_sim.py [shape]
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from selfrec_b200 import synth  # noqa: E402

torch.set_num_threads(min(32, os.cpu_count() or 1))
shape = sys.argv[1] if len(sys.argv) > 1 else "synthetic-2M"
U, I, nnz = synth.SHAPES[shape]
pu, pi = synth.make_pairs_device(U, I, nnz, 0, 1.1, "cpu")
pu, pi = pu.numpy().astype(np.int64), pi.numpy().astype(np.int64)
du, di = np.bincount(pu, minlength=U), np.bincount(pi, minlength=I)
cu, ci = np.cumsum(np.sort(du)[::-1]) / nnz, np.cumsum(np.sort(di)[::-1]) / nnz
both = np.cumsum(np.sort(np.concatenate([du, di]))[::-1]) / (2 * nnz)
print(f"{shape}: {U} x {I} x {nnz}; degree quantiles (10/50/90/99 %): items {np.quantile(di, [.1, .5, .9, .99])}, users {np.quantile(du, [.1, .5, .9, .99])}")
print("static hot set of K rows of 512 B (d = 128):")
for mb in (32, 64, 96, 126):
    K = mb * (1 << 20) // 512
    print(f"  {mb:4d} MB = {K:7d} rows: user phase (item rows) {ci[min(K, I) - 1]:.3f} of the gathers, item phase (user rows) {cu[min(K, U) - 1]:.3f}, "
          f"one mixed set {both[K - 1]:.3f}")
for K in (432, 2048):
    print(f"  ids < {K} (first-appearance ids ~ popularity): items {di[:K].sum() / nnz:.3f}, users {du[:K].sum() / nnz:.3f} of the non-zeros")
for G in (2, 4, 8):
    cs = np.cumsum(du)
    bounds = np.searchsorted(cs, np.arange(1, G) * nnz // G)
    blk = np.searchsorted(bounds, pu, side="right")
    sizes = np.diff(np.concatenate([[0], bounds, [U]]))
    ne_c = len(np.unique(blk * I + pi)) / (G * I)
    cyc = pu % G
    per = np.bincount(cyc, minlength=G)
    ne_y = len(np.unique(cyc * I + pi)) / (G * I)
    print(f"world {G}: contiguous nnz-balanced user blocks {sizes.tolist()} (non-empty partial item rows {ne_c:.3f}); "
          f"cyclic: users {[(U - g + G - 1) // G for g in range(G)]}, nnz max/mean {per.max() / per.mean():.3f} (non-empty {ne_y:.3f})")
