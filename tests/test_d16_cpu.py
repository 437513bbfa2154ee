"""Embedding size 16 without a GPU: where the SpMM epilogue's Philox noise comes from when a row lives on two lanes,
and the supported widths the Python layer and the C header state."""
import os
import re

import numpy as np
from philox_model import noise_offset, philox4x32_10, philox_noise

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_philox_noise_blocks_follow_the_two_lane_rule():
    """At d = 16 a row lives on LPR = 2 lanes, two float4 per lane: lane gl draws counter block gl for columns
    [4 gl, 4 gl + 4) and block gl + 2 for columns [8 + 4 gl, 8 + 4 gl + 4), with the view above bit 16."""
    d, lpr = 16, 2
    seed, offset, step = 0xFEDC000089ABCDEF, noise_offset(1, 3), 5
    got = philox_noise(seed, offset, step, 5, d, row_base=11, row_stride=2)
    key = (seed & 0xFFFFFFFF, seed >> 32)
    seen = set()
    for r in range(5):
        for gl in range(lpr):
            for half, blk in ((0, gl), (1, gl + lpr)):
                u = philox4x32_10((11 + 2 * r, blk | (1 << 16), 0x13, step), key)
                want = (u >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)
                c0 = half * d // 2 + 4 * gl
                assert c0 // 4 == blk  # the counter block is the column block, as at every width
                assert np.array_equal(got[r, c0:c0 + 4], want), (r, gl, half)
                seen.add(c0)
    assert sorted(seen) == [0, 4, 8, 12]  # the two lanes' four float4 cover the row exactly once


def test_d16_noise_is_the_prefix_of_the_wider_streams():
    """The counter does not depend on the width: the first 16 columns of a row's noise at d = 32 are its noise at d = 16
    (the blocks 0..3 of both)."""
    seed, offset, step = 0x0123456789ABCDEF, noise_offset(0, 2), 9
    n16 = philox_noise(seed, offset, step, 7, 16)
    n32 = philox_noise(seed, offset, step, 7, 32)
    assert n16.shape == (7, 16) and n16.dtype == np.float32
    assert np.array_equal(n16, n32[:, :16])


def test_supported_widths_agree_with_the_header_and_include_16():
    from selfrec_b200 import ops
    with open(os.path.join(ROOT, "include", "selfrec_b200.h")) as f:
        m = re.search(r"d \(embedding\.size\) must be one of ([0-9, ]+)\.", f.read())
    assert m is not None
    assert tuple(int(x) for x in m.group(1).split(",")) == ops._SUPPORTED_D
    assert ops._SUPPORTED_D == (16, 32, 64, 128, 256)
    assert 8 not in ops._SUPPORTED_D and 24 not in ops._SUPPORTED_D


def test_c_sources_list_16_in_every_width_message():
    """Every C-side width message names the same five widths as the header."""
    csrc = os.path.join(ROOT, "selfrec_b200", "csrc")
    msgs = []
    for fn in sorted(os.listdir(csrc)):
        if fn.endswith(".cu"):
            with open(os.path.join(csrc, fn)) as f:
                msgs += re.findall(r"unsupported d=%d \(([0-9, ]+)\)", f.read())
    assert len(msgs) >= 11  # spmm 3, bpr 2, infonce 1, score_topk 2, sharded 2, engine 1
    assert set(msgs) == {"16, 32, 64, 128, 256"}
