"""Embedding size 256 without a GPU: where the SpMM epilogue's Philox noise comes from when one lane group is the whole
warp, and the supported widths the Python layer and the C header state."""
import os
import re

import numpy as np
from philox_model import noise_offset, philox4x32_10, philox_noise

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_philox_noise_blocks_follow_the_whole_warp_rule():
    """At d = 256 a row lives on LPR = 32 lanes, two float4 per lane: lane gl draws counter block gl for columns
    [4 gl, 4 gl + 4) and block gl + 32 for columns [128 + 4 gl, 128 + 4 gl + 4), with the view above bit 16."""
    d, lpr = 256, 32
    seed, offset, step = 0xFEDC000089ABCDEF, noise_offset(1, 3), 5
    got = philox_noise(seed, offset, step, 3, d, row_base=11, row_stride=2)
    key = (seed & 0xFFFFFFFF, seed >> 32)
    for r in range(3):
        for gl in range(lpr):
            for half, blk in ((0, gl), (1, gl + lpr)):
                assert blk < 1 << 16  # the column block never reaches the view bits
                u = philox4x32_10((11 + 2 * r, blk | (1 << 16), 0x13, step), key)
                want = (u >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)
                c0 = half * d // 2 + 4 * gl
                assert np.array_equal(got[r, c0:c0 + 4], want), (r, gl, half)


def test_supported_widths_agree_with_the_header():
    from selfrec_b200 import ops
    with open(os.path.join(ROOT, "include", "selfrec_b200.h")) as f:
        m = re.search(r"d \(embedding\.size\) must be one of ([0-9, ]+)\.", f.read())
    assert m is not None
    assert tuple(int(x) for x in m.group(1).split(",")) == ops._SUPPORTED_D
    assert 256 in ops._SUPPORTED_D and 48 not in ops._SUPPORTED_D
