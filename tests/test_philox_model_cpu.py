"""The host model of the in-kernel Philox noise (tests/philox_model.py), without a GPU: the generator against Random123's
known-answer vectors, the unit map, and where each column of a noise row comes from."""
import numpy as np
import pytest
from philox_model import noise_offset, philox4x32_10, philox_noise, step_noise, u32_to_unit

# Random123 kat_vectors, philox4x32_10: (counter, key, output)
KAT = [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF, 0xFFFFFFFF), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]


@pytest.mark.parametrize("ctr,key,out", KAT, ids=["zeros", "ones", "pi"])
def test_philox_known_answer_vectors(ctr, key, out):
    assert philox4x32_10(ctr, key).tolist() == list(out)
    # vectorised: the same counter in every lane of an array gives the same answer in every lane
    arr = philox4x32_10(tuple(np.full((3, 5), w, dtype=np.uint32) for w in ctr), key)
    assert arr.shape == (3, 5, 4) and (arr == np.array(out, dtype=np.uint32)).all()


def test_unit_map_is_exact_and_in_range():
    u = np.array([0, 0xFF, 0x100, 0x80000000, 0xFFFFFEFF, 0xFFFFFFFF], dtype=np.uint32)
    got = u32_to_unit(u)
    assert got.dtype == np.float32
    want = [0.0, 0.0, 2.0 ** -24, 0.5, (2 ** 24 - 2) * 2.0 ** -24, 1 - 2.0 ** -24]
    assert got.astype(np.float64).tolist() == want  # every value is exact in float32
    rng = np.random.default_rng(0)
    r = rng.integers(0, 2 ** 32, 100000, dtype=np.uint64).astype(np.uint32)
    g = u32_to_unit(r).astype(np.float64)
    assert np.array_equal(g, (r >> 8).astype(np.float64) / 2 ** 24)  # the 24-bit integer survives the float32 round trip
    assert g.min() >= 0.0 and g.max() <= 1 - 2.0 ** -24


@pytest.mark.parametrize("d", [32, 64, 128])
def test_noise_columns_come_from_block_and_lane(d):
    """Column c of row r comes from Philox block c // 4 (counter word 1, with the view in its high half), lane c % 4; the
    row id, tag and step are counter words 0, 2, 3, and the seed's two words are the key."""
    seed, offset, step = 0x0123456789ABCDEF, noise_offset(1, 2), 0x7FFFFFFF
    rows = 5
    got = philox_noise(seed, offset, step, rows, d, row_base=3, row_stride=7)
    assert got.shape == (rows, d) and got.dtype == np.float32
    for r in range(rows):
        for c in range(d):
            ctr = (3 + 7 * r, (c // 4) | (1 << 16), 0x12, step)
            u = philox4x32_10(ctr, (0x89ABCDEF, 0x01234567))[c % 4]
            assert got[r, c] == np.float32(int(u) >> 8) * np.float32(2.0 ** -24), (r, c)


def test_step_pointer_is_read_as_uint32_and_keys_are_all_live():
    seed, n, d = 0x0123456789ABCDEF, 40, 32
    base = philox_noise(seed, noise_offset(0, 0), 1, n, d)
    assert np.array_equal(philox_noise(seed, noise_offset(0, 0), -1, n, d), philox_noise(seed, noise_offset(0, 0), 0xFFFFFFFF, n, d))
    assert np.array_equal(philox_noise(seed, noise_offset(0, 0), None, n, d), philox_noise(seed, noise_offset(0, 0), 0, n, d))
    others = [
        philox_noise(seed, noise_offset(0, 0), 2, n, d),                      # step
        philox_noise(seed, noise_offset(1, 0), 1, n, d),                      # view
        philox_noise(seed, noise_offset(0, 1), 1, n, d),                      # tag
        philox_noise(seed & 0xFFFFFFFF, noise_offset(0, 0), 1, n, d),        # seed high word
        philox_noise(seed ^ 1, noise_offset(0, 0), 1, n, d),                  # seed low word
        philox_noise(seed, noise_offset(0, 0), 1, n, d, row_base=1),          # row id
    ]
    for k, o in enumerate(others):
        assert (o != base).all(), k  # every value of a wrong keying differs (the seeds here have no collision)
    # row stride 0: every row draws row 0's values
    flat = philox_noise(seed, noise_offset(0, 0), 1, n, d, row_stride=0)
    assert (flat == base[0]).all()


def test_step_noise_layout():
    seed, L, N, d = 0x5EED, 3, 20, 64
    for model, views in (("SimGCL", 2), ("XSimGCL", 1)):
        t = step_noise(model, seed, L, N, d, 4)
        assert t.shape == (views, L, N, d) and t.dtype == np.float32
        for v in range(views):
            for k in range(L):
                assert np.array_equal(t[v, k], philox_noise(seed, (v << 32) | (0x10 + k), 4, N, d))
