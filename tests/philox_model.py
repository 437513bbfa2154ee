"""Host model of the in-kernel Philox noise (noise mode 2) of the SpMM epilogue, bit for bit.

For output element (row, col) of a product whose epilogue draws noise (csrc/spmm.cu, spmm_epilogue):

    ctr = (row_base + row * row_stride,  (col // 4) | (view << 16),  tag,  step)      uint32 words
    key = (seed & 0xFFFFFFFF, seed >> 32)
    u   = philox4x32_10(ctr, key)[col % 4]
    val = float32(u >> 8) * 2**-24                                                   (u32_to_unit, csrc/common.cuh)

tag and view are the low and high words of the product's philox_offset; step is the int32 the step pointer holds, read
as a uint32 (0 without a pointer).  The training step keys layer k (0-based) of view v with noise_offset(v, k) =
v << 32 | (0x10 + k) (csrc/spmm_args.cuh) and the step counter after step_begin_kernel bumped it, so the n-th step
(counted from 1) draws step n.  Mode 1 of the same epilogue reads these values from a tensor instead, and everything
after the noise values is shared code: the two modes give the same bits when mode 1 is fed philox_noise().
"""
import numpy as np

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_MASK = 0xFFFFFFFF


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al. 2011) on uint32 arrays, as csrc/common.cuh computes it.  ctr: four broadcastable
    arrays (counter words 0..3); key: two ints.  Returns uint32 [..., 4] (output words 0..3)."""
    c = [np.asarray(x, dtype=np.uint32) for x in np.broadcast_arrays(*ctr)]
    k0, k1 = int(key[0]) & _MASK, int(key[1]) & _MASK
    for _ in range(10):
        p0 = _M0 * c[0].astype(np.uint64)
        p1 = _M1 * c[2].astype(np.uint64)
        hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), p0.astype(np.uint32)
        hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), p1.astype(np.uint32)
        c = [hi1 ^ c[1] ^ np.uint32(k0), lo1, hi0 ^ c[3] ^ np.uint32(k1), lo0]
        k0, k1 = (k0 + _W0) & _MASK, (k1 + _W1) & _MASK
    return np.stack(c, -1)


def u32_to_unit(u):
    """The kernel's map of a uint32 onto [0, 1): the top 24 bits times 2^-24, exact in float32."""
    return (np.asarray(u, dtype=np.uint32) >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)


def noise_offset(view, layer):
    """philox_offset of layer `layer` (0-based) of view `view` in the training step (csrc/spmm_args.cuh)."""
    return (int(view) << 32) | (0x10 + int(layer))


def philox_noise(seed, offset, step, n_rows, d, row_base=0, row_stride=1):
    """The [n_rows, d] float32 noise the epilogue draws with philox_seed `seed`, philox_offset `offset` and a step
    pointer that holds `step` (None: no pointer).  Row r has the Philox row id row_base + r * row_stride."""
    if d % 4:
        raise ValueError("d must be a multiple of 4")
    seed, offset = int(seed), int(offset)
    tag, view = offset & _MASK, (offset >> 32) & _MASK
    stp = 0 if step is None else int(step) & _MASK
    rows = ((int(row_base) + np.arange(n_rows, dtype=np.int64) * int(row_stride)) & _MASK).astype(np.uint32)
    blk = np.arange(d // 4, dtype=np.uint32) | np.uint32((view << 16) & _MASK)
    u = philox4x32_10((rows[:, None], blk[None, :], np.uint32(tag), np.uint32(stp)), (seed & _MASK, seed >> 32))
    return u32_to_unit(u.reshape(n_rows, d))


def step_noise(model, seed, L, N, d, step):
    """The noise the training step draws at step counter `step` (the n-th step draws n), as the [views, L, N, d] tensor
    TrainEngine.set_noise_tensor takes: view v, layer k keyed by noise_offset(v, k).  SimGCL has two perturbed views,
    XSimGCL one.  SimGCL at L >= 2 draws layer 0 of both views in perturb_rows (tag 0x10) on the shared first product,
    which is the same key."""
    views = 2 if model == "SimGCL" else 1
    out = np.empty((views, L, N, d), dtype=np.float32)
    for v in range(views):
        for k in range(L):
            out[v, k] = philox_noise(seed, noise_offset(v, k), step, N, d)
    return out
