"""CPU model of disparity selection through packed keys (test_selection_model.py on the CPU, test_gpu_selection_seams.py on
the device).

Every selection path of the library ends in a packed key per pixel, (float_order_key(cost) << 32) | d:
wta_kernel<T, false>'s keys for disparity shards, wta_fold_kernel<false, false>'s running keys of a blocked context, the
keys a multi-device context's shards exchange.  The min over keys of disjoint slice ranges is claimed to be the
winner-take-all over their union (strict <, lowest d on ties, +inf and NaN never win, global d = 0 never a candidate).
This module restates the key
(psm_common.cuh::float_order_key), the one-scan key of a range of slices, the fold over a partition of the range, and
the partitions the library makes: blocks of a blocked context (block_at) and shards (sharding.shard_range)."""
import numpy as np

from primestereomatch_b200.sharding import shard_range

U64 = np.uint64
NO_WINNER = U64(0xFF800000) << U64(32)   # (+inf, 0): no cost of the range compares below +inf


def order_key(c):
    """the order-preserving uint32 of float32 costs (as uint64), -0 canonicalised to +0"""
    with np.errstate(invalid="ignore"):
        c = (np.asarray(c, np.float32) + np.float32(0.0)).astype(np.float32)
    u = c.view(np.uint32).astype(U64)
    neg = (u & U64(0x80000000)) != 0
    return np.where(neg, (~u) & U64(0xFFFFFFFF), u | U64(0x80000000))


def scan_keys(vol, d_begin=0):
    """vol[n, H, W] holds the slices d_begin .. d_begin + n - 1 -> the [H, W] uint64 keys of one strict-< scan over them,
    global d = 0 skipped; NO_WINNER where no cost is below +inf"""
    vol = np.asarray(vol, np.float32)
    mc = np.full(vol.shape[1:], np.inf, np.float32)
    md = np.zeros(vol.shape[1:], U64)
    for dl in range(vol.shape[0]):
        d = d_begin + dl
        if d == 0:
            continue
        with np.errstate(invalid="ignore"):
            better = vol[dl] < mc
        mc = np.where(better, vol[dl], mc)
        md = np.where(better, U64(d), md)
    return (order_key(mc) << U64(32)) | md


def fold(vol, blocks, d0=0):
    """vol[n, H, W] holds the slices d0 .. d0 + n - 1; blocks: (d_begin, d_count) ranges of global d covering some of
    them -> the min over the blocks' scan keys"""
    out = None
    for b, n in blocks:
        k = scan_keys(vol[b - d0:b - d0 + n], b)
        out = k if out is None else np.minimum(out, k)
    return out


def block_ranges(d_begin, d_count, B):
    """the blocks of a blocked context owning [d_begin, d_begin + d_count): B slices each from d_begin, ragged last"""
    return [(b, min(B, d_begin + d_count - b)) for b in range(d_begin, d_begin + d_count, B)]


def shard_ranges(D, n):
    return [shard_range(D, n, k) for k in range(n)]


def multi_ranges(D, n, B=None):
    """the slice ranges whose keys a multi-device context of n shards reduces: its shards, or, with blocked shards
    (psm_create_multi clamps B to each shard's count), every shard's blocks"""
    out = []
    for b, c in shard_ranges(D, n):
        out += [(b, c)] if B is None else block_ranges(b, c, min(B, c))
    return out


def disparity(keys, dtype):
    """the map a key reduction writes: the key's low 8 or 16 bits"""
    return (keys & U64(np.iinfo(dtype).max)).astype(dtype)


def seam_ties(vol, keys, ranges, d0=0):
    """the number of pixels whose winning cost also occurs, bit for bit up to the sign of zero, at another selectable
    slice on the far side of a seam between the ranges (ties that only the lowest-d rule of the fold or reduction
    decides)"""
    vol = np.asarray(vol, np.float32)
    d = (keys & U64(0xFFFFFFFF)).astype(np.int64)
    win = np.take_along_axis(vol, (d - d0)[None], 0)[0]
    part = np.full(vol.shape[0], -1)
    for k, (b, n) in enumerate(ranges):
        part[b - d0:b - d0 + n] = k
    found = np.zeros(keys.shape, bool)
    for dl in range(vol.shape[0]):
        if dl + d0 == 0 or part[dl] < 0:
            continue
        found |= (vol[dl] == win) & (part[dl] != part[d - d0]) & (d > 0)
    return int(found.sum())
