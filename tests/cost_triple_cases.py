"""CPU model of the costs beside each winner (PSM_OPT_COSTS; test_cost_triple_model.py on the CPU, test_gpu_costs.py on the
device).

The definition is a gather from the filtered volume: for the selection map m, plane k holds q(m + k - 1), bit for bit,
and the quiet NaN 0x7FC00000 where m + k - 1 lies outside [0, D).  The library never holds the whole volume on a blocked
or multi-device context, so it computes the same planes in pieces.  This module restates both:
  - gather: the definition;
  - track: wta_fold_kernel<kCosts>'s walk of a blocked context (block folds with the seam rules: a block winning on its
    first slice takes q(m - 1) from the previous block's last slice, a running winner on the previous block's last
    slice takes q(m + 1) from this block's first slice, the first block starts from the no-winner state (NaN, q(0),
    q(1)));
  - multi: cost_write_kernel's ownership on a multi-device context, every shard writing the entries it owns (unblocked
    shards from their slices, blocked shards from their tracking planes and first / last slice costs), each entry counted.
Every plane is a uint32 bit pattern, so NaN payloads and the sign of zero are compared exactly."""
import numpy as np

import selection_cases as S

U32 = np.uint32
NAN_BITS = U32(0x7FC00000)


def bits(vol):
    return np.ascontiguousarray(vol, np.float32).view(U32)


def winners(keys):
    """the disparity of packed keys, as int64"""
    return (keys & S.U64(0xFFFFFFFF)).astype(np.int64)


def gather(vol, m, d0=0, D=None):
    """vol[n, H, W] holds slices d0 .. d0 + n - 1 of a volume of D slices (default n); m[H, W] the map -> uint32 [3, H, W]:
    q(m - 1), q(m), q(m + 1), NAN_BITS outside [0, D)"""
    b = bits(vol)
    D = b.shape[0] + d0 if D is None else D
    out = np.empty((3,) + m.shape, U32)
    for k in range(3):
        d = m.astype(np.int64) + k - 1
        ok = (d >= 0) & (d < D)
        idx = np.clip(d - d0, 0, b.shape[0] - 1)
        out[k] = np.where(ok, np.take_along_axis(b, idx[None], 0)[0], NAN_BITS)
    return out


def track(vol, blocks, d0=0):
    """wta_fold_kernel<kCosts> over blocks [(d_begin, d_count), ...] (ascending, contiguous) of vol (slices d0 ..) ->
    (running keys, uint32 planes [5, H, W]: lo, ce, hi, the last slice's cost, the first slice's cost)"""
    f = np.ascontiguousarray(vol, np.float32)
    b32 = f.view(U32)
    shape = f.shape[1:]
    key = None
    planes = np.empty((5,) + shape, U32)
    for bi, (b, n) in enumerate(blocks):
        mc = np.full(shape, np.inf, np.float32)
        md = np.zeros(shape, np.int64)
        lo, ce, hi = (np.full(shape, NAN_BITS, U32) for _ in range(3))
        prev = np.full(shape, NAN_BITS, U32) if bi == 0 else planes[3].copy()
        first = None
        for dl in range(n):
            d = b + dl
            c, cf = b32[d - d0], f[d - d0]
            hi = np.where(md == d - 1, c, hi)
            if d == 0:
                ce = c.copy()
            else:
                with np.errstate(invalid="ignore"):
                    better = cf < mc
                mc = np.where(better, cf, mc)
                md = np.where(better, d, md)
                lo = np.where(better, prev, lo)
                ce = np.where(better, c, ce)
                hi = np.where(better, NAN_BITS, hi)
            prev = c.copy()
            if dl == 0:
                first = c.copy()
        v = (S.order_key(mc) << S.U64(32)) | md.astype(S.U64)
        planes[3] = prev
        if bi == 0:
            key = v
            planes[4] = first
            planes[0], planes[1], planes[2] = lo, ce, hi
        else:
            win = v < key
            planes[2] = np.where(~win & (winners(key) == b - 1), first, planes[2])
            key = np.where(win, v, key)
            for p, new in zip(range(3), (lo, ce, hi)):
                planes[p] = np.where(win, new, planes[p])
    return key, planes


def multi(vol, n, B=None):
    """a multi-device context of n shards (sharding.shard_range) over the whole vol, unblocked (B None) or every shard
    blocked at min(B, its count) -> (map, uint32 [3, H, W], writers [3, H, W]: how many shards wrote each entry)"""
    D = vol.shape[0]
    ranges = S.shard_ranges(D, n)
    local = []
    for b, c in ranges:
        if B is None:
            local.append((S.scan_keys(vol[b:b + c], b), None))
        else:
            local.append(track(vol[b:b + c], S.block_ranges(b, c, min(B, c)), b))
    m = winners(np.minimum.reduce([k for k, _ in local]))
    out = np.zeros((3,) + m.shape, U32)
    writers = np.zeros((3,) + m.shape, np.int64)
    for (b, c), (_, planes) in zip(ranges, local):
        owned = lambda d: (d >= b) & (d < b + c)   # noqa: E731
        for k in range(3):
            d = m + k - 1
            inside = (d >= 0) & (d < D)
            write = np.where(inside, owned(d), owned(m))
            if planes is None:
                src = gather(vol[b:b + c], m, b, D)[k]
            else:
                src = np.where(owned(m), planes[k], planes[4] if k == 2 else planes[3])
            val = np.where(inside, src, NAN_BITS)
            out[k] = np.where(write, val, out[k])
            writers[k] += write
    return m, out, writers


# ---- volumes ------------------------------------------------------------------------------------------------------------
SPECIAL = np.array([0x7FC00000, 0xFFC00000, 0x7FC00123, 0xFFF00001, 0x7F800001,   # NaN of both signs, with payloads
                    0x7F800000, 0xFF800000,                                        # +inf, -inf
                    0x80000000, 0x00000000,                                        # -0, +0
                    0x7F7FFFFF, 0x00000001, 0x00400000,                            # FLT_MAX, denormals
                    0x3F000000, 0x3E800000, 0x3F800000], U32)                      # 0.5, 0.25, 1


def volume(D, H=3, W=48, seed=0):
    """[D, H, W] float32 whose costs come from SPECIAL (many exact ties, -0 beside +0), with columns forced to the edges:
    every cost NaN (m = 0), the minimum at slice 1, at slice D - 1, and a tie between the first and the last slice"""
    rng = np.random.default_rng([seed, D, H, W])
    v = SPECIAL[rng.integers(0, SPECIAL.size, (D, H, W))].view(np.float32).copy()
    v[:, :, 0] = np.uint32(0x7FC00000).view(np.float32)
    v[1:, :, 1:4] = 1.0
    v[1, :, 1] = -np.inf
    v[D - 1, :, 2] = -1.0
    v[1, :, 3] = v[D - 1, :, 3] = 0.25
    return v
