"""CPU model of the runner-up away from the winner (PSM_OPT_RUNNER_UP; test_runner_up_model.py on the CPU,
test_gpu_runner_up.py on the device).

The definition: for the selection map m of a filtered volume q, the candidates are the arg-min's (d in [1, D) whose cost
compares below +inf, lowest cost first, the lowest d first on ties, -0 equal to +0), and the runner-up r is the first
candidate with |d - m| >= 2, 0 when there is none.  The planes hold r as a float and q(r) bit for bit, the quiet NaN
0x7FC00000 where r = 0.  The library never scans for r directly: every path keeps a per-pixel list of the four lowest
candidates and picks r from it.  This module restates both:
  - definition: a direct scan given m;
  - scan_list / pick: the list of one scan (wta_scan4 with the list tracked) and the pick from it (runner_up_pick);
  - fold: a blocked walk (wta_fold_kernel<kList>), each block's list inserted entry by entry into the running one;
  - multi: a multi-device context, every shard picking from its own list into its slot and the first shard taking the
    first slot of the lowest key (runner_up_write_kernel, runner_up_reduce_kernel).
Every plane is a uint32 bit pattern, so NaN payloads and the sign of zero are compared exactly."""
import numpy as np

import cost_triple_cases as CT
import selection_cases as S

U32, U64 = np.uint32, np.uint64
NAN_BITS = CT.NAN_BITS
LIST = 4


def planes(r, q_bits):
    """r [H, W] int64, q_bits [H, W] uint32 -> uint32 [2, H, W]: float(r), q(r) (NAN_BITS where r = 0)"""
    out = np.empty((2,) + r.shape, U32)
    out[0] = r.astype(np.float32).view(U32)
    out[1] = np.where(r == 0, NAN_BITS, q_bits)
    return out


def definition(vol, m):
    """the runner-up of vol[D, H, W] (float32) at map m[H, W], by a direct scan over every d with |d - m| >= 2"""
    f = np.ascontiguousarray(vol, np.float32)
    b = f.view(U32)
    m = m.astype(np.int64)
    best = np.full(m.shape, np.inf, np.float32)
    r = np.zeros(m.shape, np.int64)
    q = np.zeros(m.shape, U32)
    for d in range(1, f.shape[0]):
        with np.errstate(invalid="ignore"):
            take = (np.abs(d - m) >= 2) & (f[d] < best)
        best = np.where(take, f[d], best)
        r = np.where(take, d, r)
        q = np.where(take, b[d], q)
    return planes(r, q)


def insert(lc, ld, c, d):
    """list_insert: c (float32 [H, W]) at slices d ([H, W] or a scalar) into the sorted list (lc [4, H, W] float32, ld
    [4, H, W] int64), in place; entries of equal cost stay ahead of it, +inf and NaN never enter"""
    with np.errstate(invalid="ignore"):
        b = [c < lc[e] for e in range(LIST)]
    d = np.broadcast_to(np.asarray(d, np.int64), c.shape)
    for e in range(LIST - 1, -1, -1):
        shift = b[e - 1] if e > 0 else np.zeros_like(b[0])
        lc[e] = np.where(shift, lc[e - 1] if e > 0 else c, np.where(b[e], c, lc[e]))
        ld[e] = np.where(shift, ld[e - 1] if e > 0 else d, np.where(b[e], d, ld[e]))


def empty(shape):
    return np.full((LIST,) + shape, np.inf, np.float32), np.zeros((LIST,) + shape, np.int64)


def scan_list(vol, d_begin=0):
    """vol[n, H, W] holds slices d_begin .. d_begin + n - 1 -> the four-lowest list (lc, ld) of one scan, global d = 0
    skipped"""
    f = np.ascontiguousarray(vol, np.float32)
    lc, ld = empty(f.shape[1:])
    for dl in range(f.shape[0]):
        if d_begin + dl:
            insert(lc, ld, f[dl], d_begin + dl)
    return lc, ld


def head_key(lc, ld):
    return (S.order_key(lc[0]) << U64(32)) | ld[0].astype(U64)


def fold(vol, blocks, d0=0):
    """wta_fold_kernel<kList> over blocks [(d_begin, d_count), ...] (ascending, contiguous) of vol (slices d0 ..) -> the
    running list; a block whose head does not compare below the running list's last entry leaves it as it is"""
    f = np.ascontiguousarray(vol, np.float32)
    run = None
    for b, n in blocks:
        blc, bld = scan_list(f[b - d0:b - d0 + n], b)
        if run is None:
            run = (blc, bld)
            continue
        lc, ld = run[0].copy(), run[1].copy()
        for e in range(LIST):
            insert(lc, ld, blc[e], bld[e])
        with np.errstate(invalid="ignore"):
            enter = blc[0] < run[0][3]
        run = (np.where(enter, lc, run[0]), np.where(enter, ld, run[1]))
    return run


def pick(lc, ld, m):
    """runner_up_pick -> (r, q bits): the first entry with d != 0 and |d - m| >= 2"""
    m = m.astype(np.int64)
    r = np.zeros(m.shape, np.int64)
    q = np.full(m.shape, NAN_BITS, U32)
    for e in range(LIST - 1, -1, -1):
        ok = (ld[e] != 0) & (np.abs(ld[e] - m) >= 2)
        r = np.where(ok, ld[e], r)
        q = np.where(ok, lc[e].view(U32), q)
    return r, q


def single(vol, B=None):
    """an unblocked (B None) or blocked single-device context over the whole vol -> (map, uint32 [2, H, W])"""
    D = vol.shape[0]
    lc, ld = scan_list(vol) if B is None else fold(vol, S.block_ranges(0, D, B))
    m = ld[0]
    return m, planes(*pick(lc, ld, m))


def multi(vol, n, B=None):
    """a multi-device context of n shards over the whole vol, unblocked (B None) or every shard blocked at min(B, its
    count) -> (map, uint32 [2, H, W]) through the slots: each shard's key and cost bits, the first slot of the lowest
    key"""
    D = vol.shape[0]
    lists = []
    for b, c in S.shard_ranges(D, n):
        lists.append(scan_list(vol[b:b + c], b) if B is None else fold(vol[b:b + c], S.block_ranges(b, c, min(B, c)), b))
    m = CT.winners(np.minimum.reduce([head_key(lc, ld) for lc, ld in lists]))
    no_pick = (S.order_key(np.float32(np.inf)) << U64(32))
    best_key = best_q = None
    for lc, ld in lists:   # the slots, in shard order; a later slot wins only with a lower key
        r, q = pick(lc, ld, m)
        key = np.where(r != 0, (S.order_key(q.view(np.float32)) << U64(32)) | r.astype(U64), no_pick)
        if best_key is None:
            best_key, best_q = key, q
        else:
            take = key < best_key
            best_key, best_q = np.where(take, key, best_key), np.where(take, q, best_q)
    r = (best_key & U64(0xFFFFFFFF)).astype(np.int64)
    out = np.empty((2,) + m.shape, U32)
    out[0] = r.astype(np.float32).view(U32)
    out[1] = best_q
    return m, out


def uniqueness_brute(vol, m, ratio):
    """OpenCV's uniqueness test, brute force: valid iff no d >= 1 with |d - m| > 1 has q(d) * (100 - ratio) < 100 * q(m)
    (the reference-free restatement a caller checks the library's planes against); float64 arithmetic"""
    f = np.asarray(vol, np.float64)
    m = m.astype(np.int64)
    qm = np.take_along_axis(f, m[None], 0)[0]
    ok = np.ones(m.shape, bool)
    for d in range(1, f.shape[0]):
        with np.errstate(invalid="ignore"):
            ok &= ~((np.abs(d - m) > 1) & (f[d] * (100 - ratio) < 100 * qm))
    return ok


def uniqueness_from_planes(runner, m_cost, ratio):
    """the same test from the runner-up planes (2, H, W) float32 and q(m): valid iff r = 0 or q(r) * (100 - ratio) >=
    100 * q(m)"""
    r, qr = runner[0].astype(np.int64), runner[1].astype(np.float64)
    with np.errstate(invalid="ignore"):
        return (r == 0) | (qr * (100 - ratio) >= 100 * np.asarray(m_cost, np.float64))
