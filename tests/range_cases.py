"""CPU model of a range context over [min_disp, max_disp) (test_range_model.py on the CPU, test_gpu_range.py on the device).

The definition, given the filtered volume q of a [0, max_disp) context (slice d of a range context is bit for bit that
context's slice d):
  - selection: the arg-min over d in [max(1, min_disp), max_disp) (strict <, lowest d on ties, +inf and NaN never win),
    the absolute d in the map, 0 where nothing compares below +inf;
  - costs: entry k is q(m + k - 1), the quiet NaN 0x7FC00000 where m + k - 1 lies outside [min_disp, max_disp);
  - runner-up: the first candidate of the same order with |d - m| >= 2, 0 with a NaN cost when there is none.
The library never sees the slices below min_disp, so it computes these from the range's slices alone, in the pieces each
kind of context makes:
  - single: an unblocked context (one scan) or a blocked one (block folds from min_disp, cost tracking, list folds);
  - multi: n shards splitting [min_disp, max_disp) as sharding.shard_range(..., min_disp) does, each writing the cost
    entries it owns (cost_write_kernel's rule with the range start d_lo) and picking its runner-up into a slot.
Every plane is a uint32 bit pattern, so NaN payloads and the sign of zero are compared exactly."""
import numpy as np

import cost_triple_cases as CT
import runner_up_cases as RU
import selection_cases as S
from primestereomatch_b200.sharding import shard_range

U32, U64 = np.uint32, np.uint64
NAN_BITS = CT.NAN_BITS


def definition(vol, lo):
    """vol [D, H, W] float32, the [0, D) context's filtered volume -> (map int64 [H, W], costs uint32 [3, H, W], runner-up
    uint32 [2, H, W]) of the range context over [lo, D), by direct scans of the full volume restricted to the range"""
    f = np.ascontiguousarray(vol, np.float32)
    b = f.view(U32)
    D = f.shape[0]
    shape = f.shape[1:]
    best = np.full(shape, np.inf, np.float32)
    m = np.zeros(shape, np.int64)
    for d in range(max(1, lo), D):
        with np.errstate(invalid="ignore"):
            better = f[d] < best
        best = np.where(better, f[d], best)
        m = np.where(better, d, m)
    costs = np.empty((3,) + shape, U32)
    for k in range(3):
        d = m + k - 1
        ok = (d >= lo) & (d < D)
        costs[k] = np.where(ok, np.take_along_axis(b, np.clip(d, 0, D - 1)[None], 0)[0], NAN_BITS)
    best = np.full(shape, np.inf, np.float32)
    r = np.zeros(shape, np.int64)
    q = np.zeros(shape, U32)
    for d in range(max(1, lo), D):
        with np.errstate(invalid="ignore"):
            take = (np.abs(d - m) >= 2) & (f[d] < best)
        best = np.where(take, f[d], best)
        r = np.where(take, d, r)
        q = np.where(take, b[d], q)
    return m, costs, RU.planes(r, q)


def shard_ranges(lo, D, n):
    return [shard_range(D, n, k, min_disp=lo) for k in range(n)]


def cost_write(m, lo, D, b, c, src):
    """cost_write_kernel of the context owning [b, b + c) of [lo, D): src(k, owner_of_state) -> uint32 [H, W], the value
    it reads for entry k -> (values uint32 [3, H, W], written bool [3, H, W])"""
    mo = np.maximum(m, lo)   # the no-winner map 0 below the range: the owner of lo writes for it
    owned = lambda d: (d >= b) & (d < b + c)   # noqa: E731
    vals = np.empty((3,) + m.shape, U32)
    written = np.empty((3,) + m.shape, bool)
    for k in range(3):
        d = m + k - 1
        inside = (d >= lo) & (d < D)
        written[k] = np.where(inside, owned(d), owned(mo))
        vals[k] = np.where(inside, src(k, owned(mo)), NAN_BITS)
    return vals, written


def context(vol, lo, n=None, B=None):
    """the range context over [lo, D) of the full volume vol [D, H, W], as the library decomposes it: single-device
    (n None) or n shards, unblocked (B None) or blocked at B (clamped to each shard's count) -> (map, costs uint32
    [3, H, W], runner-up uint32 [2, H, W], writers int64 [3, H, W]: how many contexts wrote each cost entry).  Only the
    range's slices are read."""
    f = np.ascontiguousarray(vol, np.float32)
    D = f.shape[0]
    r = f[lo:]   # the slices the context holds: r[d - lo] is slice d
    parts = [(lo, D - lo)] if n is None else shard_ranges(lo, D, n)
    local = []
    for b, c in parts:
        sub = r[b - lo:b - lo + c]
        if B is None:
            keys, track = S.scan_keys(sub, b), None
            lst = RU.scan_list(sub, b)
        else:
            blocks = S.block_ranges(b, c, min(B, c))
            keys, track = CT.track(sub, blocks, b)
            lst = RU.fold(sub, blocks, b)
            assert np.array_equal(RU.head_key(*lst), keys), "the list fold's head is the key fold"
        local.append((b, c, sub, keys, track, lst))
    m = CT.winners(np.minimum.reduce([t[3] for t in local]))
    costs = np.zeros((3,) + m.shape, U32)
    writers = np.zeros((3,) + m.shape, np.int64)
    best_key = best_q = None
    no_pick = S.order_key(np.float32(np.inf)) << U64(32)
    for b, c, sub, _, track, lst in local:
        if track is None:   # an unblocked context reads q(d) from its slices
            gathered = [np.take_along_axis(CT.bits(sub), np.clip(m + k - 1 - b, 0, c - 1)[None], 0)[0] for k in range(3)]
            src = lambda k, own_state: gathered[k]   # noqa: E731
        else:               # a blocked one from its tracking planes: its own state, or the first / last slice at a seam
            src = lambda k, own_state: np.where(own_state, track[k], track[4] if k == 2 else track[3])   # noqa: E731
        vals, written = cost_write(m, lo, D, b, c, src)
        costs = np.where(written, vals, costs)
        writers += written
        rr, q = RU.pick(*lst, m)   # the pick into this context's slot; the first slot of the lowest key wins
        key = np.where(rr != 0, (S.order_key(q.view(np.float32)) << U64(32)) | rr.astype(U64), no_pick)
        if best_key is None:
            best_key, best_q = key, q
        else:
            take = key < best_key
            best_key, best_q = np.where(take, key, best_key), np.where(take, q, best_q)
    runner = np.empty((2,) + m.shape, U32)
    runner[0] = (best_key & U64(0xFFFFFFFF)).astype(np.int64).astype(np.float32).view(U32)
    runner[1] = best_q
    return m, costs, runner, writers


def min_disps(D):
    """the range starts every test covers: 0, 1, 2, 3, D / 2 and D - 1 (a range of one slice), those below D"""
    return sorted({lo for lo in (0, 1, 2, 3, D // 2, D - 1) if 0 <= lo < D})


def volume(D, lo, seed=0):
    """CT.volume with exact ties across every seam (half the columns hold three distinct costs), and, for the range start
    lo, columns forced to its edges: a winner of the full range at lo - 1 (below the range), a tie of lo - 1, lo and
    lo + 1, a range whose every cost is NaN while the slices below it are finite, and a winner at lo"""
    v = CT.volume(D, seed=seed)
    rng = np.random.default_rng([seed, D, lo, 7])
    few = np.array([0x3E800000, 0x80000000, 0x00000000], U32).view(np.float32)
    v[:, :, 24:] = few[rng.integers(0, 3, v[:, :, 24:].shape)]
    v[:, :, 4:8] = 1.0
    if lo >= 1:
        v[lo - 1, :, 4] = -np.inf
    v[max(lo - 1, 0):lo + 2, :, 5] = 0.25
    v[lo:, :, 6] = np.uint32(0xFFC00000).view(np.float32)
    v[lo, :, 7] = -0.0
    return v
