"""CPU restatement of the one-view disparity check (psm_set_disparity_check, OpenCV's cv::validateDisparity), which the
device runs as a shared-memory atomicMin per row.  Test infrastructure; pinned to cv2.validateDisparity itself by
tests/golden/golden_dcheck.json (tests/golden/make_golden_dcheck.py).

Definition, per row of one view's map m, c = the winners' costs (plane 1 of PSM_OPT_COSTS), W = width, D = max_disp:
  1. only columns x in [D, W) with m[x] != 0 take part; every other pixel keeps its value;
  2. every participating x claims column x - m[x]; per column the lowest cost wins (in the arg-min's order: the
     order-preserving key of the float, -0 equal to +0), and on equal costs the lowest x; d2[column] is the winner's m;
  3. a participating x becomes 0 when |d2[x - m[x]] - m[x]| > max_diff (as int);
  4. the right view is the mirror image: fliplr(check(fliplr(r), fliplr(c_right))).

check is the vectorised form the tests use; check_rows is the literal row loop (cv2's ascending-x loop with a strict
`>`), which the CPU tests hold the first one to.
"""
import numpy as np

MAX_DIFF = 4095   # the largest max_diff psm_set_disparity_check takes


def order_key(c):
    """the arg-min's order-preserving uint32 key of float32 costs (float_order_key): -0 becomes +0 first"""
    c = np.asarray(c, np.float32) + np.float32(0)
    u = c.view(np.uint32)
    return np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000)).astype(np.uint32)


def _args(m, c, D, max_diff):
    m, c = np.asarray(m), np.asarray(c)
    assert m.ndim == 2 and m.dtype in (np.uint8, np.uint16) and c.shape == m.shape, (m.shape, m.dtype, c.shape)
    assert D >= 1 and 0 <= max_diff <= MAX_DIFF
    return m, c


def check(m, c, D, max_diff, view=0):
    """-> the checked map of view 0 (left) or 1 (right, the mirror image), of m's dtype"""
    m, c = _args(m, c, D, max_diff)
    if view:
        return check(m[:, ::-1], c[:, ::-1], D, max_diff)[:, ::-1].copy()
    H, W = m.shape
    v = m.astype(np.int64)
    ys, xs = np.nonzero((np.arange(W) >= D)[None, :] & (v != 0))
    out = m.copy()
    if ys.size == 0:
        return out
    x2 = xs - v[ys, xs]
    order = np.lexsort((xs, order_key(c)[ys, xs], x2, ys))      # by row, column claimed, cost key, then x
    first = np.ones(order.size, bool)
    first[1:] = (ys[order][1:] != ys[order][:-1]) | (x2[order][1:] != x2[order][:-1])
    win = order[first]
    d2 = np.zeros((H, W), np.int64)
    d2[ys[win], x2[win]] = v[ys[win], xs[win]]
    bad = np.abs(d2[ys, x2] - v[ys, xs]) > max_diff
    out[ys[bad], xs[bad]] = 0
    return out


def check_rows(m, c, D, max_diff, view=0):
    """the literal row loop of the definition (small maps) -> the checked map"""
    m, c = _args(m, c, D, max_diff)
    if view:
        return check_rows(m[:, ::-1], c[:, ::-1], D, max_diff)[:, ::-1].copy()
    H, W = m.shape
    key = order_key(c).tolist()
    out = m.copy()
    for y in range(H):
        row = m[y].astype(np.int64).tolist()
        best, d2 = [None] * W, [0] * W
        for x in range(D, W):
            d = row[x]
            if d == 0:
                continue
            if best[x - d] is None or best[x - d] > key[y][x]:
                best[x - d], d2[x - d] = key[y][x], d
        for x in range(D, W):
            d = row[x]
            if d != 0 and abs(d2[x - d] - d) > max_diff:
                out[y, x] = 0
    return out


def dense_rank(c):
    """int32 dense ranks of the costs' order keys: the same order, as cv2.validateDisparity's CV_32S cost"""
    _, inv = np.unique(order_key(c).ravel(), return_inverse=True)
    return inv.reshape(np.shape(c)).astype(np.int32)


def winner_costs(vol, m):
    """plane 1 of PSM_OPT_COSTS from a filtered volume [D, H, W]: q(m) at each pixel (q(0) where m = 0)"""
    return np.take_along_axis(vol, m.astype(np.int64)[None], axis=0)[0]

