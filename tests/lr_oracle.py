"""CPU restatement of the left-right consistency check and occlusion fill (the reference's lrCheck and fillInv,
src/PP.cpp:17-143), which psm_set_lr_check runs on the device.  Test infrastructure; pinned to the reference's own
compiled PP.cpp by tests/golden/golden_lr.json (tests/golden/make_golden_lr.py).

Per row, on integer map values, W = width, mod = the non-negative (Euclidean) remainder:
  lValid[x] = l[x] == r[(x - l[x]) mod W] and l[x] >= 2
  rValid[x] = r[x] == l[(x + r[x]) mod W] and r[x] >= 2
both on the unmodified maps; then each view with its own mask: a valid pixel keeps its value, an invalid one takes
min(map[L], map[R]) of the nearest valid pixels L <= x <= R, or the one that exists; a row without a valid pixel is
unchanged.
"""
import numpy as np

MODES = {"off": 0, "fill_wmf": 1, "fill": 2}   # PSM_LR_OFF, PSM_LR_FILL_WMF, PSM_LR_FILL


def lr_check(l, r):
    """-> (lValid, rValid) as uint8 0/1 maps"""
    l, r = np.asarray(l), np.asarray(r)
    assert l.shape == r.shape and l.ndim == 2
    W = l.shape[1]
    li, ri = l.astype(np.int64), r.astype(np.int64)
    x = np.arange(W, dtype=np.int64)
    r_at = np.take_along_axis(ri, (x - li) % W, axis=1)     # numpy's % of a positive W is the Euclidean remainder
    l_at = np.take_along_axis(li, (x + ri) % W, axis=1)
    return ((li == r_at) & (li >= 2)).astype(np.uint8), ((ri == l_at) & (ri >= 2)).astype(np.uint8)


def fill(m, valid):
    """fillInv of one view -> the filled map, of m's dtype"""
    m, valid = np.asarray(m), np.asarray(valid).astype(bool)
    W = m.shape[1]
    x = np.arange(W)
    left = np.maximum.accumulate(np.where(valid, x, -1), axis=1)                       # nearest valid at or left of x
    right = np.minimum.accumulate(np.where(valid, x, W)[:, ::-1], axis=1)[:, ::-1]      # nearest valid at or right of x
    has_l, has_r = left >= 0, right < W
    vl = np.take_along_axis(m, np.clip(left, 0, W - 1), axis=1)
    vr = np.take_along_axis(m, np.clip(right, 0, W - 1), axis=1)
    return np.where(has_l & has_r, np.minimum(vl, vr), np.where(has_l, vl, np.where(has_r, vr, m))).astype(m.dtype)


def lr_check_fill(l, r):
    """-> (lValid, rValid, lFilled, rFilled)"""
    lv, rv = lr_check(l, r)
    return lv, rv, fill(l, lv), fill(r, rv)

