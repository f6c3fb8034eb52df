"""CPU restatement of OpenCV's reprojectImageTo3D(map, xyz, Q, handleMissingValues) on maps of integer disparities, the
definition psm_reproject_device / psm_read_points follow (DESIGN.md section 24), and the comparison their results
are judged by.  golden_reproject.json pins it to cv2's own results.

numpy rounds every elementwise operation on its own in fp64, so each product and each sum below is rounded separately,
in the order written, as OpenCV's loop computes it: the sum starts from +0.0, the reciprocal of h[3] is IEEE's, and each
component is rounded to float before and after its multiplication by that reciprocal."""
import hashlib

import numpy as np

MISSING_Z = np.float32(10000.0)   # reprojectImageTo3D's bigZ
CANON_NAN = np.uint32(0x7FC00000)


def reproject(m, Q, handle_missing=False):
    """(H, W) u8 / u16 map, 4 x 4 Q (any doubles) -> (H, W, 3) float32 X, Y, Z"""
    m = np.asarray(m)
    Q = np.asarray(Q, np.float64).reshape(4, 4)
    H, W = m.shape
    x = np.arange(W, dtype=np.float64)[None, :]
    y = np.arange(H, dtype=np.float64)[:, None]
    d = m.astype(np.float64)
    with np.errstate(all="ignore"):
        h = [(((0.0 + Q[i, 0] * x) + Q[i, 1] * y) + Q[i, 2] * d) + Q[i, 3] for i in range(4)]
        r = 1.0 / h[3]
        out = np.stack([(h[i].astype(np.float32).astype(np.float64) * r).astype(np.float32) for i in range(3)], axis=-1)
    if handle_missing:
        out[..., 2][m == m.min()] = MISSING_Z   # OpenCV takes the map's minimum for the missing value
    return out


def canonical(p):
    """the float bits of p with every NaN replaced by the quiet NaN 0x7FC00000"""
    u = np.ascontiguousarray(p, np.float32).view(np.uint32).copy()
    u[np.isnan(np.asarray(p))] = CANON_NAN
    return u


def sha(p):
    return hashlib.sha256(canonical(p).tobytes()).hexdigest()


def assert_points_equal(got, want, what):
    """every non-NaN value bit for bit, and NaN at exactly the same positions"""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape and got.dtype == np.float32, f"{what}: {got.shape} {got.dtype} vs {want.shape}"
    g, w = canonical(got), canonical(want)
    if not np.array_equal(g, w):
        bad = np.argwhere(g != w)
        i = tuple(bad[0])
        raise AssertionError(f"{what}: {len(bad)} of {g.size} values differ, first at {list(i)}: "
                             f"{got[i]!r} (0x{g[i]:08x}) vs {want[i]!r} (0x{w[i]:08x})")
