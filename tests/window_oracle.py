"""CPU restatement of the guided filter at any window / epsilon (test infrastructure, numpy only).

The reference fixes GIF_R_WIN = 8 and GIF_EPS = 0.0001f at compile time (include/ComFunc.h:49-50); psm_set_guided_filter
makes both run-time parameters.  This module restates, for any window K and eps, what the plain-C oracle
(oracle/stereo_oracle.c) restates for (8, 1e-4f):
  * box(src, K)         cv::boxFilter(CV_32F, Size(K, K)), anchor K/2, BORDER_REFLECT_101, in OpenCV's own summation order
                        (RowSum<float,double>: direct sums up to K = 5, sliding above; then ColumnSum<double,float>,
                        sliding; see orc_box8), so it equals cv2 even where fp64 sums are not exact;
  * box_direct(src, K)  the Fast Guided Filter's box, DEFINED as the direct order (orc_box_k); it equals cv::blur wherever
                        the fp64 sums are exact (see its docstring) and is this project's own definition beyond that;
  * cvf_preprocess      CVF::preprocess (CVF.cpp:44-70) with a K x K box;
  * guided_filter       GuidedFilter_cv (CVF.cpp:72-165), eps on the covariance diagonal, float operations in the reference's
                        order (numpy float32 arithmetic rounds every operation and never contracts to FMA);
  * cost_filter_fgf     FastGuidedFilter(img, r, eps, s) as DispEst::CostFilter_FGF drives it (see orc_cost_filter_fgf): box
                        K = 2*(r/s)+1 at the sub-sampled resolution.
Every function works on whole volumes [D, H, W] at once.  At (8, 1e-4f) the results equal the C oracle's, which
tests/test_oracle_window.py checks against the stored goldens.
"""
import numpy as np

F32 = np.float32


def reflect101(i, n):
    """cv::BORDER_REFLECT_101 index map for an integer array i, any overshoot."""
    i = np.asarray(i, np.int64)
    if n == 1:
        return np.zeros_like(i)
    period = 2 * (n - 1)
    i = np.abs(i) % period
    return np.where(i >= n, period - i, i)


def box(src, K):
    """Normalised K x K box of the last two axes of a float32 array, OpenCV's order of fp64 operations."""
    src = np.asarray(src, F32)
    if K == 1:                     # OpenCV copies
        return src.copy()
    H, W = src.shape[-2:]
    a = K // 2
    scale = 1.0 / float(K * K)
    # RowSum: padded row p[i] = src[reflect101(i - a)], s = p[0] + ... + p[K-1], then s += p[i+K] - p[i]; rows up to 5
    # wide OpenCV sums directly, p[i] + p[i+1] + ... + p[i+K-1] left to right (both checked against cv2 by
    # tests/test_fgf_numerics.py on data where the two orders differ)
    cols = reflect101(np.arange(W + K - 1) - a, W)
    prow = src[..., cols].astype(np.float64)
    if K <= 5:
        rs = prow[..., 0:W]
        for i in range(1, K):
            rs = rs + prow[..., i:i + W]
    else:
        rs = np.empty(src.shape, np.float64)
        acc = np.zeros(src.shape[:-1], np.float64)
        for i in range(K):
            acc = acc + prow[..., i]
        rs[..., 0] = acc
        for i in range(W - 1):
            acc = acc + (prow[..., i + K] - prow[..., i])
            rs[..., i + 1] = acc
    # ColumnSum: SUM = rows -a .. K-2-a; per output row s0 = SUM + newest, out = (float)(s0 * scale), SUM = s0 - oldest
    out = np.empty(src.shape, F32)
    SUM = np.zeros(src.shape[:-2] + (W,), np.float64)
    for r in range(K - 1):
        SUM = SUM + rs[..., reflect101(r - a, H), :]
    for y in range(H):
        s0 = SUM + rs[..., reflect101(y + K - 1 - a, H), :]
        out[..., y, :] = (s0 * scale).astype(F32)
        SUM = s0 - rs[..., reflect101(y - a, H), :]
    return out


def cvf_preprocess(img3, K=8):
    """-> rgb[3,H,W], mean_I[3,H,W], var_I[6,H,W] (rr, rg, rb, gg, gb, bb)"""
    img3 = np.asarray(img3, F32)
    rgb = np.ascontiguousarray(np.moveaxis(img3, -1, 0))
    mean = box(rgb, K)
    var = []
    for c in range(3):
        for cp in range(c, 3):
            var.append(box(rgb[c] * rgb[cp], K) - mean[c] * mean[cp])
    return rgb, mean, np.stack(var)


def guided_filter(rgb, mean, var, p, K=8, eps=1e-4, want_ab=False):
    """GuidedFilter_cv of p ([H,W] or [D,H,W]) -> q (or (q, a[..., 3, H, W], b) with want_ab)."""
    p = np.asarray(p, F32)
    eps = F32(eps)
    mean_p = box(p, K)
    cov = [box(rgb[c] * p, K) - mean[c] * mean_p for c in range(3)]
    c0, c1, c2 = cov
    a11 = var[0] + eps; a12 = var[1]; a13 = var[2]
    a21 = var[1]; a22 = var[3] + eps; a23 = var[4]
    a31 = var[2]; a32 = var[4]; a33 = var[5] + eps
    DET = a11 * (a33 * a22 - a32 * a23) - a21 * (a33 * a12 - a32 * a13) + a31 * (a23 * a12 - a22 * a13)
    DET = F32(1) / DET
    a0 = DET * (c0 * (a33 * a22 - a32 * a23) + c1 * (a31 * a23 - a33 * a21) + c2 * (a32 * a21 - a31 * a22))
    a1 = DET * (c0 * (a32 * a13 - a33 * a12) + c1 * (a33 * a11 - a31 * a13) + c2 * (a31 * a12 - a32 * a11))
    a2 = DET * (c0 * (a23 * a12 - a22 * a13) + c1 * (a21 * a13 - a23 * a11) + c2 * (a22 * a11 - a21 * a12))
    b = mean_p
    for c, ac in enumerate((a0, a1, a2)):
        b = b - ac * mean[c]
    q = box(b, K)
    for c, ac in enumerate((a0, a1, a2)):
        q = q + box(ac, K) * rgb[c]
    if want_ab:
        return q, np.stack([a0, a1, a2], axis=-3), b
    return q


def cost_filter(l, r, lv, rv, K=8, eps=1e-4):
    """CVF::preprocess per view, then GuidedFilter_cv of every slice -> filtered (lVol, rVol)."""
    out = []
    for img, vol in ((l, lv), (r, rv)):
        rgb, mean, var = cvf_preprocess(img, K)
        out.append(guided_filter(rgb, mean, var, vol, K, eps))
    return out[0], out[1]


def wta(vol):
    """DispSel.cpp:83-109: argmin over d >= 1, strict <, ties to the lowest d, 0 when nothing is below +inf."""
    vol = np.asarray(vol, F32)
    best = np.full(vol.shape[1:], np.inf, F32)
    dis = np.zeros(vol.shape[1:], np.uint8)
    for d in range(1, vol.shape[0]):
        m = vol[d] < best
        best = np.where(m, vol[d], best)
        dis[m] = d
    return dis


# ---- Fast Guided Filter (fastguidedfilter.cpp:121-198 with r, eps, s; the C restatement is orc_cost_filter_fgf) -----------
def box_direct(src, K):
    """The Fast Guided Filter's K x K box as orc_box_k defines it: per pixel, from 0.0, the K reflected taps of a row left
    to right in fp64, then the K row sums top to bottom, * 1/(K*K) in double, one rounding.

    cv::blur slides most of its fp64 sums (box above), so the two agree exactly when every fp64 sum either order forms
    is exact.  That holds when all values are integer multiples of 2^q and below 2^Q in magnitude with
    Q - q + ceil(log2(K*K)) <= 53: every partial sum is then a multiple of 2^q of magnitude at most 2^(q+53).  For
    normal floats (a float in [2^e, 2^(e+1)) is a multiple of 2^(e-23)) this allows the exponents of the nonzero values
    to span 29 - ceil(log2(K*K)) binary orders of magnitude: 20 at K = 17, 16 at K = 65.  Beyond that the direct order
    is this project's definition, not cv::blur's."""
    src = np.asarray(src, F32)
    H, W = src.shape[-2:]
    a = K // 2
    rows = np.zeros(src.shape, np.float64)
    for dx in range(-a, K - a):
        rows = rows + src[..., reflect101(np.arange(W) + dx, W)].astype(np.float64)
    acc = np.zeros(src.shape, np.float64)
    for dy in range(-a, K - a):
        acc = acc + rows[..., reflect101(np.arange(H) + dy, H), :]
    return (acc * (1.0 / (float(K) * K))).astype(F32)


def _fgf_plan(W, H, s):
    w2, h2 = W // s, H // s
    ifx, ify = 1.0 / (w2 / W), 1.0 / (h2 / H)
    xs = np.minimum(np.floor(np.arange(w2) * ifx).astype(np.int64), W - 1)
    ys = np.minimum(np.floor(np.arange(h2) * ify).astype(np.int64), H - 1)

    def lin(n, n2):
        sc = n2 / n
        f = ((np.arange(n) + 0.5) * sc - 0.5).astype(F32)
        i = np.floor(f).astype(np.int64)
        f = (f - i.astype(F32)).astype(F32)
        return i, f

    ix, fx = lin(W, w2)
    lo = ix < 0
    fx[lo] = 0; ix[lo] = 0
    hi = ix >= w2 - 1
    fx[hi] = 0; ix[hi] = w2 - 1
    lx0, lx1 = ix, np.minimum(ix + 1, w2 - 1)
    iy, fy = lin(H, h2)
    ly0, ly1 = np.clip(iy, 0, h2 - 1), np.clip(iy + 1, 0, h2 - 1)
    return xs, ys, lx0, lx1, fx, ly0, ly1, fy


def _fgf_up(lo, plan):
    _, _, lx0, lx1, fx, ly0, ly1, fy = plan
    tmp = lo[..., lx0] * (F32(1) - fx) + lo[..., lx1] * fx
    b0, b1 = (F32(1) - fy)[:, None], fy[:, None]
    return tmp[..., ly0, :] * b0 + tmp[..., ly1, :] * b1


def fgf_filter_volume(img3, vol, r=8, eps=1e-4, s=4):
    """FastGuidedFilter(img, r, eps, s) of every slice of vol [D,H,W] -> filtered volume."""
    img3 = np.asarray(img3, F32)
    vol = np.asarray(vol, F32)
    H, W = vol.shape[-2:]
    K = 2 * (r // s) + 1
    plan = _fgf_plan(W, H, s)
    xs, ys = plan[0], plan[1]
    orig = np.moveaxis(img3, -1, 0)
    Ic = orig[:, ys][:, :, xs]
    m = box_direct(Ic, K)
    pa, pb = (0, 0, 0, 1, 1, 2), (0, 1, 2, 1, 2, 2)
    var = []
    for v in range(6):
        bx = box_direct(Ic[pa[v]] * Ic[pb[v]], K)
        mm = m[pa[v]] * m[pb[v]]
        if pa[v] == pb[v]:
            var.append(((bx.astype(np.float64) - mm.astype(np.float64)) + float(F32(eps))).astype(F32))
        else:
            var.append(bx - mm)
    rr, rg, rb, gg, gb, bb = var
    irr = gg * bb - gb * gb; irg = gb * rb - rg * bb; irb = rg * gb - gg * rb
    igg = rr * bb - rb * rb; igb = rb * rg - rr * gb; ibb = rr * gg - rg * rg
    det = (irr * rr + irg * rg) + irb * rb
    inv = [irr / det, irg / det, irb / det, igg / det, igb / det, ibb / det]
    p2 = vol[:, ys][:, :, xs]
    mp = box_direct(p2, K)
    mIp = [box_direct(Ic[k] * p2, K) for k in range(3)]
    c0, c1, c2 = (mIp[k] - m[k] * mp for k in range(3))
    ar = (inv[0] * c0 + inv[1] * c1) + inv[2] * c2
    ag = (inv[1] * c0 + inv[3] * c1) + inv[4] * c2
    ab = (inv[2] * c0 + inv[4] * c1) + inv[5] * c2
    b = ((mp - ar * m[0]) - ag * m[1]) - ab * m[2]
    q = None
    for k, ak in enumerate((ar, ag, ab)):
        prod = _fgf_up(box_direct(ak, K), plan) * orig[k]
        q = prod if q is None else q + prod
    return q + _fgf_up(box_direct(b, K), plan)


def cost_filter_fgf(l, r, lv, rv, window=8, eps=1e-4, s=4):
    return fgf_filter_volume(l, lv, window, eps, s), fgf_filter_volume(r, rv, window, eps, s)
