"""CPU restatement of the cost-volume construction at any matching-cost setting (test infrastructure, numpy only).

The reference compiles ALPHA_32F = 0.9f into CVC.cpp and leaves the truncation by TAU_1_32F / TAU_2_32F commented out
(src/CVC.cpp:24-25, 36-37); psm_set_matching_cost makes all three run-time parameters.  This module restates, for any
(alpha, tau_color, tau_grad), what the plain-C oracle (oracle/stereo_oracle.c) restates for (0.9f, off, off):
  * preprocess      CVC::preprocess (CVC.cpp:41-46): cv::cvtColor RGB2GRAY on the BGR image as OpenCV's SIMD path computes
                    it, fma(c2, .114, fma(c0, .299, c1 * .587)), then Sobel dx = 1, ksize = 1 with BORDER_REFLECT_101;
  * cost_volumes    buildCV_left / buildCV_right (CVC.cpp:122-179, the right view with the caller's swapped arguments,
                    DispEst.cpp:260) of whole volumes: interior pixels in float, border pixels with the BC_32F = 1.0
                    differences in double rounded once, then `if (clr > tau_color) clr = tau_color` (and the same for grd),
                    then alpha * clr + (1 - alpha) * grd, every float operation rounded separately.
At the defaults the volumes equal the C oracle's, which tests/test_oracle_cost.py checks against the stored goldens.
"""
import numpy as np

F32 = np.float32
F64 = np.float64
DEFAULT = (0.9, np.inf, np.inf)


def fma32(a, b, c):
    """fmaf(a, b, c) on float32 arrays: the product is exact in float64, the sum is rounded to odd in float64 (exact
    remainder by TwoSum), and the one rounding to float32 after that is the correctly rounded fma (53 >= 24 + 2 bits)."""
    a, b, c = (np.asarray(v, F32).astype(F64) for v in (a, b, c))
    p = a * b
    s = p + c
    bv = s - p
    e = (p - (s - bv)) + (c - bv)
    inexact = np.isfinite(s) & (e != 0) & ((s.view(np.int64) & 1) == 0)
    s = np.where(inexact, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return s.astype(F32)


def reflect101(i, n):
    i = np.asarray(i, np.int64)
    if n == 1:
        return np.zeros_like(i)
    period = 2 * (n - 1)
    i = np.abs(i) % period
    return np.where(i >= n, period - i, i)


def preprocess(img3):
    """CVC::preprocess of an HxWx3 float32 image -> x-gradient of the gray image [H, W]."""
    img3 = np.asarray(img3, F32)
    c0, c1, c2 = img3[..., 0], img3[..., 1], img3[..., 2]
    gray = fma32(c2, F32(0.114), fma32(c0, F32(0.299), c1 * F32(0.587)))
    W = gray.shape[1]
    x = np.arange(W)
    return gray[:, reflect101(x + 1, W)] - gray[:, reflect101(x - 1, W)]


def _weigh(clr, grd, alpha, tau_color, tau_grad):
    alpha, tau_color, tau_grad = F32(alpha), F32(tau_color), F32(tau_grad)
    clr = np.where(clr > tau_color, tau_color, clr)     # NaN > tau is False: a NaN difference stays NaN
    grd = np.where(grd > tau_grad, tau_grad, grd)
    return alpha * clr + (F32(1) - alpha) * grd


def _cost(sC, oC, sG, oG, k):
    """CVC.cpp:18-27 with the truncation restored."""
    clr = (np.abs(sC[..., 0] - oC[..., 0]) + np.abs(sC[..., 1] - oC[..., 1])) + np.abs(sC[..., 2] - oC[..., 2])
    return _weigh(clr, np.abs(sG - oG), *k)


def _border(sC, sG, k):
    """CVC.cpp:30-39: BC_32F is a double literal -> double differences, one rounding, then the float truncation."""
    c = sC.astype(F64)
    clr = ((np.abs(c[..., 0] - 1.0) + np.abs(c[..., 1] - 1.0)) + np.abs(c[..., 2] - 1.0)).astype(F32)
    grd = np.abs(sG.astype(F64) - 1.0).astype(F32)
    return _weigh(clr, grd, *k)


def cost_volumes(l, r, D, alpha=0.9, tau_color=np.inf, tau_grad=np.inf, d_begin=0, d_count=None, grads=None):
    """Raw cost volumes (lVol, rVol), each [d_count, H, W], for the global disparities [d_begin, d_begin + d_count)."""
    l, r = np.asarray(l, F32), np.asarray(r, F32)
    H, W, _ = l.shape
    d_count = D - d_begin if d_count is None else d_count
    lg, rg = (preprocess(l), preprocess(r)) if grads is None else grads
    k = (alpha, tau_color, tau_grad)
    lb, rb = _border(l, lg, k), _border(r, rg, k)
    lv = np.empty((d_count, H, W), F32)
    rv = np.empty((d_count, H, W), F32)
    for i in range(d_count):
        d = min(d_begin + i, W)
        lv[i, :, :d] = lb[:, :d]
        lv[i, :, d:] = _cost(l[:, d:], r[:, :W - d], lg[:, d:], rg[:, :W - d], k)
        rv[i, :, W - d:] = rb[:, W - d:]
        rv[i, :, :W - d] = _cost(r[:, :W - d], l[:, d:], rg[:, :W - d], lg[:, d:], k)
    return lv, rv
