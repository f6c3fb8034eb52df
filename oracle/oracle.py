"""ctypes loader for the CPU oracle (oracle/libstereo_oracle.so).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  The product package never imports this module.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

_f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
_u8p = np.ctypeslib.ndpointer(dtype=np.uint8, flags="C_CONTIGUOUS")
_u32p = np.ctypeslib.ndpointer(dtype=np.uint32, flags="C_CONTIGUOUS")
_f64p = np.ctypeslib.ndpointer(dtype=np.float64, flags="C_CONTIGUOUS")

# the post-filter's weight types (JointWMF.h:503-508 numbering, as psm_set_post_filter takes them)
WEIGHTS = {"exp": 0, "iv1": 1, "iv2": 2, "off": 5}
_PP_TABLE_MAX = 3 * 63 * 63 + 1
_MAP_BYTES = {np.dtype(np.uint8): 1, np.dtype(np.uint16): 2}
# The reference's compile-time constants (ORC_GIF_R_WIN, ORC_GIF_EPS, ORC_ALPHA, no truncation) are the defaults of the
# keyword arguments window, eps, alpha, tau_color and tau_grad below.
INF = float("inf")


def build():
    """Compile the oracle with its Makefile (gcc, seconds)."""
    subprocess.run(["make", "-C", _HERE, "-s"], check=True)


def lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, "libstereo_oracle.so")
        if not os.path.exists(path):
            build()
        L = C.CDLL(path)
        L.orc_u8_to_f32.argtypes = [_u8p, _f32p, C.c_size_t]
        L.orc_rgb2gray.argtypes = [_f32p, C.c_int, C.c_int, _f32p, C.c_int]
        L.orc_sobel_x.argtypes = [_f32p, C.c_int, C.c_int, _f32p]
        L.orc_cvc_preprocess.argtypes = [_f32p, C.c_int, C.c_int, _f32p, C.c_int]
        for fn in (L.orc_buildcv_left, L.orc_buildcv_right):
            fn.argtypes = [_f32p, _f32p, _f32p, _f32p, C.c_int, C.c_int, C.c_int, _f32p]
        for fn in (L.orc_box, L.orc_box_k):
            fn.argtypes = [_f32p, C.c_int, C.c_int, C.c_int, _f32p]
        L.orc_cvf_preprocess.argtypes = [_f32p, C.c_int, C.c_int, C.c_int, _f32p, _f32p, _f32p]
        L.orc_guided_filter.argtypes = [_f32p, _f32p, _f32p, C.c_int, C.c_int, C.c_int, C.c_float, _f32p, _f32p, _f32p]
        L.orc_wta.argtypes = [_f32p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int]
        L.orc_cost_const.argtypes = [_f32p, _f32p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.c_float, C.c_float, C.c_float, _f32p, _f32p, _f32p, _f32p]
        L.orc_cost_filter.argtypes = [_f32p, _f32p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float,
                                      _f32p, _f32p]
        L.orc_disp_select.argtypes = [_f32p, _f32p, C.c_int, C.c_int, C.c_int, _u8p, _u8p]
        L.orc_pipeline.argtypes = [_f32p, _f32p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                   C.c_float, C.c_float, C.c_float, C.c_int, C.c_float,
                                   _f32p, _f32p, _u8p, _u8p, _f64p]
        L.orc_cost_filter_fgf.argtypes = [_f32p, _f32p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float,
                                          _f32p, _f32p]
        L.orc_pp_weight_table.argtypes = [C.c_float, C.c_int, _u32p]
        L.orc_wmf.argtypes = [C.c_void_p, C.c_int, _u8p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int, C.c_int,
                              C.c_void_p]
        L.orc_f32_to_u8x255.argtypes = [_f32p, _u8p, C.c_size_t]
        for name in ("orc_cost_const", "orc_cost_filter", "orc_cost_filter_fgf", "orc_disp_select", "orc_pipeline",
                     "orc_pp_weight_table", "orc_wmf"):
            getattr(L, name).restype = C.c_int
        _LIB = L
    return _LIB


def _c(a, dt=np.float32):
    return np.ascontiguousarray(a, dtype=dt)


def u8_to_f32(img_u8):
    src = _c(img_u8, np.uint8)
    dst = np.empty(src.shape, np.float32)
    lib().orc_u8_to_f32(src.reshape(-1), dst.reshape(-1), src.size)
    return dst


def rgb2gray(img3, gray_mode=0):
    img3 = _c(img3)
    H, W, _ = img3.shape
    out = np.empty((H, W), np.float32)
    lib().orc_rgb2gray(img3, W, H, out, gray_mode)
    return out


def sobel_x(gray):
    gray = _c(gray)
    H, W = gray.shape
    out = np.empty((H, W), np.float32)
    lib().orc_sobel_x(gray, W, H, out)
    return out


def cvc_preprocess(img3, gray_mode=0):
    img3 = _c(img3)
    H, W, _ = img3.shape
    out = np.empty((H, W), np.float32)
    lib().orc_cvc_preprocess(img3, W, H, out, gray_mode)
    return out


def box(src, K):
    """cv::boxFilter(src, -1, (K, K)) of one plane, in OpenCV's order of fp64 operations (orc_box)"""
    src = _c(src)
    H, W = src.shape
    out = np.empty((H, W), np.float32)
    lib().orc_box(src, W, H, K, out)
    return out


def box8(src):
    return box(src, 8)


def box_direct(src, K):
    """the Fast Guided Filter's K x K box of one plane: direct fp64 sums (orc_box_k; stereo_oracle.h says when it equals
    box)"""
    src = _c(src)
    H, W = src.shape
    out = np.empty((H, W), np.float32)
    lib().orc_box_k(src, W, H, K, out)
    return out


def cvf_preprocess(img3, *, window=8):
    """-> rgb[3,H,W], mean[3,H,W], var[6,H,W]"""
    img3 = _c(img3)
    H, W, _ = img3.shape
    rgb = np.empty((3, H, W), np.float32)
    mean = np.empty((3, H, W), np.float32)
    var = np.empty((6, H, W), np.float32)
    lib().orc_cvf_preprocess(img3, W, H, window, rgb, mean, var)
    return rgb, mean, var


def guided_filter(rgb, mean, var, p, want_ab=False, *, window=8, eps=1e-4):
    """GuidedFilter_cv of one slice p[H,W] or of every slice of a volume p[D,H,W]
    -> q  (or (q, a[3,H,W], b[H,W]) with want_ab; a[D,3,H,W], b[D,H,W] for a volume)"""
    rgb, mean, var = _c(rgb), _c(mean), _c(var)
    q = _c(p).copy()
    H, W = q.shape[-2:]
    a = np.empty(q.shape[:-2] + (3, H, W), np.float32)
    b = np.empty(q.shape, np.float32)
    for qs, as_, bs in zip(q.reshape(-1, H, W), a.reshape(-1, 3, H, W), b.reshape(-1, H, W)):
        lib().orc_guided_filter(rgb, mean, var, W, H, window, eps, qs, as_, bs)
    return (q, a, b) if want_ab else q


def _map_bytes(dtype):
    try:
        return _MAP_BYTES[np.dtype(dtype)]
    except KeyError:
        raise TypeError(f"disparity maps are uint8 or uint16, not {np.dtype(dtype)}") from None


def wta(vol, dtype=np.uint8):
    """vol[D, H, W] -> arg-min map over d in [1, D); uint8 keeps the low byte as the reference does, uint16 all of it"""
    vol = _c(vol)
    D, H, W = vol.shape
    out = np.empty((H, W), dtype)
    lib().orc_wta(vol, W, H, D, out.ctypes.data_as(C.c_void_p), _map_bytes(dtype))
    return out


def cost_const(l, r, D, threads=8, gray_mode=0, *, alpha=0.9, tau_color=INF, tau_grad=INF, d_begin=0, d_count=None):
    """-> lGrd, rGrd, lVol, rVol  (raw cost volumes [d_count,H,W] of the disparities [d_begin, d_begin + d_count), all
    of [0, D) by default)"""
    l, r = _c(l), _c(r)
    H, W, _ = l.shape
    d_count = D - d_begin if d_count is None else d_count
    lg = np.empty((H, W), np.float32)
    rg = np.empty((H, W), np.float32)
    lv = np.empty((d_count, H, W), np.float32)
    rv = np.empty((d_count, H, W), np.float32)
    rc = lib().orc_cost_const(l, r, W, H, d_begin, d_count, threads, gray_mode, alpha, tau_color, tau_grad, lg, rg, lv, rv)
    assert rc == 0
    return lg, rg, lv, rv


def cost_filter(l, r, lv, rv, threads=8, *, window=8, eps=1e-4):
    """filters copies of the volumes -> lVolF, rVolF"""
    l, r = _c(l), _c(r)
    lv, rv = _c(lv).copy(), _c(rv).copy()
    D, H, W = lv.shape
    rc = lib().orc_cost_filter(l, r, W, H, D, threads, window, eps, lv, rv)
    assert rc == 0
    return lv, rv


def disp_select(lv, rv):
    lv, rv = _c(lv), _c(rv)
    D, H, W = lv.shape
    ld = np.empty((H, W), np.uint8)
    rd = np.empty((H, W), np.uint8)
    lib().orc_disp_select(lv, rv, W, H, D, ld, rd)
    return ld, rd


def pipeline(l, r, D, threads=8, gray_mode=0, keep_volumes=False, *, alpha=0.9, tau_color=INF, tau_grad=INF, window=8,
             eps=1e-4):
    """Full CVC->CVF->WTA.  -> dict(lDis, rDis, times_ms=[cvc,cvf,wta], [lVol, rVol])"""
    l, r = _c(l), _c(r)
    H, W, _ = l.shape
    lv = np.empty((D, H, W), np.float32)
    rv = np.empty((D, H, W), np.float32)
    ld = np.empty((H, W), np.uint8)
    rd = np.empty((H, W), np.uint8)
    t = np.zeros(3, np.float64)
    rc = lib().orc_pipeline(l, r, W, H, D, threads, gray_mode, alpha, tau_color, tau_grad, window, eps, lv, rv, ld, rd, t)
    assert rc == 0
    out = {"lDis": ld, "rDis": rd, "times_ms": t.tolist()}
    if keep_volumes:
        out["lVol"], out["rVol"] = lv, rv
    return out


def to_u8x255(img3_f32):
    """convertTo(CV_8UC3, 255) (src/PP.cpp:416-417): saturate_cast<uchar>(cvRound(v * 255)), half to even; 0 where the
    float product is NaN or >= 2^31 (x86 cvRound's INT_MIN)"""
    img3 = _c(img3_f32)
    img8 = np.empty(img3.shape, np.uint8)
    lib().orc_f32_to_u8x255(img3.reshape(-1), img8.reshape(-1), img3.size)
    return img8


def weight_table(sigma=25.5, weight="exp"):
    """the post-filter's 2^-22 fixed-point weight table at (sigma, weight), as uint32"""
    t = np.zeros(_PP_TABLE_MAX, np.uint32)
    n = lib().orc_pp_weight_table(sigma, WEIGHTS[weight], t)
    return t[:n].copy()


def post_process(img3_f32, disp, r=9, sigma=25.5, iterations=1, weight="exp", threads=8):
    """One view of the post-filter, JointWMF::filter at (r, sigma, iterations, weight) as PP::processDM drives it
    (src/PP.cpp:414-422, defaults: its live code), un-clustered restatement (see stereo_oracle.c).  img3_f32: float BGR
    feature image in [0, 1]; disp: a uint8 or uint16 map -> the filtered map, of disp's dtype."""
    img8 = to_u8x255(img3_f32)
    disp = np.ascontiguousarray(disp)
    H, W = disp.shape
    out = np.empty((H, W), disp.dtype)
    rc = lib().orc_wmf(disp.ctypes.data_as(C.c_void_p), _map_bytes(disp.dtype), img8, W, H, int(r), float(sigma),
                       int(iterations), WEIGHTS[weight], int(threads), out.ctypes.data_as(C.c_void_p))
    assert rc == 0
    return out


def cost_filter_fgf(l, r, lv, rv, s=4, threads=8, *, window=8, eps=1e-4):
    """DispEst::CostFilter_FGF (FastGuidedFilter(img, window, eps, s)) on copies of the volumes -> lVolF, rVolF"""
    l, r = _c(l), _c(r)
    lv, rv = _c(lv).copy(), _c(rv).copy()
    D, H, W = lv.shape
    rc = lib().orc_cost_filter_fgf(l, r, W, H, D, threads, s, window, eps, lv, rv)
    assert rc == 0
    return lv, rv
