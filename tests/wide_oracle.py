"""ctypes loader for tests/wide_oracle.c: the CPU restatement of the 16-bit-map stages (orc_wta16, orc_wmf16; TEST
INFRASTRUCTURE).  The C source is compiled on first use into a temporary directory, with the oracle's flags
(-O3 -ffp-contract=off -fno-fast-math), so that nothing is written into the tree."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "wide_oracle.c")
_LIB = None

WEIGHTS = {"exp": 0, "iv1": 1, "iv2": 2, "off": 5}

_u8p = np.ctypeslib.ndpointer(dtype=np.uint8, flags="C_CONTIGUOUS")
_u16p = np.ctypeslib.ndpointer(dtype=np.uint16, flags="C_CONTIGUOUS")
_f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")


def lib():
    global _LIB
    if _LIB is None:
        src = open(_SRC, "rb").read()
        tag = hashlib.sha256(src).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), f"psm_wide_oracle_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        path = os.path.join(d, f"libwide_oracle_{tag}.so")
        if not os.path.exists(path):
            tmp = f"{path}.{os.getpid()}.tmp"
            cc = os.environ.get("CC", "gcc")
            subprocess.run([cc, "-O3", "-std=c11", "-fPIC", "-pthread", "-ffp-contract=off", "-fno-fast-math", "-shared",
                            "-o", tmp, _SRC, "-lm", "-lpthread"], check=True)
            os.replace(tmp, path)
        L = C.CDLL(path)
        L.orc_wta16.argtypes = [_f32p, C.c_int, C.c_int, C.c_int, _u16p]
        L.orc_wmf16.argtypes = [_u16p, _u8p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int, C.c_int, _u16p]
        _LIB = L
    return _LIB


def wta16(vol):
    """vol[D, H, W] float32 -> u16 arg-min map over d in [1, D)"""
    vol = np.ascontiguousarray(vol, np.float32)
    D, H, W = vol.shape
    out = np.empty((H, W), np.uint16)
    lib().orc_wta16(vol, W, H, D, out)
    return out


def to_u8x255(img3_f32):
    """convertTo(CV_8UC3, 255) (src/PP.cpp:416-417): saturate_cast<uchar>(cvRound(v * 255)), half to even"""
    q = np.rint(np.asarray(img3_f32, np.float32) * np.float32(255.0))
    return np.clip(q, 0, 255).astype(np.uint8)


def post_process16(img3_f32, disp, r=9, sigma=25.5, iterations=1, weight="exp", threads=8):
    """One view of the post-filter on a u16 map at (r, sigma, iterations, weight), float BGR feature image in [0,1]."""
    img8 = np.ascontiguousarray(to_u8x255(img3_f32))
    disp = np.ascontiguousarray(disp, np.uint16)
    H, W = disp.shape
    out = np.empty((H, W), np.uint16)
    rc = lib().orc_wmf16(disp, img8, W, H, int(r), float(sigma), int(iterations), WEIGHTS[weight], int(threads), out)
    assert rc == 0
    return out


def argmin_volume(W, H, D, seed, lo=256):
    """Seeded synthetic volume [D, H, W] whose arg-mins spread over [1, D) with most of them >= lo (when D > lo), and
    with exact ties (the lowest d must win) and +inf / NaN slices mixed in.  -> (vol, intended arg-min)"""
    rng = np.random.default_rng(seed)
    vol = rng.uniform(1.0, 2.0, (D, H, W)).astype(np.float32)
    want = rng.integers(max(1, min(lo, D - 1)) if D > lo else 1, D, (H, W))
    low = rng.random((H, W)) < 0.2
    want = np.where(low, rng.integers(1, D, (H, W)), want)
    yy, xx = np.mgrid[0:H, 0:W]
    vol[want, yy, xx] = 0.5
    # a tie at a higher d never wins
    hi = np.minimum(want + 1 + rng.integers(0, 7, (H, W)), D - 1)
    tie = (rng.random((H, W)) < 0.3) & (hi > want)
    vol[hi[tie], yy[tie], xx[tie]] = 0.5
    vol[0] = 0.0                                        # d = 0 is never a candidate
    vol[:, 0, 0] = np.inf                               # nothing below +inf: 0
    vol[:, 0, 1] = np.nan
    return vol, want


def widen(disp_u8, seed):
    """A wide map from a D = 64 map: 8 * d plus a seeded offset in [0, 8) that is constant on 8 x 8 blocks (values up to
    511, piecewise constant like a real disparity map)."""
    rng = np.random.default_rng(seed)
    H, W = disp_u8.shape
    off = np.repeat(np.repeat(rng.integers(0, 8, ((H + 7) // 8, (W + 7) // 8)), 8, 0), 8, 1)[:H, :W]
    return (disp_u8.astype(np.uint16) * 8 + off).astype(np.uint16)
