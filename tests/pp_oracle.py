"""ctypes loader for tests/pp_oracle.c: the CPU restatement of the post-filter at any psm_set_post_filter setting
(TEST INFRASTRUCTURE).  The C source is compiled on first use into a temporary directory, with the oracle's flags
(-O3 -ffp-contract=off -fno-fast-math), so that nothing is written into the tree."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "pp_oracle.c")
_LIB = None

WEIGHTS = {"exp": 0, "iv1": 1, "iv2": 2, "off": 5}
DEFAULT = (9, 25.5, 1, "exp")

_u8p = np.ctypeslib.ndpointer(dtype=np.uint8, flags="C_CONTIGUOUS")
_u32p = np.ctypeslib.ndpointer(dtype=np.uint32, flags="C_CONTIGUOUS")


def lib():
    global _LIB
    if _LIB is None:
        src = open(_SRC, "rb").read()
        tag = hashlib.sha256(src).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), f"psm_pp_oracle_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        path = os.path.join(d, f"libpp_oracle_{tag}.so")
        if not os.path.exists(path):
            tmp = f"{path}.{os.getpid()}.tmp"
            cc = os.environ.get("CC", "gcc")
            subprocess.run([cc, "-O3", "-std=c11", "-fPIC", "-pthread", "-ffp-contract=off", "-fno-fast-math", "-shared",
                            "-o", tmp, _SRC, "-lm", "-lpthread"], check=True)
            os.replace(tmp, path)
        L = C.CDLL(path)
        L.pp_table_size.argtypes = [C.c_int]
        L.pp_weight_table.argtypes = [C.c_float, C.c_int, _u32p]
        L.pp_wmf.argtypes = [_u8p, _u8p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int, C.c_int, _u8p]
        _LIB = L
    return _LIB


def weight_table(sigma=25.5, weight="exp"):
    t = np.zeros(lib().pp_table_size(WEIGHTS[weight]), np.uint32)
    lib().pp_weight_table(sigma, WEIGHTS[weight], t)
    return t


def table_sha(sigma=25.5, weight="exp"):
    return hashlib.sha256(weight_table(sigma, weight).tobytes()).hexdigest()


def to_u8x255(img3_f32):
    """convertTo(CV_8UC3, 255) (src/PP.cpp:416-417): saturate_cast<uchar>(cvRound(v * 255)), half to even"""
    q = np.rint(np.asarray(img3_f32, np.float32) * np.float32(255.0))
    return np.clip(q, 0, 255).astype(np.uint8)


def post_process(img3_f32, disp, r=9, sigma=25.5, iterations=1, weight="exp", threads=8):
    """One view of the post-filter at (r, sigma, iterations, weight), float BGR feature image in [0,1]."""
    img8 = np.ascontiguousarray(to_u8x255(img3_f32))
    disp = np.ascontiguousarray(disp, np.uint8)
    H, W = disp.shape
    out = np.empty((H, W), np.uint8)
    rc = lib().pp_wmf(disp, img8, W, H, int(r), float(sigma), int(iterations), WEIGHTS[weight], int(threads), out)
    assert rc == 0
    return out
