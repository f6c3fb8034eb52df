"""Golden vectors for the full-resolution guided filter on the inputs of tests/gif_cases.py -- TEST INFRASTRUCTURE.

CVF::preprocess (reference src/CVF.cpp:44-70), GuidedFilter_cv (CVF.cpp:72-165) and DispSel::CVSelect
(src/DispSel.cpp:83-109) are followed call by call through the REAL cv2 primitives: boxFilter (CV_32F, 8 x 8, default
anchor and border), multiply, subtract, add.  The per-pixel solve of CVF.cpp:102-149 is plain float arithmetic and is
written out in numpy float32 (every operation rounded, none contracted).  IPP is disabled so that the box filter runs
OpenCV's own code (its running fp64 sums), whatever the build.

The inputs are the ones where the summation order matters: +inf, -inf, NaN, 1e30, a 1e15 band, |N| exp(U(-40, 10)),
mixed signs with -0.0 and ties as costs (guide: the near-black pair as 8-bit images), and the near-black float pair, its
8-bit version and a float pair with NaN / inf pixels as images (costs: orc_cost_const of the pair).  NaN payloads are not
part of the result: every NaN is written as the canonical quiet NaN before hashing.

Writes tests/golden/golden_gif.json: sha256 of the preprocess planes, of every filtered slice and of the WTA map.
Run: python tests/golden/make_golden_gif.py"""
import hashlib
import json
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
f32 = np.float32
R = (8, 8)
EPS = f32(0.0001)
D_COST, D_IMAGE = 5, 4


def canon(a):
    a = np.array(a, copy=True)
    if a.dtype == np.float32:
        a[np.isnan(a)] = f32(np.nan)
    return a


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(canon(a)).tobytes()).hexdigest()


def preprocess(img):                                            # CVF.cpp:44-70
    rgb = cv2.split(img)
    mean = [cv2.boxFilter(c, -1, R) for c in rgb]
    var = []
    for c in range(3):
        for cp in range(c, 3):
            v = cv2.boxFilter(cv2.multiply(rgb[c], rgb[cp]), -1, R)
            var.append(cv2.subtract(v, cv2.multiply(mean[c], mean[cp])))
    return rgb, mean, var


def guided_filter(rgb, mean_I, var_I, p):                       # CVF.cpp:72-165
    mean_p = cv2.boxFilter(p, -1, R)
    mean_Ip = [cv2.boxFilter(cv2.multiply(rgb[c], p), -1, R) for c in range(3)]
    c0, c1, c2 = (cv2.subtract(mean_Ip[c], cv2.multiply(mean_I[c], mean_p)) for c in range(3))
    v = var_I
    a11, a12, a13 = v[0] + EPS, v[1], v[2]
    a21, a22, a23 = v[1], v[3] + EPS, v[4]
    a31, a32, a33 = v[2], v[4], v[5] + EPS
    det = a11 * (a33 * a22 - a32 * a23) - a21 * (a33 * a12 - a32 * a13) + a31 * (a23 * a12 - a22 * a13)
    det = f32(1) / det
    a = [det * (c0 * (a33 * a22 - a32 * a23) + c1 * (a31 * a23 - a33 * a21) + c2 * (a32 * a21 - a31 * a22)),
         det * (c0 * (a32 * a13 - a33 * a12) + c1 * (a33 * a11 - a31 * a13) + c2 * (a31 * a12 - a32 * a11)),
         det * (c0 * (a23 * a12 - a22 * a13) + c1 * (a21 * a13 - a23 * a11) + c2 * (a22 * a11 - a21 * a12))]
    for c in range(3):
        mean_p = cv2.subtract(mean_p, cv2.multiply(a[c], mean_I[c]))
    q = cv2.boxFilter(mean_p, -1, R)
    for c in range(3):
        q = cv2.add(q, cv2.multiply(cv2.boxFilter(a[c], -1, R), rgb[c]))
    return q


def cv_select(vol):                                             # DispSel.cpp:83-109
    best = np.full(vol.shape[1:], np.inf, f32)                  # (float)DBL_MAX
    dis = np.zeros(vol.shape[1:], np.uint8)
    for d in range(1, vol.shape[0]):
        m = vol[d] < best
        best = np.where(m, vol[d], best)
        dis[m] = d
    return dis


def filter_volume(img, vol):
    rgb, mean, var = preprocess(img)
    return np.stack([guided_filter(rgb, mean, var, vol[d]) for d in range(vol.shape[0])]), mean, var


def entry(img, vol):
    with np.errstate(all="ignore"):
        q, mean, var = filter_volume(img, vol)
    return {"mean": sha(np.stack(mean)), "var": sha(np.stack(var)), "slices": [sha(s) for s in q],
            "wta": sha(cv_select(q)), "nan": int(np.isnan(q).sum())}


def inputs():
    """-> {name: (guide image, raw cost volume)} for every cost kind and image kind of gif_cases"""
    import gif_cases as GC
    from oracle import oracle as O
    guide = O.u8_to_f32(GC.to_u8(GC.dark_pair(GC.W, GC.H, seed=11)[0]))
    out = {f"cost_{k}": (guide, GC.costs(k, D_COST, seed=1)) for k in GC.COST_KINDS}
    for k in GC.IMAGE_KINDS:
        _, (l, r) = GC.images(k)
        with np.errstate(all="ignore"):
            vol = O.cost_const(l, r, D_IMAGE)[2]
        out[f"image_{k}"] = (l, vol)
    return out


def golden_text():
    """the contents of golden_gif.json, computed now"""
    threads, ipp = cv2.getNumThreads(), cv2.ipp.useIPP()
    cv2.setNumThreads(1)
    cv2.ipp.setUseIPP(False)
    try:
        out = {"cv2": cv2.__version__, "ipp": False, "cases": {}}
        for name, (img, vol) in inputs().items():
            out["cases"][name] = entry(img, vol)
    finally:
        cv2.setNumThreads(threads)
        cv2.ipp.setUseIPP(ipp)
    return json.dumps(out, indent=1, sort_keys=True) + "\n"


def main():
    text = golden_text()
    with open(os.path.join(HERE, "golden_gif.json"), "w") as f:
        f.write(text)
    print(json.dumps({k: v["nan"] for k, v in json.loads(text)["cases"].items()}))


if __name__ == "__main__":
    main()
