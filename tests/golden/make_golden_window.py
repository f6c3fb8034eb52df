"""Golden vectors for the guided filter at other windows and epsilons than the reference's compile-time GIF_R_WIN = 8 and
GIF_EPS = 0.0001f (include/ComFunc.h:49-50) -- TEST INFRASTRUCTURE.

The reference cannot be rebuilt with another window (ComFunc.h defines GIF_R_WIN unconditionally), so the other windows
are pinned by OpenCV itself: CVF::preprocess and GuidedFilter_cv (CVF.cpp:44-165) restated with cv2.boxFilter(p, -1,
(k, k)) and float32 element-wise operations in CVF.cpp order; the Fast Guided Filter branch by make_golden_fgf.py's
call-by-call restatement with FastGuidedFilter(img, r = window, eps, s).  IPP is disabled, as in make_golden_fgf.py.

Writes tests/golden/golden_window.json: per case and scene the sha256 of mean_I / var_I (left view), both filtered volumes
and both WTA maps, Cones and Teddy at D = 64.
Run: python tests/golden/make_golden_window.py"""
import hashlib
import json
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)
from make_golden_fgf import FastGuidedFilterColor  # noqa: E402

f32 = np.float32
GIF_CASES = [(4, 1e-4), (9, 1e-4), (16, 1e-4), (32, 1e-4), (8, 1e-3)]
FGF_CASES = [(16, 1e-4, 4), (32, 1e-4, 2)]


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def preprocess(img, k):                                    # CVF.cpp:44-70
    rgb = cv2.split(img)
    box = lambda x: cv2.boxFilter(x, -1, (k, k))
    mean = [box(c) for c in rgb]
    var = []
    for c in range(3):
        for cp in range(c, 3):
            var.append(box(rgb[c] * rgb[cp]) - mean[c] * mean[cp])
    return rgb, mean, var


def guided_filter(rgb, mean, var, p, k, eps):              # CVF.cpp:72-165
    box = lambda x: cv2.boxFilter(x, -1, (k, k))
    eps = f32(eps)
    mean_p = box(p)
    cov = [box(rgb[c] * p) - mean[c] * mean_p for c in range(3)]
    c0, c1, c2 = cov
    a11, a12, a13 = var[0] + eps, var[1], var[2]
    a21, a22, a23 = var[1], var[3] + eps, var[4]
    a31, a32, a33 = var[2], var[4], var[5] + eps
    DET = a11 * (a33 * a22 - a32 * a23) - a21 * (a33 * a12 - a32 * a13) + a31 * (a23 * a12 - a22 * a13)
    DET = f32(1) / DET
    a = [DET * (c0 * (a33 * a22 - a32 * a23) + c1 * (a31 * a23 - a33 * a21) + c2 * (a32 * a21 - a31 * a22)),
         DET * (c0 * (a32 * a13 - a33 * a12) + c1 * (a33 * a11 - a31 * a13) + c2 * (a31 * a12 - a32 * a11)),
         DET * (c0 * (a23 * a12 - a22 * a13) + c1 * (a21 * a13 - a23 * a11) + c2 * (a22 * a11 - a21 * a12))]
    b = mean_p
    for c in range(3):
        b = b - a[c] * mean[c]
    q = box(b)
    for c in range(3):
        q = q + box(a[c]) * rgb[c]
    return q


def main():
    cv2.setNumThreads(1)
    cv2.ipp.setUseIPP(False)
    from oracle import oracle as O
    out = {"cv2": cv2.__version__, "ipp": False, "D": 64, "cases": {}}
    scenes = {}
    for scene in ("Cones", "Teddy"):
        s_ = scene.lower()
        l8 = cv2.imread(os.path.join(HERE, f"{s_}_im2.png"), cv2.IMREAD_COLOR)
        r8 = cv2.imread(os.path.join(HERE, f"{s_}_im6.png"), cv2.IMREAD_COLOR)
        l, r = O.u8_to_f32(l8), O.u8_to_f32(r8)
        _, _, lraw, rraw = O.cost_const(l, r, 64)
        scenes[scene] = (l, r, lraw, rraw)
    for (k, eps) in GIF_CASES:
        name = f"gif_w{k}_eps{eps:g}"
        case = {"params": {"kind": "gif", "window": k, "eps": eps}}
        for scene, (l, r, lraw, rraw) in scenes.items():
            vols = []
            for img, raw in ((l, lraw), (r, rraw)):
                rgb, mean, var = preprocess(img, k)
                if img is l:
                    lmean, lvar = np.stack(mean), np.stack(var)
                vols.append(np.stack([guided_filter(rgb, mean, var, raw[d], k, eps) for d in range(raw.shape[0])]))
            case[scene] = {"lMean": sha(lmean), "lVar": sha(lvar), "lFilt": sha(vols[0]), "rFilt": sha(vols[1]),
                           "lDis": sha(O.wta(vols[0])), "rDis": sha(O.wta(vols[1]))}
        out["cases"][name] = case
        print(name, flush=True)
    for (k, eps, s) in FGF_CASES:
        name = f"fgf_w{k}_eps{eps:g}_s{s}"
        case = {"params": {"kind": "fgf", "window": k, "eps": eps, "s": s}}
        for scene, (l, r, lraw, rraw) in scenes.items():
            fl = FastGuidedFilterColor(l, k, float(f32(eps)), s)
            fr = FastGuidedFilterColor(r, k, float(f32(eps)), s)
            lf = np.stack([fl.filter(lraw[d]) for d in range(lraw.shape[0])])
            rf = np.stack([fr.filter(rraw[d]) for d in range(rraw.shape[0])])
            case[scene] = {"lFilt": sha(lf), "rFilt": sha(rf), "lDis": sha(O.wta(lf)), "rDis": sha(O.wta(rf))}
        out["cases"][name] = case
        print(name, flush=True)
    with open(os.path.join(HERE, "golden_window.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
