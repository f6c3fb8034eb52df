"""Golden vectors for the stages that read a float frame, on frames outside [0, 1] -- TEST INFRASTRUCTURE.

1. The post-filter's colour quantisation, PP.cpp:416-417 `img.convertTo(img8UC3, CV_8UC3, 255)`, i.e.
   saturate_cast<uchar>(cvRound(fl(v * 255))).  Python has no binding for Mat::convertTo; two cv2 calls reach the same
   float -> u8 conversion with the product rounded to float, and they must agree on every value:
     cv2.multiply(img, <float32 array of 255>, dtype=CV_8U)  and  cv2.addWeighted(img, 255, img, 0, 0, dtype=CV_8U).
   (cv2.multiply(img, 255) with a scalar is NOT the same: it forms the product in double, and differs from convertTo at
   the floats just above (k + 0.5) / 255.)  The table holds float bit patterns and their u8 results, in rows of 67 (the
   SIMD path plus a ragged scalar tail): every (k + 0.5) / 255 float and both its neighbours, the floats around 2^31/255,
   2^63/255 and FLT_MAX/255, +-0, subnormals, +-inf, NaNs of both signs with payloads, negative values, values just above 1.
2. CVC::preprocess (CVC.cpp:41-46): cv2.cvtColor(RGB2GRAY) then cv2.Sobel(CV_32F, dx = 1, ksize = 1, BORDER_REFLECT_101)
   of both views of every frame of tests/image_cases.py (sha256, NaN payloads canonicalised).
cv2 runs on one thread.  The table is computed with IPP off and on, and the two must agree.  The gradients are computed
as make_golden.py computes them, with cv2's default IPP setting: gray_mode 0 of the oracle is that build's RGB2GRAY.

Writes tests/golden/golden_image.json.  Run: python tests/golden/make_golden_image.py"""
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
F32 = np.float32
ROW = 67


def canon(a):
    a = np.array(a, copy=True)
    if a.dtype == np.float32:
        a[np.isnan(a)] = F32(np.nan)
    return a


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(canon(a)).tobytes()).hexdigest()


def _around(x, n=3):
    """the float nearest x and its n neighbours either side"""
    c = F32(x)
    out = [c]
    lo = hi = c
    for _ in range(n):
        if not np.isfinite(hi):
            break
        with np.errstate(over="ignore"):
            lo, hi = np.nextafter(lo, F32(-np.inf)), np.nextafter(hi, F32(np.inf))
        out += [lo, hi]
    return out


def table_values():
    """the float32 values of the quantisation table"""
    k = np.arange(256)
    half = ((k + 0.5) / 255).astype(F32)
    v = list(half) + list(np.nextafter(half, F32(np.inf))) + list(np.nextafter(half, F32(-np.inf)))
    v += list((k / 255).astype(F32))
    for x in (2.0 ** 31 / 255, 8421504.0, 8421505.0, 2.0 ** 63 / 255, float(np.finfo(F32).max) / 255, 1e10, 1.3e36):
        v += _around(x)
    v += _around(np.finfo(F32).max, 1) + [F32(3.4e38)]
    v += [F32(0.0), F32(-0.0), F32(np.inf), F32(-np.inf), F32(1e-45), F32(2.0 ** -149 * 5), F32(1e-40), F32(1.1754942e-38),
          F32(np.finfo(F32).tiny), F32(-1e-45), F32(-1e-40)]
    v += [F32(x) for x in (-1e-30, -0.001, -0.5 / 255, -1.5 / 255, -0.5, -1, -255, -1e10, -8421505, -3.4e38)]
    v += _around(1.0, 4) + [F32(x) for x in (1.0001, 1.002, 1.7, 2, 255, 256, 1e5)]
    nans = np.array([0x7FC00000, 0xFFC00000, 0x7FC01234, 0xFFC01234, 0x7F800001, 0xFF800001, 0x7FBFFFFF, 0xFFFFFFFF],
                    np.uint32).view(F32)
    v += list(nans)
    v = np.array(v, F32)
    pad = (-len(v)) % ROW + ROW - 3          # a ragged last row: ROW - 3 values
    return np.concatenate([v, ((np.arange(pad) * 37 % 256 + 0.5) / 255).astype(F32)])


def quantise(v):
    """-> the u8 values cv2 gives for v (1-D float32), both ways, asserting they agree"""
    rows = [v[i:i + ROW].reshape(1, -1) for i in range(0, len(v), ROW)]
    a = np.concatenate([cv2.multiply(r, np.full_like(r, 255), dtype=cv2.CV_8U).ravel() for r in rows])
    b = np.concatenate([cv2.addWeighted(r, 255, r, 0, 0, dtype=cv2.CV_8U).ravel() for r in rows])
    assert np.array_equal(a, b), f"multiply and addWeighted differ at {v.view(np.uint32)[a != b]}"
    c = cv2.multiply(v.reshape(-1, 1), np.full((len(v), 1), 255, F32), dtype=cv2.CV_8U).ravel()   # a column: scalar path
    assert np.array_equal(a, c), "row and column conversions differ"
    return a


def preprocess(img):                                           # CVC.cpp:41-46
    g = cv2.cvtColor(img, cv2.COLOR_RGB2GRAY)
    return cv2.Sobel(g, cv2.CV_32F, 1, 0, ksize=1, borderType=cv2.BORDER_REFLECT_101)


def frames():
    """-> {name: (left, right)}: every frame of image_cases"""
    import image_cases as IC
    out = {}
    for kind in IC.KINDS:
        for size, (W, H, D) in (("main", IC.MAIN), ("narrow", IC.NARROW), ("point", IC.POINT)):
            out[f"{kind}_{size}"] = IC.frame(kind, W, H, D)
        out[f"{kind}_wide"] = IC.wide_frame(kind)
    return out


def golden_text():
    """the contents of golden_image.json, computed now"""
    threads, ipp = cv2.getNumThreads(), cv2.ipp.useIPP()
    cv2.setNumThreads(1)
    try:
        v = table_values()
        cv2.ipp.setUseIPP(False)
        q = quantise(v)
        cv2.ipp.setUseIPP(True)
        assert np.array_equal(q, quantise(v)), "the conversion depends on IPP"
        cv2.ipp.setUseIPP(ipp)
        out = {"cv2": cv2.__version__, "ipp": bool(cv2.ipp.useIPP()), "row": ROW,
               "u8x255": {"bits": [int(b) for b in v.view(np.uint32)], "u8": [int(x) for x in q]},
               "gradients": {}}
        with np.errstate(all="ignore"):
            for name, (l, r) in frames().items():
                out["gradients"][name] = [sha(preprocess(l)), sha(preprocess(r))]
    finally:
        cv2.setNumThreads(threads)
        cv2.ipp.setUseIPP(ipp)
    return json.dumps(out, indent=None, sort_keys=True, separators=(",", ":")) + "\n"


def main():
    text = golden_text()
    with open(os.path.join(HERE, "golden_image.json"), "w") as f:
        f.write(text)
    t = json.loads(text)["u8x255"]
    print(f"{len(t['u8'])} table values, {len(json.loads(text)['gradients'])} frames")


if __name__ == "__main__":
    main()
