#!/usr/bin/env python
"""Pin the rectification restatement (tests/rectify_oracle.py) to OpenCV's own cv2.remap and the reference's crop,
without needing cv2 at test time.

Cases:
  - "rigs": cv2.stereoRectify + initUndistortRectifyMap(..., CV_16SC2) for made-up K, D, R, T, at alpha 0 and 1, with and
    without CALIB_ZERO_DISPARITY: the reference camera's 1344 x 376 and a 640 x 480 rig ("big"), and an 80 x 48 rig
    ("small").  Each view's maps are cropped to crop_box(roi1, roi2) and applied to a seeded random frame.  cv2.remap
    of the whole frame, then the crop, is compared with the oracle on the cropped maps.  Small rigs keep their whole
    maps in the npz.  Big rigs keep three bands of rows of the cropped maps, and the digest of cv2's whole cropped
    output; their frames are re-made from the seed (np.random.default_rng(seed).integers(0, 256, (SH, SW, 3))).
  - "random": maps from cv2.convertMaps of seeded float maps whose coordinates reach far outside the source, and that
    hit -1, SW - 1 and SH - 1 exactly; raw int16 / uint16 maps with a above 1023; 1 x 1 sources and outputs; sources
    larger and smaller than the output.
Every entry records the sha256 of cv2's result (the band's rows for the bands).  The script fails unless the oracle
equals cv2 on every case, and unless remapping with a cropped map equals cropping the remapped frame.

Output (committed): tests/golden/golden_rectify.json, tests/golden/rectify_cases.npz
"""
import hashlib
import json
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import rectify_oracle as RO  # noqa: E402

BAND_ROWS = 4


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def frame(seed, sw, sh):
    return np.random.default_rng(seed).integers(0, 256, (sh, sw, 3), dtype=np.uint8)


def rig(w, h, alpha, zero_disparity):
    """stereoRectify of a made-up rig of w x h: -> (maps of each view (xy, a), crop box)"""
    s = w / 1344.0
    K1 = np.array([[700.1 * s, 0, w / 2 + 3.3 * s], [0, 699.8 * s, h / 2 + 1.4 * s], [0, 0, 1]])
    K2 = np.array([[701.5 * s, 0, w / 2 - 4.1 * s], [0, 700.9 * s, h / 2 - 2.2 * s], [0, 0, 1]])
    D1 = np.array([-0.17, 0.027, 0.0004, -0.0003, 0.0])
    D2 = np.array([-0.168, 0.025, -0.0002, 0.0005, 0.0])
    R = cv2.Rodrigues(np.array([0.003, -0.008, 0.002]))[0]
    T = np.array([-119.9, 0.3, -0.5])
    flags = cv2.CALIB_ZERO_DISPARITY if zero_disparity else 0
    R1, R2, P1, P2, _, roi1, roi2 = cv2.stereoRectify(K1, D1, K2, D2, (w, h), R, T, flags=flags, alpha=alpha)
    maps = [cv2.initUndistortRectifyMap(K, D, Rr, P, (w, h), cv2.CV_16SC2) for K, D, Rr, P in
            ((K1, D1, R1, P1), (K2, D2, R2, P2))]
    return maps, RO.crop_box(roi1, roi2)


def check(src, xy, a):
    """cv2.remap of src through (xy, a), asserted equal to the oracle -> cv2's output"""
    want = cv2.remap(src, xy, a, cv2.INTER_LINEAR)
    got = RO.remap(src, xy, a)
    assert np.array_equal(got, want), "oracle differs from cv2.remap"
    return want


def rig_cases(arrays, cases):
    for (w, h, kind) in ((1344, 376, "big"), (640, 480, "big"), (80, 48, "small")):
        for alpha in (0, 1):
            for zero in (True, False):
                name = f"rig_{w}x{h}_a{alpha}_{'zero' if zero else 'shift'}"
                maps, box = rig(w, h, alpha, zero)
                seed = len(cases) + 100
                entry = {"name": name, "kind": "rig", "src": [w, h], "box": list(box), "seed": seed, "views": []}
                for v, (xy, a) in enumerate(maps):
                    src = frame(seed + v, w, h)
                    whole = cv2.remap(src, xy, a, cv2.INTER_LINEAR)
                    cxy, ca = RO.crop(xy, box), RO.crop(a, box)
                    out = check(src, cxy, ca)
                    assert np.array_equal(out, RO.crop(whole, box)), "crop-then-remap differs from remap-then-crop"
                    view = {"sha256": digest(out)}
                    if kind == "small":
                        arrays[f"{name}_{v}_xy"], arrays[f"{name}_{v}_a"] = xy, a   # uncropped: the tests crop them
                    else:
                        H = box[3]
                        bands = [0, H // 2 - BAND_ROWS // 2, H - BAND_ROWS]
                        view["bands"] = []
                        for k, y in enumerate(bands):
                            arrays[f"{name}_{v}_band{k}_xy"] = cxy[y:y + BAND_ROWS]
                            arrays[f"{name}_{v}_band{k}_a"] = ca[y:y + BAND_ROWS]
                            view["bands"].append({"y": y, "sha256": digest(out[y:y + BAND_ROWS])})
                    entry["views"].append(view)
                entry["full_maps"] = kind == "small"
                cases.append(entry)


def random_cases(arrays, cases):
    rng = np.random.default_rng(7)

    def add(name, src, xy, a):
        out = check(src, xy, a)
        arrays[f"{name}_src"], arrays[f"{name}_xy"], arrays[f"{name}_a"] = src, xy, a
        cases.append({"name": name, "kind": "random", "src": [src.shape[1], src.shape[0]], "sha256": digest(out)})

    for k in range(24):   # convertMaps of float maps reaching 3 px and far outside the source, and its exact edges
        sw, sh = (int(v) for v in rng.integers(1, 60, 2))
        w, h = (int(v) for v in rng.integers(1, 60, 2))
        reach = 3.0 if k % 3 else 40.0
        mx = rng.uniform(-1 - reach, sw + reach, (h, w)).astype(np.float32)
        my = rng.uniform(-1 - reach, sh + reach, (h, w)).astype(np.float32)
        edge = rng.random((h, w)) < 0.25
        mx[edge] = rng.choice(np.array([-1, 0, sw - 1, sw], np.float32), edge.sum())
        my[edge] = rng.choice(np.array([-1, 0, sh - 1, sh], np.float32), edge.sum())
        xy, a = cv2.convertMaps(mx, my, cv2.CV_16SC2)
        add(f"convert{k}", rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8), xy, a)
    for k in range(8):   # raw maps: a above 1023 (remap reads its low 10 bits), any int16 coordinates near the source
        sw, sh = (int(v) for v in rng.integers(1, 40, 2))
        w, h = (int(v) for v in rng.integers(1, 40, 2))
        xy = np.stack([rng.integers(-3, sw + 3, (h, w)), rng.integers(-3, sh + 3, (h, w))], -1).astype(np.int16)
        if k == 0:
            xy[0, 0] = (-32768, 32767)
        a = rng.integers(0, 65536, (h, w)).astype(np.uint16)
        add(f"raw{k}", rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8), xy, a)
    one = np.array([[[200, 17, 99]]], np.uint8)
    for name, xy, a in (("one_in", np.zeros((1, 1, 2), np.int16), np.zeros((1, 1), np.uint16)),
                        ("one_half", np.zeros((1, 1, 2), np.int16), np.array([[16 * 32 + 16]], np.uint16)),
                        ("one_left", np.array([[[-1, 0]]], np.int16), np.array([[5 * 32 + 27]], np.uint16))):
        add(name, one, xy, a)
    src = rng.integers(0, 256, (30, 50, 3), dtype=np.uint8)
    add("one_out_of_many", src, np.array([[[49, 29]]], np.int16), np.array([[1023]], np.uint16))
    mx, my = np.meshgrid(np.linspace(-2, 5, 64, dtype=np.float32), np.linspace(-2, 3, 40, dtype=np.float32))
    xy, a = cv2.convertMaps(mx, my, cv2.CV_16SC2)
    add("source_smaller", rng.integers(0, 256, (2, 4, 3), dtype=np.uint8), xy, a)
    mx, my = np.meshgrid(np.linspace(10.3, 70.9, 16, dtype=np.float32), np.linspace(5.1, 40.2, 9, dtype=np.float32))
    xy, a = cv2.convertMaps(mx, my, cv2.CV_16SC2)
    add("source_larger", rng.integers(0, 256, (60, 90, 3), dtype=np.uint8), xy, a)


def main():
    arrays, cases = {}, []
    rig_cases(arrays, cases)
    random_cases(arrays, cases)
    np.savez_compressed(os.path.join(HERE, "rectify_cases.npz"), **arrays)
    with open(os.path.join(HERE, "golden_rectify.json"), "w") as f:
        json.dump({"cv2": cv2.__version__, "band_rows": BAND_ROWS, "cases": cases}, f, indent=1)
        f.write("\n")
    print(f"{len(cases)} cases, npz {os.path.getsize(os.path.join(HERE, 'rectify_cases.npz'))} bytes")


if __name__ == "__main__":
    main()
