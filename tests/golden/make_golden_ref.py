#!/usr/bin/env python
"""Record what the reference's OWN compiled code (oracle/_ref, built by `make -C oracle ref` from a checkout of
PRiMEStereoMatch) returns for the inputs of tests/test_oracle_ref.py and the reference parts of tests/test_pp.py, so
that those tests pin the C port to the reference without needing the reference at test time.

Outputs (committed):
  tests/golden/ref_outputs.json   sha256 of every reference result the tests compare with, and the colour counts
  tests/golden/ref_pp_teddy.npz   the reference's post-processed Teddy left map (natural image: compared by agreement)

Every result that the reference computes in more than one way (thread counts, the non-pthread twins) is checked
here to agree before it is recorded once.
"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from conftest import read_png  # noqa: E402
from oracle import oracle as O  # noqa: E402
from oracle import ref as R  # noqa: E402


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def posterise(img8, masks=(0xE0, 0xE0, 0xC0)):
    return (img8 & np.array(masks, np.uint8)).astype(np.uint8)


def scene(name):
    s = name.lower()
    l8 = read_png(os.path.join(HERE, f"{s}_im2.png"))
    r8 = read_png(os.path.join(HERE, f"{s}_im6.png"))
    return l8, r8, O.u8_to_f32(l8), O.u8_to_f32(r8)


def main():
    if not R.available():
        raise SystemExit("oracle/_ref is not built: `make -C oracle ref REF=<PRiMEStereoMatch checkout>`")
    out = {"scenes": {}, "pp": {}}
    keys = ("lGrd", "rGrd", "lRaw", "rRaw", "lVol", "rVol", "lDis", "rDis")
    for name in ("Cones", "Teddy"):
        l8, r8, l, r = scene(name)
        ref = R.pipeline(l, r, 64, threads=8, keep=True)
        out["scenes"][name] = {k: sha(ref[k]) for k in keys}
        ld, rd = ref["lDis"], ref["rDis"]
        pp = {}
        for view, img8, disp in (("l", l8, ld), ("r", r8, rd)):
            want, ncol = R.post_process(O.u8_to_f32(posterise(img8)), disp)
            pp[view] = {"sha": sha(want), "colours": ncol}
        out["pp"][name] = pp
        if name == "Teddy":
            want, ncol = R.post_process(l, ld)
            out["pp"]["Teddy_natural_colours"] = ncol
            np.savez_compressed(os.path.join(HERE, "ref_pp_teddy.npz"), lpp=want)

    # Teddy crop, D = 12: thread counts (remainder batches) and the non-pthread twins agree
    _, _, l, r = scene("Teddy")
    l, r = l[:60, :128].copy(), r[:60, :128].copy()
    base = R.pipeline(l, r, 12, threads=8, keep=True)
    for t in (1, 3):
        other = R.pipeline(l, r, 12, threads=t, keep=True)
        for k in ("lRaw", "rRaw", "lVol", "rVol", "lDis", "rDis"):
            assert np.array_equal(base[k], other[k]), (t, k)
    for d in (0, 5, 11):
        assert np.array_equal(R.buildcv(l, r, d, right=False), base["lRaw"][d])
        assert np.array_equal(R.buildcv(l, r, d, right=True), base["rRaw"][d])
    assert np.array_equal(R.wta(base["lVol"], thread_variant=True, threads=4), base["lDis"])
    assert np.array_equal(R.wta(base["lVol"]), base["lDis"])
    out["teddy_crop_D12"] = {k: sha(base[k]) for k in ("lRaw", "rRaw", "lVol", "rVol", "lDis", "rDis")}

    # GuidedFilter_cv on signed, wide-range costs
    rng = np.random.default_rng(8)
    H, W = 48, 77
    img = rng.random((H, W, 3), dtype=np.float32)
    gf = {}
    for scale in (1.0, 1e-4, 300.0):
        p = (rng.normal(0, 1, (H, W)) * scale).astype(np.float32)
        gf[repr(scale)] = sha(R.guided_filter(img, p))
    out["guided_filter_48x77"] = gf

    # gray-mode switch on a Cones crop, D = 6
    _, _, l, r = scene("Cones")
    l, r = l[:40, :90].copy(), r[:40, :90].copy()
    out["gray_mode_cones_crop_D6"] = {}
    for gm in (0, 1):
        ref = R.pipeline(l, r, 6, gray_mode=gm, keep=True)
        out["gray_mode_cones_crop_D6"][str(gm)] = {k: sha(ref[k]) for k in ("lGrd", "lRaw", "rRaw")}

    with open(os.path.join(HERE, "ref_outputs.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote ref_outputs.json, ref_pp_teddy.npz")


if __name__ == "__main__":
    main()
