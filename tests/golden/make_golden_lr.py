#!/usr/bin/env python
"""Pin the left-right check and fill restatement (tests/lr_oracle.py) to the reference's OWN src/PP.cpp (lrCheck and
fillInv, and PP::processDM with its lines 405-406 restored), without needing the reference at test time.

Needs a checkout of PRiMEStereoMatch (REF, default /root/reference) and a C++ compiler with OpenMP: ref_lr_driver.cpp
is compiled with REF/src/PP.cpp (unmodified) against REF/include and oracle/shim with the flags of oracle/Makefile's
_ref build, into a temporary directory.

Cases (every one keeps l[x] <= x + W, where the reference's (x - d + W) % W is defined):
  - "scenes": the D = 64 winner-take-all maps of Cones and Teddy (which equal the reference's, golden.json): sha256 of
    both masks and both filled maps, from the reference and from the restatement;
  - "processdm": posterised Cones / Teddy (<= 256 distinct 6-bit colours, as golden_pp.json) through check, fill and
    JointWMF::filter at a few post-filter settings: per view the restatement's sha256 (lr_oracle.lr_check_fill, then
    oracle.post_process), the reference's, and the number of pixels where they differ;
  - "synthetic": seeded small pairs of mostly consistent maps (widths 1 .. 256, rows without a valid pixel, rows valid
    only at the first or last column, wrap-around both ways, values 0 and 1), inputs in lr_cases.npz: sha256 of the
    reference's masks and filled maps.

Output (committed): tests/golden/golden_lr.json, tests/golden/lr_cases.npz
"""
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from conftest import read_png  # noqa: E402
from oracle import oracle as O  # noqa: E402
import lr_oracle as LR  # noqa: E402
import pp_chain as PP  # noqa: E402

REF = os.environ.get("REF", "/root/reference")

# (radius, sigma, iterations, weight) of the post-filter after the fill
SETTINGS = [(9, 25.5, 1, "exp"), (16, 25.5, 1, "exp"), (9, 25.5, 2, "exp"), (9, 25.5, 1, "iv2"), (5, 10.0, 1, "off")]
SYNTH_SIZES = [(1, 3), (2, 4), (3, 5), (7, 6), (31, 4), (33, 7), (255, 3), (256, 5), (64, 1), (100, 9)]


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def posterise(img8, masks=(0xE0, 0xE0, 0xC0)):
    return (img8 & np.array(masks, np.uint8)).astype(np.uint8)


def synthetic_case(W, H, seed):
    """A pair of u8 maps with l[x] <= x + W (the reference's domain): random values made mostly consistent, then the
    special rows: row 0 has no valid pixel, row 1 (H > 1) is valid only at column 0 (left view), row 2 (H > 2) only at
    column W - 1 (left view)."""
    rng = np.random.default_rng(seed)
    x = np.arange(W)
    hi = np.minimum(255, x + W)                                   # l[x] <= x + W
    l = (rng.random((H, W)) * (hi + 1)).astype(np.int64)
    r = rng.integers(0, min(255, 2 * W) + 1, (H, W))
    for y in range(H):
        for xx in np.flatnonzero(rng.random(W) < 0.7):         # make most left pixels consistent
            r[y, (xx - l[y, xx]) % W] = l[y, xx]
    small = rng.random((H, W)) < 0.05                              # values 0 and 1 are never valid
    l[small] = rng.integers(0, 2, int(small.sum()))
    l[0] = rng.integers(0, 2, W)
    r[0] = rng.integers(0, 2, W)
    for y, col in ((1, 0), (2, W - 1)):
        if y < H:
            d = int(min(hi[col], max(2, W // 2 + 1)))
            l[y] = 0
            r[y] = 0
            if d >= 2:
                l[y, col] = d
                r[y, (col - d) % W] = d
    return l.astype(np.uint8), r.astype(np.uint8)


def ref_lib(tmp):
    shim = os.path.join(ROOT, "oracle", "shim")
    so = os.path.join(tmp, "libref_lr.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    obj = os.path.join(tmp, "stereo_oracle.o")
    subprocess.run(["gcc", "-O3", "-std=c11", "-fPIC", "-pthread", "-ffp-contract=off", "-fno-fast-math", "-c", "-o", obj,
                    os.path.join(ROOT, "oracle", "stereo_oracle.c")], check=True)
    subprocess.run([cxx, "-O3", "-std=c++11", "-fPIC", "-pthread", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-w",
                    "-I" + shim, "-I" + os.path.join(REF, "include"), "-shared", "-o", so,
                    os.path.join(HERE, "ref_lr_driver.cpp"), os.path.join(REF, "src", "PP.cpp"),
                    os.path.join(shim, "opencv_shim.cpp"), obj, "-lm", "-lpthread"], check=True)
    L = C.CDLL(so)
    f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
    u8p = np.ctypeslib.ndpointer(dtype=np.uint8, flags="C_CONTIGUOUS")
    L.ref_lr_check_fill.argtypes = [u8p, u8p, C.c_int, C.c_int, u8p, u8p, u8p, u8p]
    L.ref_process_dm_lr.argtypes = [f32p, f32p, u8p, u8p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int, u8p, u8p]
    return L


def ref_check_fill(L, l, r):
    H, W = l.shape
    out = [np.empty((H, W), np.uint8) for _ in range(4)]
    assert L.ref_lr_check_fill(np.ascontiguousarray(l), np.ascontiguousarray(r), W, H, *out) == 0
    return out


def hashes(arrs):
    return dict(zip(("lValid", "rValid", "lFill", "rFill"), (sha(a) for a in arrs)))


def main():
    if not os.path.exists(os.path.join(REF, "src", "PP.cpp")):
        raise SystemExit(f"{REF}/src/PP.cpp not found: set REF to a PRiMEStereoMatch checkout")
    out = {"scenes": {}, "processdm": {"inputs": "posterised (0xE0, 0xE0, 0xC0) Cones / Teddy, D = 64 WTA maps",
                                       "settings": []}, "synthetic": []}
    cases = {}
    with tempfile.TemporaryDirectory() as tmp:
        L = ref_lib(tmp)
        wta = {}
        for name in ("Cones", "Teddy"):
            s = name.lower()
            l8 = read_png(os.path.join(HERE, f"{s}_im2.png"))
            r8 = read_png(os.path.join(HERE, f"{s}_im6.png"))
            res = O.pipeline(O.u8_to_f32(l8), O.u8_to_f32(r8), 64, threads=8)
            ld, rd = res["lDis"], res["rDis"]
            wta[name] = (O.u8_to_f32(posterise(l8)), O.u8_to_f32(posterise(r8)), ld, rd)
            ref, mine = ref_check_fill(L, ld, rd), LR.lr_check_fill(ld, rd)
            out["scenes"][name] = {"ref": hashes(ref), "restatement": hashes(mine),
                                   "valid_pixels": [int(ref[0].sum()), int(ref[1].sum())]}
            print(name, "restatement equals the reference:", out["scenes"][name]["ref"] == out["scenes"][name]["restatement"])
        for (radius, sigma, it, weight) in SETTINGS:
            ent = {"radius": radius, "sigma": float(sigma).hex(), "iterations": it, "weight": weight, "scenes": {}}
            for name, (li, ri, ld, rd) in wta.items():
                H, W = ld.shape
                want_l, want_r = np.empty((H, W), np.uint8), np.empty((H, W), np.uint8)
                assert L.ref_process_dm_lr(li, ri, ld, rd, W, H, radius, sigma, it, O.WEIGHTS[weight], want_l, want_r) == 0
                got_l, got_r, _ = PP.chain(li, ri, ld, rd, lr=1, setting=(radius, sigma, it, weight))
                ent["scenes"][name] = {v: {"sha": sha(g), "ref_sha": sha(w), "differ": int((g != w).sum())}
                                       for v, g, w in (("l", got_l, want_l), ("r", got_r, want_r))}
            print((radius, sigma, it, weight), {k: [v["differ"] for v in s.values()] for k, s in ent["scenes"].items()},
                  flush=True)
            out["processdm"]["settings"].append(ent)
        for i, (W, H) in enumerate(SYNTH_SIZES):
            l, r = synthetic_case(W, H, seed=100 + i)
            key = f"{W}x{H}"
            cases[f"{key}_l"], cases[f"{key}_r"] = l, r
            ref = ref_check_fill(L, l, r)
            out["synthetic"].append({"key": key, "W": W, "H": H, "ref": hashes(ref),
                                     "valid_pixels": [int(ref[0].sum()), int(ref[1].sum())]})
            print(key, "restatement equals the reference:", hashes(ref) == hashes(LR.lr_check_fill(l, r)), flush=True)
    np.savez_compressed(os.path.join(HERE, "lr_cases.npz"), **cases)
    with open(os.path.join(HERE, "golden_lr.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote golden_lr.json, lr_cases.npz")


if __name__ == "__main__":
    main()
