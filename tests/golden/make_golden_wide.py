#!/usr/bin/env python
"""Pin the restatements on 16-bit maps (oracle.wta and oracle.post_process with uint16 maps) to the reference's OWN
code, without needing the reference at test time.

Needs a checkout of PRiMEStereoMatch (REF, default /root/reference):
  - oracle/_ref (oracle/Makefile target `ref`: src/DispSel.cpp compiled unmodified) for the selection;
  - a C++ compiler with OpenMP: ref_wmf32f_driver.cpp is compiled against REF/include (JointWMF.h unmodified) and
    oracle/shim with the flags of oracle/Makefile's _ref build, into a temporary directory.

Records (committed as tests/golden/golden_wide.json):
  wta:  seeded volumes (wide_cases.argmin_volume) at D in {300, 511, 600, 1024}: the sha256 of DispSel::CVSelect's
        uchar map, which must equal the low byte of the u16 orc_wta, and how many arg-mins exceed 255;
  wmf:  posterised Cones / Teddy (<= 256 six-bit colours, so the reference's colour clustering is exact), both views,
        with wide maps (wide_cases.widen of the D = 64 maps, values up to 511, max_disp 512): for each setting the sha256
        of orc_wmf, of JointWMF::filter on the map as CV_32F with nI = 512, and the number of pixels where they
        differ (the reference's float cut-point search; 0 expected, as at these settings in golden_pp.json);
  loop: JointWMF::filter on the D = 64 maps as CV_32F (nI = 256) against the CV_8U path's hashes in golden_pp.json.
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
from oracle import ref as R  # noqa: E402
from wide_cases import argmin_volume, widen  # noqa: E402

REF = os.environ.get("REF", "/root/reference")

WTA_CASES = [(300, 48, 32, 1), (511, 40, 24, 2), (600, 37, 21, 3), (1024, 24, 16, 4)]   # (D, W, H, seed)
WIDE_MAX_DISP = 512
# (radius, sigma, iterations, weight)
SETTINGS = [
    (9, 25.5, 1, "exp"),
    (4, 25.5, 1, "exp"),
    (16, 25.5, 1, "exp"),
    (9, 10.0, 1, "exp"),
    (9, 25.5, 3, "exp"),
    (9, 25.5, 1, "iv1"),
    (9, 25.5, 1, "iv2"),
    (9, 25.5, 1, "off"),
    (20, 25.5, 2, "iv2"),
]
LOOP_KEYS = ["9/0x1.9800000000000p+4/1/exp", "16/0x1.9800000000000p+4/1/exp", "9/0x1.9800000000000p+4/1/iv1"]


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def posterise(img8, masks=(0xE0, 0xE0, 0xC0)):
    return (img8 & np.array(masks, np.uint8)).astype(np.uint8)


def key(r, sigma, it, weight):
    return f"{r}/{float(sigma).hex()}/{it}/{weight}"


def ref_lib(tmp):
    shim = os.path.join(ROOT, "oracle", "shim")
    so = os.path.join(tmp, "libref_wmf32f.so")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    obj = os.path.join(tmp, "stereo_oracle.o")
    subprocess.run(["gcc", "-O3", "-std=c11", "-fPIC", "-pthread", "-ffp-contract=off", "-fno-fast-math", "-c", "-o", obj,
                    os.path.join(ROOT, "oracle", "stereo_oracle.c")], check=True)
    subprocess.run([cxx, "-O3", "-std=c++11", "-fPIC", "-pthread", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-w",
                    "-I" + shim, "-I" + os.path.join(REF, "include"), "-shared", "-o", so,
                    os.path.join(HERE, "ref_wmf32f_driver.cpp"), os.path.join(shim, "opencv_shim.cpp"), obj, "-lm",
                    "-lpthread"], check=True)
    L = C.CDLL(so)
    f32p = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")
    L.ref_wmf32f.argtypes = [f32p, f32p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int, C.c_int, f32p,
                             C.POINTER(C.c_int)]
    return L


def ref_filter(L, img, disp, r, sigma, it, weight, nI):
    H, W = disp.shape
    out = np.empty((H, W), np.float32)
    n = C.c_int(0)
    assert L.ref_wmf32f(img, np.ascontiguousarray(disp, np.float32), W, H, r, sigma, nI, it, O.WEIGHTS[weight], out,
                        C.byref(n)) == 0
    assert n.value <= 256
    assert np.array_equal(out, np.rint(out)), "the CV_32F path returned a value that is not one of the map's"
    return out


def main():
    if not os.path.exists(os.path.join(REF, "include", "JointWMF.h")) or not R.available():
        raise SystemExit(f"{REF}: needs a PRiMEStereoMatch checkout (set REF) and `make -C oracle ref`")
    out = {"wta": [], "wmf": {"inputs": "posterised (0xE0, 0xE0, 0xC0) Cones / Teddy; maps wide_oracle.widen(D = 64 WTA map, "
                                        "seed 7 left / 8 right), max_disp 512", "max_disp": WIDE_MAX_DISP, "settings": []},
           "loop": []}
    for D, W, H, seed in WTA_CASES:
        vol, _ = argmin_volume(W, H, D, seed)
        mine = O.wta(vol, np.uint16)
        ref8 = R.wta(vol)
        assert np.array_equal((mine & 0xFF).astype(np.uint8), ref8), f"D={D}: low byte differs from DispSel"
        out["wta"].append({"D": D, "W": W, "H": H, "seed": seed, "ref_sha": sha(ref8), "sha16": sha(mine),
                           "above_255": int((mine > 255).sum())})
        print("wta", D, "above 255:", int((mine > 255).sum()), flush=True)
    inputs = {}
    for name in ("Cones", "Teddy"):
        s = name.lower()
        l8 = read_png(os.path.join(HERE, f"{s}_im2.png"))
        r8 = read_png(os.path.join(HERE, f"{s}_im6.png"))
        res = O.pipeline(O.u8_to_f32(l8), O.u8_to_f32(r8), 64, threads=8)
        inputs[name] = {"l": (O.u8_to_f32(posterise(l8)), res["lDis"], widen(res["lDis"], 7)),
                        "r": (O.u8_to_f32(posterise(r8)), res["rDis"], widen(res["rDis"], 8))}
    with open(os.path.join(HERE, "golden_pp.json")) as f:
        gpp = {e["key"]: e for e in json.load(f)["settings"]}
    with tempfile.TemporaryDirectory() as tmp:
        L = ref_lib(tmp)
        for (r, sigma, it, weight) in SETTINGS:
            ent = {"key": key(r, sigma, it, weight), "radius": r, "sigma": float(sigma).hex(), "iterations": it,
                   "weight": weight, "scenes": {}}
            for name, views in inputs.items():
                ent["scenes"][name] = {}
                for view, (img, _, wide) in views.items():
                    want = ref_filter(L, img, wide, r, sigma, it, weight, WIDE_MAX_DISP).astype(np.uint16)
                    got = O.post_process(img, wide, r, sigma, it, weight)
                    ent["scenes"][name][view] = {"sha": sha(got), "ref_sha": sha(want), "differ": int((got != want).sum()),
                                                 "max": int(got.max())}
            print(ent["key"], {k: [v["differ"] for v in s.values()] for k, s in ent["scenes"].items()}, flush=True)
            out["wmf"]["settings"].append(ent)
        for k in LOOP_KEYS:
            g = gpp[k]
            r, sigma, it, weight = g["radius"], float.fromhex(g["sigma"]), g["iterations"], g["weight"]
            ent = {"key": k, "scenes": {}}
            for name, views in inputs.items():
                ent["scenes"][name] = {}
                for view, (img, d8, _) in views.items():
                    f32 = ref_filter(L, img, d8, r, sigma, it, weight, 256).astype(np.uint8)
                    ent["scenes"][name][view] = {"ref32f_sha": sha(f32), "ref8u_sha": g["scenes"][name][view]["ref_sha"]}
                    assert sha(f32) == g["scenes"][name][view]["ref_sha"], f"{k} {name} {view}: CV_32F path != CV_8U path"
            out["loop"].append(ent)
            print("loop", k, "CV_32F == CV_8U", flush=True)
    with open(os.path.join(HERE, "golden_wide.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote golden_wide.json")


if __name__ == "__main__":
    main()
