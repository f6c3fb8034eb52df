"""Wide disparity ranges (psm_create_u16) on one GPU; prints one JSON line.

Workload: the synthetic 1920 x 1080 stereo pair of bench.py (synth.stereo_pair_u8) at
  D = 256 on a u8 context and on a u16 context (the like-for-like comparison of the two map formats),
  D = 512 and D = 1024 on a u16 context (D = 1024 is skipped, and the line says so, when cudaMemGetInfo shows less free
  memory than its four volumes need).
Per configuration: `steps` timed frames after `warmup` (ingest -> CVC -> CVF -> WTA -> post-filter at the default), CUDA
events around the whole loop on the context's stream -> ms per frame and frames per second; the median stage times
(psm_stage_ms) of CVC, CVF, WTA and the post-filter at the default (radius 9) and at radius 16.
Parity: before the line is printed, rows [0, 16) of both maps of every configuration are compared with the CPU oracle
(oracle/ CVC + guided filter, tests/wide_oracle.c arg-min) run on rows [0, 32): the filtered costs of those rows depend on
rows < 25 only.

Usage: python bench_wide_disparity.py [--steps 10] [--warmup 2]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

W, H = 1920, 1080
CONFIGS = [(256, 8), (256, 16), (512, 16), (1024, 16)]
BAND, CROP = 16, 32


def volume_bytes(D):
    wp = (W + 32 + 12 + 31) // 32 * 32   # a bound on the padded row pitch (kPadLeft + kPadRight, 128-byte rows)
    return 4 * (wp * H * D + 64) * 4     # four float volumes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    from bench import device_info
    from primestereomatch_b200 import DispEst, capi, synth
    from oracle import oracle as O
    import wide_oracle as WO
    if not torch.cuda.is_available() or capi.lib().psm_device_count() < 1:
        raise SystemExit("bench_wide_disparity.py needs a CUDA device")
    L = capi.lib()
    pairs, results = {}, []
    for D, bits in CONFIGS:
        res = {"D": D, "map_bits": bits, "skipped": None}
        free, _ = torch.cuda.mem_get_info()
        if volume_bytes(D) * 1.1 > free:
            res["skipped"] = f"needs about {volume_bytes(D) / 2**30:.1f} GiB for its volumes, {free / 2**30:.1f} GiB free"
            results.append(res)
            continue
        if D not in pairs:
            l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=W * 1000003 + H * 1009 + D)
            pairs[D] = (synth.to_f32(l8), synth.to_f32(r8))
        l, r = pairs[D]
        with DispEst(l, r, D, map_bits=bits) as de:
            stream = torch.cuda.Stream()
            capi.check(L.psm_set_stream(de.handle, C.c_void_p(stream.cuda_stream)), de.handle)

            def frame():
                de.CostConst_GPU(); de.CostFilter_GPU()
                capi.check(L.psm_disp_select_device(de.handle), de.handle)
                capi.check(L.psm_post_process_device(de.handle), de.handle)

            for _ in range(args.warmup):
                frame()
            torch.cuda.synchronize()
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record(stream)
            for _ in range(args.steps):
                frame()
            ev1.record(stream)
            torch.cuda.synchronize()
            ms = ev0.elapsed_time(ev1) / args.steps
            st = {k: [] for k in ("cvc", "cvf", "wta", "pp_r9")}
            for _ in range(args.steps):
                frame()
                for k, s in (("cvc", 1), ("cvf", 2), ("wta", 3), ("pp_r9", 5)):
                    st[k].append(de.stage_ms(s))
            de.setPostFilter(16)
            st["pp_r16"] = []
            for _ in range(args.steps):
                capi.check(L.psm_post_process_device(de.handle), de.handle)
                st["pp_r16"].append(de.stage_ms(5))
            de.setPostFilter(9)
            res.update({"ms_per_frame": round(ms, 3), "fps": round(1000.0 / ms, 2), "launches_per_frame": None,
                        "stage_ms": {k: round(float(np.median(v)), 4) for k, v in st.items()}})
            n0 = de.launch_count(); frame(); res["launches_per_frame"] = de.launch_count() - n0
            de.DispSelect_GPU()
            ld, rd = de.lDisMap[:BAND].astype(np.uint16), de.rDisMap[:BAND].astype(np.uint16)
            res["max_disparity_in_map"] = int(max(de.lDisMap.max(), de.rDisMap.max()))
        lc, rc = np.ascontiguousarray(l[:CROP]), np.ascontiguousarray(r[:CROP])
        _, _, lraw, rraw = O.cost_const(lc, rc, D)
        lf, rf = O.cost_filter(lc, rc, lraw, rraw)
        del lraw, rraw
        res["band_parity"] = bool(np.array_equal(ld, WO.wta16(lf)[:BAND]) and np.array_equal(rd, WO.wta16(rf)[:BAND]))
        del lf, rf
        results.append(res)
        print(json.dumps({"progress": res}), file=sys.stderr, flush=True)
    if not all(r["band_parity"] for r in results if not r["skipped"]):
        raise SystemExit("band parity failed: " + json.dumps(results))
    gpu = device_info(0)
    line = {"workload": "wide_disparity_1920x1080", "gpu": gpu, "steps": args.steps, "warmup": args.warmup,
            "configs": results}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
