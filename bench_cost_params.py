"""Cost of the matching-cost setting (psm_set_matching_cost) on one GPU; prints one JSON line.

Frame: the synthetic 1920 x 1080 x 128 stereo pair of bench.py (both views), device-resident inputs.  Configurations:
(0.9, inf, inf) is the default and runs the tuned cost-volume kernel; (0.9, 1e30, 1e30) runs the parameterised kernel on
the same values, the like-for-like comparison of the two; (0.11, 0.21, 0.008) and (0.5, inf, inf) are other settings.
Each configuration is timed in two alternating rounds.  Per configuration and round: ms per frame (set images -> CVC ->
CVF -> WTA, CUDA events) and the median CVC stage time (psm_stage_ms stage 1), plus the raw volumes of a top row band
against the CPU restatement tests/cost_oracle.py.  Quality: %BP (non-occluded, left map) of Cones and Teddy at D = 64 for
a small grid of settings, from the GPU maps (the metric of bench_gif_window.py).

Usage: python bench_cost_params.py [--steps 20] [--warmup 3] [--no-quality]
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

INF = float("inf")
CONFIGS = [(0.9, INF, INF), (0.9, 1e30, 1e30), (0.11, 0.21, 0.008), (0.5, INF, INF)]
QUALITY_GRID = [(0.9, INF, INF), (0.9, 0.028, 0.008), (0.9, 0.084, 0.008), (0.9, 0.3, 0.03), (0.5, INF, INF),
                (0.11, 0.21, 0.008), (0.0, INF, INF), (1.0, INF, INF)]
ROUNDS = 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-quality", action="store_true")
    args = ap.parse_args()
    import torch
    from bench import device_info
    from bench_gif_window import bad_pixels_nonocc, read_png
    from primestereomatch_b200 import DispEst, capi, synth
    from oracle import oracle as O
    import cost_oracle as CO
    if not torch.cuda.is_available() or capi.lib().psm_device_count() < 1:
        raise SystemExit("bench_cost_params.py needs a CUDA device")
    W, H, D = 1920, 1080, 128
    l8, r8, _ = synth.stereo_pair_u8(W, H, D)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    ld_dev, rd_dev = torch.from_numpy(l).cuda(), torch.from_numpy(r).cuda()
    step = W * 3 * 4
    L = capi.lib()
    band, band_ds = 24, (0, 1, 64, 127)
    num = lambda v: "inf" if v == INF else v   # noqa: E731  (strict JSON has no Infinity)
    results = {str(c): {"alpha": c[0], "tau_color": num(c[1]), "tau_grad": num(c[2]),
                        "kernel": "tuned" if c == CONFIGS[0] else "parameterised",
                        "ms_per_frame": [], "cvc_ms": [], "band_parity": True} for c in CONFIGS}
    for _ in range(ROUNDS):
        for cost in CONFIGS:
            res = results[str(cost)]
            with DispEst(l, r, D) as de:
                de.setMatchingCost(*cost)
                stream = torch.cuda.Stream()   # the context runs on this stream, so the events below bracket the frames
                capi.check(L.psm_set_stream(de.handle, C.c_void_p(stream.cuda_stream)), de.handle)

                def frame():
                    capi.check(L.psm_set_images_device(de.handle, ld_dev.data_ptr(), step, rd_dev.data_ptr(), step), de.handle)
                    capi.check(L.psm_cost_const(de.handle), de.handle)
                    capi.check(L.psm_cost_filter(de.handle), de.handle)
                    capi.check(L.psm_disp_select_device(de.handle), de.handle)

                for _ in range(args.warmup):
                    frame()
                torch.cuda.synchronize()
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ev0.record(stream)
                for _ in range(args.steps):
                    frame()
                ev1.record(stream)
                torch.cuda.synchronize()
                res["ms_per_frame"].append(round(ev0.elapsed_time(ev1) / args.steps, 3))
                kms = []
                for _ in range(args.steps):   # stage 1 = CVC alone (psm_stage_ms waits for each frame)
                    frame()
                    kms.append(de.stage_ms(1))
                res["cvc_ms"].append(round(float(np.median(kms)), 4))
                if len(res["cvc_ms"]) == 1:   # raw volumes of the top row band against the CPU restatement
                    de.CostConst_GPU()
                    lv, rv = CO.cost_volumes(l[:band], r[:band], D, *cost)
                    for d in band_ds:
                        ok = (np.array_equal(de.read_cost_slice(0, d)[:band], lv[d])
                              and np.array_equal(de.read_cost_slice(1, d)[:band], rv[d]))
                        res["band_parity"] = res["band_parity"] and bool(ok)
            print(json.dumps({"progress": {"cost": str(cost), "ms_per_frame": res["ms_per_frame"][-1],
                                           "cvc_ms": res["cvc_ms"][-1]}}), file=sys.stderr, flush=True)
    quality = None
    if not args.no_quality:
        quality = {}
        g = os.path.join(ROOT, "tests", "golden")
        for scene in ("Cones", "Teddy"):
            s = scene.lower()
            ls, rs = O.u8_to_f32(read_png(os.path.join(g, f"{s}_im2.png"))), O.u8_to_f32(read_png(os.path.join(g, f"{s}_im6.png")))
            gt, occl = read_png(os.path.join(g, f"{s}_disp2.png"), True), read_png(os.path.join(g, f"{s}_occl.png"), True)
            quality[scene] = {}
            for cost in QUALITY_GRID:
                with DispEst(ls, rs, 64) as de:
                    de.setMatchingCost(*cost)
                    de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
                    quality[scene][str(cost)] = round(bad_pixels_nonocc(de.lDisMap, gt, occl), 3)
    gpu = device_info(0)
    try:   # SM clock right after the timed work and the card's maximum: part of every absolute number above
        import subprocess
        q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        gpu["sm_clock_mhz"], gpu["max_sm_clock_mhz"] = float(q[0]), float(q[1])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        gpu["sm_clock_mhz"] = gpu["max_sm_clock_mhz"] = None
    line = {"workload": "matching_cost_C4_1920x1080x128", "gpu": gpu, "steps": args.steps, "warmup": args.warmup,
            "rounds": ROUNDS, "configs": list(results.values()), "bp_nonocc_left_D64": quality}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
