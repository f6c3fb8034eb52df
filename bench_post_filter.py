"""Cost of the post-filter setting (psm_set_post_filter) on one GPU; prints one JSON line.

Maps: the winner-take-all maps of the synthetic 1920 x 1080 x 128 stereo pair of bench.py (both views), computed once.
Configurations: (9, 25.5, 1, exp) is the default and runs the tuned kernel pair (the first H100 figure for this stage);
(9, nextafterf(25.5, inf), 1, exp) runs the generic-radius kernel on the same filter, the like-for-like comparison of the
two; radius 16 and 32, iv2 and 3 iterations are other settings.  Each configuration is timed in two alternating rounds.
Per configuration and round: ms per call of psm_post_process_device (CUDA events around `steps` calls on the context's
stream) and the median stage-5 time (psm_stage_ms, all passes of both views); in the first round the top 64 rows of both
filtered maps are checked against the CPU restatement tests/pp_oracle.c run on rows [0, 64 + iterations * radius)
(exact: the clipped windows of those rows lie inside).  Quality: %BP (non-occluded, left map) of Cones and Teddy at
D = 64 after post-processing, for a small grid of filter settings at the default matching cost and at
(0.11, 0.21, 0.008), the metric of bench_gif_window.py.

Usage: python bench_post_filter.py [--steps 20] [--warmup 3] [--no-quality]
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
SIGMA_NEXT = float(np.nextafter(np.float32(25.5), np.float32(np.inf)))
CONFIGS = [(9, 25.5, 1, "exp"), (9, SIGMA_NEXT, 1, "exp"), (16, 25.5, 1, "exp"), (32, 25.5, 1, "exp"),
           (9, 25.5, 1, "iv2"), (9, 25.5, 3, "exp")]
QUALITY_GRID = [None, (9, 25.5, 1, "exp"), (4, 25.5, 1, "exp"), (16, 25.5, 1, "exp"), (32, 25.5, 1, "exp"),
                (9, 10.0, 1, "exp"), (9, 80.0, 1, "exp"), (16, 10.0, 1, "exp"), (9, 25.5, 3, "exp"),
                (9, 25.5, 1, "iv1"), (9, 25.5, 1, "iv2"), (9, 25.5, 1, "off")]
COSTS = [(0.9, INF, INF), (0.11, 0.21, 0.008)]
ROUNDS = 2
BAND = 64


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
    import pp_oracle as P
    if not torch.cuda.is_available() or capi.lib().psm_device_count() < 1:
        raise SystemExit("bench_post_filter.py needs a CUDA device")
    W, H, D = 1920, 1080, 128
    l8, r8, _ = synth.stereo_pair_u8(W, H, D)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    L = capi.lib()
    results = {str(c): {"radius": c[0], "sigma": c[1], "iterations": c[2], "weight": c[3],
                        "kernel": "tuned" if c[:2] == (9, 25.5) and c[3] == "exp" else "generic",
                        "ms_per_call": [], "stage5_ms": [], "band_parity": None} for c in CONFIGS}
    with DispEst(l, r, D) as de:
        stream = torch.cuda.Stream()   # the context runs on this stream, so the events below bracket the calls
        capi.check(L.psm_set_stream(de.handle, C.c_void_p(stream.cuda_stream)), de.handle)
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        ld, rd = de.lDisMap.copy(), de.rDisMap.copy()
        for _ in range(ROUNDS):
            for cfg in CONFIGS:
                res = results[str(cfg)]
                de.setPostFilter(*cfg)
                call = lambda: capi.check(L.psm_post_process_device(de.handle), de.handle)   # noqa: E731
                for _ in range(args.warmup):
                    call()
                torch.cuda.synchronize()
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ev0.record(stream)
                for _ in range(args.steps):
                    call()
                ev1.record(stream)
                torch.cuda.synchronize()
                res["ms_per_call"].append(round(ev0.elapsed_time(ev1) / args.steps, 3))
                kms = []
                for _ in range(args.steps):   # psm_stage_ms waits for each call
                    call()
                    kms.append(de.stage_ms(5))
                res["stage5_ms"].append(round(float(np.median(kms)), 4))
                if res["band_parity"] is None:
                    de.PostProcess_GPU()
                    rows = BAND + cfg[2] * cfg[0]
                    ok = True
                    for img, dmap, got in ((l, ld, de.lDisMap), (r, rd, de.rDisMap)):
                        want = P.post_process(img[:rows], dmap[:rows], *cfg)[:BAND]
                        ok = ok and bool(np.array_equal(got[:BAND], want))
                    res["band_parity"] = ok
                print(json.dumps({"progress": {"cfg": str(cfg), "ms_per_call": res["ms_per_call"][-1],
                                               "stage5_ms": res["stage5_ms"][-1]}}), file=sys.stderr, flush=True)
    quality = None
    if not args.no_quality:
        quality = {}
        g = os.path.join(ROOT, "tests", "golden")
        for cost in COSTS:
            qc = quality[str(cost)] = {}
            for scene in ("Cones", "Teddy"):
                s = scene.lower()
                ls = O.u8_to_f32(read_png(os.path.join(g, f"{s}_im2.png")))
                rs = O.u8_to_f32(read_png(os.path.join(g, f"{s}_im6.png")))
                gt, occl = read_png(os.path.join(g, f"{s}_disp2.png"), True), read_png(os.path.join(g, f"{s}_occl.png"), True)
                qc[scene] = {}
                with DispEst(ls, rs, 64) as de:
                    de.setMatchingCost(*cost)
                    de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
                    for pf in QUALITY_GRID:
                        if pf is None:
                            de.DispSelect_GPU()
                        else:
                            de.setPostFilter(*pf)
                            de.PostProcess_GPU()
                        qc[scene]["no post-filter" if pf is None else str(pf)] = round(bad_pixels_nonocc(de.lDisMap, gt, occl), 3)
    gpu = device_info(0)
    try:   # SM clock right after the timed work and the card's maximum: part of every absolute number above
        import subprocess
        q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        gpu["sm_clock_mhz"], gpu["max_sm_clock_mhz"] = float(q[0]), float(q[1])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        gpu["sm_clock_mhz"] = gpu["max_sm_clock_mhz"] = None
    line = {"workload": "post_filter_1920x1080_wta_D128", "gpu": gpu, "steps": args.steps, "warmup": args.warmup,
            "rounds": ROUNDS, "configs": list(results.values()), "bp_nonocc_left_D64": quality}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
