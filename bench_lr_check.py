"""Cost and quality of the left-right check and occlusion fill (psm_set_lr_check) on one GPU; prints one JSON line.

Maps: the winner-take-all maps of the synthetic 1920 x 1080 stereo pair of bench.py (both views), at D = 128 on a u8
context and at D = 256 on a u16 context (psm_create_u16), computed once per context.  Modes 0 (post-filter alone, the
default), 1 (check + fill + post-filter) and 2 (check + fill alone: exactly one launch of the new kernel, so its stage-5
time is the kernel's time) at the default post-filter, timed in two alternating rounds.  Per mode and round: ms per call
of psm_post_process_device (CUDA events around `steps` calls on the context's stream) and the median stage-5 time
(psm_stage_ms); the medians over the rounds are reported, and for mode 2 the achieved bandwidth of the algorithmic
traffic (both maps read, both filled maps and both masks written: 6 bytes per pixel on u8 maps, 10 on u16).  In the
first round the top 64 rows of both output maps are checked against the CPU restatement (tests/lr_oracle.py, whose fill
is row-local, then oracle.post_process on rows [0, 64 + 9)).  Quality: %BP (non-occluded, left map; the metric of
bench_gif_window.py) of Cones and Teddy at D = 64 from the GPU maps, at the default matching cost and at
(0.11, 0.21, 0.008): no post-processing, check/fill, post-filter, check/fill + post-filter, with the post-filter at the
default and at radius 16.

Usage: python bench_lr_check.py [--steps 20] [--warmup 3] [--no-quality]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

INF = float("inf")
WORKLOADS = [(128, 8), (256, 16)]        # (D, map bits)
MODES = (0, 1, 2)
COSTS = [(0.9, INF, INF), (0.11, 0.21, 0.008)]
FILTERS = [(9, 25.5, 1, "exp"), (16, 25.5, 1, "exp")]
ROUNDS = 2
BAND = 64


def gpu_clocks():
    """power limit and SM clocks as nvidia-smi shows them (None where it does not)"""
    fields = ("power.limit", "clocks.sm", "clocks.max.sm")
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=" + ",".join(fields), "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        return {k: float(v) for k, v in zip(("power_limit_w", "sm_clock_mhz", "max_sm_clock_mhz"), q)}
    except (OSError, ValueError, subprocess.SubprocessError):
        return {"power_limit_w": None, "sm_clock_mhz": None, "max_sm_clock_mhz": None}


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
    import lr_oracle as LR
    if not torch.cuda.is_available() or capi.lib().psm_device_count() < 1:
        raise SystemExit("bench_lr_check.py needs a CUDA device")
    W, H = 1920, 1080
    L = capi.lib()
    results = []
    for D, bits in WORKLOADS:
        l8, r8, _ = synth.stereo_pair_u8(W, H, D)
        l, r = synth.to_f32(l8), synth.to_f32(r8)
        per_mode = {m: {"mode": m, "ms_per_call": [], "stage5_ms": [], "band_parity": None} for m in MODES}
        with DispEst(l, r, D, map_bits=bits) as de:
            stream = torch.cuda.Stream()   # the context runs on this stream, so the events below bracket the calls
            capi.check(L.psm_set_stream(de.handle, C.c_void_p(stream.cuda_stream)), de.handle)
            de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
            ld, rd = de.lDisMap.copy(), de.rDisMap.copy()
            for _ in range(ROUNDS):
                for m in MODES:
                    res = per_mode[m]
                    de.setLRCheck(m)
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
                    res["ms_per_call"].append(ev0.elapsed_time(ev1) / args.steps)
                    kms = []
                    for _ in range(args.steps):   # psm_stage_ms waits for each call
                        call()
                        kms.append(de.stage_ms(5))
                    res["stage5_ms"].append(float(np.median(kms)))
                    if res["band_parity"] is None:
                        de.PostProcess_GPU()
                        rows = BAND + 9
                        ok = True
                        for img, dmap, got, v in ((l, ld, de.lDisMap, 0), (r, rd, de.rDisMap, 1)):
                            want = LR.lr_check_fill(ld[:rows], rd[:rows])[2 + v] if m else dmap[:rows]
                            if m != 2:
                                want = O.post_process(img[:rows], want)
                            ok = ok and bool(np.array_equal(got[:BAND], want[:BAND]))
                        res["band_parity"] = ok
                    print(json.dumps({"progress": {"D": D, "mode": m, "ms_per_call": res["ms_per_call"][-1],
                                                   "stage5_ms": res["stage5_ms"][-1]}}), file=sys.stderr, flush=True)
        for res in per_mode.values():
            res["ms_per_call_median"] = round(float(np.median(res["ms_per_call"])), 4)
            res["stage5_ms_median"] = round(float(np.median(res["stage5_ms"])), 4)
            res["ms_per_call"] = [round(x, 4) for x in res["ms_per_call"]]
            res["stage5_ms"] = [round(x, 4) for x in res["stage5_ms"]]
        bytes_per_px = 6 if bits == 8 else 10
        kern = per_mode[2]["stage5_ms_median"]
        results.append({"D": D, "map_bits": bits, "modes": list(per_mode.values()),
                        "lr_kernel_ms": kern, "lr_kernel_bytes": bytes_per_px * W * H,
                        "lr_kernel_gbs": round(bytes_per_px * W * H / (kern * 1e-3) / 1e9, 1) if kern > 0 else None})
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
                q = qc[scene] = {}
                with DispEst(ls, rs, 64) as de:
                    de.setMatchingCost(*cost)
                    de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
                    q["WTA"] = round(bad_pixels_nonocc(de.lDisMap, gt, occl), 3)
                    de.setLRCheck(2); de.PostProcess_GPU()
                    q["WTA + check/fill"] = round(bad_pixels_nonocc(de.lDisMap, gt, occl), 3)
                    for pf in FILTERS:
                        de.setPostFilter(*pf)
                        for m, name in ((0, "post-filter"), (1, "check/fill + post-filter")):
                            de.setLRCheck(m); de.PostProcess_GPU()
                            q[f"WTA + {name} {pf}"] = round(bad_pixels_nonocc(de.lDisMap, gt, occl), 3)
    gpu = device_info(0)
    gpu.update(gpu_clocks())
    line = {"workload": "lr_check_1920x1080_wta", "gpu": gpu, "steps": args.steps, "warmup": args.warmup,
            "rounds": ROUNDS, "workloads": results, "bp_nonocc_left_D64": quality}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
