"""Cost and quality of the one-view disparity check (psm_set_disparity_check) on one GPU; prints one JSON line.

Maps: the winner-take-all maps of the synthetic 1920 x 1080 stereo pair of bench.py (both views, PSM_OPT_COSTS on), at
D = 128 on a u8 context and at D = 256 on a u16 context.  Stage configurations, timed in alternating rounds:
PSM_DCHECK_ONLY (the new kernel alone, so its stage-5 time is its own), the default post-filter alone, and
PSM_DCHECK_FIRST + the default post-filter, at max_diff 1 (StereoSGBM's disp12MaxDiff in the reference's matcher).  Per
configuration and round: ms per call of psm_post_process_device (CUDA events around `steps` calls on the context's
stream) and the median stage-5 time (psm_stage_ms); the medians over the rounds are reported.  Frames, timed the same
way (psm_cost_const, psm_cost_filter, psm_disp_select_device, psm_post_process_device per frame, no host copies): a
left-only frame with check + fill + the default post-filter against a two-view frame with the left-right check + fill +
the default post-filter.  Parity, in the first round: the whole PSM_DCHECK_ONLY maps against tests/dcheck_oracle.py on
the context's own selection maps and costs.

Quality, from the GPU's D = 64 maps of Cones and Teddy at the default matching cost: the %BP of
bench_gif_window.bad_pixels_nonocc of the left map after the one-view check alone (checked pixels are 0), check + fill
and check + fill + the default post-filter on a left-only context, next to the two-view left-right check + fill and
check + fill + post-filter.

Usage: python bench_disp_check.py [--steps 20] [--warmup 3] [--no-quality]
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

WORKLOADS = [(128, 8), (256, 16)]        # (D, map bits)
MAX_DIFF = 1
ROUNDS = 3


def timed(stream, call, steps, warmup, stage=None):
    """-> (ms per call, median stage-5 ms of `stage`'s context or None)"""
    import torch
    for _ in range(warmup):
        call()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(stream)
    for _ in range(steps):
        call()
    ev1.record(stream)
    torch.cuda.synchronize()
    kms = None
    if stage is not None:
        kms = []
        for _ in range(steps):   # psm_stage_ms waits for each call
            call()
            kms.append(stage.stage_ms(5))
        kms = float(np.median(kms))
    return ev0.elapsed_time(ev1) / steps, kms


def summarise(res):
    for k in [k for k in ("ms_per_call", "stage5_ms") if k in res]:
        res[k + "_median"] = round(float(np.median(res[k])), 4)
        res[k] = [round(x, 4) for x in res[k]]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-quality", action="store_true")
    args = ap.parse_args()
    import torch
    from bench import device_info
    from bench_gif_window import bad_pixels_nonocc, read_png
    from bench_lr_check import gpu_clocks
    from primestereomatch_b200 import DispEst, capi, synth
    from oracle import oracle as O
    import dcheck_oracle as DC
    if not torch.cuda.is_available() or capi.lib().psm_device_count() < 1:
        raise SystemExit("bench_disp_check.py needs a CUDA device")
    W, H = 1920, 1080
    L = capi.lib()
    stages = {"only": (capi.PSM_DCHECK_ONLY, capi.PSM_LR_OFF), "post-filter": (capi.PSM_DCHECK_OFF, capi.PSM_LR_OFF),
              "first + post-filter": (capi.PSM_DCHECK_FIRST, capi.PSM_LR_OFF)}
    frames = {"two views, lr check + fill + post-filter": ("both", capi.PSM_DCHECK_OFF),
              "left only, check + fill + post-filter": ("left", capi.PSM_DCHECK_FIRST)}
    results, parity = [], True
    for D, bits in WORKLOADS:
        l8, r8, _ = synth.stereo_pair_u8(W, H, D)
        l, r = synth.to_f32(l8), synth.to_f32(r8)
        per = {name: {"config": name, "ms_per_call": [], "stage5_ms": []} for name in stages}
        fper = {name: {"frame": name, "ms_per_call": []} for name in frames}
        ctxs = {}
        for views in ("both", "left"):
            de = ctxs[views] = DispEst(l, r, D, map_bits=bits)
            de.stream = torch.cuda.Stream()   # the context runs on this stream, so the events bracket the calls
            capi.check(L.psm_set_stream(de.handle, C.c_void_p(de.stream.cuda_stream)), de.handle)
            if views == "left":
                de.setViews("left")
            de.setCostOutput(True)
            de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        de = ctxs["both"]
        ld, rd, lc, rc = de.lDisMap.copy(), de.rDisMap.copy(), de.lCosts[1].copy(), de.rCosts[1].copy()
        want = DC.check(ld, lc, D, MAX_DIFF), DC.check(rd, rc, D, MAX_DIFF, view=1)
        removed = [round(100.0 * np.count_nonzero(w != m) / m.size, 3) for w, m in zip(want, (ld, rd))]
        post = lambda c: capi.check(L.psm_post_process_device(c.handle), c.handle)   # noqa: E731

        def frame(c):
            for f in (L.psm_cost_const, L.psm_cost_filter, L.psm_disp_select_device, L.psm_post_process_device):
                capi.check(f(c.handle), c.handle)
        for rnd in range(ROUNDS):
            for name, (mode, lr) in stages.items():
                de.setDisparityCheck(mode, MAX_DIFF); de.setLRCheck(lr)
                ms, k = timed(de.stream, lambda: post(de), args.steps, args.warmup, de)
                per[name]["ms_per_call"].append(ms)
                per[name]["stage5_ms"].append(k)
                if rnd == 0 and mode == capi.PSM_DCHECK_ONLY:
                    de.PostProcess_GPU()
                    parity = parity and bool(np.array_equal(de.lDisMap, want[0]) and np.array_equal(de.rDisMap, want[1]))
                print(json.dumps({"progress": {"D": D, "config": name, "ms_per_call": ms, "stage5_ms": k}}),
                      file=sys.stderr, flush=True)
            for name, (views, mode) in frames.items():
                c = ctxs[views]
                c.setDisparityCheck(mode, MAX_DIFF); c.setLRCheck(capi.PSM_LR_FILL_WMF)
                ms, _ = timed(c.stream, lambda: frame(c), max(1, args.steps // 2), 1)
                fper[name]["ms_per_call"].append(ms)
                print(json.dumps({"progress": {"D": D, "frame": name, "ms_per_call": ms}}), file=sys.stderr, flush=True)
        for c in ctxs.values():
            c.close()
        results.append({"D": D, "map_bits": bits, "max_diff": MAX_DIFF, "checked_pct": removed,
                        "stages": [summarise(x) for x in per.values()], "frames": [summarise(x) for x in fper.values()]})
    quality = None
    if not args.no_quality:
        quality = {}
        g = os.path.join(ROOT, "tests", "golden")
        for scene in ("Cones", "Teddy"):
            s = scene.lower()
            ls = O.u8_to_f32(read_png(os.path.join(g, f"{s}_im2.png")))
            rs = O.u8_to_f32(read_png(os.path.join(g, f"{s}_im6.png")))
            gt, occl = read_png(os.path.join(g, f"{s}_disp2.png"), True), read_png(os.path.join(g, f"{s}_occl.png"), True)
            q = quality[scene] = {}
            for views, rows in (("both", ((capi.PSM_DCHECK_OFF, capi.PSM_LR_FILL, "two views: lr check + fill"),
                                          (capi.PSM_DCHECK_OFF, capi.PSM_LR_FILL_WMF, "two views: lr check + fill + r9"))),
                                ("left", ((capi.PSM_DCHECK_ONLY, capi.PSM_LR_OFF, "left only: check"),
                                          (capi.PSM_DCHECK_FIRST, capi.PSM_LR_FILL, "left only: check + fill"),
                                          (capi.PSM_DCHECK_FIRST, capi.PSM_LR_FILL_WMF, "left only: check + fill + r9")))):
                with DispEst(ls, rs, 64) as de:
                    if views == "left":
                        de.setViews("left")
                    de.setCostOutput(True)
                    de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
                    if views == "both":
                        q["WTA"] = round(bad_pixels_nonocc(de.lDisMap, gt, occl), 3)
                    for mode, lr, name in rows:
                        de.setDisparityCheck(mode, MAX_DIFF); de.setLRCheck(lr); de.PostProcess_GPU()
                        q[name] = round(bad_pixels_nonocc(de.lDisMap, gt, occl), 3)
    gpu = device_info(0)
    gpu.update(gpu_clocks())
    line = {"workload": "disp_check_1920x1080_wta", "gpu": gpu, "steps": args.steps, "warmup": args.warmup,
            "rounds": ROUNDS, "parity": parity, "workloads": results, "bp_nonocc_D64_left_max_diff_1": quality}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
