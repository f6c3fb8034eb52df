"""Cost and quality of speckle removal (psm_set_speckle_filter) on one GPU; prints one JSON line.

Maps: the winner-take-all maps of the synthetic 1920 x 1080 stereo pair of bench.py (both views), at D = 128 on a u8
context and at D = 256 on a u16 context, computed once per context; and two adversarial u8 maps injected through
one-hot cost slices: a constant map (one map-wide blob per view) and a checkerboard at max_diff = 0 (one blob per
pixel).  Configurations, timed in alternating rounds: PSM_SPECKLE_ONLY (the four new kernels alone, so its stage-5 time
is theirs), the default post-filter alone, and PSM_SPECKLE_FIRST + the default post-filter, at (max_size, max_diff) =
(400, 2).  Per configuration and round: ms per call of psm_post_process_device (CUDA events around `steps` calls on the
context's stream) and the median stage-5 time (psm_stage_ms); the medians over the rounds are reported.  Parity, in the
first round: the whole PSM_SPECKLE_ONLY maps against tests/speckle_oracle.py, and the top 64 rows of the FIRST +
post-filter maps against the oracle's post-filter of rows [0, 64 + 9) of the oracle's speckle-filtered maps.

Quality, from the GPU's D = 64 left maps of Cones and Teddy at the default matching cost: over the non-occluded pixels
from column 65 on (the region bench_gif_window.bad_pixels_nonocc scores), the share kept (map value not 0) and the
share of kept pixels that are bad (|min(4 m, 255) - gt| > 4), without speckle removal and at (50, 1), (100, 1) and
(400, 2); then the %BP of bad_pixels_nonocc after check + fill and after check + fill + the default post-filter, without
and with PSM_SPECKLE_FIRST at (400, 2).

Usage: python bench_speckle.py [--steps 20] [--warmup 3] [--no-quality]
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
SETTING = (400, 2)
QUALITY_SETTINGS = [(50, 1), (100, 1), (400, 2)]
ROUNDS = 3
BAND = 64


def timed(de, stream, steps, warmup):
    """-> (ms per call of psm_post_process_device, median stage-5 ms)"""
    import torch
    from primestereomatch_b200 import capi
    L = capi.lib()
    call = lambda: capi.check(L.psm_post_process_device(de.handle), de.handle)   # noqa: E731
    for _ in range(warmup):
        call()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(stream)
    for _ in range(steps):
        call()
    ev1.record(stream)
    torch.cuda.synchronize()
    kms = []
    for _ in range(steps):   # psm_stage_ms waits for each call
        call()
        kms.append(de.stage_ms(5))
    return ev0.elapsed_time(ev1) / steps, float(np.median(kms))


def summarise(res):
    for k in ("ms_per_call", "stage5_ms"):
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
    import speckle_oracle as SP
    if not torch.cuda.is_available() or capi.lib().psm_device_count() < 1:
        raise SystemExit("bench_speckle.py needs a CUDA device")
    W, H = 1920, 1080
    L = capi.lib()
    configs = {"only": (capi.PSM_SPECKLE_ONLY, 0), "post-filter": (capi.PSM_SPECKLE_OFF, 0),
               "first + post-filter": (capi.PSM_SPECKLE_FIRST, 0)}
    results, parity = [], True
    for D, bits in WORKLOADS:
        l8, r8, _ = synth.stereo_pair_u8(W, H, D)
        l, r = synth.to_f32(l8), synth.to_f32(r8)
        per = {name: {"config": name, "ms_per_call": [], "stage5_ms": []} for name in configs}
        with DispEst(l, r, D, map_bits=bits) as de:
            stream = torch.cuda.Stream()   # the context runs on this stream, so the events bracket the calls
            capi.check(L.psm_set_stream(de.handle, C.c_void_p(stream.cuda_stream)), de.handle)
            de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
            ld, rd = de.lDisMap.copy(), de.rDisMap.copy()
            want = [SP.filter_speckles(m, *SETTING) for m in (ld, rd)]
            removed = [round(100.0 * np.count_nonzero(w != m) / m.size, 3) for w, m in zip(want, (ld, rd))]
            for rnd in range(ROUNDS):
                for name, (mode, lr) in configs.items():
                    de.setSpeckleFilter(mode, *SETTING); de.setLRCheck(lr)
                    ms, k = timed(de, stream, args.steps, args.warmup)
                    per[name]["ms_per_call"].append(ms)
                    per[name]["stage5_ms"].append(k)
                    if rnd == 0:
                        de.PostProcess_GPU()
                        if mode == capi.PSM_SPECKLE_ONLY:
                            ok = np.array_equal(de.lDisMap, want[0]) and np.array_equal(de.rDisMap, want[1])
                        elif mode == capi.PSM_SPECKLE_FIRST:
                            rows = BAND + 9
                            ok = all(np.array_equal(got[:BAND], O.post_process(img[:rows], w[:rows])[:BAND])
                                     for got, img, w in ((de.lDisMap, l, want[0]), (de.rDisMap, r, want[1])))
                        else:
                            ok = True
                        parity = parity and bool(ok)
                    print(json.dumps({"progress": {"D": D, "config": name, "ms_per_call": ms, "stage5_ms": k}}),
                          file=sys.stderr, flush=True)
        results.append({"D": D, "map_bits": bits, "setting": SETTING, "removed_pct": removed,
                        "configs": [summarise(x) for x in per.values()]})
    # adversarial maps: a map-wide blob and a blob per pixel, injected through one-hot cost slices
    const = np.full((H, W), 2, np.uint8)
    chk = (1 + (np.indices((H, W)).sum(0) % 2)).astype(np.uint8)
    adversarial = []
    l8, r8, _ = synth.stereo_pair_u8(W, H, 4)
    with DispEst(synth.to_f32(l8), synth.to_f32(r8), 3) as de:
        stream = torch.cuda.Stream()
        capi.check(L.psm_set_stream(de.handle, C.c_void_p(stream.cuda_stream)), de.handle)
        for name, m, setting in (("constant", const, (400, 2)), ("checkerboard", chk, (400, 0))):
            de.CostConst_GPU(); de.CostFilter_GPU()
            for d in range(3):
                s = (m != d).astype(np.float32)
                de.write_cost_slice(0, d, s); de.write_cost_slice(1, d, s)
            de.DispSelect_GPU()
            de.setSpeckleFilter(capi.PSM_SPECKLE_ONLY, *setting)
            res = {"map": name, "setting": setting, "ms_per_call": [], "stage5_ms": []}
            for _ in range(ROUNDS):
                ms, k = timed(de, stream, args.steps, args.warmup)
                res["ms_per_call"].append(ms); res["stage5_ms"].append(k)
            de.PostProcess_GPU()
            parity = parity and bool(np.array_equal(de.lDisMap, SP.filter_speckles(m, *setting)))
            adversarial.append(summarise(res))
    quality = None
    if not args.no_quality:
        quality = {}
        g = os.path.join(ROOT, "tests", "golden")
        for scene in ("Cones", "Teddy"):
            s = scene.lower()
            ls = O.u8_to_f32(read_png(os.path.join(g, f"{s}_im2.png")))
            rs = O.u8_to_f32(read_png(os.path.join(g, f"{s}_im6.png")))
            gt, occl = read_png(os.path.join(g, f"{s}_disp2.png"), True), read_png(os.path.join(g, f"{s}_occl.png"), True)
            region = occl > 0
            region[:, :65] = False
            q = quality[scene] = {"kept_pct / bad_among_kept_pct": {}, "bp_nonocc": {}}
            with DispEst(ls, rs, 64) as de:
                de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
                for setting in [None] + QUALITY_SETTINGS:
                    if setting is None:
                        m = de.lDisMap.copy()
                    else:
                        de.setSpeckleFilter(capi.PSM_SPECKLE_ONLY, *setting); de.PostProcess_GPU()
                        m = de.lDisMap.copy()
                    kept = region & (m != 0)
                    bad = kept & (np.abs(np.minimum(4 * m.astype(np.int32), 255) - gt.astype(np.int32)) > 4)
                    q["kept_pct / bad_among_kept_pct"][str(setting or "none (WTA)")] = [
                        round(100.0 * kept.sum() / region.sum(), 2), round(100.0 * bad.sum() / kept.sum(), 2)]
                for sp, sname in ((capi.PSM_SPECKLE_OFF, "no speckle removal"), (capi.PSM_SPECKLE_FIRST, f"speckle {SETTING}")):
                    for lr, lname in ((capi.PSM_LR_FILL, "fill"), (capi.PSM_LR_FILL_WMF, "fill + r9 post-filter")):
                        de.setSpeckleFilter(sp, *SETTING); de.setLRCheck(lr); de.PostProcess_GPU()
                        q["bp_nonocc"][f"{sname}, {lname}"] = round(bad_pixels_nonocc(de.lDisMap, gt, occl), 3)
    gpu = device_info(0)
    gpu.update(gpu_clocks())
    line = {"workload": "speckle_1920x1080_wta", "gpu": gpu, "steps": args.steps, "warmup": args.warmup,
            "rounds": ROUNDS, "band_parity": parity, "workloads": results, "adversarial_u8": adversarial,
            "quality_D64_left": quality}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
