"""Cost of the uniqueness test and the median (psm_set_uniqueness_check, psm_set_median_blur) and of the reference's
whole StereoSGBM post-processing on one GPU; prints one JSON line.  With --quality-only it prints the quality numbers
instead, which need no GPU: the device equals the CPU restatements bit for bit (tests/test_gpu_unique_median.py).

Maps: the winner-take-all maps of the synthetic 1920 x 1080 stereo pair of bench.py (PSM_OPT_COSTS and
PSM_OPT_RUNNER_UP on), at D = 128 on a u8 context and at D = 256 on a u16 context, on both views and on the left view
alone.  Stage configurations, timed in alternating rounds: PSM_UNIQUE_ONLY at ratio 10, PSM_MEDIAN_ONLY at ksize 3 and
5, the reference's SGBM set (uniqueness 10 -> disparity check 1 -> median 3 -> speckle (100, 32) PSM_SPECKLE_ONLY, no
weighted median) and the default post-filter alone.  Per configuration and round: ms per call of
psm_post_process_device (CUDA events around `steps` calls on the context's stream) and the median stage-5 time
(psm_stage_ms); the medians over the rounds are reported.  Frames: a left-only TorchStereo.match(post_process=True) with
the SGBM set against one with disparity check + fill + the default post-filter, timed the same way.

Quality (--quality-only), from the oracle's D = 64 maps of Cones and Teddy: the share of pixels kept (non-zero and
unchanged) and the %BP among the kept non-occluded pixels (bench_gif_window.bad_pixels_nonocc's threshold), for
uniqueness 5 / 10 / 15 alone, the disparity check + speckle removal of DESIGN §23 / §26, and the full SGBM set.

Usage: python bench_sgbm_post.py [--steps 20] [--warmup 3] | --quality-only
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
ROUNDS = 3
SGBM = dict(uniqueness=(1, 10), dcheck=(1, 1), median=(1, 3), speckle=(2, 100, 32))


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


def configure(de, uniqueness=(0, 10), dcheck=(0, 1), median=(0, 3), speckle=(0, 0, 0), lr=0):
    de.setUniquenessCheck(*uniqueness); de.setDisparityCheck(*dcheck); de.setMedianBlur(*median)
    de.setSpeckleFilter(*speckle); de.setLRCheck(lr)


STAGES = {"unique only 10": dict(uniqueness=(2, 10)), "median only 3": dict(median=(2, 3)),
          "median only 5": dict(median=(2, 5)), "sgbm set": SGBM, "post-filter": {}}


def quality():
    from bench_gif_window import read_png
    from oracle import oracle as O
    import sgbm_chain as SC
    import runner_up_cases as RU
    g = os.path.join(ROOT, "tests", "golden")
    out = {}
    for scene in ("Cones", "Teddy"):
        s = scene.lower()
        l = O.u8_to_f32(read_png(os.path.join(g, f"{s}_im2.png")))
        r = O.u8_to_f32(read_png(os.path.join(g, f"{s}_im6.png")))
        gt, occl = read_png(os.path.join(g, f"{s}_disp2.png"), True), read_png(os.path.join(g, f"{s}_occl.png"), True)
        _, _, lraw, rraw = O.cost_const(l, r, 64)
        lf, rf = O.cost_filter(l, r, lraw, rraw)
        ld, rd = O.disp_select(lf, rf)
        qm = [np.take_along_axis(v, m.astype(np.int64)[None], 0)[0] for v, m in ((lf, ld), (rf, rd))]
        qr = [RU.definition(v, m)[1].view(np.float32) for v, m in ((lf, ld), (rf, rd))]
        settings = {"WTA": {}, **{f"uniqueness {k}": dict(uniqueness=(2, k)) for k in (5, 10, 15)},
                    "dcheck 1 + speckle (100, 1)": dict(dcheck=(1, 1), speckle=(2, 100, 1)),
                    "sgbm set": SGBM}
        q = out[scene] = {}
        for name, kw in settings.items():
            m = SC.chain(l, r, ld, rd, costs=qm, runner=qr, D=64, **kw)[0] if kw else ld
            kept = (m == ld) & (m != 0)
            nonocc = occl > 0
            nonocc[:, :65] = False
            disp = np.minimum(m.astype(np.int32) * 4, 255)
            err = np.abs(disp - gt.astype(np.int32)) > 4
            sel = kept & nonocc
            q[name] = {"kept_pct": round(100.0 * np.count_nonzero(kept) / kept.size, 2),
                       "bp_among_kept_pct": round(100.0 * np.count_nonzero(err & sel) / max(1, np.count_nonzero(sel)), 2)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--quality-only", action="store_true")
    args = ap.parse_args()
    if args.quality_only:
        print(json.dumps({"workload": "sgbm_post_quality_D64", "quality": quality()}), flush=True)
        return
    import torch
    from bench import device_info
    from bench_lr_check import gpu_clocks
    from primestereomatch_b200 import DispEst, capi, synth
    from primestereomatch_b200.torch_stereo import TorchStereo
    import sgbm_chain as SC
    if not torch.cuda.is_available() or capi.lib().psm_device_count() < 1:
        raise SystemExit("bench_sgbm_post.py needs a CUDA device")
    W, H = 1920, 1080
    L = capi.lib()
    results, parity = [], True
    for D, bits in WORKLOADS:
        l8, r8, _ = synth.stereo_pair_u8(W, H, D)
        l, r = synth.to_f32(l8), synth.to_f32(r8)
        for views in ("both", "left"):
            per = {name: {"config": name, "ms_per_call": [], "stage5_ms": []} for name in STAGES}
            de = DispEst(l, r, D, map_bits=bits)
            de.stream = torch.cuda.Stream()   # the context runs on this stream, so the events bracket the calls
            capi.check(L.psm_set_stream(de.handle, C.c_void_p(de.stream.cuda_stream)), de.handle)
            if views == "left":
                de.setViews("left")
            de.setCostOutput(True); de.setRunnerUpOutput(True)
            de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
            ld = de.lDisMap.copy()
            qm, qr = de.lCosts[1].copy(), de.lRunnerUp[1].copy()
            post = lambda: capi.check(L.psm_post_process_device(de.handle), de.handle)   # noqa: E731
            for rnd in range(ROUNDS):
                for name, kw in STAGES.items():
                    configure(de, **kw)
                    ms, k = timed(de.stream, post, args.steps, args.warmup, de)
                    per[name]["ms_per_call"].append(ms)
                    per[name]["stage5_ms"].append(k)
                    if rnd == 0 and name == "sgbm set":   # the left map against the restatement
                        de.PostProcess_GPU()
                        exp = SC.chain(None, None, ld, None, costs=(qm, None), runner=(qr, None), D=D, **kw)[0]
                        parity = parity and bool(np.array_equal(de.lDisMap, exp))
                    print(json.dumps({"progress": {"D": D, "views": views, "config": name, "ms_per_call": ms,
                                                   "stage5_ms": k}}), file=sys.stderr, flush=True)
            de.close()
            results.append({"D": D, "map_bits": bits, "views": views, "stages": [summarise(x) for x in per.values()]})
        # frames: a left-only TorchStereo frame with the SGBM set against check + fill + the default post-filter
        lt, rt = torch.from_numpy(l8).cuda(), torch.from_numpy(r8).cuda()
        fper = {}
        with TorchStereo(W, H, D, map_bits=bits) as ts:
            ts.setViews("left")
            frames = {"left only, sgbm set": lambda: configure(ts, **SGBM),
                      "left only, check + fill + post-filter": lambda: configure(ts, dcheck=(1, 1), lr=1)}
            stream = torch.cuda.current_stream()
            for rnd in range(ROUNDS):
                for name, setup in frames.items():
                    setup()
                    ms, _ = timed(stream, lambda: ts.match(lt, rt, post_process=True), max(1, args.steps // 2), 1)
                    fper.setdefault(name, {"frame": name, "ms_per_call": []})["ms_per_call"].append(ms)
                    print(json.dumps({"progress": {"D": D, "frame": name, "ms_per_call": ms}}), file=sys.stderr,
                          flush=True)
        results.append({"D": D, "map_bits": bits, "frames": [summarise(x) for x in fper.values()]})
    gpu = device_info(0)
    gpu.update(gpu_clocks())
    print(json.dumps({"workload": "sgbm_post_1920x1080_wta", "gpu": gpu, "steps": args.steps, "warmup": args.warmup,
                      "rounds": ROUNDS, "parity": parity, "workloads": results}), flush=True)


if __name__ == "__main__":
    main()
