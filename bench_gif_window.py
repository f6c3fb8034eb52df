"""Cost of the guided-filter window (psm_set_guided_filter) on one GPU; prints one JSON line.

Frame: the synthetic 1920 x 1080 x 128 stereo pair of bench.py (both views), device-resident inputs.  Configurations:
(8, 1e-4) runs the tuned 8 x 8 kernels; (8, 2e-4) runs the generic-window kernel at the same window, the only like-for-like
comparison of the two; windows 12, 16, 24 and 32 (eps 1e-4) show how the generic kernel scales with the window.
Per configuration: ms per frame (set images -> CVC -> CVF -> WTA, CUDA events), CVF kernel ms (psm_stage_ms stage 4), the
algorithmic bytes of the filter (8 B per voxel + 48 B per pixel per view) over the kernel time as a fraction of the
H100 SXM data-sheet 3.35 TB/s, and the maps of the top row band against the CPU restatement.  Quality: %BP (non-occluded,
left map) of Cones and Teddy at D = 64 per window, the metric of tests/test_oracle.py::test_bad_pixel_metric_matches_golden
restated in numpy.

Usage: python bench_gif_window.py [--steps 20] [--warmup 3] [--no-quality]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

CONFIGS = [(8, 1e-4), (8, 2e-4), (12, 1e-4), (16, 1e-4), (24, 1e-4), (32, 1e-4)]
HBM_GBS = 3350.0   # H100 SXM data sheet


def read_png(path, gray=False):
    try:
        import cv2
        return cv2.imread(path, cv2.IMREAD_GRAYSCALE if gray else cv2.IMREAD_UNCHANGED)
    except ImportError:
        from PIL import Image
        a = np.array(Image.open(path).convert("L") if gray else Image.open(path))
        return a[:, :, ::-1].copy() if a.ndim == 3 else a


def bad_pixels_nonocc(ld, gt, occl):
    """StereoMatch.cpp:275-311: convertScaleAbs(map, 4), absdiff with the ground truth, first 65 columns cleared,
    THRESH_TOZERO at 4, multiply by the occlusion mask with scale 1/255, percentage of non-zero pixels."""
    disp = np.minimum(ld.astype(np.int32) * 4, 255)
    e = np.abs(disp - gt.astype(np.int32))
    e[:, :65] = 0
    e = np.where(e > 4, e, 0)
    v = np.rint(e.astype(np.float64) * occl.astype(np.float64) / 255.0)
    return float(np.count_nonzero(v)) * 100.0 / gt.size


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-quality", action="store_true")
    args = ap.parse_args()
    import torch
    from bench import device_info
    from primestereomatch_b200 import DispEst, capi, synth
    from oracle import oracle as O
    if not torch.cuda.is_available() or capi.lib().psm_device_count() < 1:
        raise SystemExit("bench_gif_window.py needs a CUDA device")
    W, H, D = 1920, 1080, 128
    l8, r8, _ = synth.stereo_pair_u8(W, H, D)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    ld_dev, rd_dev = torch.from_numpy(l).cuda(), torch.from_numpy(r).cuda()
    step = W * 3 * 4
    L = capi.lib()
    voxels = 2 * D * W * H
    alg_bytes = 8 * voxels + 2 * 48 * W * H
    results = []
    for window, eps in CONFIGS:
        with DispEst(l, r, D) as de:
            de.setGuidedFilter(window, eps)
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
            ms_frame = ev0.elapsed_time(ev1) / args.steps
            kms = []
            for _ in range(args.steps):   # kernel time of the filter alone (psm_stage_ms waits for each frame)
                frame()
                kms.append(de.stage_ms(4))
            # maps of the top row band against the CPU oracle at this window (raw costs + filter + WTA)
            de.DispSelect_GPU()
            band = 32
            c1 = band + 2 * window + 8
            _, _, lraw, rraw = O.cost_const(np.ascontiguousarray(l[:c1]), np.ascontiguousarray(r[:c1]), D)
            lf, rf = O.cost_filter(l[:c1], r[:c1], lraw, rraw, window=window, eps=eps)
            parity = bool(np.array_equal(de.lDisMap[:band], O.wta(lf)[:band]) and np.array_equal(de.rDisMap[:band], O.wta(rf)[:band]))
            kernel_ms = float(np.median(kms))
            results.append({"window": window, "eps": eps, "path": "tuned 8x8" if (window, eps) == (8, 1e-4) else "generic",
                            "ms_per_frame": round(ms_frame, 3), "cvf_kernel_ms": round(kernel_ms, 3),
                            "cvf_hbm_fraction": round(alg_bytes / (kernel_ms * 1e-3) / (HBM_GBS * 1e9), 3),
                            "band_parity": parity})
        print(json.dumps({"progress": results[-1]}), file=sys.stderr, flush=True)
    quality = None
    if not args.no_quality:
        quality = {}
        g = os.path.join(ROOT, "tests", "golden")
        for scene in ("Cones", "Teddy"):
            s = scene.lower()
            l8s, r8s = read_png(os.path.join(g, f"{s}_im2.png")), read_png(os.path.join(g, f"{s}_im6.png"))
            ls, rs = O.u8_to_f32(l8s), O.u8_to_f32(r8s)
            gt, occl = read_png(os.path.join(g, f"{s}_disp2.png"), True), read_png(os.path.join(g, f"{s}_occl.png"), True)
            quality[scene] = {}
            for window in sorted({w for w, _ in CONFIGS} | {4}):
                with DispEst(ls, rs, 64) as de:
                    de.setGuidedFilter(window, 1e-4)
                    de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
                    quality[scene][str(window)] = round(bad_pixels_nonocc(de.lDisMap, gt, occl), 3)
    line = {"workload": "gif_window_C4_1920x1080x128", "gpu": device_info(0), "steps": args.steps, "warmup": args.warmup,
            "hbm_peak_gbs": HBM_GBS, "algorithmic_bytes": alg_bytes, "configs": results, "bp_nonocc_left_D64": quality}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
