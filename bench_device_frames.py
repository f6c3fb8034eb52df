"""Frames already in GPU memory: TorchStereo on device tensors against the host upload and the device-host round trip;
prints one JSON line.

Three arms per workload, each on its own context, with both views and the default filter:
  a. host_u8: pinned host u8 frames through psm_set_images_u8, CVC, filter, psm_disp_select into host maps;
  b. torch_hwc_bgr / torch_chw_rgb: device u8 tensors, (H, W, 3) BGR and torchvision's (3, H, W) RGB, through
     TorchStereo.match (psm_set_images_device_planes ... psm_copy_maps_device), maps left on the device;
  c. roundtrip_u8: what a GPU-decode user does without (b): the device tensor goes to the host (.cpu()), then arm a,
     then both maps back to the device (.cuda()).
A frame is timed on the host clock from its first call to its maps being complete (the host copy returned, or torch's
stream synchronised).  Every round runs one frame of each arm in turn, so drift on a shared card hits all alike;
frames/s is 1000 over the median frame time, and stage 0 (ingest) the median of psm_stage_ms(0).  Workloads:
1920 x 1080 at D = 128 and 450 x 375 at D = 64 on the synthetic pair of bench.py (synth.stereo_pair_u8).  Before the line
is printed every arm's maps must equal arm a's.  "ingest_kernels_ms" times the ingest alone (stage 0, median over
--steps calls on one context with nothing else queued), by entry point: interleaved frames (f32 through
psm_set_images_device, u8 through psm_set_images_u8_async after its upload has finished, then psm_set_images_commit)
and psm_set_images_device_planes on the same pixels as HWC BGR u8 / f32 and CHW RGB u8 tensors.  The GPU name and power
limit are read in the same run.

Usage: python bench_device_frames.py [--steps 50] [--warmup 5]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

WORKLOADS = [(1920, 1080, 128), (450, 375, 64)]
ARMS = ("host_u8", "torch_hwc_bgr", "torch_chw_rgb", "roundtrip_u8")


def ingest_only(L, capi, torch, de, pinned, hwc, chw, W, steps):
    """median stage-0 ms of each ingest path on one context (see the module text)"""
    from primestereomatch_b200.torch_stereo import frame_layout
    h = de.handle
    f32 = [t.float().div_(255.0).contiguous() for t in hwc]   # not the convertTo rounding: only the timing matters here
    H = hwc[0].shape[0]

    def planes(pair, ch):
        pix, lf, row, col, _ = frame_layout(pair[0], H, W, ch)
        _, rf, _, _, _ = frame_layout(pair[1], H, W, ch)
        return lambda: capi.check(L.psm_set_images_device_planes(h, pix, (C.c_void_p * 3)(*lf[0]),
                                                                 (C.c_void_p * 3)(*rf[0]), row, col), h)

    def commit_u8():
        capi.check(L.psm_set_images_u8_async(h, pinned[0].data_ptr(), W * 3, pinned[1].data_ptr(), W * 3), h)
        de.sync()
        capi.check(L.psm_set_images_commit(h), h)

    paths = {
        "device_f32": lambda: capi.check(L.psm_set_images_device(h, f32[0].data_ptr(), W * 12, f32[1].data_ptr(),
                                                                 W * 12), h),
        "async_commit_u8": commit_u8,
        "planes_hwc_bgr_u8": planes(hwc, "bgr"),
        "planes_hwc_bgr_f32": planes(f32, "bgr"),
        "planes_chw_rgb_u8": planes(chw, "rgb"),
    }
    torch.cuda.synchronize()
    out = {}
    for name, call in paths.items():
        ms = []
        for _ in range(steps):
            call()
            ms.append(de.stage_ms(0))
        out[name] = round(float(np.median(ms)), 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    from bench import device_info
    from primestereomatch_b200 import DispEst, TorchStereo, capi, synth
    if not torch.cuda.is_available() or capi.lib().psm_device_count() < 1:
        raise SystemExit("bench_device_frames.py needs a CUDA device")
    L = capi.lib()
    results, failures = [], []

    for W, H, D in WORKLOADS:
        l8, r8, _ = synth.stereo_pair_u8(W, H, D)
        pinned = [torch.from_numpy(a.copy()).pin_memory() for a in (l8, r8)]
        hwc = [torch.from_numpy(a).cuda() for a in (l8, r8)]
        chw = [t.flip(2).permute(2, 0, 1).contiguous() for t in hwc]
        host_maps = {a: [np.zeros((H, W), np.uint8) for _ in range(2)] for a in ("host_u8", "roundtrip_u8")}
        ctx = {"host_u8": DispEst(l8, r8, D), "roundtrip_u8": DispEst(l8, r8, D),
               "torch_hwc_bgr": TorchStereo(W, H, D), "torch_chw_rgb": TorchStereo(W, H, D)}
        dev_maps = {}
        try:
            def host_frame(h, lp, rp, m):
                capi.check(L.psm_set_images_u8(h, lp, W * 3, rp, W * 3), h)
                capi.check(L.psm_cost_const(h), h)
                capi.check(L.psm_cost_filter(h), h)
                capi.check(L.psm_disp_select(h, m[0].ctypes.data_as(C.c_void_p), W, m[1].ctypes.data_as(C.c_void_p), W), h)

            def frame(arm):
                if arm == "host_u8":
                    host_frame(ctx[arm].handle, pinned[0].data_ptr(), pinned[1].data_ptr(), host_maps[arm])
                elif arm == "roundtrip_u8":
                    l, r = hwc[0].cpu(), hwc[1].cpu()
                    host_frame(ctx[arm].handle, l.data_ptr(), r.data_ptr(), host_maps[arm])
                    dev_maps[arm] = tuple(torch.from_numpy(m).cuda() for m in host_maps[arm])
                else:
                    src, ch = (hwc, "bgr") if arm == "torch_hwc_bgr" else (chw, "rgb")
                    dev_maps[arm] = ctx[arm].match(src[0], src[1], channels=ch)
                    torch.cuda.current_stream().synchronize()

            def timed(arm):
                t0 = time.perf_counter()
                frame(arm)
                return (time.perf_counter() - t0) * 1e3, ctx[arm].stage_ms(0)

            for _ in range(args.warmup):
                for arm in ARMS:
                    frame(arm)
            samples = {arm: [] for arm in ARMS}
            for _ in range(args.steps):
                for arm in ARMS:
                    samples[arm].append(timed(arm))
            torch.cuda.synchronize()
            want = host_maps["host_u8"]
            same = {}
            for arm in ARMS[1:]:
                got = [m.cpu().numpy() for m in dev_maps[arm]]
                same[arm] = bool(all(np.array_equal(g, w) for g, w in zip(got, want)))
                if not same[arm]:
                    failures.append(f"{W}x{H}x{D} {arm}: maps differ from host_u8")
            ent = {"W": W, "H": H, "D": D, "maps_identical_to_host_u8": same}
            for arm in ARMS:
                ms = float(np.median([s[0] for s in samples[arm]]))
                ent[arm] = {"fps": round(1000.0 / ms, 2), "frame_ms": round(ms, 3),
                            "stage0_ms": round(float(np.median([s[1] for s in samples[arm]])), 4)}
            ent["ingest_kernels_ms"] = ingest_only(L, capi, torch, ctx["roundtrip_u8"], pinned, hwc, chw, W, args.steps)
            ent["roundtrip_over_torch_hwc_ms"] = round(ent["roundtrip_u8"]["frame_ms"] - ent["torch_hwc_bgr"]["frame_ms"], 3)
            results.append(ent)
            print(json.dumps({"progress": ent}), file=sys.stderr, flush=True)
        finally:
            torch.cuda.synchronize()
            for c in ctx.values():
                c.close()

    if failures:
        raise SystemExit("parity failed: " + "; ".join(failures))
    print(json.dumps({"workload": "device_frames", "gpu": device_info(0), "steps": args.steps, "warmup": args.warmup,
                      "results": results}), flush=True)


if __name__ == "__main__":
    main()
