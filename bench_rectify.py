"""Cost of rectification in ingest (psm_set_rectify) on one GPU; prints one JSON line.

Maps: a closed-form pinhole + radial-distortion rig (synth.rectify_maps), so no cv2 is needed.  Frames: bench.py's
synthetic pair, of the source size.  Workloads, each with rectification on and off in alternating rounds:
  - "crop_1080p": a 1920 x 1080 crop of a 2200 x 1300 source;
  - "camera_sbs": the reference camera's side-by-side frame, one 2688 x 376 tensor whose two 1344 x 376 halves are the
    views, rectified into a 1248 x 336 crop.
"on" feeds the raw frames (device planes, rectified in ingest); "off" feeds the oracle's rectified frames to a context
without maps (device planes, contiguous HWC).  Stage 0 (psm_stage_ms 0: one ingest_kernel and one halo pass per view)
is read after each of `steps` calls, following `warmup` calls; the medians over the steps, then over the rounds, are
reported.  Parity, in the first round: the planes and gradients of both views of the two contexts are equal bit for bit.

TorchStereo.match: ms per frame at D = 128 at 1920 x 1080, raw frames with rectification against the rectified frames
without it, in alternating rounds (CUDA events around `frames` calls on torch's current stream), maps checked equal.

Usage: python bench_rectify.py [--steps 200] [--warmup 20] [--frames 10]
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

ROUNDS = 3
WORKLOADS = {"crop_1080p": ((1920, 1080), (2200, 1300), False), "camera_sbs": ((1248, 336), (1344, 376), True)}


def event_ms(stream, n, call):
    import torch
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(stream)
    for _ in range(n):
        call()
    ev1.record(stream)
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--frames", type=int, default=10)
    args = ap.parse_args()
    import torch
    from bench import device_info
    from bench_lr_check import gpu_clocks
    from primestereomatch_b200 import DispEst, capi, synth
    from primestereomatch_b200.torch_stereo import TorchStereo, frame_layout
    import rectify_oracle as RO
    if not torch.cuda.is_available() or capi.lib().psm_device_count() < 1:
        raise SystemExit("bench_rectify.py needs a CUDA device")
    L = capi.lib()
    parity = True

    def planes_call(de, lt, rt, hw):
        pix, lf, row, col, _ = frame_layout(lt, *hw)
        _, rf, _, _, _ = frame_layout(rt, *hw)
        lp, rp = (C.c_void_p * 3)(*lf[0]), (C.c_void_p * 3)(*rf[0])
        return lambda: capi.check(L.psm_set_images_device_planes(de.handle, pix, lp, rp, row, col), de.handle)

    results = []
    for name, ((W, H), (SW, SH), sbs) in WORKLOADS.items():
        l8, r8, _ = synth.stereo_pair_u8(SW, SH, 64)
        maps = [synth.rectify_maps(W, H, SW, SH, view=v) for v in range(2)]
        lo, ro = RO.remap(l8, *maps[0]), RO.remap(r8, *maps[1])
        if sbs:
            cam = torch.from_numpy(np.concatenate([l8, r8], axis=1)).cuda()
            raw = (cam[:, :SW], cam[:, SW:])
        else:
            raw = (torch.from_numpy(l8).cuda(), torch.from_numpy(r8).cuda())
        rect_frames = (torch.from_numpy(lo).cuda(), torch.from_numpy(ro).cuda())
        per = {"on": [], "off": []}
        with DispEst(lo, ro, 64) as on, DispEst(lo, ro, 64) as off:
            on.setRectify(maps[0], maps[1], (SW, SH))
            calls = {"on": (on, planes_call(on, *raw, (SH, SW))), "off": (off, planes_call(off, *rect_frames, (H, W)))}
            for rnd in range(ROUNDS):
                for arm, (de, call) in calls.items():
                    for _ in range(args.warmup):
                        call()
                    de.sync()
                    ms = []
                    for _ in range(args.steps):
                        call()
                        ms.append(de.stage_ms(0))
                    per[arm].append(float(np.median(ms)))
                if rnd == 0:
                    for view in (0, 1):
                        for plane in (0, 1, 2, 12):
                            a, b = on.read_guide_plane(view, plane), off.read_guide_plane(view, plane)
                            parity &= bool(np.array_equal(a.view(np.uint32), b.view(np.uint32)))
        results.append({"workload": name, "width": W, "height": H, "src_width": SW, "src_height": SH,
                        "side_by_side": sbs, "stage0_ms_on": [round(x, 4) for x in per["on"]],
                        "stage0_ms_off": [round(x, 4) for x in per["off"]],
                        "stage0_ms_on_median": round(float(np.median(per["on"])), 4),
                        "stage0_ms_off_median": round(float(np.median(per["off"])), 4)})

    W, H, SW, SH, D = 1920, 1080, 2200, 1300, 128
    l8, r8, _ = synth.stereo_pair_u8(SW, SH, D)
    maps = [synth.rectify_maps(W, H, SW, SH, view=v) for v in range(2)]
    lo, ro = RO.remap(l8, *maps[0]), RO.remap(r8, *maps[1])
    raw = (torch.from_numpy(l8).cuda(), torch.from_numpy(r8).cuda())
    pre = (torch.from_numpy(lo).cuda(), torch.from_numpy(ro).cuda())
    frame = {"raw frames, rectify on": [], "rectified frames, rectify off": []}
    with TorchStereo(W, H, D) as on, TorchStereo(W, H, D) as off:
        on.setRectify(maps[0], maps[1], (SW, SH))
        arms = {"raw frames, rectify on": (on, raw), "rectified frames, rectify off": (off, pre)}
        stream = torch.cuda.current_stream()
        for rnd in range(ROUNDS):
            outs = []
            for arm, (ts, frames) in arms.items():
                call = lambda: ts.match(*frames)   # noqa: E731
                outs.append(call())
                torch.cuda.synchronize()
                frame[arm].append(round(event_ms(stream, args.frames, call), 3))
            if rnd == 0:
                parity &= all(torch.equal(a, b) for a, b in zip(outs[0], outs[1]))
    torch_res = {k: {"ms_per_frame": v, "median": float(np.median(v))} for k, v in frame.items()}

    info = device_info(0)
    print(json.dumps({"bench": "rectify", "gpu": info["name"], **gpu_clocks(), "steps": args.steps,
                      "warmup": args.warmup, "rounds": ROUNDS, "parity": parity, "ingest": results,
                      "torch_stereo_d128_1080p": torch_res}))


if __name__ == "__main__":
    main()
