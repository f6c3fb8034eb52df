"""Cost of YUV frames converted in ingest (psm_set_images_yuv / _device_yuv) on one GPU; prints one JSON line.

Frames: bench.py's synthetic pair turned into YUV (yuv_oracle.from_bgr); every BGR arm is fed the oracle's conversion of
the same YUV frames (yuv_oracle.bgr), so both arms compute the same planes and maps.  Workloads, in alternating rounds:
  - "stage0_1080p": stage 0 (psm_stage_ms 0: one ingest_kernel and one halo pass per view) of 1920 x 1080 device frames,
    NV12 and YUYV (psm_set_images_device_yuv) against the BGR frame as device planes (contiguous HWC).  The median over
    `steps` calls after `warmup` calls, then over the rounds.
  - "camera_sbs_rectified": the reference camera's side-by-side 2688 x 376 YUYV tensor, its halves rectified into a
    1248 x 336 crop (synth.rectify_maps), against the same frame as a BGR side-by-side tensor, also rectified.
  - "torch_stereo_d128_1080p": TorchStereo.match at D = 128 from NV12 tensors against BGR tensors: ms per frame (CUDA
    events around `frames` calls on torch's current stream).
  - "host_frame_d128_1080p": one whole frame from pinned host frames -- psm_set_images_yuv (NV12, YUYV) or
    psm_set_images_u8 (BGR), psm_cost_const, psm_cost_filter and psm_disp_select into host maps -- ms per frame by the
    host clock over `frames` frames, and the ms of the upload call alone (it returns once the copy has read the frame).
Parity, in the first round of each: planes and gradients (stage 0) or maps equal bit for bit.

Usage: python bench_yuv.py [--steps 200] [--warmup 20] [--frames 10]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

ROUNDS = 3


def event_ms(stream, n, call):
    import torch
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(stream)
    for _ in range(n):
        call()
    ev1.record(stream)
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / n


def med(xs, nd=4):
    return round(float(np.median(xs)), nd)


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
    from primestereomatch_b200.torch_stereo import TorchStereo, frame_layout, yuv_layout
    import rectify_oracle as RO
    import yuv_oracle as YO
    if not torch.cuda.is_available() or capi.lib().psm_device_count() < 1:
        raise SystemExit("bench_yuv.py needs a CUDA device")
    L = capi.lib()
    parity = True

    def planes_call(de, lt, rt, hw):
        pix, lf, row, col, _ = frame_layout(lt, *hw)
        _, rf, _, _, _ = frame_layout(rt, *hw)
        lp, rp = (C.c_void_p * 3)(*lf[0]), (C.c_void_p * 3)(*rf[0])
        return lambda: capi.check(L.psm_set_images_device_planes(de.handle, pix, lp, rp, row, col), de.handle)

    def yuv_call(de, lt, rt, hw, fmt):
        sampling, lf, *steps, _ = yuv_layout(lt, *hw, fmt)
        _, rf, *_ = yuv_layout(rt, *hw, fmt)
        lp, rp = (C.c_void_p * 3)(*lf[0]), (C.c_void_p * 3)(*rf[0])
        return lambda: capi.check(L.psm_set_images_device_yuv(de.handle, sampling, lp, rp, *steps), de.handle)

    def same_planes(a, b):
        return all(np.array_equal(a.read_guide_plane(v, p).view(np.uint32), b.read_guide_plane(v, p).view(np.uint32))
                   for v in (0, 1) for p in (0, 1, 2, 12))

    def stage0(arms, ref):
        """arms: {name: (DispEst, call)} -> {name: [median stage-0 ms per round]}; parity against arms[ref]"""
        nonlocal parity
        per = {k: [] for k in arms}
        for rnd in range(ROUNDS):
            for arm, (de, call) in arms.items():
                for _ in range(args.warmup):
                    call()
                de.sync()
                ms = []
                for _ in range(args.steps):
                    call()
                    ms.append(de.stage_ms(0))
                per[arm].append(float(np.median(ms)))
            if rnd == 0:
                for arm, (de, _) in arms.items():
                    parity &= same_planes(de, arms[ref][0])
        return {k: {"per_round": [round(x, 4) for x in v], "median": med(v)} for k, v in per.items()}

    out = {}
    # stage 0 of 1920 x 1080 device frames
    W, H = 1920, 1080
    l8, r8, _ = synth.stereo_pair_u8(W, H, 64)
    yuv = {f: tuple(YO.from_bgr(i, f) for i in (l8, r8)) for f in ("nv12", "yuyv")}
    bgr = tuple(YO.bgr(f, "nv12") for f in yuv["nv12"])
    bgr2 = tuple(YO.bgr(f, "yuyv") for f in yuv["yuyv"])
    with DispEst(*bgr, 64) as dn, DispEst(*bgr2, 64) as dy, DispEst(*bgr, 64) as db, DispEst(*bgr2, 64) as db2:
        dev = {f: tuple(torch.from_numpy(x).cuda() for x in v) for f, v in yuv.items()}
        t_bgr = tuple(torch.from_numpy(x).cuda() for x in bgr)
        t_bgr2 = tuple(torch.from_numpy(x).cuda() for x in bgr2)
        out["stage0_1080p"] = {
            **stage0({"nv12": (dn, yuv_call(dn, *dev["nv12"], (H, W), "nv12")),
                      "bgr_planes": (db, planes_call(db, *t_bgr, (H, W)))}, "bgr_planes"),
            **stage0({"yuyv": (dy, yuv_call(dy, *dev["yuyv"], (H, W), "yuyv")),
                      "bgr_planes_of_yuyv": (db2, planes_call(db2, *t_bgr2, (H, W)))}, "bgr_planes_of_yuyv")}

    # the reference camera's side-by-side frame, rectified
    (W, H), (SW, SH) = (1248, 336), (1344, 376)
    l8, r8, _ = synth.stereo_pair_u8(SW, SH, 64)
    maps = [synth.rectify_maps(W, H, SW, SH, view=v) for v in range(2)]
    fy = tuple(YO.from_bgr(i, "yuyv") for i in (l8, r8))
    fb = tuple(YO.bgr(f, "yuyv") for f in fy)
    lo, ro = (RO.remap(b, *m) for b, m in zip(fb, maps))
    cam_y = torch.from_numpy(np.concatenate(fy, axis=1)).cuda()
    cam_b = torch.from_numpy(np.concatenate(fb, axis=1)).cuda()
    with DispEst(lo, ro, 64) as ry, DispEst(lo, ro, 64) as rb:
        for de in (ry, rb):
            de.setRectify(maps[0], maps[1], (SW, SH))
        out["camera_sbs_rectified"] = stage0(
            {"yuyv": (ry, yuv_call(ry, cam_y[:, :SW], cam_y[:, SW:], (SH, SW), "yuyv")),
             "bgr_planes": (rb, planes_call(rb, cam_b[:, :SW], cam_b[:, SW:], (SH, SW)))}, "bgr_planes")

    # TorchStereo.match at D = 128
    W, H, D = 1920, 1080, 128
    l8, r8, _ = synth.stereo_pair_u8(W, H, D)
    fn = tuple(YO.from_bgr(i, "nv12") for i in (l8, r8))
    fb = tuple(YO.bgr(f, "nv12") for f in fn)
    arms = {"nv12": tuple(torch.from_numpy(x).cuda() for x in fn), "bgr": tuple(torch.from_numpy(x).cuda() for x in fb)}
    frame = {k: [] for k in arms}
    with TorchStereo(W, H, D) as ts:
        stream = torch.cuda.current_stream()
        for rnd in range(ROUNDS):
            maps_out = []
            for arm, frames in arms.items():
                kw = {"yuv": "nv12"} if arm == "nv12" else {}
                call = lambda: ts.match(*frames, **kw)   # noqa: E731
                maps_out.append(call())
                torch.cuda.synchronize()
                frame[arm].append(round(event_ms(stream, args.frames, call), 3))
            if rnd == 0:
                parity &= all(torch.equal(a, b) for a, b in zip(*maps_out))
    out["torch_stereo_d128_1080p"] = {k: {"ms_per_frame": v, "median": med(v, 3)} for k, v in frame.items()}

    # a whole frame from pinned host frames
    host = {f: tuple(torch.from_numpy(YO.from_bgr(i, f)).pin_memory() for i in (l8, r8)) for f in ("nv12", "yuyv")}
    host["bgr"] = tuple(torch.from_numpy(YO.bgr(host["nv12"][k].numpy(), "nv12")).pin_memory() for k in range(2))
    host["bgr_of_yuyv"] = tuple(torch.from_numpy(YO.bgr(host["yuyv"][k].numpy(), "yuyv")).pin_memory() for k in range(2))
    lmap, rmap = (torch.empty((H, W), dtype=torch.uint8).pin_memory() for _ in range(2))
    res = {k: {"frame_ms": [], "upload_ms": []} for k in host}
    with DispEst(*fb, D) as de:
        h = de.handle

        def upload(arm):
            l, r = host[arm]
            if arm.startswith("bgr"):
                return L.psm_set_images_u8(h, l.data_ptr(), l.stride(0), r.data_ptr(), r.stride(0))
            return L.psm_set_images_yuv(h, capi.YUV_FORMATS[arm], l.data_ptr(), l.stride(0), r.data_ptr(), r.stride(0))

        def whole(arm):
            t0 = time.perf_counter()
            capi.check(upload(arm), h)
            t1 = time.perf_counter()
            for rc in (L.psm_cost_const(h), L.psm_cost_filter(h),
                       L.psm_disp_select(h, lmap.data_ptr(), W, rmap.data_ptr(), W)):
                capi.check(rc, h)
            return t1 - t0, time.perf_counter() - t0

        for rnd in range(ROUNDS):
            got = {}
            for arm in host:
                whole(arm)
                up, tot = zip(*(whole(arm) for _ in range(args.frames)))
                res[arm]["upload_ms"].append(round(1e3 * float(np.median(up)), 3))
                res[arm]["frame_ms"].append(round(1e3 * float(np.median(tot)), 3))
                got[arm] = (lmap.clone(), rmap.clone())
            if rnd == 0:
                parity &= all(torch.equal(a, b) for a, b in zip(got["nv12"], got["bgr"]))
                parity &= all(torch.equal(a, b) for a, b in zip(got["yuyv"], got["bgr_of_yuyv"]))
    out["host_frame_d128_1080p"] = {k: {**v, "frame_ms_median": med(v["frame_ms"], 3),
                                        "upload_ms_median": med(v["upload_ms"], 3)} for k, v in res.items()}

    info = device_info(0)
    print(json.dumps({"bench": "yuv", "gpu": info["name"], **gpu_clocks(), "steps": args.steps, "warmup": args.warmup,
                      "frames": args.frames, "rounds": ROUNDS, "parity": parity, **out}))


if __name__ == "__main__":
    main()
