"""Cost of Bayer frames demosaiced in ingest (psm_set_images_bayer / _device_bayer) on one GPU; prints one JSON line.

Frames: bench.py's synthetic pair turned into RGGB mosaics (bayer_oracle.from_bgr); every BGR arm is fed the oracle's
demosaicing of the same raw frames (bayer_oracle.bgr), so both arms compute the same planes and maps.  Workloads, in
alternating rounds:
  - "stage0_1080p": stage 0 (psm_stage_ms 0: one ingest_kernel and one halo pass per view) of 1920 x 1080 device frames,
    bilinear and edge-aware (psm_set_images_device_bayer), against the BGR frame as device planes (contiguous HWC).  The
    median over `steps` calls after `warmup` calls, then over the rounds.
  - "camera_sbs_rectified": the reference camera's side-by-side 2688 x 376 raw tensor, its halves rectified into a
    1248 x 336 crop (synth.rectify_maps), against the same frame as a BGR side-by-side tensor, also rectified.
  - "host_frame_d128_1080p": one whole frame from pinned host frames -- psm_set_images_bayer (bilinear, EA) or
    psm_set_images_u8 (BGR), psm_cost_const, psm_cost_filter and psm_disp_select into host maps -- ms per frame by the
    host clock over `frames` frames, and the ms of the upload call alone (it returns once the copy has read the frame).
Parity, in the first round of each: planes and gradients (stage 0) or maps equal bit for bit.

Usage: python bench_bayer.py [--steps 200] [--warmup 20] [--frames 10]
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
    from primestereomatch_b200.torch_stereo import bayer_layout, frame_layout
    import bayer_oracle as BO
    import rectify_oracle as RO
    if not torch.cuda.is_available() or capi.lib().psm_device_count() < 1:
        raise SystemExit("bench_bayer.py needs a CUDA device")
    L = capi.lib()
    parity = True

    def planes_call(de, lt, rt, hw):
        pix, lf, row, col, _ = frame_layout(lt, *hw)
        _, rf, _, _, _ = frame_layout(rt, *hw)
        lp, rp = (C.c_void_p * 3)(*lf[0]), (C.c_void_p * 3)(*rf[0])
        return lambda: capi.check(L.psm_set_images_device_planes(de.handle, pix, lp, rp, row, col), de.handle)

    def bayer_call(de, lt, rt, hw, method):
        p, m, lf, row, col, _ = bayer_layout(lt, *hw, "rggb", method)
        _, _, rf, _, _, _ = bayer_layout(rt, *hw, "rggb", method)
        return lambda: capi.check(L.psm_set_images_device_bayer(de.handle, p, m, lf[0], rf[0], row, col), de.handle)

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
    raw = tuple(BO.from_bgr(i, "rggb") for i in (l8, r8))
    bgr = {m: tuple(BO.bgr(f, "rggb", m) for f in raw) for m in BO.METHODS}
    dev = tuple(torch.from_numpy(x).cuda() for x in raw)
    with DispEst(*bgr["bilinear"], 64) as dbl, DispEst(*bgr["ea"], 64) as dea, \
            DispEst(*bgr["bilinear"], 64) as pbl, DispEst(*bgr["ea"], 64) as pea:
        t_bgr = {m: tuple(torch.from_numpy(x).cuda() for x in v) for m, v in bgr.items()}
        out["stage0_1080p"] = {
            **stage0({"bilinear": (dbl, bayer_call(dbl, *dev, (H, W), "bilinear")),
                      "bgr_planes": (pbl, planes_call(pbl, *t_bgr["bilinear"], (H, W)))}, "bgr_planes"),
            **stage0({"ea": (dea, bayer_call(dea, *dev, (H, W), "ea")),
                      "bgr_planes_of_ea": (pea, planes_call(pea, *t_bgr["ea"], (H, W)))}, "bgr_planes_of_ea")}

    # the reference camera's side-by-side frame, rectified
    (W, H), (SW, SH) = (1248, 336), (1344, 376)
    l8, r8, _ = synth.stereo_pair_u8(SW, SH, 64)
    maps = [synth.rectify_maps(W, H, SW, SH, view=v) for v in range(2)]
    fr = tuple(BO.from_bgr(i, "rggb") for i in (l8, r8))
    fb = tuple(BO.bgr(f, "rggb") for f in fr)
    lo, ro = (RO.remap(b, *m) for b, m in zip(fb, maps))
    cam_r = torch.from_numpy(np.concatenate(fr, axis=1)).cuda()
    cam_b = torch.from_numpy(np.concatenate(fb, axis=1)).cuda()
    with DispEst(lo, ro, 64) as rr, DispEst(lo, ro, 64) as rb:
        for de in (rr, rb):
            de.setRectify(maps[0], maps[1], (SW, SH))
        out["camera_sbs_rectified"] = stage0(
            {"bilinear": (rr, bayer_call(rr, cam_r[:, :SW], cam_r[:, SW:], (SH, SW), "bilinear")),
             "bgr_planes": (rb, planes_call(rb, cam_b[:, :SW], cam_b[:, SW:], (SH, SW)))}, "bgr_planes")

    # a whole frame from pinned host frames
    W, H, D = 1920, 1080, 128
    l8, r8, _ = synth.stereo_pair_u8(W, H, D)
    raw = tuple(BO.from_bgr(i, "rggb") for i in (l8, r8))
    host = {m: tuple(torch.from_numpy(f).pin_memory() for f in raw) for m in BO.METHODS}
    host["bgr"] = tuple(torch.from_numpy(BO.bgr(f, "rggb")).pin_memory() for f in raw)
    host["bgr_of_ea"] = tuple(torch.from_numpy(BO.bgr(f, "rggb", "ea")).pin_memory() for f in raw)
    lmap, rmap = (torch.empty((H, W), dtype=torch.uint8).pin_memory() for _ in range(2))
    res = {k: {"frame_ms": [], "upload_ms": []} for k in host}
    with DispEst(*(h.numpy() for h in host["bgr"]), D) as de:
        h = de.handle

        def upload(arm):
            l, r = host[arm]
            if arm.startswith("bgr"):
                return L.psm_set_images_u8(h, l.data_ptr(), l.stride(0), r.data_ptr(), r.stride(0))
            return L.psm_set_images_bayer(h, capi.PSM_BAYER_RGGB, capi.DEMOSAIC_METHODS[arm], l.data_ptr(), l.stride(0),
                                          r.data_ptr(), r.stride(0))

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
                parity &= all(torch.equal(a, b) for a, b in zip(got["bilinear"], got["bgr"]))
                parity &= all(torch.equal(a, b) for a, b in zip(got["ea"], got["bgr_of_ea"]))
    out["host_frame_d128_1080p"] = {k: {**v, "frame_ms_median": med(v["frame_ms"], 3),
                                        "upload_ms_median": med(v["upload_ms"], 3)} for k, v in res.items()}

    info = device_info(0)
    print(json.dumps({"bench": "bayer", "gpu": info["name"], **gpu_clocks(), "steps": args.steps, "warmup": args.warmup,
                      "frames": args.frames, "rounds": ROUNDS, "parity": parity, **out}))


if __name__ == "__main__":
    main()
