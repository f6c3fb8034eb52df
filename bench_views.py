"""Left-only frames (PSM_OPT_VIEWS = PSM_VIEWS_LEFT) against two-view frames on one GPU; prints one JSON line.

For each workload two contexts of the same geometry are alive at once, one computing both views and one the left view
alone, and they run in turn, one frame each per round, so that drift on a shared card hits both alike.  Reported per
setting: frames per second from the median frame time, and the medians of psm_stage_ms stages 0-3 (ingest, CVC, filter,
selection).  Workloads, at 1920 x 1080 on the synthetic pair of bench.py (synth.stereo_pair_u8):
  1. c4_device: D = 128, float frames already on the device (psm_set_images_device), maps left on the device;
  2. c4_host_u8: D = 128 end to end from pinned u8 host frames: the next frame's upload (psm_set_images_u8_async) overlaps
     the current frame, psm_set_images_commit ingests it, and the maps come back to pinned host memory;
  3. d256_device: as 1 at D = 256;
  4. blocked_d2048: as 1 at D = 2048 with 16-bit maps on a blocked context of 128 slices per block.
Frame times are CUDA events on the contexts' stream for the device workloads and the host clock around a frame that
ends with its maps on the host for workload 2.  Before the line is printed the left maps of the two settings must be
identical on every workload.  The GPU name, power limit and SM clock are read in the same run.

Usage: python bench_views.py [--steps 100] [--warmup 5]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

W, H = 1920, 1080
WORKLOADS = [("c4_device", 128, None), ("c4_host_u8", 128, None), ("d256_device", 256, None), ("blocked_d2048", 2048, 128)]


def sm_clock(index):
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                              str(index)], capture_output=True, text=True, timeout=20).stdout.strip()
        cur, mx = (float(x) for x in out.split(","))
        return {"sm_clock_mhz": cur, "sm_clock_max_mhz": mx}
    except Exception:
        return {"sm_clock_mhz": None, "sm_clock_max_mhz": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    from bench import device_info
    from primestereomatch_b200 import DispEst, capi, synth
    if not torch.cuda.is_available() or capi.lib().psm_device_count() < 1:
        raise SystemExit("bench_views.py needs a CUDA device")
    L = capi.lib()
    stream = torch.cuda.Stream()
    results, failures, clocks = [], [], []

    for name, D, block in WORKLOADS:
        l8, r8, _ = synth.stereo_pair_u8(W, H, D)
        host = name == "c4_host_u8"
        bits = 16 if D > 256 else 8
        mdt = np.uint16 if bits == 16 else np.uint8
        ctxs = {v: DispEst(l8, r8, D, map_bits=bits, block_slices=block) for v in ("both", "left")}
        try:
            dev = [torch.from_numpy(synth.to_f32(a)).cuda().contiguous() for a in (l8, r8)]
            pinned = [torch.from_numpy(a.copy()).pin_memory() for a in (l8, r8)]
            maps = {v: [torch.zeros((H, W), dtype=torch.uint8 if bits == 8 else torch.int16).pin_memory()
                        for _ in range(2)] for v in ctxs}
            for v, de in ctxs.items():
                capi.check(L.psm_set_stream(de.handle, C.c_void_p(stream.cuda_stream)), de.handle)
                de.setViews(v)
            step = W * 3 * 4
            sel = L.psm_disp_select_u16 if bits == 16 else L.psm_disp_select

            def upload_async(de):
                p = [t.data_ptr() for t in pinned]
                capi.check(L.psm_set_images_u8_async(de.handle, p[0], W * 3, p[1], W * 3), de.handle)

            def frame(v):
                de, h = ctxs[v], ctxs[v].handle
                if host:
                    capi.check(L.psm_set_images_commit(h), h)
                else:
                    capi.check(L.psm_set_images_device(h, dev[0].data_ptr(), step, dev[1].data_ptr(), step), h)
                capi.check(L.psm_cost_const(h), h)
                capi.check(L.psm_cost_filter(h), h)
                if host:
                    upload_async(de)   # the next frame's copy overlaps this frame's selection and the map copy
                    m = maps[v]
                    right = m[1].data_ptr() if v == "both" else None
                    capi.check(sel(h, m[0].data_ptr(), W * m[0].element_size(), right, W * m[1].element_size()), h)
                else:
                    capi.check(L.psm_disp_select_device(h), h)

            def timed(v):
                de = ctxs[v]
                if host:
                    t0 = time.perf_counter(); frame(v); ms = (time.perf_counter() - t0) * 1e3
                else:
                    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    ev0.record(stream); frame(v); ev1.record(stream)
                    torch.cuda.synchronize()
                    ms = ev0.elapsed_time(ev1)
                return (ms,) + tuple(de.stage_ms(s) for s in range(4))

            if host:
                for de in ctxs.values():
                    upload_async(de)
            for _ in range(args.warmup):
                for v in ctxs:
                    frame(v)
            torch.cuda.synchronize()
            samples = {v: [] for v in ctxs}
            for _ in range(args.steps):
                for v in ctxs:
                    samples[v].append(timed(v))
            clocks.append(sm_clock(0))
            left = {}
            for v, de in ctxs.items():
                de.sync()
                ld = np.zeros((H, W), mdt)
                rd = np.zeros((H, W), mdt) if v == "both" else None
                capi.check(sel(de.handle, ld.ctypes.data_as(C.c_void_p), ld.strides[0],
                               None if rd is None else rd.ctypes.data_as(C.c_void_p), W * ld.itemsize), de.handle)
                left[v] = ld
            same = bool(np.array_equal(left["both"], left["left"]))
            if not same:
                failures.append(f"{name}: the left-only left map differs from the two-view one")
            ent = {"workload": name, "D": D, "block_slices": block, "map_bits": bits, "left_maps_identical": same}
            for v in ctxs:
                med = [float(np.median([s[i] for s in samples[v]])) for i in range(5)]
                ent[v] = {"fps": round(1000.0 / med[0], 2), "frame_ms": round(med[0], 3),
                          "stage_ms": {k: round(x, 3) for k, x in zip(("ingest", "cvc", "cvf", "wta"), med[1:])}}
            ent["speedup"] = round(ent["left"]["fps"] / ent["both"]["fps"], 3)
            results.append(ent)
            print(json.dumps({"progress": ent}), file=sys.stderr, flush=True)
        finally:
            torch.cuda.synchronize()
            for de in ctxs.values():
                de.close()

    if failures:
        raise SystemExit("parity failed: " + "; ".join(failures))
    line = {"workload": "views_1920x1080", "gpu": device_info(0), "clocks_after_each_workload": clocks, "steps": args.steps,
            "warmup": args.warmup, "results": results}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
