"""Multi-device contexts (psm_create_multi) against the single-device context; prints one JSON line.

Workload: the synthetic 1920 x 1080 pair of bench.py (synth.stereo_pair_u8), u8 frames uploaded from the host.  A frame
is ingest -> CVC -> CVF -> selection (maps left on the device, psm_disp_select_device), timed on the host clock from
the upload to psm_sync, which waits for every shard.  A multi-device context cannot run on a caller's stream, so host
time is the one clock both kinds share.
  1. One GPU: the single-device context and multi-device contexts with n = 2 and 4 shards co-located on device 0, at
     D = 128 and 256 (unblocked), and at D = 2048 with block_slices 128 (16-bit maps, every shard blocked).  All
     contexts of one D are alive at once and run in turn, one frame each per round, so that drift on a shared card hits
     every kind alike; medians over the rounds.  This is the cost of splitting the range and of ordering the shards by
     events on one card.
  2. Several GPUs: frames per second of contexts over devices [0, k) for k = 1, 2, 4, 8 (up to the devices present) at
     D = 128, 256 and 4096 (block_slices 128); k = 1 is the single-device context.  With one GPU visible this section
     says "unmeasured".
  3. Parity, before the line is printed: every multi-device map equals the single-device map of its D and blocking, and
     rows [0, 16) of the single-device maps at D = 128, 256 and 2048 equal the CPU oracle's (oracle/ CVC, guided filter
     and 16-bit arg-min on rows [0, 32): the filtered costs of rows < 16 depend on rows < 25 only).

Usage: python bench_multi_device.py [--steps 10] [--warmup 2]
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

W, H = 1920, 1080
ONE_GPU = ((128, None), (256, None), (2048, 128))   # (D, block_slices)
SHARDS = (2, 4)
SCALING = ((128, None), (256, None), (4096, 128))
BAND = 16


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    from bench import device_info
    from oracle import oracle as O
    from primestereomatch_b200 import DispEst, capi, synth
    L = capi.lib()
    ngpu = L.psm_device_count()
    if not torch.cuda.is_available() or ngpu < 1:
        raise SystemExit("bench_multi_device.py needs a CUDA device")

    def frame(de):
        de.CostConst_GPU(); de.CostFilter_GPU()
        capi.check(L.psm_disp_select_device(de.handle), de.handle)

    def timed(de):
        t0 = time.perf_counter()
        frame(de)
        de.sync()
        return 1000.0 * (time.perf_counter() - t0)

    def maps(de):
        de.DispSelect_GPU()
        return de.lDisMap.copy(), de.rDisMap.copy()

    failures = []

    def same(got, want, what):
        ok = bool(np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]))
        if not ok:
            failures.append(f"{what}: maps differ from the single-device context's")
        return ok

    def check_band(got, l8, r8, D, what):
        lc, rc = (synth.to_f32(np.ascontiguousarray(a[:2 * BAND])) for a in (l8, r8))
        _, _, lraw, rraw = O.cost_const(lc, rc, D)
        lf, rf = O.cost_filter(lc, rc, lraw, rraw)
        del lraw, rraw
        ok = bool(np.array_equal(got[0][:BAND].astype(np.uint16), O.wta(lf, np.uint16)[:BAND])
                  and np.array_equal(got[1][:BAND].astype(np.uint16), O.wta(rf, np.uint16)[:BAND]))
        if not ok:
            failures.append(f"{what}: rows [0, {BAND}) differ from the oracle")
        return ok

    def make(l8, r8, D, block, devices):
        bits = 16 if D > 256 else 8
        if devices is None or len(devices) == 1:
            return DispEst(l8, r8, D, map_bits=bits, block_slices=block, device=0 if devices is None else devices[0])
        return DispEst(l8, r8, D, map_bits=bits, block_slices=block, devices=devices)

    one_gpu = []
    for D, block in ONE_GPU:
        l8, r8, _ = synth.stereo_pair_u8(W, H, min(D, 256))
        kinds = [1] + list(SHARDS)
        ctxs = {n: make(l8, r8, D, block, None if n == 1 else [0] * n) for n in kinds}
        try:
            for de in ctxs.values():
                for _ in range(args.warmup):
                    frame(de)
                de.sync()
            samples = {n: [] for n in kinds}
            for _ in range(args.steps):
                for n in kinds:
                    samples[n].append(timed(ctxs[n]))
            want = maps(ctxs[1])
            band_ok = check_band(want, l8, r8, D, f"D={D} single")
            for n in kinds:
                fr = float(np.median(samples[n]))
                ent = {"D": D, "block_slices": block, "shards_on_device_0": n, "frame_ms": round(fr, 3),
                       "fps": round(1000.0 / fr, 2), "stage3_ms": round(ctxs[n].stage_ms(3), 3)}
                if n == 1:
                    ent["band_parity"] = band_ok
                    base = fr
                else:
                    ent["maps_equal_single"] = same(maps(ctxs[n]), want, f"D={D} block {block} n={n}")
                    ent["frame_overhead_pct"] = round(100 * (fr / base - 1), 2)
                one_gpu.append(ent)
                print(json.dumps({"progress": ent}), file=sys.stderr, flush=True)
        finally:
            for de in ctxs.values():
                de.close()
            torch.cuda.synchronize()

    scaling = "unmeasured: one GPU visible"
    if ngpu >= 2:
        scaling = []
        for D, block in SCALING:
            l8, r8, _ = synth.stereo_pair_u8(W, H, min(D, 256))
            want = None
            for k in (1, 2, 4, 8):
                if k > ngpu:
                    break
                with make(l8, r8, D, block, list(range(k))) as de:
                    for _ in range(args.warmup):
                        frame(de)
                    de.sync()
                    fr = float(np.median([timed(de) for _ in range(args.steps)]))
                    got = maps(de)
                ent = {"D": D, "block_slices": block, "devices": k, "frame_ms": round(fr, 3), "fps": round(1000.0 / fr, 2)}
                if want is None:
                    want = got
                else:
                    ent["maps_equal_single"] = same(got, want, f"D={D} on {k} devices")
                scaling.append(ent)
                print(json.dumps({"progress": ent}), file=sys.stderr, flush=True)

    if failures:
        raise SystemExit("parity failed: " + "; ".join(failures))
    line = {"workload": "multi_device_1920x1080_u8", "gpu": device_info(0), "gpus_visible": ngpu, "steps": args.steps,
            "warmup": args.warmup, "parity": "passed", "one_gpu": one_gpu, "scaling": scaling}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
