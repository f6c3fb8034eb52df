"""Blocked contexts (psm_create_blocked) on one GPU; prints one JSON line.

Workload: the synthetic 1920 x 1080 pair of bench.py (synth.stereo_pair_u8), both views, default filter, u8 frames
uploaded from the host.  A frame is ingest -> CVC -> CVF -> WTA (maps left on the device); the post-filter consumes the
maps and does not depend on blocking, so it is left out.
  1. Overhead: at D = 128 and 256, the unblocked context and blocked ones with block_slices 16, 32, 64 and 128, all
     alive at once and run in turn, one frame each per round, so that drift on a shared card hits every kind alike.
     Medians over the rounds of the frame time (CUDA events on the context's stream) and of stages 1, 2 and 3
     (psm_stage_ms).  On a blocked context stage 1 builds the first block only, stage 2 builds the other blocks and
     folds every block's winner-take-all, and stage 3 reduces the running keys, so stage 2 alone is not comparable:
     "volume_ms" is the sum of the three on either kind.
  2. Reach: at D = 2048, 2560 and 4096 with 16-bit maps, block_slices 128 and 256: frames per second, and the device
     memory the context took (cudaMemGetInfo before creation and after one frame, so lazy allocations count) next to what
     the four volumes of an unblocked context would need.  That footprint is only computed, never allocated.
  3. Parity, before the line is printed: every blocked map equals the unblocked map of its D (section 1), and rows
     [0, 16) of both maps of the unblocked context (section 1) and of one blocked context per D (section 2) equal the CPU
     oracle's (oracle/ CVC, guided filter and 16-bit arg-min on rows [0, 32): the filtered costs of rows < 16 depend on
     rows < 25 only); the other block size's maps equal that context's.

Usage: python bench_blocked.py [--steps 10] [--warmup 2]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

W, H = 1920, 1080
OVERHEAD_D, OVERHEAD_BLOCKS = (128, 256), (16, 32, 64, 128)
REACH_D, REACH_BLOCKS = (2048, 2560, 4096), (128, 256)
BAND = 16


def pitch(width):
    """psm's row pitch in floats (pitch_for_width in psm_kernels.cuh)"""
    w4 = (width + 3) & ~3
    return 32 + ((max(w4 + 12, 120) + 31) & ~31)


def unblocked_volume_bytes(D):
    return 4 * D * H * pitch(W) * 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    from bench import device_info
    from oracle import oracle as O
    from primestereomatch_b200 import DispEst, capi, synth
    if not torch.cuda.is_available() or capi.lib().psm_device_count() < 1:
        raise SystemExit("bench_blocked.py needs a CUDA device")
    L = capi.lib()
    stream = torch.cuda.Stream()

    def bind(de):
        capi.check(L.psm_set_stream(de.handle, C.c_void_p(stream.cuda_stream)), de.handle)

    def frame(de):
        de.CostConst_GPU(); de.CostFilter_GPU()
        capi.check(L.psm_disp_select_device(de.handle), de.handle)

    def timed(de):
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(stream); frame(de); ev1.record(stream)
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1), de.stage_ms(1), de.stage_ms(2), de.stage_ms(3)

    def maps(de):
        de.DispSelect_GPU()
        return de.lDisMap.copy(), de.rDisMap.copy()

    failures = []

    def check_band(de, l8, r8, D, what):
        got = maps(de)
        lc, rc = (synth.to_f32(np.ascontiguousarray(a[:2 * BAND])) for a in (l8, r8))
        _, _, lraw, rraw = O.cost_const(lc, rc, D)
        lf, rf = O.cost_filter(lc, rc, lraw, rraw)
        del lraw, rraw
        ld, rd = O.wta(lf, np.uint16)[:BAND], O.wta(rf, np.uint16)[:BAND]
        ok = bool(np.array_equal(got[0][:BAND].astype(np.uint16), ld) and np.array_equal(got[1][:BAND].astype(np.uint16), rd))
        if not ok:
            failures.append(f"{what}: rows [0, {BAND}) differ from the oracle")
        return got, ok

    overhead = []
    for D in OVERHEAD_D:
        l8, r8, _ = synth.stereo_pair_u8(W, H, D)
        kinds = [None] + [b for b in OVERHEAD_BLOCKS if b <= D]
        ctxs = {b: DispEst(l8, r8, D, block_slices=b) for b in kinds}
        try:
            for de in ctxs.values():
                bind(de)
                for _ in range(args.warmup):
                    frame(de)
            torch.cuda.synchronize()
            samples = {b: [] for b in kinds}
            for _ in range(args.steps):
                for b in kinds:
                    samples[b].append(timed(ctxs[b]))
            want, ok = check_band(ctxs[None], l8, r8, D, f"D={D} unblocked")
            for b in kinds:
                fr, s1, s2, s3 = (float(np.median([s[i] for s in samples[b]])) for i in range(4))
                vol = float(np.median([s[1] + s[2] + s[3] for s in samples[b]]))
                ent = {"D": D, "block_slices": b, "frame_ms": round(fr, 3), "stage1_ms": round(s1, 3),
                       "stage2_ms": round(s2, 3), "stage3_ms": round(s3, 3), "volume_ms": round(vol, 3)}
                if b is None:
                    ent["band_parity"] = ok
                    base = (fr, vol)
                else:
                    got = maps(ctxs[b])
                    same = bool(np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]))
                    if not same:
                        failures.append(f"D={D} block {b}: maps differ from the unblocked context's")
                    ent.update({"maps_equal_unblocked": same, "frame_overhead_pct": round(100 * (fr / base[0] - 1), 2),
                                "volume_overhead_pct": round(100 * (vol / base[1] - 1), 2)})
                overhead.append(ent)
                print(json.dumps({"progress": ent}), file=sys.stderr, flush=True)
        finally:
            for de in ctxs.values():
                de.close()
            torch.cuda.synchronize()

    reach = []
    for D in REACH_D:
        l8, r8, _ = synth.stereo_pair_u8(W, H, D)
        first = None
        for b in REACH_BLOCKS:
            torch.cuda.synchronize()
            free0, _ = torch.cuda.mem_get_info()
            with DispEst(l8, r8, D, map_bits=16, block_slices=b) as de:
                bind(de)
                frame(de)
                torch.cuda.synchronize()
                free1, _ = torch.cuda.mem_get_info()
                for _ in range(args.warmup):
                    frame(de)
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ev0.record(stream)
                for _ in range(args.steps):
                    frame(de)
                ev1.record(stream)
                torch.cuda.synchronize()
                ms = ev0.elapsed_time(ev1) / args.steps
                ent = {"D": D, "block_slices": b, "map_bits": 16, "frame_ms": round(ms, 2), "fps": round(1000.0 / ms, 2),
                       "stage2_ms": round(de.stage_ms(2), 2), "context_gib": round((free0 - free1) / 2**30, 2),
                       "unblocked_volumes_gib": round(unblocked_volume_bytes(D) / 2**30, 1)}
                if first is None:
                    first, ok = check_band(de, l8, r8, D, f"D={D} block {b}")
                    ent["band_parity"] = ok
                else:
                    got = maps(de)
                    same = bool(np.array_equal(got[0], first[0]) and np.array_equal(got[1], first[1]))
                    if not same:
                        failures.append(f"D={D} block {b}: maps differ from block {REACH_BLOCKS[0]}")
                    ent["maps_equal_block_%d" % REACH_BLOCKS[0]] = same
                ent["max_disparity_in_map"] = int(max(first[0].max(), first[1].max()))
            reach.append(ent)
            print(json.dumps({"progress": ent}), file=sys.stderr, flush=True)

    if failures:
        raise SystemExit("parity failed: " + "; ".join(failures))
    line = {"workload": "blocked_1920x1080", "gpu": device_info(0), "steps": args.steps, "warmup": args.warmup,
            "parity": "passed", "overhead": overhead, "reach": reach}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
