"""The cost of PSM_OPT_RUNNER_UP (each pixel's runner-up away from the winner) on one GPU; prints one JSON line.

Workload: the synthetic 1920 x 1080 pair of bench.py (synth.stereo_pair_u8), both views, default filter, u8 frames
uploaded from the host; a frame is ingest -> CVC -> CVF -> WTA (maps left on the device), and with the option on also
the runner-up into device tensors (psm_copy_runner_up_device).  Six configurations, the ones whose path differs:
  - D = 128 unblocked (the selection kernel keeps the four-lowest lists in its one read of the volume);
  - D = 2048 at block_slices 128 and D = 128 at block_slices 16 (the block fold keeps the running lists; the small
    blocks move them most often per slice);
  - two shards co-located on device 0 at D = 256 (a list scan of every shard's slices, the slots and their reduce);
  - D = 128 unblocked and D = 128 at block_slices 16 with PSM_OPT_COSTS on in both contexts (what the runner-up adds
    to the costs; blocked, the block fold tracks the costs and the running lists in one read).
For each, one context with the option off and one with it on are alive at once and run in turn, one frame each per
round, so that drift on a shared card hits both alike.  Medians over the rounds of the frame time (CUDA events around
the frame on the first device's stream after psm_wait_stream, psm_signal_stream back).  Before the line is printed, the
maps of the two contexts are compared (they must be identical).

Usage: python bench_runner_up.py [--steps 10] [--warmup 2]
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
CONFIGS = [("unblocked D=128", 128, {}, False), ("blocked D=2048 B=128", 2048, dict(block_slices=128), False),
           ("blocked D=128 B=16", 128, dict(block_slices=16), False), ("2 shards D=256", 256, dict(devices=[0, 0]), False),
           ("unblocked D=128, costs on in both", 128, {}, True),
           ("blocked D=128 B=16, costs on in both", 128, dict(block_slices=16), True)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    from bench import device_info
    from primestereomatch_b200 import DispEst, capi, synth
    if not torch.cuda.is_available() or capi.lib().psm_device_count() < 1:
        raise SystemExit("bench_runner_up.py needs a CUDA device")
    L = capi.lib()
    stream = torch.cuda.current_stream(0)
    sp = C.c_void_p(stream.cuda_stream)
    runner = torch.empty((2, 2, H, W), dtype=torch.float32, device="cuda:0")
    costs = torch.empty((2, 3, H, W), dtype=torch.float32, device="cuda:0")

    def frame(de, on):
        capi.check(L.psm_wait_stream(de.handle, sp), de.handle)
        de.CostConst_GPU(); de.CostFilter_GPU()
        capi.check(L.psm_disp_select_device(de.handle), de.handle)
        if de.cost_output:
            capi.check(L.psm_copy_costs_device(de.handle, costs[0].data_ptr(), costs[1].data_ptr(), W * 4), de.handle)
        if on:
            capi.check(L.psm_copy_runner_up_device(de.handle, runner[0].data_ptr(), runner[1].data_ptr(), W * 4),
                       de.handle)
        capi.check(L.psm_signal_stream(de.handle, sp), de.handle)

    def timed(de, on):
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(stream); frame(de, on); ev1.record(stream)
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1)

    out, failures = [], []
    for name, D, kw, with_costs in CONFIGS:
        l8, r8, _ = synth.stereo_pair_u8(W, H, min(D, 256))
        bits = 16 if D > 256 else 8
        off, on = DispEst(l8, r8, D, map_bits=bits, **kw), DispEst(l8, r8, D, map_bits=bits, **kw)
        try:
            on.setRunnerUpOutput(True)
            if with_costs:
                off.setCostOutput(True)
                on.setCostOutput(True)
            for _ in range(args.warmup):
                frame(off, False); frame(on, True)
            torch.cuda.synchronize()
            t = {False: [], True: []}
            for _ in range(args.steps):
                for de, flag in ((off, False), (on, True)):
                    t[flag].append(timed(de, flag))
            off.DispSelect_GPU(); on.DispSelect_GPU()
            same = bool(np.array_equal(off.lDisMap, on.lDisMap) and np.array_equal(off.rDisMap, on.rDisMap))
            if not same:
                failures.append(f"{name}: the maps differ with the option on")
            m_off, m_on = float(np.median(t[False])), float(np.median(t[True]))
            out.append({"config": name, "frame_ms_off": round(m_off, 3), "frame_ms_on": round(m_on, 3),
                        "overhead_pct": round(100.0 * (m_on - m_off) / m_off, 2),
                        "spread_ms_off": round(float(np.max(t[False]) - np.min(t[False])), 3), "maps_identical": same})
        finally:
            off.close(); on.close()
    print(json.dumps({"bench": "runner_up", "device": device_info(0), "W": W, "H": H, "steps": args.steps,
                      "results": out, "ok": not failures, "failures": failures}))
    if failures:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
