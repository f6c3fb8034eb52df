"""Range contexts (psm_create_range) against the full range on one GPU; prints one JSON line.

Workload: the synthetic 1920 x 1080 pair of bench.py (synth.stereo_pair_u8), both views, default filter, u8 frames
uploaded from the host; a frame is ingest -> CVC -> CVF -> WTA, maps left on the device.  Four pairs of contexts, a
[0, max_disp) context against one over the upper half of its range, the rig whose nearest background sits at a known
depth:
  - u8 maps: [0, 256) against [128, 256), and against [129, 256), a start that is not a multiple of 4 (the cost
    construction's grouped path needs one);
  - u16 maps: [0, 512) against [256, 512);
  - blocked at B = 128: [0, 2048) against [1024, 2048).
Both contexts of a pair are alive at once and run in turn, one frame each per round, so that drift on a shared card hits
both alike.  Medians over the rounds of the frame time (CUDA events around the frame on the device's stream, after
psm_wait_stream, psm_signal_stream back).  Device memory per context is the drop in the device's free memory across its
creation.  Before the line is printed, the range context's maps are checked against the arg-min over [min_disp, max_disp)
of the full context's filtered volume (unblocked pairs: read in place through psm_device_ptr), or, for the blocked pair,
against the keys of a blocked context owning those slices of the full problem (psm_create_blocked with d_begin = min_disp).

Usage: python bench_range.py [--steps 15] [--warmup 3]
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
CONFIGS = [("u8 [128, 256)", 256, 128, {}), ("u8 [129, 256)", 256, 129, {}), ("u16 [256, 512)", 512, 256, {}),
           ("blocked B=128 [1024, 2048)", 2048, 1024, dict(block_slices=128))]


class _Dev:
    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = dict(shape=shape, typestr="<f4", data=(ptr, False), version=2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    from bench import device_info
    from primestereomatch_b200 import DispEst, capi, synth
    if not torch.cuda.is_available() or capi.lib().psm_device_count() < 1:
        raise SystemExit("bench_range.py needs a CUDA device")
    L = capi.lib()
    stream = torch.cuda.current_stream(0)
    sp = C.c_void_p(stream.cuda_stream)

    def frame(de):
        capi.check(L.psm_wait_stream(de.handle, sp), de.handle)
        de.CostConst_GPU(); de.CostFilter_GPU()
        capi.check(L.psm_disp_select_device(de.handle), de.handle)
        capi.check(L.psm_signal_stream(de.handle, sp), de.handle)

    def timed(de):
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(stream); frame(de); ev1.record(stream)
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1)

    def created(make):
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info(0)[0]
        de = make()
        torch.cuda.synchronize()
        return de, free0 - torch.cuda.mem_get_info(0)[0]

    def restricted_argmin(de, lo, D):
        """the arg-min over [lo, D) of the full unblocked context's filtered volumes (NaN and +inf never win, lowest d on
        ties, 0 where nothing wins)"""
        ptr, pitch = C.c_void_p(), C.c_size_t()
        out = []
        for v in (0, 1):
            capi.check(L.psm_device_ptr(de.handle, v, C.byref(ptr), C.byref(pitch)), de.handle)
            vol = torch.as_tensor(_Dev(ptr.value, (D, H, pitch.value)), device="cuda:0")[lo:, :, :W]
            vol = torch.nan_to_num(vol, nan=float("inf"))
            best, idx = vol.min(dim=0)   # the first index of the minimum on CUDA
            out.append(torch.where(torch.isinf(best) & (best > 0), 0, idx + lo).cpu().numpy())
        return out

    def shard_keys(l8, r8, D, lo, bits, kw):
        """the maps of the keys of a context owning [lo, D) of the full problem"""
        with DispEst(l8, r8, D, map_bits=bits, d_begin=lo, d_count=D - lo, **kw) as sh:
            sh.CostConst_GPU(); sh.CostFilter_GPU()
            keys = torch.empty((2, H * W), dtype=torch.int64, device="cuda:0")
            capi.check(L.psm_disp_select_keys(sh.handle, keys[0].data_ptr(), keys[1].data_ptr()), sh.handle)
            sh.sync()
            return [(keys[v] & 0xFFFFFFFF).view(H, W).cpu().numpy() for v in (0, 1)]

    out, failures = [], []
    for name, D, lo, kw in CONFIGS:
        l8, r8, _ = synth.stereo_pair_u8(W, H, min(D, 256))
        bits = 16 if D > 256 else 8
        full, mem_full = created(lambda: DispEst(l8, r8, D, map_bits=bits, **kw))
        rng, mem_rng = created(lambda: DispEst(l8, r8, D, map_bits=bits, min_disp=lo, **kw))
        try:
            for _ in range(args.warmup):
                frame(full); frame(rng)
            torch.cuda.synchronize()
            t = {"full": [], "range": []}
            for _ in range(args.steps):
                for de, key in ((full, "full"), (rng, "range")):
                    t[key].append(timed(de))
            rng.DispSelect_GPU()
            if kw.get("block_slices"):
                want = shard_keys(l8, r8, D, lo, bits, kw)
            else:
                full.CostConst_GPU(); full.CostFilter_GPU(); full.sync()
                want = restricted_argmin(full, lo, D)
            same = bool(np.array_equal(rng.lDisMap, want[0]) and np.array_equal(rng.rDisMap, want[1]))
            if not same:
                failures.append(f"{name}: the range context's maps differ from the restricted arg-min")
            m_full, m_rng = float(np.median(t["full"])), float(np.median(t["range"]))
            out.append({"config": name, "max_disp": D, "min_disp": lo, "frame_ms_full": round(m_full, 3),
                        "frame_ms_range": round(m_rng, 3), "time_ratio": round(m_rng / m_full, 3),
                        "spread_ms_full": round(float(np.max(t["full"]) - np.min(t["full"])), 3),
                        "spread_ms_range": round(float(np.max(t["range"]) - np.min(t["range"])), 3),
                        "mem_mib_full": round(mem_full / 2**20, 1), "mem_mib_range": round(mem_rng / 2**20, 1),
                        "maps_ok": same})
        finally:
            full.close(); rng.close()
    print(json.dumps({"bench": "range", "device": device_info(0), "W": W, "H": H, "steps": args.steps,
                      "results": out, "ok": not failures, "failures": failures}))
    if failures:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
