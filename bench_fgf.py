"""Time of the Fast Guided Filter stage (psm_cost_filter_fgf, psm_stage_ms stage 4: guide, low-resolution and
up-sampling kernels of both views) on one GPU; prints one JSON line.

Frame: the synthetic 1920 x 1080 x 128 stereo pair of bench.py, CVC costs, window 8, s = 1, 2, 4, 8 (boxes 17, 9, 5, 3).
With --baseline PATH, a second build of libprime_stereo_b200.so (for example one made from an earlier commit) is loaded
beside the in-tree one and the two are timed alternately, round by round, in the same process on the same card, and
their filtered volumes are compared on the timed frame (slices 0, 64, 127 of both views, bit for bit).

Usage: python bench_fgf.py [--steps 20] [--warmup 3] [--rounds 5] [--baseline PATH]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

RATES = [1, 2, 4, 8]
W, H, D = 1920, 1080, 128


def load(path):
    """the C-ABI of the library at `path`, with capi's argument types"""
    from primestereomatch_b200 import capi
    saved = capi.LIB_PATH, capi._lib
    capi.LIB_PATH, capi._lib = path, None
    try:
        return capi.lib()
    finally:
        capi.LIB_PATH, capi._lib = saved


class Ctx:
    def __init__(self, L, l, r):
        from primestereomatch_b200 import capi
        self.L, self.capi = L, capi
        self.h = C.c_void_p()
        self.ok(L.psm_create(C.byref(self.h), W, H, D, 0))
        self.ok(L.psm_set_images(self.h, l.ctypes.data, l.strides[0], r.ctypes.data, r.strides[0]))

    def ok(self, rc):
        if rc != 0:
            text = self.L.psm_last_error(self.h) if self.h else b"?"
            raise self.capi.PsmError(rc, text.decode() if text else "?")

    def fgf_ms(self, s):
        """one CVC + FGF frame -> FGF stage ms (device events)"""
        self.ok(self.L.psm_cost_const(self.h))
        self.ok(self.L.psm_cost_filter_fgf(self.h, s))
        ms = C.c_float()
        self.ok(self.L.psm_stage_ms(self.h, 4, C.byref(ms)))
        return ms.value

    def slice(self, view, d):
        out = np.empty((H, W), np.float32)
        self.ok(self.L.psm_read_cost_slice(self.h, view, d, out.ctypes.data, out.strides[0]))
        return out

    def close(self):
        self.L.psm_destroy(self.h)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="timed frames per build, rate and round")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5, help="alternations of the builds per rate")
    ap.add_argument("--baseline", help="path of a second libprime_stereo_b200.so to time against the in-tree one")
    args = ap.parse_args()
    from bench import device_info
    from primestereomatch_b200 import capi, synth
    if capi.lib().psm_device_count() < 1:
        raise SystemExit("bench_fgf.py needs a CUDA device")
    l8, r8, _ = synth.stereo_pair_u8(W, H, D)
    l, r = np.ascontiguousarray(synth.to_f32(l8)), np.ascontiguousarray(synth.to_f32(r8))
    builds = {"tree": Ctx(capi.lib(), l, r)}
    if args.baseline:
        builds["baseline"] = Ctx(load(os.path.abspath(args.baseline)), l, r)
    results = []
    try:
        for s in RATES:
            times = {name: [] for name in builds}
            for name, ctx in builds.items():
                for _ in range(args.warmup):
                    ctx.fgf_ms(s)
            for _ in range(args.rounds):
                for name, ctx in builds.items():
                    times[name] += [ctx.fgf_ms(s) for _ in range(args.steps)]
            row = {"s": s, "box": 2 * (8 // s) + 1}
            for name, t in times.items():
                row[f"{name}_ms_median"] = round(float(np.median(t)), 4)
                row[f"{name}_ms_min"] = round(float(np.min(t)), 4)
            if "baseline" in builds:
                row["tree_over_baseline"] = round(row["tree_ms_median"] / row["baseline_ms_median"], 3)
                row["same_bits"] = all(np.array_equal(builds["tree"].slice(v, d).view(np.uint32),
                                                      builds["baseline"].slice(v, d).view(np.uint32))
                                       for v in (0, 1) for d in (0, 64, 127))
            results.append(row)
            print(json.dumps({"progress": row}), file=sys.stderr, flush=True)
    finally:
        for ctx in builds.values():
            ctx.close()
    print(json.dumps({"workload": f"fgf_stage_{W}x{H}x{D}", "gpu": device_info(0), "steps": args.steps,
                      "warmup": args.warmup, "rounds": args.rounds, "results": results}), flush=True)


if __name__ == "__main__":
    main()
