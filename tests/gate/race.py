"""Two contexts' frames with one thread's shared-memory limit set held open while the other thread sets it (run by
tests/test_gpu_threads.py under LD_PRELOAD=libsmem_gate.so, without torch).

argv: a JSON file {"gate", "min_bytes", "timeout_ms", "frames" (an .npz of la, ra, lb, rb u8 frames), "out" (an .npz to
write), "a", "b"}, where "a" and "b" each give a context: {"D", "kwargs" (DispEst's), "window", "eps", "fgf" (a rate or
null), "volumes" (read the raw and filtered volumes)}.  The contexts are created on this thread.  Thread A runs a's
frame with the gate armed at min_bytes; once A is held, thread B runs b's.  Writes each context's outputs to "out" and
prints one JSON line: each frame's error (null when it returned PSM_OK), whether A was held, whether the gate reached the
CUDA runtime, and its counters."""
import ctypes as C
import json
import os
import sys
import threading

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from primestereomatch_b200 import DispEst, capi  # noqa: E402


def frame(de, spec, l8, r8, out, name):
    try:
        de.setInputImages(l8, r8)
        de.CostConst_GPU()
        if spec["volumes"]:
            out[name + "_lraw"], out[name + "_rraw"] = de.read_cost_volume(0), de.read_cost_volume(1)
        if spec["fgf"]:
            de.setSubsampleRate(spec["fgf"])
            de.CostFilter_FGF_GPU()
        else:
            de.CostFilter_GPU()
        if spec["volumes"]:
            out[name + "_lvol"], out[name + "_rvol"] = de.read_cost_volume(0), de.read_cost_volume(1)
        de.DispSelect_GPU()
        out[name + "_lmap"], out[name + "_rmap"] = de.lDisMap.copy(), de.rDisMap.copy()
        return None
    except capi.PsmError as e:
        return f"code {e.code}: {e}"


def main():
    with open(sys.argv[1]) as f:
        spec = json.load(f)
    gate = C.CDLL(spec["gate"])
    fr = np.load(spec["frames"])
    ctxs = {}
    for name in ("a", "b"):
        s = spec[name]
        blank = np.zeros(fr["l" + name].shape, np.uint8)
        ctxs[name] = DispEst(blank, blank, s["D"], **s["kwargs"])
        if s["window"] is not None:
            ctxs[name].setGuidedFilter(s["window"], s["eps"])
    out, errors = {}, {}

    def run(name):
        errors[name] = frame(ctxs[name], spec[name], fr["l" + name], fr["r" + name], out, name)

    gate.gate_arm(spec["min_bytes"], spec["timeout_ms"])
    ta = threading.Thread(target=run, args=("a",))
    ta.start()
    held = bool(gate.gate_wait_held(10000))
    tb = threading.Thread(target=run, args=("b",))
    tb.start()
    ta.join()
    tb.join()
    n = [C.c_int() for _ in range(3)]
    gate.gate_stats(*(C.byref(x) for x in n))
    for de in ctxs.values():
        de.close()
    np.savez(spec["out"], **out)
    print(json.dumps({"errors": errors, "held": held, "forwards": gate.gate_forwards(),
                      "gate": dict(zip(("holds", "releases", "timeouts"), (x.value for x in n)))}))


if __name__ == "__main__":
    main()
