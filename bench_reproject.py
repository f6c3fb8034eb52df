"""Cost of reprojection to 3D points (psm_reproject_device) on one GPU; prints one JSON line.

Maps: the winner-take-all maps of the synthetic 1920 x 1080 stereo pair of bench.py (both views), at D = 128 on a u8
context and at D = 256 on a u16 context, computed once per context.  Q: a stereoRectify-shaped matrix with cx - cx' != 0.
Per workload, with handle_missing off and on in alternating rounds: ms per psm_reproject_device call over both views
(CUDA events around `steps` calls on the context's stream, after `warmup` calls); the medians over the rounds are
reported.  Bytes are the algorithm's, from shapes: the maps read once (twice with handle_missing: the min-reduction reads
them first) and 12 bytes per pixel written; achieved GB/s and the share of the H100 SXM's 3.35 TB/s HBM3 bandwidth follow
from the median time.  Parity, in the first round: both full-frame views against tests/reproject_oracle.py.

TorchStereo.match: ms per frame at D = 128 without and with points=(Q, Q), in alternating rounds (CUDA events around
`frames` calls on torch's current stream).

Usage: python bench_reproject.py [--steps 200] [--warmup 20] [--frames 10]
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

WORKLOADS = [(128, 8), (256, 16)]        # (D, map bits)
ROUNDS = 3
HBM_BYTES_PER_S = 3.35e12                # H100 SXM data sheet
# stereoRectify's Q for a 1920 x 1080 rig (f = 1400 px, baseline 0.12 m, cx - cx' = 3.5 px)
Q = np.array([[1.0, 0.0, 0.0, -960.25], [0.0, 1.0, 0.0, -541.75], [0.0, 0.0, 0.0, 1400.0],
              [0.0, 0.0, 1.0 / 0.12, 3.5 / 0.12]], np.float64)


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
    from primestereomatch_b200.torch_stereo import TorchStereo
    import reproject_oracle as RP
    if not torch.cuda.is_available() or capi.lib().psm_device_count() < 1:
        raise SystemExit("bench_reproject.py needs a CUDA device")
    W, H = 1920, 1080
    npix = W * H
    L = capi.lib()
    q = (C.c_double * 16)(*Q.ravel())
    results, parity = [], True
    for D, bits in WORKLOADS:
        l8, r8, _ = synth.stereo_pair_u8(W, H, D)
        mb = bits // 8
        per = {hm: {"handle_missing": bool(hm), "ms_per_call": []} for hm in (0, 1)}
        with DispEst(synth.to_f32(l8), synth.to_f32(r8), D, map_bits=bits) as de:
            stream = torch.cuda.Stream()   # the context runs on this stream, so the events bracket the calls
            capi.check(L.psm_set_stream(de.handle, C.c_void_p(stream.cuda_stream)), de.handle)
            de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
            maps = (de.lDisMap.copy(), de.rDisMap.copy())
            out = [torch.empty((H, W, 3), dtype=torch.float32, device="cuda") for _ in range(2)]
            for rnd in range(ROUNDS):
                for hm in (0, 1):
                    call = lambda: capi.check(L.psm_reproject_device(de.handle, 0, q, q, hm, out[0].data_ptr(),   # noqa: E731
                                                                     out[1].data_ptr(), 12 * W), de.handle)
                    for _ in range(args.warmup):
                        call()
                    torch.cuda.synchronize()
                    per[hm]["ms_per_call"].append(event_ms(stream, args.steps, call))
                    if rnd == 0:
                        call()
                        torch.cuda.synchronize()
                        for v in (0, 1):
                            try:
                                RP.assert_points_equal(out[v].cpu().numpy(), RP.reproject(maps[v], Q, hm), "bench")
                            except AssertionError:
                                parity = False
        for hm, res in per.items():
            ms = float(np.median(res["ms_per_call"]))
            nbytes = 2 * npix * mb * (2 if hm else 1) + 2 * npix * 12
            res.update(D=D, map_bits=bits, views=2, bytes=nbytes, ms_per_call_median=round(ms, 4),
                       ms_per_call=[round(x, 4) for x in res["ms_per_call"]],
                       gb_per_s=round(nbytes / (ms * 1e-3) / 1e9, 1),
                       share_of_hbm_peak=round(nbytes / (ms * 1e-3) / HBM_BYTES_PER_S, 3))
            results.append(res)

    D = 128
    l8, r8, _ = synth.stereo_pair_u8(W, H, D)
    lt, rt = torch.from_numpy(l8).cuda(), torch.from_numpy(r8).cuda()
    frame = {"without points": [], "with points": []}
    with TorchStereo(W, H, D) as ts:
        stream = torch.cuda.current_stream()
        for rnd in range(ROUNDS):
            for name, pts in (("without points", None), ("with points", (Q, Q))):
                call = lambda: ts.match(lt, rt, points=pts)   # noqa: E731
                call()
                torch.cuda.synchronize()
                frame[name].append(round(event_ms(stream, args.frames, call), 3))
    torch_res = {k: {"ms_per_frame": v, "median": float(np.median(v))} for k, v in frame.items()}

    info = device_info(0)
    print(json.dumps({"bench": "reproject", "gpu": info["name"], **gpu_clocks(), "width": W, "height": H,
                      "steps": args.steps, "warmup": args.warmup, "rounds": ROUNDS, "q": Q.ravel().tolist(),
                      "parity": parity, "reproject": results, "torch_stereo_d128": torch_res}))


if __name__ == "__main__":
    main()
