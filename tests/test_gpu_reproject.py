"""GPU: reprojection to 3D points (psm_reproject_device / psm_read_points) through the C-ABI against the CPU restatement
tests/reproject_oracle.py (pinned to cv2.reprojectImageTo3D by golden_reproject.json): every golden case on both
views and both map sources, both map formats, a 1080p map, every kind of context, padded rows, argument and state
errors, the maps and selection outputs left untouched, launch counts, TorchStereo and the C++ demo.

Equality: every non-NaN value bit for bit and NaN at the same positions (the device's NaN payload is its own).  Maps are
injected as tests/test_gpu_speckle.py does: one-hot cost slices written with psm_write_cost_slice."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from primestereomatch_b200 import DispEst, capi, synth
import reproject_oracle as RP

pytestmark = pytest.mark.gpu

with open(os.path.join(GOLDEN, "golden_reproject.json")) as f:
    GOLD = json.load(f)
CASES = np.load(os.path.join(GOLDEN, "reproject_cases.npz"))
QS = {k[2:]: CASES[k] for k in CASES.files if k.startswith("q_")}
MAPS = {k[4:]: CASES[k] for k in CASES.files if k.startswith("map_")}
Q0, Q1 = QS["rectify_shift"], QS["rectify_zero"]
ONLY = capi.PSM_SPECKLE_ONLY


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def qbuf(q):
    return None if q is None else (C.c_double * 16)(*np.asarray(q, np.float64).ravel())


def images(W, H, seed):
    rng = np.random.default_rng(seed)
    l8 = (rng.integers(0, 4, (H, W, 3)) * 85).astype(np.uint8)
    return synth.to_f32(l8), synth.to_f32(np.roll(l8, -1, axis=1).copy())


def inject_maps(de, ld, rd=None):
    assert de.CostConst_GPU() == 0 and de.CostFilter_GPU() == 0
    for d in range(de.d_begin, de.d_begin + de.d_count):
        de.write_cost_slice(0, d, np.where(ld == 0, np.inf, ld != d).astype(np.float32))
        if rd is not None:
            de.write_cost_slice(1, d, np.where(rd == 0, np.inf, rd != d).astype(np.float32))
    assert de.DispSelect_GPU() == 0
    assert np.array_equal(de.lDisMap, ld)


def context_for(m):
    H, W = m.shape
    bits = 16 if m.dtype == np.uint16 else 8
    return DispEst(*images(W, H, seed=W + H), max(int(m.max()) + 1, 2), map_bits=bits)


def device_maps(de, which):
    import torch
    dt = torch.uint16 if de.map_bits == 16 else torch.uint8
    both = de.rDisMap is not None
    lt = torch.empty((de.hei, de.wid), dtype=dt, device="cuda")
    rt = torch.empty_like(lt) if both else None
    row = de.wid * lt.element_size()
    capi.check(capi.lib().psm_copy_maps_device(de.handle, which, lt.data_ptr(), row, rt.data_ptr() if both else None, row),
               de.handle)
    de.sync()
    return lt.cpu().numpy(), (rt.cpu().numpy() if both else None)


def device_points(de, which, ql, qr, hm, pad=0):
    """psm_reproject_device into CUDA buffers with rows of 12 W + pad bytes -> (left, right) (H, W, 3) host arrays,
    and the untouched gap bytes of each row"""
    import torch
    H, W = de.hei, de.wid
    step = 12 * W + pad
    bufs = [None if q is None else torch.full((H * step // 4 + 1,), -7.0, dtype=torch.float32, device="cuda")
            for q in (ql, qr)]
    rc = capi.lib().psm_reproject_device(de.handle, which, qbuf(ql), qbuf(qr), int(hm),
                                         *[None if b is None else b.data_ptr() for b in bufs], step)
    capi.check(rc, de.handle)
    de.sync()
    out = []
    for b in bufs:
        if b is None:
            out.append(None)
            continue
        raw = b.cpu().numpy()[:H * step // 4].reshape(H, step // 4)
        assert (raw[:, 3 * W:] == -7.0).all(), "bytes between the rows were written"
        assert raw.size * 4 < b.numel() * 4 and b.cpu().numpy()[-1] == -7.0
        out.append(raw[:, :3 * W].reshape(H, W, 3).copy())
    return out


def check_views(de, which, ld, rd, q, hm, what, pad=0):
    gl, gr = device_points(de, which, q, q if rd is not None else None, hm, pad)
    RP.assert_points_equal(gl, RP.reproject(ld, q, hm), f"{what} left")
    if rd is not None:
        RP.assert_points_equal(gr, RP.reproject(rd, q, hm), f"{what} right")
    return gl, gr


# ---- cv2's own results --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", sorted(MAPS))
def test_synthetic_golden_cases(key):
    """every golden map with every Q, handle_missing off and on: the left view against cv2's hash, the right (the
    map upside down) against the restatement; then the post-processed maps (speckle removal alone, so zeros remain,
    and the default post-filter) through psm_read_points"""
    m = MAPS[key]
    gold = {(e["q"], e["hm"]): e["sha"] for e in GOLD["synthetic"] if e["map"] == key}
    rd = m[::-1].copy()
    with context_for(m) as de:
        inject_maps(de, m, rd)
        for (qk, hm), sha in sorted(gold.items()):
            gl, _ = check_views(de, 0, m, rd, QS[qk], hm, f"{key} {qk} hm {hm}")
            assert RP.sha(gl) == sha, (key, qk, hm)
        for setting in ((ONLY, 2, 0), (capi.PSM_SPECKLE_OFF, 0, 0)):
            de.setSpeckleFilter(*setting)
            assert de.PostProcess_GPU() == 0
            pl, pr = de.lDisMap.copy(), de.rDisMap.copy()
            for qk in ("rectify_shift", "nan", "w_row_zero"):
                for hm in (False, True):
                    for view, mm in (("left", pl), ("right", pr)):
                        RP.assert_points_equal(de.reproject(QS[qk], view, "post", hm), RP.reproject(mm, QS[qk], hm),
                                               f"{key} post {setting} {qk} {view} hm {hm}")


@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_scenes_against_the_golden(scene, scenes, oracle_scene_results):
    _, _, l, r = scenes[scene]
    ref = oracle_scene_results[scene]
    with DispEst(l, r, 64) as de:
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        assert np.array_equal(de.lDisMap, ref["ld"]) and np.array_equal(de.rDisMap, ref["rd"])
        for e in (e for e in GOLD["scenes"] if e["scene"] == scene):
            got = de.reproject(QS[e["q"]], "left" if e["view"] == "l" else "right", "selection", bool(e["hm"]))
            assert RP.sha(got) == e["sha"], (scene, e)
        de.PostProcess_GPU()
        check_views(de, 1, de.lDisMap, de.rDisMap, Q0, True, f"{scene} post-processed")


def test_full_1080p_maps_both_formats():
    H, W = 1080, 1920
    rng = np.random.default_rng(5)
    for bits, D in ((8, 12), (16, 12)):
        dt = np.uint16 if bits == 16 else np.uint8
        ld = rng.integers(0, D, (H, W)).astype(dt)
        rd = rng.integers(1, D, (H, W)).astype(dt)
        with DispEst(*images(W, H, seed=1), D, map_bits=bits) as de:
            inject_maps(de, ld, rd)
            for q in (Q0, QS["random1"]):
                for hm in (False, True):
                    check_views(de, 0, ld, rd, q, hm, f"1080p u{bits} hm {hm}")


# ---- every kind of context; nothing else changes -------------------------------------------------------------------------
KINDS = [("unblocked", {}), ("blocked", {"block_slices": 16}), ("multi", {"devices": [0, 0]}),
         ("multi-blocked", {"devices": [0, 0, 0], "block_slices": 8}), ("range", {"min_disp": 17}),
         ("left-only", {}), ("u16", {"map_bits": 16}), ("u16 range multi", {"map_bits": 16, "min_disp": 5, "devices": [0, 0]})]


@pytest.mark.parametrize("kind,kw", KINDS, ids=[k for k, _ in KINDS])
def test_context_kinds(kind, kw):
    W, H, D = 200, 120, 64
    l, r = synth.stereo_pair_f32(W, H, D, seed=8)[:2]
    L = capi.lib()
    with DispEst(l, r, D, **kw) as de:
        left_only = kind == "left-only"
        if left_only:
            de.setViews("left")
        de.setCostOutput(True); de.setRunnerUpOutput(True)
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        de.setLRCheck(0 if left_only else 1)
        de.PostProcess_GPU()
        sel, post = device_maps(de, 0), device_maps(de, 1)
        costs, runner = de._read_output(L.psm_read_costs, 3), de._read_output(L.psm_read_runner_up, 2)
        masks = (de.lValid.copy(), de.rValid.copy())
        if "range" in kind:
            nz = sel[0][sel[0] != 0]
            assert nz.size and nz.min() >= kw["min_disp"], "not absolute disparities"
        for which, maps in ((0, sel), (1, post)):
            for hm in (False, True):
                check_views(de, which, maps[0], maps[1], Q0, hm, f"{kind} which {which} hm {hm}", pad=8)
                RP.assert_points_equal(de.reproject(Q1, "left", ("selection", "post")[which], hm),
                                       RP.reproject(maps[0], Q1, hm), f"{kind} read_points which {which}")
        assert all(np.array_equal(a, b) for a, b in zip(device_maps(de, 0), sel) if a is not None)
        assert all(np.array_equal(a, b) for a, b in zip(device_maps(de, 1), post) if a is not None)
        for got, was in ((de._read_output(L.psm_read_costs, 3), costs), (de._read_output(L.psm_read_runner_up, 2), runner)):
            for v in (0,) if left_only else (0, 1):
                assert got[v].tobytes() == was[v].tobytes(), f"{kind}: costs / runner-up of view {v} changed"
        if not left_only:
            mask = np.zeros((H, W), np.uint8)
            for v in (0, 1):
                capi.check(L.psm_read_valid_mask(de.handle, v, ptr(mask), W), de.handle)
                assert np.array_equal(mask, masks[v]), f"{kind}: mask {v} changed"
        else:
            import torch
            buf = torch.empty((H, W, 3), dtype=torch.float32, device="cuda")
            assert L.psm_reproject_device(de.handle, 0, None, qbuf(Q0), 0, None, buf.data_ptr(), 12 * W) == capi.PSM_ESTATE
            out = np.empty((H, W, 3), np.float32)
            assert L.psm_read_points(de.handle, 1, 1, qbuf(Q0), 0, ptr(out), 12 * W) == capi.PSM_ESTATE
            check_views(de, 0, sel[0], None, Q0, True, "left-only after the refusal")


def test_disparity_shard_after_the_fused_exchange():
    W, H, D, SPLIT = 96, 64, 48, 20
    l, r = synth.stereo_pair_f32(W, H, D, seed=4)[:2]
    L = capi.lib()
    des = [DispEst(l, r, D, d_begin=0, d_count=SPLIT), DispEst(l, r, D, d_begin=SPLIT, d_count=D - SPLIT)]
    try:
        bufs = (C.c_void_p * 2)()
        for k, de in enumerate(des):
            p = C.c_void_p()
            capi.check(L.psm_p2p_create_buffer(de.handle, 2, C.byref(p)), de.handle)
            bufs[k] = p.value
        for k, de in enumerate(des):
            capi.check(L.psm_p2p_set_peers(de.handle, bufs, 2, k), de.handle)
        for de in des:
            de.CostConst_GPU(); de.CostFilter_GPU()
        for de in des:
            capi.check(L.psm_disp_select_keys_p2p(de.handle), de.handle)
        for de in des:
            de.sync()
        for de in des:
            capi.check(L.psm_disp_reduce_p2p(de.handle), de.handle)
        for de in des:
            de.sync()
        with DispEst(l, r, D) as whole:
            whole.CostConst_GPU(); whole.CostFilter_GPU(); whole.DispSelect_GPU()
            want = (whole.lDisMap.copy(), whole.rDisMap.copy())
        for k, de in enumerate(des):
            assert [np.array_equal(a, b) for a, b in zip(device_maps(de, 0), want)] == [True, True]
            check_views(de, 0, *want, Q0, True, f"fused shard {k}")
    finally:
        for de in des:
            de.close()


# ---- arguments, states, launches -----------------------------------------------------------------------------------------
def test_invalid_arguments_and_states():
    import torch
    H, W = 30, 40
    ld, rd = (np.random.default_rng(s).integers(0, 16, (H, W)).astype(np.uint8) for s in (1, 2))
    L = capi.lib()
    q = qbuf(Q0)
    buf = torch.zeros((2, H * W * 3 + 4), dtype=torch.float32, device="cuda")
    lp, rp = buf[0].data_ptr(), buf[1].data_ptr()
    host = np.zeros((H, W * 3 + 1), np.float32)
    with DispEst(*images(W, H, seed=2), 16) as de:
        h = de.handle
        before = de.launch_count()
        assert L.psm_reproject_device(h, 0, q, q, 0, lp, rp, 12 * W) == capi.PSM_ESTATE     # no selection yet
        assert L.psm_read_points(h, 1, 0, q, 0, ptr(host), host.strides[0]) == capi.PSM_ESTATE
        inject_maps(de, ld, rd)
        assert L.psm_reproject_device(h, 1, q, None, 0, lp, None, 12 * W) == capi.PSM_ESTATE  # no post-process yet
        n = de.launch_count()
        bad = {"Q without a buffer": (0, q, q, 0, lp, None, 12 * W),
               "buffer without a Q": (0, None, q, 0, lp, rp, 12 * W),
               "no view": (0, None, None, 0, None, None, 12 * W),
               "which 2": (2, q, q, 0, lp, rp, 12 * W), "which -1": (-1, q, None, 0, lp, None, 12 * W),
               "handle_missing 2": (0, q, q, 2, lp, rp, 12 * W),
               "short row_step": (0, q, q, 0, lp, rp, 12 * W - 4),
               "row_step not a multiple of 4": (0, q, None, 0, lp, None, 12 * W + 2),
               "misaligned left": (0, q, q, 0, lp + 2, rp, 12 * W),
               "misaligned right": (0, q, q, 0, lp, rp + 1, 12 * W)}
        for what, args in bad.items():
            assert L.psm_reproject_device(h, *args) == capi.PSM_EINVAL and L.psm_last_error(h), what
        for what, args in {"view 2": (0, 2, q, 0, ptr(host), 12 * W), "view -1": (0, -1, q, 0, ptr(host), 12 * W),
                           "null Q": (0, 0, None, 0, ptr(host), 12 * W), "null dst": (0, 0, q, 0, None, 12 * W),
                           "which 3": (3, 0, q, 0, ptr(host), 12 * W), "hm -1": (0, 0, q, -1, ptr(host), 12 * W),
                           "short step": (0, 0, q, 0, ptr(host), 12 * W - 1)}.items():
            assert L.psm_read_points(h, *args) == capi.PSM_EINVAL, what
        assert L.psm_reproject_device(None, 0, q, q, 0, lp, rp, 12 * W) == capi.PSM_EINVAL
        assert L.psm_read_points(None, 0, 0, q, 0, ptr(host), 12 * W) == capi.PSM_EINVAL
        assert de.launch_count() == n, "a refused call launched"
        assert not buf.any().item(), "a refused call wrote"
        with pytest.raises(capi.PsmError):
            de.reproject(Q0, "middle", "selection")
        with pytest.raises(capi.PsmError):
            de.reproject(Q0, "left", "final")
        # the context is still usable, and an unpadded host destination works too
        check_views(de, 0, ld, rd, Q0, True, "after the refusals")
        assert L.psm_read_points(h, 0, 1, q, 0, ptr(host), host.strides[0]) == 0
        RP.assert_points_equal(host[:, :3 * W].reshape(H, W, 3), RP.reproject(rd, Q0), "read_points padded host rows")
        assert (host[:, 3 * W] == 0).all()
        assert before <= n


def test_launch_counts():
    H, W = 20, 30
    for kw in ({}, {"devices": [0, 0]}, {"block_slices": 4}):
        with DispEst(*images(W, H, seed=3), 8, **kw) as de:
            de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
            de.PostProcess_GPU()
            for which in (0, 1):
                for hm, views in ((0, "l"), (0, "lr"), (1, "l"), (1, "lr"), (1, "r")):
                    n = de.launch_count()
                    device_points(de, which, Q0 if "l" in views else None, Q0 if "r" in views else None, hm)
                    assert de.launch_count() - n == 1 + hm, (kw, which, hm, views)
                    n = de.launch_count()
                    de.reproject(Q0, "left", ("selection", "post")[which], bool(hm))
                    assert de.launch_count() - n == 1 + hm


# ---- TorchStereo and the demo ----------------------------------------------------------------------------------------------
def test_torch_stereo_points_on_a_held_back_stream_and_a_batch():
    import torch
    from primestereomatch_b200.torch_stereo import TorchStereo
    W, H, D = 160, 96, 48
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=13)
    lt, rt = torch.from_numpy(l8).cuda(), torch.from_numpy(r8).cuda()
    with TorchStereo(W, H, D) as ts, DispEst(l8, r8, D) as de:                # the same pixels, uploaded from the host
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        sel = (de.reproject(Q0, "left", "selection", True), de.reproject(Q1, "right", "selection", True))
        de.PostProcess_GPU()
        post = de.reproject(Q0, "left", "post")
        torch.cuda.synchronize()
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            torch.cuda._sleep(20_000_000)                                   # the frames' stream is held back
            lm, rm, lp, rp = ts.match(lt, rt, points=(Q0, Q1), handle_missing=True)
        torch.cuda.synchronize()
        assert lp.shape == (H, W, 3) and lp.dtype == torch.float32
        RP.assert_points_equal(lp.cpu().numpy(), sel[0], "TorchStereo left points")
        RP.assert_points_equal(rp.cpu().numpy(), sel[1], "TorchStereo right points")
        out = ts.match(lt, rt, post_process=True, costs=True, points=(Q0, None))
        assert len(out) == 6 and out[5] is None
        RP.assert_points_equal(out[4].cpu().numpy(), post, "TorchStereo post-processed points")
        lb, rb = torch.stack([lt, lt]), torch.stack([rt, rt])
        _, _, bl, br = ts.match(lb, rb, points=(None, Q1), handle_missing=True)
        assert bl is None and br.shape == (2, H, W, 3)
        for b in range(2):
            RP.assert_points_equal(br[b].cpu().numpy(), sel[1], f"TorchStereo batch frame {b}")
        with pytest.raises((TypeError, ValueError)):
            ts.match(lt, rt, points=(None, None))
        with pytest.raises(TypeError):
            ts.match(lt, rt, points=Q0)


def test_cpp_demo_points_flag(tmp_path, scenes, oracle_scene_results):
    exe = os.path.join(ROOT, "primestereomatch_b200", "host", "dispest_demo")
    if not os.path.exists(exe):
        pytest.skip("dispest_demo not built")
    _, _, l, r = scenes["Cones"]
    H, W, _ = l.shape
    l.tofile(tmp_path / "l.f32"); r.tofile(tmp_path / "r.f32")
    Q0.astype(np.float64).tofile(tmp_path / "q.f64")
    tail = [str(W), str(H), "64", str(tmp_path / "l.f32"), str(tmp_path / "r.f32"), str(tmp_path / "l.u8"),
            str(tmp_path / "r.u8")]
    out = subprocess.run([exe, "--points", str(tmp_path / "q.f64"), str(tmp_path / "p.xyz")] + tail,
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    final = np.fromfile(tmp_path / "l.u8", np.uint8).reshape(H, W)
    got = np.fromfile(tmp_path / "p.xyz", np.float32).reshape(H, W, 3)
    RP.assert_points_equal(got, RP.reproject(final, Q0), "demo --points")
