"""GPU: rectification in ingest (psm_set_rectify) against the CPU restatement, bit for bit.

The core check: a context that rectifies raw camera frames holds the same channel planes and gradient, and computes the
same maps, as a context of the same kind fed the oracle's rectified frame (rectify_oracle.remap) through
psm_set_images_u8.  It covers every golden case, every entry path, every kind of context, launch counts, every rejected
argument, switching off, TorchStereo and the demo."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import rectify_cases
import rectify_oracle as RO
from primestereomatch_b200 import DispEst, capi, synth
from test_gpu_parity import assert_same

torch = pytest.importorskip("torch")

from primestereomatch_b200.torch_stereo import TorchStereo, frame_layout  # noqa: E402

pytestmark = pytest.mark.gpu

CASES = rectify_cases.load()
D = 64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEMO = os.path.join(ROOT, "primestereomatch_b200", "host", "dispest_demo")


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def rectified(srcs, maps):
    return tuple(RO.remap(s, *m) for s, m in zip(srcs, maps))


def scene_rig(scenes, name, margin=(36, 22)):
    """a scene's pair as raw frames of a synthetic rig: (srcs, maps), the maps cropping margin px off each side"""
    l8, r8, _, _ = scenes[name]
    SH, SW = l8.shape[:2]
    W, H = SW - 2 * margin[0], SH - 2 * margin[1]
    return (l8, r8), tuple(synth.rectify_maps(W, H, SW, SH, view=v) for v in range(2))


def pair(srcs, maps, d=D, kw=None, setup=None):
    """(rect, plain): DispEst contexts of one kind, rect rectifying srcs through maps, plain fed the oracle's frames"""
    kw = kw or {}
    lo, ro = rectified(srcs, maps)
    rect, plain = DispEst(lo, ro, d, **kw), DispEst(lo, ro, d, **kw)
    for de in (rect, plain):
        if setup:
            setup(de)
    SH, SW = srcs[0].shape[:2]
    rect.setRectify(maps[0], maps[1], (SW, SH))
    rect.setInputImages(*srcs)
    return rect, plain


def compare_planes(a, b, what, views=(0, 1)):
    for view in views:
        for plane in (0, 1, 2, 12):
            assert_same(a.read_guide_plane(view, plane).view(np.uint32), b.read_guide_plane(view, plane).view(np.uint32),
                        f"{what} view {view} plane {plane}")


def run_maps(de, post=False):
    de.CostFilter_GPU()
    de.DispSelect_GPU()
    if post:
        de.PostProcess_GPU()


def compare_maps(a, b, what):
    assert_same(a.lDisMap, b.lDisMap, what + " lDisMap")
    if b.rDisMap is not None:
        assert_same(a.rDisMap, b.rDisMap, what + " rDisMap")


# -- every golden case: planes and gradient ---------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_planes_every_golden_case(case):
    name, srcs, maps, _ = case
    rect, plain = pair(srcs, maps, d=4)
    with rect, plain:
        rect.CostConst_GPU()
        plain.CostConst_GPU()
        compare_planes(rect, plain, name)


# -- maps after the post-filter on the scenes -------------------------------------------------------------------------
@pytest.mark.parametrize("setup", ["lr1", "lr2", "speckle", "speckle_lr1"])
@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_scene_maps_after_post_process(scene, setup, scenes):
    srcs, maps = scene_rig(scenes, scene)

    def configure(de):
        if setup.endswith("lr1"):
            de.setLRCheck(1)
        if setup == "lr2":
            de.setLRCheck(2)
        if setup.startswith("speckle"):
            de.setSpeckleFilter(1, 100, 1)

    rect, plain = pair(srcs, maps, setup=configure)
    with rect, plain:
        for de in (rect, plain):
            de.CostConst_GPU()
            run_maps(de, post=True)
        compare_maps(rect, plain, f"{scene} {setup}")
        if setup != "speckle":
            assert_same(rect.lValid, plain.lValid, "lValid")
            assert_same(rect.rValid, plain.rValid, "rValid")


# -- every entry path --------------------------------------------------------------------------------------------------
def device_layout(img, layout):
    """(tensor, channels) of a BGR numpy frame in one of the layouts psm_set_images_device_planes reads"""
    t = torch.from_numpy(np.ascontiguousarray(img)).cuda()
    if layout == "hwc_bgr":
        return t, "bgr"
    if layout == "hwc_rgb":
        return t.flip(2).contiguous(), "rgb"
    if layout == "chw_rgb":
        return t.flip(2).permute(2, 0, 1).contiguous(), "rgb"
    if layout == "bgra":
        return torch.cat([t, torch.full_like(t[:, :, :1], 77)], 2).contiguous(), "bgr"
    raise ValueError(layout)


def set_planes(de, lt, rt, channels, hw):
    L = capi.lib()
    pix, lf, row, col, _ = frame_layout(lt, *hw, channels)
    _, rf, row2, col2, _ = frame_layout(rt, *hw, channels)
    assert (row, col) == (row2, col2)
    capi.check(L.psm_set_images_device_planes(de.handle, pix, (C.c_void_p * 3)(*lf[0]), (C.c_void_p * 3)(*rf[0]), row,
                                              col), de.handle)


def feed(de, srcs, path):
    """the frame pair srcs into de through one entry path, then psm_cost_const"""
    L = capi.lib()
    l, r = (np.ascontiguousarray(s) for s in srcs)
    hw = l.shape[:2]
    if path == "u8":
        de.setInputImages(l, r)
        de.CostConst_GPU()
        return
    if path == "u8_async":
        capi.check(L.psm_set_images_u8_async(de.handle, ptr(l), l.strides[0], ptr(r), r.strides[0]), de.handle)
        capi.check(L.psm_set_images_commit(de.handle), de.handle)
    elif path == "side_by_side":
        t = torch.from_numpy(np.concatenate([l, r], axis=1)).cuda()
        W = l.shape[1]
        set_planes(de, t[:, :W], t[:, W:], "bgr", hw)
    else:
        (lt, ch), (rt, _) = device_layout(l, path), device_layout(r, path)
        set_planes(de, lt, rt, ch, hw)
    torch.cuda.synchronize()
    capi.check(L.psm_cost_const(de.handle), de.handle)


PATHS = ["u8", "u8_async", "hwc_bgr", "hwc_rgb", "chw_rgb", "bgra", "side_by_side"]


@pytest.mark.parametrize("path", PATHS)
def test_entry_paths(path, scenes):
    srcs, maps = scene_rig(scenes, "Cones")
    rect, plain = pair(srcs, maps)
    with rect, plain:
        feed(rect, srcs, path)
        plain.CostConst_GPU()
        compare_planes(rect, plain, path)
        for de in (rect, plain):
            run_maps(de)
        compare_maps(rect, plain, path)


# -- every kind of context ---------------------------------------------------------------------------------------------
CONTEXTS = {
    "unblocked": (D, {}, None),
    "blocked": (D, dict(block_slices=24), None),
    "u16_d300": (300, dict(map_bits=16), None),
    "range": (D, dict(min_disp=16), None),
    "left_only": (D, {}, lambda de: de.setViews("left")),
    "multi2": (D, dict(devices=[0, 0]), None),
    "multi3": (D, dict(devices=[0, 0, 0]), None),
    "multi2_blocked": (D, dict(devices=[0, 0], block_slices=20), None),
    "multi3_blocked": (D, dict(devices=[0, 0, 0], block_slices=7), None),
}


@pytest.mark.parametrize("path", ["u8", "hwc_bgr"])
@pytest.mark.parametrize("name", list(CONTEXTS))
def test_context_kinds(name, path, scenes):
    d, kw, setup = CONTEXTS[name]
    srcs, maps = scene_rig(scenes, "Teddy")
    rect, plain = pair(srcs, maps, d, kw, setup)
    with rect, plain:
        feed(rect, srcs, path)
        plain.CostConst_GPU()
        views = (0,) if name == "left_only" else (0, 1)
        compare_planes(rect, plain, name, views)
        for de in (rect, plain):
            run_maps(de, post=True)
        compare_maps(rect, plain, name)


# -- launch counts -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name, path", [(n, p) for n in ("unblocked", "blocked", "multi2")
                                         for p in ("u8", "u8_async", "hwc_bgr", "side_by_side")
                                         if not (n == "multi2" and p == "u8_async")])   # no async upload on multi-device
def test_launch_counts(name, path, scenes):
    d, kw, setup = CONTEXTS[name]
    srcs, maps = scene_rig(scenes, "Cones")
    rect, plain = pair(srcs, maps, d, kw, setup)
    # a multi-device context's other shards receive the rectified frame as planes, never run an ingest of their own:
    # its count is that of the same context fed device planes
    plain_path = "hwc_bgr" if kw.get("devices") else path
    with rect, plain:
        for de, p, frames in ((rect, path, srcs), (plain, plain_path, rectified(srcs, maps))):
            n0 = de.launch_count()
            feed(de, frames, p)
            run_maps(de, post=True)
            de.sync()
            de.n = de.launch_count() - n0
        assert rect.n == plain.n


# -- arguments ---------------------------------------------------------------------------------------------------------
def set_rectify(de, sw, sh, maps, steps=None):
    L = capi.lib()
    arrs = [m for pair_ in maps for m in pair_]
    steps = steps or [a.strides[0] if a is not None else 0 for a in arrs]
    args = []
    for a, s in zip(arrs, steps):
        args += [None if a is None else ptr(a), s]
    return L.psm_set_rectify(de.handle, sw, sh, *args)


def test_rejected_arguments_leave_the_context_unchanged(scenes):
    srcs, maps = scene_rig(scenes, "Cones")
    SH, SW = srcs[0].shape[:2]
    rect, plain = pair(srcs, maps)
    H, W = maps[0][1].shape
    with rect, plain:
        xy, a = maps[0]
        bad = [
            (SW, SH, ((None, a), maps[1]), None),                          # null map while turning on
            (SW, SH, (maps[0], (xy, None)), None),
            (SW, SH, (maps[0], maps[1]), [W * 4 - 1, W * 2, W * 4, W * 2]),   # steps below a row
            (SW, SH, (maps[0], maps[1]), [W * 4, W * 2, W * 4, W * 2 - 1]),
            (0, SH, maps, None),                                            # source sides outside 1..32767
            (SW, 32768, maps, None),
            (-1, SH, maps, None),
            (0, 0, maps, None),                                             # mixes of zero and non-zero
            (0, 0, ((None, None), (None, None)), [0, 0, 4, 0]),
            (SW, SH, ((None, None), (None, None)), [0, 0, 0, 0]),
        ]
        for sw, sh, m, steps in bad:
            assert set_rectify(rect, sw, sh, m, steps) == capi.PSM_EINVAL, (sw, sh, steps)
        # still rectifying with the maps of the setRectify call
        rect.CostConst_GPU()
        plain.CostConst_GPU()
        compare_planes(rect, plain, "after rejected arguments")


def test_pending_upload_is_a_state_error(scenes):
    L = capi.lib()
    srcs, maps = scene_rig(scenes, "Cones")
    rect, plain = pair(srcs, maps)
    with rect, plain:
        l, r = srcs
        capi.check(L.psm_set_images_u8_async(rect.handle, ptr(l), l.strides[0], ptr(r), r.strides[0]), rect.handle)
        assert set_rectify(rect, 0, 0, ((None, None), (None, None))) == capi.PSM_ESTATE
        capi.check(L.psm_set_images_commit(rect.handle), rect.handle)
        capi.check(L.psm_cost_const(rect.handle), rect.handle)
        plain.CostConst_GPU()
        compare_planes(rect, plain, "after the state error")


@pytest.mark.parametrize("name", ["unblocked", "multi2"])
def test_float_frames_and_short_steps_are_refused(name, scenes):
    L = capi.lib()
    d, kw, _ = CONTEXTS[name]
    srcs, maps = scene_rig(scenes, "Cones")
    rect, plain = pair(srcs, maps, d, kw)
    SH, SW = srcs[0].shape[:2]
    H, W = maps[0][1].shape
    with rect, plain:
        f = np.zeros((SH, SW, 3), np.float32)
        fw = np.zeros((H, W, 3), np.float32)
        h = rect.handle
        for img in (f, fw):
            assert L.psm_set_images(h, ptr(img), img.strides[0], ptr(img), img.strides[0]) == capi.PSM_EINVAL
            assert "8-bit" in L.psm_last_error(h).decode()
            t = torch.from_numpy(img).cuda()
            assert L.psm_set_images_device(h, t.data_ptr(), img.strides[0], t.data_ptr(), img.strides[0]) == capi.PSM_EINVAL
            p = (C.c_void_p * 3)(t.data_ptr(), t.data_ptr() + 4, t.data_ptr() + 8)
            assert L.psm_set_images_device_planes(h, capi.PSM_PIX_F32, p, p, img.strides[0], 12) == capi.PSM_EINVAL
            if name == "unblocked":
                assert L.psm_set_images_async(h, ptr(img), img.strides[0], ptr(img), img.strides[0]) == capi.PSM_EINVAL
        l = np.ascontiguousarray(srcs[0])
        assert L.psm_set_images_u8(h, ptr(l), SW * 3 - 1, ptr(l), SW * 3) == capi.PSM_EINVAL
        t = torch.from_numpy(l).cuda()
        p = (C.c_void_p * 3)(t.data_ptr(), t.data_ptr() + 1, t.data_ptr() + 2)
        assert L.psm_set_images_device_planes(h, capi.PSM_PIX_U8, p, p, (SW - 1) * 3, 3) == capi.PSM_EINVAL
        assert L.psm_set_images_device_planes(h, capi.PSM_PIX_U8, p, p, (SW - 1) * 3 + 1, 3) == capi.PSM_OK
        rect.setInputImages(*srcs)
        rect.CostConst_GPU()
        plain.CostConst_GPU()
        compare_planes(rect, plain, "after refused frames")


@pytest.mark.parametrize("name", ["unblocked", "blocked", "multi2"])
def test_switching_off_equals_a_never_set_context(name, scenes):
    d, kw, _ = CONTEXTS[name]
    srcs, maps = scene_rig(scenes, "Teddy")
    lo, ro = rectified(srcs, maps)
    rect, plain = pair(srcs, maps, d, kw)
    with rect, plain:
        rect.CostConst_GPU()
        rect.setRectify(None, None, None)
        rect.setInputImages(lo, ro)
        for de in (rect, plain):
            n0 = de.launch_count()
            de.CostConst_GPU()
            run_maps(de, post=True)
            de.sync()
            de.n = de.launch_count() - n0
        assert rect.n == plain.n
        compare_planes(rect, plain, "off")
        compare_maps(rect, plain, "off")
        f = synth.to_f32(lo), synth.to_f32(ro)   # float frames are accepted again
        rect.setInputImages(*f)
        plain.setInputImages(*f)
        for de in (rect, plain):
            de.CostConst_GPU()
        compare_planes(rect, plain, "off, float frames")


# -- TorchStereo and the demo ------------------------------------------------------------------------------------------
def test_torch_stereo_points_on_a_side_by_side_frame(scenes):
    srcs, maps = scene_rig(scenes, "Cones")
    lo, ro = rectified(srcs, maps)
    H, W = lo.shape[:2]
    SH, SW = srcs[0].shape[:2]
    Q = np.array([[1, 0, 0, -W / 2], [0, 1, 0, -H / 2], [0, 0, 0, 400.0], [0, 0, 1 / 0.12, 0]])
    with TorchStereo(W, H, D) as rect, TorchStereo(W, H, D) as plain:
        rect.setRectify(maps[0], maps[1], (SW, SH))
        cam = torch.from_numpy(np.concatenate(srcs, axis=1)).cuda()
        with pytest.raises(ValueError):
            rect.match(cam[:, :SW].float(), cam[:, SW:].float())
        with pytest.raises(ValueError):   # frames of the context's size, not the source's
            rect.match(torch.from_numpy(lo).cuda(), torch.from_numpy(ro).cuda())
        got = rect.match(cam[:, :SW], cam[:, SW:], post_process=True, points=(Q, Q))
        want = plain.match(torch.from_numpy(lo).cuda(), torch.from_numpy(ro).cuda(), post_process=True, points=(Q, Q))
        torch.cuda.synchronize()
        for g, w, what in zip(got, want, ("lmap", "rmap", "lpts", "rpts")):
            assert_same(g.cpu().numpy().view(np.uint8), w.cpu().numpy().view(np.uint8), what)


def test_demo_rectifies(tmp_path, scenes):
    srcs, maps = scene_rig(scenes, "Cones")
    lo, ro = rectified(srcs, maps)
    H, W = lo.shape[:2]
    SH, SW = srcs[0].shape[:2]
    files = {}
    for name, arr in (("l.u8", srcs[0]), ("r.u8", srcs[1]), ("l.f32", synth.to_f32(lo)), ("r.f32", synth.to_f32(ro))):
        files[name] = str(tmp_path / name)
        np.ascontiguousarray(arr).tofile(files[name])
    for v, name in enumerate(("l.map", "r.map")):
        files[name] = str(tmp_path / name)
        with open(files[name], "wb") as f:
            f.write(np.ascontiguousarray(maps[v][0]).tobytes() + np.ascontiguousarray(maps[v][1]).tobytes())
    out = {k: str(tmp_path / k) for k in ("rl", "rr", "pl", "pr")}
    subprocess.run([DEMO, "--rectify", str(SW), str(SH), files["l.map"], files["r.map"], str(W), str(H), str(D),
                    files["l.u8"], files["r.u8"], out["rl"], out["rr"]], check=True, capture_output=True)
    subprocess.run([DEMO, str(W), str(H), str(D), files["l.f32"], files["r.f32"], out["pl"], out["pr"]], check=True,
                   capture_output=True)
    for a, b in (("rl", "pl"), ("rr", "pr")):
        got, want = np.fromfile(out[a], np.uint8), np.fromfile(out[b], np.uint8)
        assert got.size == W * H
        assert_same(got, want, a)
