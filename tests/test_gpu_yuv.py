"""GPU: YUV frames converted in ingest (psm_set_images_yuv, _yuv_async, psm_set_images_device_yuv, TorchStereo.match(yuv=))
against the CPU restatement, bit for bit.

The core check: a context fed a YUV frame holds the same channel planes and gradient, and computes the same maps, as a
context of the same kind fed the oracle's BGR frame (yuv_oracle.bgr, then rectify_oracle.remap with rectification on)
through psm_set_images_u8.  It covers every format through every entry path, every kind of context, rectification, the
halves of one side-by-side frame, every (Y, U, V) triple, format switches on one context, launch counts, every rejected
argument, a held-back compute stream and the demo."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import rectify_oracle as RO
import yuv_oracle as YO
from primestereomatch_b200 import DispEst, capi, synth
from test_gpu_parity import assert_same

torch = pytest.importorskip("torch")

from primestereomatch_b200.torch_stereo import TorchStereo, yuv_layout  # noqa: E402

pytestmark = pytest.mark.gpu

D = 64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEMO = os.path.join(ROOT, "primestereomatch_b200", "host", "dispest_demo")
CODE = capi.YUV_FORMATS


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def scene_yuv(scenes, name, fmt, size=(448, 372)):
    """a scene's pair as YUV frames of fmt, cropped to size (W, H)"""
    l8, r8, _, _ = scenes[name]
    W, H = size
    return tuple(YO.from_bgr(np.ascontiguousarray(img[:H, :W]), fmt) for img in (l8, r8))


def expected(frames, fmt, maps=None):
    """the BGR frames a YUV pair stands for, rectified through maps when given"""
    out = tuple(YO.bgr(f, fmt) for f in frames)
    return out if maps is None else tuple(RO.remap(o, *m) for o, m in zip(out, maps))


def pair(frames, fmt, d=D, kw=None, setup=None, maps=None):
    """(yuv, plain): DispEst contexts of one kind; plain holds the oracle's BGR frames, yuv is set up to take frames"""
    kw = kw or {}
    lo, ro = expected(frames, fmt, maps)
    yuv, plain = DispEst(lo, ro, d, **kw), DispEst(lo, ro, d, **kw)
    for de in (yuv, plain):
        if setup:
            setup(de)
    if maps is not None:
        SW, SH = YO.size(frames[0], fmt)
        yuv.setRectify(maps[0], maps[1], (SW, SH))
    return yuv, plain


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


def set_device(handle, lt, rt, fmt, hw):
    """psm_set_images_device_yuv of two tensors, laid out by yuv_layout"""
    H, W = hw
    sampling, lf, *steps, _ = yuv_layout(lt, H, W, fmt)
    _, rf, *steps2, _ = yuv_layout(rt, H, W, fmt)
    assert steps == steps2
    return capi.lib().psm_set_images_device_yuv(handle, sampling, (C.c_void_p * 3)(*lf[0]), (C.c_void_p * 3)(*rf[0]),
                                                *steps)


def feed(de, frames, fmt, path):
    """the YUV pair into de through one entry path, then psm_cost_const"""
    L = capi.lib()
    l, r = (np.ascontiguousarray(f) for f in frames)
    W, H = YO.size(l, fmt)
    if path == "host":
        de.setInputImagesYUV(l, r, fmt)
        de.CostConst_GPU()
        return
    if path == "async":
        capi.check(L.psm_set_images_yuv_async(de.handle, CODE[fmt], ptr(l), l.strides[0], ptr(r), r.strides[0]), de.handle)
        capi.check(L.psm_set_images_commit(de.handle), de.handle)
    elif path == "device":
        capi.check(set_device(de.handle, torch.from_numpy(l).cuda(), torch.from_numpy(r).cuda(), fmt, (H, W)), de.handle)
    elif path == "side_by_side":   # both views in one frame, left | right
        t = torch.from_numpy(np.concatenate([l, r], axis=1)).cuda()
        capi.check(set_device(de.handle, t[:, :W], t[:, W:], fmt, (H, W)), de.handle)
    else:
        raise ValueError(path)
    torch.cuda.synchronize()
    capi.check(L.psm_cost_const(de.handle), de.handle)


# -- every format through every entry path -----------------------------------------------------------------------------
# planar 4:2:0 frames (I420, YV12) pack their chroma rows, so the halves of a side-by-side one are not two frames
@pytest.mark.parametrize("fmt, path", [(f, p) for f in YO.FORMATS for p in ("host", "async", "device", "side_by_side")
                                       if not (p == "side_by_side" and f in ("i420", "yv12"))])
def test_formats_and_entry_paths(fmt, path, scenes):
    frames = scene_yuv(scenes, "Cones", fmt)
    yuv, plain = pair(frames, fmt)
    with yuv, plain:
        feed(yuv, frames, fmt, path)
        plain.CostConst_GPU()
        compare_planes(yuv, plain, f"{fmt} {path}")
        for de in (yuv, plain):
            run_maps(de)
        compare_maps(yuv, plain, f"{fmt} {path}")


@pytest.mark.parametrize("fmt", YO.FORMATS)
def test_torch_stereo(fmt, scenes):
    frames = scene_yuv(scenes, "Teddy", fmt)
    lo, ro = expected(frames, fmt)
    H, W = lo.shape[:2]
    with TorchStereo(W, H, D) as yt, TorchStereo(W, H, D) as bt:
        lt, rt = (torch.from_numpy(f).cuda() for f in frames)
        got = yt.match(lt, rt, yuv=fmt, post_process=True)
        want = bt.match(torch.from_numpy(lo).cuda(), torch.from_numpy(ro).cuda(), post_process=True)
        # a batch of two: the pair, then the pair swapped
        gb = yt.match(torch.stack([lt, rt]), torch.stack([rt, lt]), yuv=fmt)
        wb = bt.match(torch.from_numpy(np.stack([lo, ro])).cuda(), torch.from_numpy(np.stack([ro, lo])).cuda())
        torch.cuda.synchronize()
        for g, w, what in zip(got + gb, want + wb, ("lmap", "rmap", "batch lmap", "batch rmap")):
            assert_same(g.cpu().numpy(), w.cpu().numpy(), f"{fmt} {what}")
        with pytest.raises(ValueError):   # a BGR tensor is not a YUV frame
            yt.match(torch.from_numpy(lo).cuda(), torch.from_numpy(ro).cuda(), yuv=fmt)


# -- every kind of context, with and without rectification --------------------------------------------------------------
CONTEXTS = {
    "unblocked": (D, {}, None),
    "blocked": (D, dict(block_slices=24), None),
    "u16_d300": (300, dict(map_bits=16), None),
    "range": (D, dict(min_disp=16), None),
    "left_only": (D, {}, lambda de: de.setViews("left")),
    "multi2": (D, dict(devices=[0, 0]), None),
    "multi3_blocked": (D, dict(devices=[0, 0, 0], block_slices=7), None),
}


def rig(frames, fmt, margin=(36, 22)):
    """the maps of a synthetic rig that crops margin px off each side of the frames"""
    SW, SH = YO.size(frames[0], fmt)
    W, H = SW - 2 * margin[0], SH - 2 * margin[1]
    return tuple(synth.rectify_maps(W, H, SW, SH, view=v) for v in range(2))


@pytest.mark.parametrize("rectify", [False, True], ids=["plain", "rectify"])
@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("name", list(CONTEXTS))
def test_context_kinds(name, path, rectify, scenes):
    d, kw, setup = CONTEXTS[name]
    fmt = "yuyv" if rectify else "nv12"
    frames = scene_yuv(scenes, "Teddy", fmt)
    maps = rig(frames, fmt) if rectify else None
    yuv, plain = pair(frames, fmt, d, kw, setup, maps)
    with yuv, plain:
        feed(yuv, frames, fmt, path)
        plain.CostConst_GPU()
        views = (0,) if name == "left_only" else (0, 1)
        compare_planes(yuv, plain, name, views)
        for de in (yuv, plain):
            run_maps(de, post=True)
        compare_maps(yuv, plain, name)


@pytest.mark.parametrize("fmt", ["yuyv", "nv12", "uyvy", "nv21"])
@pytest.mark.parametrize("path", ["host", "async", "side_by_side"])
def test_rectified_entry_paths(fmt, path, scenes):
    frames = scene_yuv(scenes, "Cones", fmt)
    maps = rig(frames, fmt)
    yuv, plain = pair(frames, fmt, maps=maps)
    with yuv, plain:
        feed(yuv, frames, fmt, path)
        plain.CostConst_GPU()
        compare_planes(yuv, plain, f"{fmt} {path} rectified")
        for de in (yuv, plain):
            run_maps(de)
        compare_maps(yuv, plain, f"{fmt} {path} rectified")


@pytest.mark.parametrize("fmt", ["yuyv", "nv12"])
def test_torch_stereo_side_by_side_camera_frame(fmt, scenes):
    """one side-by-side camera frame, rectified on the device: TorchStereo on its two halves"""
    frames = scene_yuv(scenes, "Cones", fmt)
    maps = rig(frames, fmt)
    lo, ro = expected(frames, fmt, maps)
    H, W = lo.shape[:2]
    SW, SH = YO.size(frames[0], fmt)
    Q = np.array([[1, 0, 0, -W / 2], [0, 1, 0, -H / 2], [0, 0, 0, 400.0], [0, 0, 1 / 0.12, 0]])
    with TorchStereo(W, H, D) as yt, TorchStereo(W, H, D) as bt:
        yt.setRectify(maps[0], maps[1], (SW, SH))
        cam = torch.from_numpy(np.concatenate(frames, axis=1)).cuda()
        small = torch.from_numpy(YO.frame(0, fmt, W, H)).cuda()
        with pytest.raises(ValueError):   # frames of the context's size, not the source's
            yt.match(small, small, yuv=fmt)
        got = yt.match(cam[:, :SW], cam[:, SW:], yuv=fmt, post_process=True, points=(Q, Q))
        want = bt.match(torch.from_numpy(lo).cuda(), torch.from_numpy(ro).cuda(), post_process=True, points=(Q, Q))
        torch.cuda.synchronize()
        for g, w, what in zip(got, want, ("lmap", "rmap", "lpts", "rpts")):
            assert_same(g.cpu().numpy().view(np.uint8), w.cpu().numpy().view(np.uint8), what)


# -- every (Y, U, V) triple --------------------------------------------------------------------------------------------
def test_every_triple_through_the_device():
    frame = YO.all_triples()
    want = YO.all_triples_bgr()
    t = torch.from_numpy(frame).cuda()
    zeros = np.zeros((4096, 4096, 3), np.uint8)
    with DispEst(zeros, zeros, 4) as yuv, DispEst(want, want, 4) as plain:
        capi.check(set_device(yuv.handle, t, t, "yuyv", (4096, 4096)), yuv.handle)
        plain.CostConst_GPU()
        torch.cuda.synchronize()
        for plane in (0, 1, 2, 12):
            assert_same(yuv.read_guide_plane(0, plane).view(np.uint32), plain.read_guide_plane(0, plane).view(np.uint32),
                        f"plane {plane}")
        # and the planes are the triples' BGR as to_f32 scales it
        for c in range(3):
            assert_same(yuv.read_guide_plane(1, c), want[..., c].astype(np.float32) * np.float32(1 / 255.0), f"channel {c}")


# -- formats switched between frames on one live context ---------------------------------------------------------------
@pytest.mark.parametrize("name", ["unblocked", "multi2"])
def test_format_switches(name, scenes):
    d, kw, _ = CONTEXTS[name]
    seq = [("nv12", "host"), ("yuyv", "device"), ("bgr", "host"), ("i420", "host"), ("uyvy", "device"),
           ("yv12", "async"), ("nv21", "device"), ("yvyu", "async"), ("bgr", "host")]
    l8, r8, _, _ = scenes["Teddy"]
    crop = tuple(np.ascontiguousarray(i[:372, :448]) for i in (l8, r8))
    with DispEst(*crop, d, **kw) as live:
        for k, (fmt, path) in enumerate(seq):
            if path == "async" and name == "multi2":
                path = "host"   # no asynchronous upload on multi-device contexts
            scene = "Cones" if k % 2 else "Teddy"
            if fmt == "bgr":
                lo, ro = (np.ascontiguousarray(i[:372, :448]) for i in scenes[scene][:2])
                live.setInputImages(lo, ro)
                live.CostConst_GPU()
            else:
                frames = scene_yuv(scenes, scene, fmt)
                lo, ro = expected(frames, fmt)
                feed(live, frames, fmt, path)
            with DispEst(lo, ro, d, **kw) as plain:
                plain.CostConst_GPU()
                compare_planes(live, plain, f"step {k} {fmt}")
                for de in (live, plain):
                    run_maps(de, post=True)
                compare_maps(live, plain, f"step {k} {fmt}")


# -- launch counts -----------------------------------------------------------------------------------------------------
def feed_bgr_device(de, imgs):
    from primestereomatch_b200.torch_stereo import frame_layout
    lt, rt = (torch.from_numpy(np.ascontiguousarray(i)).cuda() for i in imgs)
    H, W = imgs[0].shape[:2]
    pix, lf, row, col, _ = frame_layout(lt, H, W)
    _, rf, _, _, _ = frame_layout(rt, H, W)
    capi.check(capi.lib().psm_set_images_device_planes(de.handle, pix, (C.c_void_p * 3)(*lf[0]), (C.c_void_p * 3)(*rf[0]),
                                                       row, col), de.handle)
    torch.cuda.synchronize()
    capi.check(capi.lib().psm_cost_const(de.handle), de.handle)


@pytest.mark.parametrize("name, path", [(n, p) for n in ("unblocked", "blocked", "multi2")
                                         for p in ("host", "async", "device")
                                         if not (n == "multi2" and p == "async")])
@pytest.mark.parametrize("rectify", [False, True], ids=["plain", "rectify"])
def test_launch_counts(name, path, rectify, scenes):
    d, kw, setup = CONTEXTS[name]
    fmt = "nv12"
    frames = scene_yuv(scenes, "Cones", fmt)
    maps = rig(frames, fmt) if rectify else None
    yuv, plain = pair(frames, fmt, d, kw, setup, maps)
    # one ingest launch and one halo pass per view, as for u8 frames; a multi-device context's other shards receive the
    # first shard's planes, as for device BGR planes
    with yuv, plain:
        counts = []
        for de, f in ((yuv, lambda: feed(yuv, frames, fmt, path)),
                      (plain, lambda: plain.CostConst_GPU() if not kw.get("devices") and path != "device"
                       else feed_bgr_device(plain, expected(frames, fmt, maps)))):
            n0 = de.launch_count()
            f()
            run_maps(de, post=True)
            de.sync()
            counts.append(de.launch_count() - n0)
        assert counts[0] == counts[1]


# -- arguments ---------------------------------------------------------------------------------------------------------
def test_rejected_arguments_leave_the_context_unchanged(scenes):
    L = capi.lib()
    fmt = "nv12"
    frames = scene_yuv(scenes, "Cones", fmt)
    yuv, plain = pair(frames, fmt)
    l, r = frames
    W, H = YO.size(l, fmt)
    with yuv, plain:
        feed(yuv, frames, fmt, "host")
        plain.CostConst_GPU()
        h = yuv.handle
        bad_host = [
            (0, ptr(l), W, ptr(r), W),                      # unknown formats
            (8, ptr(l), W, ptr(r), W),
            (-1, ptr(l), W, ptr(r), W),
            (CODE["nv12"], None, W, ptr(r), W),             # null frames
            (CODE["nv12"], ptr(l), W, None, W),
            (CODE["nv12"], ptr(l), W - 1, ptr(r), W),       # steps below a row
            (CODE["yuyv"], ptr(l), 2 * W - 1, ptr(r), 2 * W),
            (CODE["i420"], ptr(l), W + 2, ptr(r), W + 2),   # planar formats are contiguous
            (CODE["yv12"], ptr(l), W, ptr(r), W + 2),
        ]
        for args in bad_host:
            assert L.psm_set_images_yuv(h, *args) == capi.PSM_EINVAL, args[0]
            assert L.psm_set_images_yuv_async(h, *args) == capi.PSM_EINVAL, args[0]
        t = torch.from_numpy(l).cuda()
        p = t.data_ptr()
        yuv3 = (C.c_void_p * 3)(p, p + H * W, p + H * W + 1)
        null = (C.c_void_p * 3)(p, None, p + 1)
        bad_device = [
            (0, yuv3, yuv3, W, 1, W, 2),                    # unknown sampling
            (3, yuv3, yuv3, W, 1, W, 2),
            (capi.PSM_YUV_420, None, yuv3, W, 1, W, 2),     # null pointers
            (capi.PSM_YUV_420, yuv3, null, W, 1, W, 2),
            (capi.PSM_YUV_420, yuv3, yuv3, W - 1, 1, W, 2),   # steps below a row
            (capi.PSM_YUV_420, yuv3, yuv3, W, 1, W - 2, 2),
            (capi.PSM_YUV_420, yuv3, yuv3, W, 0, W, 2),       # zero column steps
            (capi.PSM_YUV_420, yuv3, yuv3, W, 1, W, 0),
            (capi.PSM_YUV_422, yuv3, yuv3, 2 * W, 2, 2 * W, 1 << 62),   # a row span that overflows
        ]
        for args in bad_device:
            assert L.psm_set_images_device_yuv(h, *args) == capi.PSM_EINVAL, args
        # still the frame of the first call
        capi.check(L.psm_cost_const(h), h)
        compare_planes(yuv, plain, "after rejected arguments")
        # the least steps a row spans are accepted
        assert L.psm_set_images_device_yuv(h, capi.PSM_YUV_420, yuv3, yuv3, W, 1, (W // 2 - 1) * 2 + 1, 2) == 0


@pytest.mark.parametrize("fmt, size", [("nv12", (63, 40)), ("yuyv", (63, 40)), ("nv12", (64, 39)), ("i420", (64, 39))])
def test_odd_sizes_are_refused(fmt, size):
    L = capi.lib()
    W, H = size
    img = np.zeros((H, W, 3), np.uint8)
    buf = np.zeros(4 * W * H, np.uint8)
    t = torch.zeros(4 * W * H, dtype=torch.uint8, device="cuda")
    p = t.data_ptr()
    with DispEst(img, img, 16) as de:
        h = de.handle
        step = W if fmt in YO.FORMATS_420 else 2 * W
        assert L.psm_set_images_yuv(h, CODE[fmt], ptr(buf), step, ptr(buf), step) == capi.PSM_EINVAL
        assert L.psm_set_images_yuv_async(h, CODE[fmt], ptr(buf), step, ptr(buf), step) == capi.PSM_EINVAL
        three = (C.c_void_p * 3)(p, p + 1, p + 2)
        sampling = capi.PSM_YUV_420 if fmt in YO.FORMATS_420 else capi.PSM_YUV_422
        assert L.psm_set_images_device_yuv(h, sampling, three, three, 4 * W, 1, 4 * W, 2) == capi.PSM_EINVAL
        assert "even" in L.psm_last_error(h).decode()
    if fmt == "yuyv" or H % 2 == 0:
        return
    # an odd height is fine for 4:2:2
    with DispEst(img, img, 16) as de:
        three = (C.c_void_p * 3)(p, p + 1, p + 3)
        assert L.psm_set_images_device_yuv(de.handle, capi.PSM_YUV_422, three, three, 2 * W, 2, 2 * W, 4) == capi.PSM_OK


def test_pending_upload_and_multi_device_async(scenes):
    L = capi.lib()
    fmt = "yuyv"
    frames = scene_yuv(scenes, "Cones", fmt)
    l, r = frames
    yuv, plain = pair(frames, fmt)
    with yuv, plain:
        h = yuv.handle
        capi.check(L.psm_set_images_yuv_async(h, CODE[fmt], ptr(l), l.strides[0], ptr(r), r.strides[0]), h)
        assert L.psm_set_images_yuv_async(h, CODE[fmt], ptr(l), l.strides[0], ptr(r), r.strides[0]) == capi.PSM_ESTATE
        assert L.psm_set_images_u8_async(h, ptr(l), l.strides[0], ptr(r), r.strides[0]) == capi.PSM_ESTATE
        capi.check(L.psm_set_images_commit(h), h)
        capi.check(L.psm_cost_const(h), h)
        plain.CostConst_GPU()
        compare_planes(yuv, plain, "after the state error")
    lo, ro = expected(frames, fmt)
    with DispEst(lo, ro, D, devices=[0, 0]) as multi:
        assert L.psm_set_images_yuv_async(multi.handle, CODE[fmt], ptr(l), l.strides[0], ptr(r),
                                          r.strides[0]) == capi.PSM_EINVAL


# -- a held-back compute stream ----------------------------------------------------------------------------------------
HOLD_MS = 250.0


def test_held_back_stream(scenes):
    """each YUV entry path issued while the context's stream is held back by a spin (as in test_gpu_stream_order): the
    host calls return once the caller's buffers are read, before the spin ends, and the device path reads the frame the
    held stream writes after psm_wait_stream"""
    L = capi.lib()
    fmt = "nv12"
    s = torch.cuda.Stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(s):
        torch.cuda._sleep(1_000_000)
        e0.record(s)
        torch.cuda._sleep(50_000_000)
        e1.record(s)
    e1.synchronize()
    cycles_per_ms = 50_000_000 / e0.elapsed_time(e1)

    def hold():
        done = torch.cuda.Event()
        with torch.cuda.stream(s):
            torch.cuda._sleep(int(HOLD_MS * cycles_per_ms))
            done.record(s)
        return done

    a, b = scene_yuv(scenes, "Cones", fmt), scene_yuv(scenes, "Teddy", fmt)
    W, H = YO.size(a[0], fmt)
    with DispEst(*expected(a, fmt), D) as live:
        h = live.handle
        capi.check(L.psm_set_stream(h, C.c_void_p(s.cuda_stream)), h)
        # outside the hold: the first asynchronous upload allocates the second staging set
        l, r = (np.array(f) for f in a)
        capi.check(L.psm_set_images_yuv_async(h, CODE[fmt], ptr(l), l.strides[0], ptr(r), r.strides[0]), h)
        capi.check(L.psm_set_images_commit(h), h)
        live.sync()
        for path, cur, other in (("host", b, a), ("async", a, b), ("device", b, a)):
            l, r = (np.array(f) for f in cur)
            done = hold()
            if path == "host":
                capi.check(L.psm_set_images_yuv(h, CODE[fmt], ptr(l), l.strides[0], ptr(r), r.strides[0]), h)
            elif path == "async":
                capi.check(L.psm_set_images_yuv_async(h, CODE[fmt], ptr(l), l.strides[0], ptr(r), r.strides[0]), h)
                capi.check(L.psm_set_images_commit(h), h)
            else:
                lt, rt = (torch.zeros(f.shape, dtype=torch.uint8, device="cuda") for f in cur)
                src = [torch.from_numpy(f).pin_memory() for f in (l, r)]
                with torch.cuda.stream(s):   # the frame is written on the held stream, after the spin
                    lt.copy_(src[0], non_blocking=True)
                    rt.copy_(src[1], non_blocking=True)
                capi.check(L.psm_wait_stream(h, C.c_void_p(s.cuda_stream)), h)
                capi.check(set_device(h, lt, rt, fmt, (H, W)), h)
            assert not done.query(), f"the hold ended before the {path} frame was issued"
            if path != "device":
                l[...], r[...] = other   # the caller reuses its buffers at once
            capi.check(L.psm_cost_const(h), h)
            run_maps(live)
            with DispEst(*expected(cur, fmt), D) as plain:
                plain.CostConst_GPU()
                run_maps(plain)
                compare_maps(live, plain, f"held {path}")
        torch.cuda.synchronize()


# -- the demo ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt, rectify", [("nv12", False), ("i420", False), ("yuyv", True)])
def test_demo(fmt, rectify, tmp_path, scenes):
    frames = scene_yuv(scenes, "Cones", fmt)
    maps = rig(frames, fmt) if rectify else None
    lo, ro = expected(frames, fmt, maps)
    H, W = lo.shape[:2]
    files = {}
    for name, arr in (("l.yuv", frames[0]), ("r.yuv", frames[1]), ("l.f32", synth.to_f32(lo)),
                      ("r.f32", synth.to_f32(ro))):
        files[name] = str(tmp_path / name)
        np.ascontiguousarray(arr).tofile(files[name])
    pre = []
    if rectify:
        for v, name in enumerate(("l.map", "r.map")):
            files[name] = str(tmp_path / name)
            with open(files[name], "wb") as f:
                f.write(np.ascontiguousarray(maps[v][0]).tobytes() + np.ascontiguousarray(maps[v][1]).tobytes())
        SW, SH = YO.size(frames[0], fmt)
        pre = ["--rectify", str(SW), str(SH), files["l.map"], files["r.map"]]
    out = {k: str(tmp_path / k) for k in ("yl", "yr", "pl", "pr")}
    subprocess.run([DEMO] + pre + ["--yuv", fmt, str(W), str(H), str(D), files["l.yuv"], files["r.yuv"], out["yl"],
                                   out["yr"]], check=True, capture_output=True)
    subprocess.run([DEMO, str(W), str(H), str(D), files["l.f32"], files["r.f32"], out["pl"], out["pr"]], check=True,
                   capture_output=True)
    for a, b in (("yl", "pl"), ("yr", "pr")):
        got, want = np.fromfile(out[a], np.uint8), np.fromfile(out[b], np.uint8)
        assert got.size == W * H
        assert_same(got, want, a)
