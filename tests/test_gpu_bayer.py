"""GPU: Bayer frames demosaiced in ingest (psm_set_images_bayer, _bayer_async, psm_set_images_device_bayer,
TorchStereo.match(bayer=)) against the CPU restatement, bit for bit.

The core check: a context fed a Bayer frame holds the same channel planes and gradient, and computes the same maps, as a
context of the same kind fed the oracle's BGR frame (bayer_oracle.bgr, then rectify_oracle.remap with rectification on)
through psm_set_images_u8.  It covers every pattern and method through every entry path, every kind of context,
rectification, strided frames and the halves of one side-by-side frame, frames below 3 x 3, switches between Bayer, YUV
and BGR frames on one context, launch counts, every rejected argument, a held-back compute stream and the demo."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import bayer_oracle as BO
import rectify_oracle as RO
import yuv_oracle as YO
from primestereomatch_b200 import DispEst, capi, synth
from test_gpu_parity import assert_same

torch = pytest.importorskip("torch")

from primestereomatch_b200.torch_stereo import TorchStereo, bayer_layout  # noqa: E402

pytestmark = pytest.mark.gpu

D = 64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEMO = os.path.join(ROOT, "primestereomatch_b200", "host", "dispest_demo")
CODES = [(p, m) for m in BO.METHODS for p in BO.PATTERNS]
PAT, MET = capi.BAYER_PATTERNS, capi.DEMOSAIC_METHODS


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def scene_raw(scenes, name, pattern, size=(448, 372)):
    """a scene's pair as Bayer frames of the pattern, cropped to size (W, H)"""
    l8, r8, _, _ = scenes[name]
    W, H = size
    return tuple(BO.from_bgr(img[:H, :W], pattern) for img in (l8, r8))


def expected(frames, pattern, method, maps=None):
    """the BGR frames a Bayer pair stands for, rectified through maps when given"""
    out = tuple(BO.bgr(f, pattern, method) for f in frames)
    return out if maps is None else tuple(RO.remap(o, *m) for o, m in zip(out, maps))


def pair(frames, pattern, method, d=D, kw=None, setup=None, maps=None):
    """(bayer, plain): DispEst contexts of one kind; plain holds the oracle's BGR frames, bayer is set up to take frames"""
    kw = kw or {}
    lo, ro = expected(frames, pattern, method, maps)
    bayer, plain = DispEst(lo, ro, d, **kw), DispEst(lo, ro, d, **kw)
    for de in (bayer, plain):
        if setup:
            setup(de)
    if maps is not None:
        SH, SW = frames[0].shape
        bayer.setRectify(maps[0], maps[1], (SW, SH))
    return bayer, plain


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


def set_device(handle, lt, rt, pattern, method):
    """psm_set_images_device_bayer of two tensors, laid out by bayer_layout"""
    H, W = lt.shape[-2:]
    p, m, lf, row, col, _ = bayer_layout(lt, H, W, pattern, method)
    _, _, rf, row2, col2, _ = bayer_layout(rt, H, W, pattern, method)
    assert (row, col) == (row2, col2)
    return capi.lib().psm_set_images_device_bayer(handle, p, m, lf[0], rf[0], row, col)


def feed(de, frames, pattern, method, path):
    """the Bayer pair into de through one entry path, then psm_cost_const"""
    L = capi.lib()
    l, r = (np.ascontiguousarray(f) for f in frames)
    H, W = l.shape
    if path == "host":
        de.setInputImagesBayer(l, r, pattern, method)
        de.CostConst_GPU()
        return
    if path == "async":
        capi.check(L.psm_set_images_bayer_async(de.handle, PAT[pattern], MET[method], ptr(l), l.strides[0], ptr(r),
                                                r.strides[0]), de.handle)
        capi.check(L.psm_set_images_commit(de.handle), de.handle)
    elif path == "device":
        capi.check(set_device(de.handle, torch.from_numpy(l).cuda(), torch.from_numpy(r).cuda(), pattern, method),
                   de.handle)
    elif path == "strided":   # every other column of a padded buffer: a column step of 2 and a longer row step
        views = []
        for f in (l, r):
            buf = torch.zeros(H, 2 * W + 6, dtype=torch.uint8, device="cuda")
            views.append(buf[:, 0:2 * W:2])
            views[-1].copy_(torch.from_numpy(f).cuda())
        capi.check(set_device(de.handle, views[0], views[1], pattern, method), de.handle)
    elif path == "side_by_side":   # both views in one frame, left | right
        t = torch.from_numpy(np.concatenate([l, r], axis=1)).cuda()
        capi.check(set_device(de.handle, t[:, :W], t[:, W:], pattern, method), de.handle)
    else:
        raise ValueError(path)
    torch.cuda.synchronize()
    capi.check(L.psm_cost_const(de.handle), de.handle)


# -- every pattern and method through every entry path ------------------------------------------------------------------
@pytest.mark.parametrize("path", ["host", "async", "device", "strided", "side_by_side"])
@pytest.mark.parametrize("pattern, method", CODES)
def test_codes_and_entry_paths(pattern, method, path, scenes):
    frames = scene_raw(scenes, "Cones", pattern)
    bayer, plain = pair(frames, pattern, method)
    with bayer, plain:
        feed(bayer, frames, pattern, method, path)
        plain.CostConst_GPU()
        compare_planes(bayer, plain, f"{pattern} {method} {path}")
        for de in (bayer, plain):
            run_maps(de)
        compare_maps(bayer, plain, f"{pattern} {method} {path}")


@pytest.mark.parametrize("pattern, method", CODES)
def test_torch_stereo(pattern, method, scenes):
    frames = scene_raw(scenes, "Teddy", pattern)
    lo, ro = expected(frames, pattern, method)
    H, W = lo.shape[:2]
    with TorchStereo(W, H, D) as bt, TorchStereo(W, H, D) as pt:
        lt, rt = (torch.from_numpy(f).cuda() for f in frames)
        got = bt.match(lt, rt, bayer=pattern, demosaic=method, post_process=True)
        want = pt.match(torch.from_numpy(lo).cuda(), torch.from_numpy(ro).cuda(), post_process=True)
        # a batch of two: the pair, then the pair swapped
        gb = bt.match(torch.stack([lt, rt]), torch.stack([rt, lt]), bayer=pattern, demosaic=method)
        wb = pt.match(torch.from_numpy(np.stack([lo, ro])).cuda(), torch.from_numpy(np.stack([ro, lo])).cuda())
        torch.cuda.synchronize()
        for g, w, what in zip(got + gb, want + wb, ("lmap", "rmap", "batch lmap", "batch rmap")):
            assert_same(g.cpu().numpy(), w.cpu().numpy(), f"{pattern} {method} {what}")
        with pytest.raises(ValueError):   # a BGR tensor is not a Bayer frame
            bt.match(torch.from_numpy(lo).cuda(), torch.from_numpy(ro).cuda(), bayer=pattern)


def test_side_by_side_half_at_an_odd_column(scenes):
    """a half that starts at an odd column of an RGGB frame is a GRBG frame of its own"""
    l, r = scene_raw(scenes, "Cones", "rggb", size=(449, 372))
    frames = (np.ascontiguousarray(l[:, 1:]), np.ascontiguousarray(r[:, 1:]))
    bayer, plain = pair(frames, "grbg", "ea")
    with bayer, plain:
        t = torch.from_numpy(np.concatenate([l, r], axis=1)).cuda()
        capi.check(set_device(bayer.handle, t[:, 1:449], t[:, 450:], "grbg", "ea"), bayer.handle)
        torch.cuda.synchronize()
        capi.check(capi.lib().psm_cost_const(bayer.handle), bayer.handle)
        plain.CostConst_GPU()
        compare_planes(bayer, plain, "odd-column half")


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


def rig(frames, margin=(36, 22)):
    """the maps of a synthetic rig that crops margin px off each side of the frames"""
    SH, SW = frames[0].shape
    W, H = SW - 2 * margin[0], SH - 2 * margin[1]
    return tuple(synth.rectify_maps(W, H, SW, SH, view=v) for v in range(2))


@pytest.mark.parametrize("rectify", [False, True], ids=["plain", "rectify"])
@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("name", list(CONTEXTS))
def test_context_kinds(name, path, rectify, scenes):
    d, kw, setup = CONTEXTS[name]
    pattern, method = ("gbrg", "ea") if rectify else ("rggb", "bilinear")
    frames = scene_raw(scenes, "Teddy", pattern)
    maps = rig(frames) if rectify else None
    bayer, plain = pair(frames, pattern, method, d, kw, setup, maps)
    with bayer, plain:
        feed(bayer, frames, pattern, method, path)
        plain.CostConst_GPU()
        views = (0,) if name == "left_only" else (0, 1)
        compare_planes(bayer, plain, name, views)
        for de in (bayer, plain):
            run_maps(de, post=True)
        compare_maps(bayer, plain, name)


@pytest.mark.parametrize("pattern, method", [("rggb", "ea"), ("bggr", "bilinear"), ("grbg", "bilinear"), ("gbrg", "ea")])
@pytest.mark.parametrize("path", ["host", "async", "side_by_side"])
def test_rectified_entry_paths(pattern, method, path, scenes):
    frames = scene_raw(scenes, "Cones", pattern)
    maps = rig(frames)
    bayer, plain = pair(frames, pattern, method, maps=maps)
    with bayer, plain:
        feed(bayer, frames, pattern, method, path)
        plain.CostConst_GPU()
        compare_planes(bayer, plain, f"{pattern} {method} {path} rectified")
        for de in (bayer, plain):
            run_maps(de)
        compare_maps(bayer, plain, f"{pattern} {method} {path} rectified")


@pytest.mark.parametrize("method", BO.METHODS)
def test_torch_stereo_side_by_side_camera_frame(method, scenes):
    """one side-by-side raw camera frame, rectified on the device: TorchStereo on its two halves"""
    pattern = "bggr"
    frames = scene_raw(scenes, "Cones", pattern)
    maps = rig(frames)
    lo, ro = expected(frames, pattern, method, maps)
    H, W = lo.shape[:2]
    SH, SW = frames[0].shape
    Q = np.array([[1, 0, 0, -W / 2], [0, 1, 0, -H / 2], [0, 0, 0, 400.0], [0, 0, 1 / 0.12, 0]])
    with TorchStereo(W, H, D) as bt, TorchStereo(W, H, D) as pt:
        bt.setRectify(maps[0], maps[1], (SW, SH))
        cam = torch.from_numpy(np.concatenate(frames, axis=1)).cuda()
        small = torch.zeros(H, W, dtype=torch.uint8, device="cuda")
        with pytest.raises(ValueError):   # frames of the context's size, not the source's
            bt.match(small, small, bayer=pattern, demosaic=method)
        got = bt.match(cam[:, :SW], cam[:, SW:], bayer=pattern, demosaic=method, post_process=True, points=(Q, Q))
        want = pt.match(torch.from_numpy(lo).cuda(), torch.from_numpy(ro).cuda(), post_process=True, points=(Q, Q))
        torch.cuda.synchronize()
        for g, w, what in zip(got, want, ("lmap", "rmap", "lpts", "rpts")):
            assert_same(g.cpu().numpy().view(np.uint8), w.cpu().numpy().view(np.uint8), what)


# -- frames below 3 x 3 and at the 3 x 3 edge ---------------------------------------------------------------------------
@pytest.mark.parametrize("size", [(1, 1), (2, 2), (2, 9), (9, 2), (3, 3), (4, 3), (3, 7)])
@pytest.mark.parametrize("path", ["host", "device"])
def test_small_frames(size, path):
    """every output is 0 below 3 x 3, as cv2 gives; at and just above it the border clamp covers the whole frame"""
    W, H = size
    for k, (pattern, method) in enumerate(CODES):
        frames = (BO.frame(10 * k + 1, W, H), BO.frame(10 * k + 2, W, H))
        bayer, plain = pair(frames, pattern, method, d=2)
        with bayer, plain:
            feed(bayer, frames, pattern, method, path)
            plain.CostConst_GPU()
            compare_planes(bayer, plain, f"{size} {pattern} {method}")
            for de in (bayer, plain):
                run_maps(de)
            compare_maps(bayer, plain, f"{size} {pattern} {method}")


@pytest.mark.parametrize("src", [(2, 9), (9, 2), (1, 1), (3, 3)])
def test_small_rectified_source(src):
    """a source frame below or at 3 x 3 read through the maps of a 24 x 16 context"""
    SW, SH = src
    rng = np.random.default_rng(SW * 10 + SH)
    maps = []
    for v in range(2):   # taps spread over the source and beyond it
        xy = np.stack([rng.integers(-2, SW + 1, (16, 24)), rng.integers(-2, SH + 1, (16, 24))], -1).astype(np.int16)
        maps.append((xy, rng.integers(0, 1024, (16, 24)).astype(np.uint16)))
    for pattern, method in CODES:
        frames = (BO.frame(3, SW, SH), BO.frame(4, SW, SH))
        bayer, plain = pair(frames, pattern, method, d=8, maps=maps)
        with bayer, plain:
            feed(bayer, frames, pattern, method, "host")
            plain.CostConst_GPU()
            compare_planes(bayer, plain, f"{src} {pattern} {method}")


# -- Bayer, YUV and BGR frames switched between frames on one live context ----------------------------------------------
@pytest.mark.parametrize("name", ["unblocked", "multi2"])
def test_format_switches(name, scenes):
    d, kw, _ = CONTEXTS[name]
    seq = [("rggb", "host"), ("nv12", "host"), ("bgr", "host"), ("gbrg", "device"), ("yuyv", "device"),
           ("bggr", "async"), ("bgr", "host"), ("grbg", "host")]
    l8, r8, _, _ = scenes["Teddy"]
    crop = tuple(np.ascontiguousarray(i[:372, :448]) for i in (l8, r8))
    L = capi.lib()
    with DispEst(*crop, d, **kw) as live:
        for k, (fmt, path) in enumerate(seq):
            if path == "async" and name == "multi2":
                path = "host"   # no asynchronous upload on multi-device contexts
            scene = "Cones" if k % 2 else "Teddy"
            if fmt == "bgr":
                lo, ro = (np.ascontiguousarray(i[:372, :448]) for i in scenes[scene][:2])
                live.setInputImages(lo, ro)
                live.CostConst_GPU()
            elif fmt in YO.FORMATS:
                l8s, r8s = (np.ascontiguousarray(i[:372, :448]) for i in scenes[scene][:2])
                frames = tuple(YO.from_bgr(i, fmt) for i in (l8s, r8s))
                lo, ro = (YO.bgr(f, fmt) for f in frames)
                if path == "host":
                    live.setInputImagesYUV(*frames, fmt)
                    live.CostConst_GPU()
                else:
                    lt, rt = (torch.from_numpy(f).cuda() for f in frames)
                    from primestereomatch_b200.torch_stereo import yuv_layout
                    sampling, lf, *steps, _ = yuv_layout(lt, 372, 448, fmt)
                    _, rf, *_ = yuv_layout(rt, 372, 448, fmt)
                    capi.check(L.psm_set_images_device_yuv(live.handle, sampling, (C.c_void_p * 3)(*lf[0]),
                                                           (C.c_void_p * 3)(*rf[0]), *steps), live.handle)
                    torch.cuda.synchronize()
                    capi.check(L.psm_cost_const(live.handle), live.handle)
            else:
                method = "ea" if k % 2 else "bilinear"
                frames = scene_raw(scenes, scene, fmt)
                lo, ro = expected(frames, fmt, method)
                feed(live, frames, fmt, method, path)
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
    pattern, method = "grbg", "ea"
    frames = scene_raw(scenes, "Cones", pattern)
    maps = rig(frames) if rectify else None
    bayer, plain = pair(frames, pattern, method, d, kw, setup, maps)
    # one ingest launch and one halo pass per view, as for u8 frames; a multi-device context's other shards receive the
    # first shard's planes, as for device BGR planes
    with bayer, plain:
        counts = []
        for de, f in ((bayer, lambda: feed(bayer, frames, pattern, method, path)),
                      (plain, lambda: plain.CostConst_GPU() if not kw.get("devices") and path != "device"
                       else feed_bgr_device(plain, expected(frames, pattern, method, maps)))):
            n0 = de.launch_count()
            f()
            run_maps(de, post=True)
            de.sync()
            counts.append(de.launch_count() - n0)
        assert counts[0] == counts[1]


# -- arguments ---------------------------------------------------------------------------------------------------------
def test_rejected_arguments_leave_the_context_unchanged(scenes):
    L = capi.lib()
    pattern, method = "rggb", "bilinear"
    frames = scene_raw(scenes, "Cones", pattern)
    bayer, plain = pair(frames, pattern, method)
    l, r = (np.ascontiguousarray(f) for f in frames)
    H, W = l.shape
    rg, bl = capi.PSM_BAYER_RGGB, capi.PSM_DEMOSAIC_BILINEAR
    with bayer, plain:
        feed(bayer, frames, pattern, method, "host")
        plain.CostConst_GPU()
        h = bayer.handle
        other = frames[::-1]   # a different frame, so that an accepted call would show
        lo, ro = (np.ascontiguousarray(f) for f in other)
        bad_host = [
            (0, bl, ptr(lo), W, ptr(ro), W),             # unknown patterns
            (5, bl, ptr(lo), W, ptr(ro), W),
            (-1, bl, ptr(lo), W, ptr(ro), W),
            (rg, 0, ptr(lo), W, ptr(ro), W),             # unknown methods
            (rg, 3, ptr(lo), W, ptr(ro), W),
            (rg, bl, None, W, ptr(ro), W),               # null frames
            (rg, bl, ptr(lo), W, None, W),
            (rg, bl, ptr(lo), W - 1, ptr(ro), W),        # steps below a row
            (rg, bl, ptr(lo), W, ptr(ro), 0),
        ]
        for args in bad_host:
            assert L.psm_set_images_bayer(h, *args) == capi.PSM_EINVAL, args[:2]
            assert L.psm_set_images_bayer_async(h, *args) == capi.PSM_EINVAL, args[:2]
        t = torch.from_numpy(lo).cuda()
        p = t.data_ptr()
        bad_device = [
            (0, bl, p, p, W, 1),                         # unknown pattern and method
            (5, bl, p, p, W, 1),
            (rg, 0, p, p, W, 1),
            (rg, 3, p, p, W, 1),
            (rg, bl, None, p, W, 1),                     # null pointers
            (rg, bl, p, None, W, 1),
            (rg, bl, p, p, W, 0),                        # zero column step
            (rg, bl, p, p, W - 1, 1),                    # steps below a row
            (rg, bl, p, p, 2 * (W - 1), 2),
            (rg, bl, p, p, 4 * W, 1 << 62),              # a row span that overflows
        ]
        for args in bad_device:
            assert L.psm_set_images_device_bayer(h, *args) == capi.PSM_EINVAL, args
        # still the frame of the first call
        capi.check(L.psm_cost_const(h), h)
        compare_planes(bayer, plain, "after rejected arguments")
        # the least steps a row spans are accepted
        assert L.psm_set_images_device_bayer(h, rg, bl, p, p, W, 1) == capi.PSM_OK
        assert L.psm_set_images_bayer(h, rg, bl, ptr(lo), W, ptr(ro), W) == capi.PSM_OK
        torch.cuda.synchronize()


def test_pending_upload_and_multi_device_async(scenes):
    L = capi.lib()
    pattern, method = "bggr", "ea"
    frames = scene_raw(scenes, "Cones", pattern)
    l, r = (np.ascontiguousarray(f) for f in frames)
    bayer, plain = pair(frames, pattern, method)
    args = (PAT[pattern], MET[method], ptr(l), l.strides[0], ptr(r), r.strides[0])
    with bayer, plain:
        h = bayer.handle
        capi.check(L.psm_set_images_bayer_async(h, *args), h)
        assert L.psm_set_images_bayer_async(h, *args) == capi.PSM_ESTATE
        assert L.psm_set_images_u8_async(h, ptr(l), l.strides[0], ptr(r), r.strides[0]) == capi.PSM_ESTATE
        capi.check(L.psm_set_images_commit(h), h)
        capi.check(L.psm_cost_const(h), h)
        plain.CostConst_GPU()
        compare_planes(bayer, plain, "after the state error")
    lo, ro = expected(frames, pattern, method)
    with DispEst(lo, ro, D, devices=[0, 0]) as multi:
        assert L.psm_set_images_bayer_async(multi.handle, *args) == capi.PSM_EINVAL


# -- a held-back compute stream ----------------------------------------------------------------------------------------
HOLD_MS = 250.0


def test_held_back_stream(scenes):
    """each Bayer entry path issued while the context's stream is held back by a spin (as in test_gpu_stream_order): the
    host calls return once the caller's buffers are read, before the spin ends, and the device path reads the frame the
    held stream writes after psm_wait_stream"""
    L = capi.lib()
    pattern, method = "rggb", "ea"
    code = (PAT[pattern], MET[method])
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

    a, b = scene_raw(scenes, "Cones", pattern), scene_raw(scenes, "Teddy", pattern)
    with DispEst(*expected(a, pattern, method), D) as live:
        h = live.handle
        capi.check(L.psm_set_stream(h, C.c_void_p(s.cuda_stream)), h)
        # outside the hold: the first asynchronous upload allocates the second staging set
        l, r = (np.array(f) for f in a)
        capi.check(L.psm_set_images_bayer_async(h, *code, ptr(l), l.strides[0], ptr(r), r.strides[0]), h)
        capi.check(L.psm_set_images_commit(h), h)
        live.sync()
        for path, cur, other in (("host", b, a), ("async", a, b), ("device", b, a)):
            l, r = (np.array(f) for f in cur)
            done = hold()
            if path == "host":
                capi.check(L.psm_set_images_bayer(h, *code, ptr(l), l.strides[0], ptr(r), r.strides[0]), h)
            elif path == "async":
                capi.check(L.psm_set_images_bayer_async(h, *code, ptr(l), l.strides[0], ptr(r), r.strides[0]), h)
                capi.check(L.psm_set_images_commit(h), h)
            else:
                lt, rt = (torch.zeros(f.shape, dtype=torch.uint8, device="cuda") for f in cur)
                src = [torch.from_numpy(f).pin_memory() for f in (l, r)]
                with torch.cuda.stream(s):   # the frame is written on the held stream, after the spin
                    lt.copy_(src[0], non_blocking=True)
                    rt.copy_(src[1], non_blocking=True)
                capi.check(L.psm_wait_stream(h, C.c_void_p(s.cuda_stream)), h)
                capi.check(set_device(h, lt, rt, pattern, method), h)
            assert not done.query(), f"the hold ended before the {path} frame was issued"
            if path != "device":
                l[...], r[...] = other   # the caller reuses its buffers at once
            capi.check(L.psm_cost_const(h), h)
            run_maps(live)
            with DispEst(*expected(cur, pattern, method), D) as plain:
                plain.CostConst_GPU()
                run_maps(plain)
                compare_maps(live, plain, f"held {path}")
        torch.cuda.synchronize()


# -- the demo ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pattern, method, rectify", [("rggb", "bilinear", False), ("gbrg", "ea", False),
                                                      ("bggr", "ea", True)])
def test_demo(pattern, method, rectify, tmp_path, scenes):
    frames = scene_raw(scenes, "Cones", pattern)
    maps = rig(frames) if rectify else None
    lo, ro = expected(frames, pattern, method, maps)
    H, W = lo.shape[:2]
    files = {}
    for name, arr in (("l.raw", frames[0]), ("r.raw", frames[1]), ("l.f32", synth.to_f32(lo)),
                      ("r.f32", synth.to_f32(ro))):
        files[name] = str(tmp_path / name)
        np.ascontiguousarray(arr).tofile(files[name])
    pre = []
    if rectify:
        for v, name in enumerate(("l.map", "r.map")):
            files[name] = str(tmp_path / name)
            with open(files[name], "wb") as f:
                f.write(np.ascontiguousarray(maps[v][0]).tobytes() + np.ascontiguousarray(maps[v][1]).tobytes())
        SH, SW = frames[0].shape
        pre = ["--rectify", str(SW), str(SH), files["l.map"], files["r.map"]]
    pre += ["--bayer", pattern] + (["--ea"] if method == "ea" else [])
    out = {k: str(tmp_path / k) for k in ("bl", "br", "pl", "pr")}
    subprocess.run([DEMO] + pre + [str(W), str(H), str(D), files["l.raw"], files["r.raw"], out["bl"], out["br"]],
                   check=True, capture_output=True)
    subprocess.run([DEMO, str(W), str(H), str(D), files["l.f32"], files["r.f32"], out["pl"], out["pr"]], check=True,
                   capture_output=True)
    for a, b in (("bl", "pl"), ("br", "pr")):
        got, want = np.fromfile(out[a], np.uint8), np.fromfile(out[b], np.uint8)
        assert got.size == W * H
        assert_same(got, want, a)
    bad = subprocess.run([DEMO, "--bayer", "bg", str(W), str(H), str(D), files["l.raw"], files["r.raw"], out["bl"],
                          out["br"]], capture_output=True)
    assert bad.returncode == 2 and b"unknown --bayer pattern" in bad.stderr
