"""GPU: device frames in any 8-bit or float layout (psm_set_images_device_planes), the stream-ordering calls
(psm_wait_stream / psm_signal_stream), maps into device buffers (psm_copy_maps_device) and TorchStereo.

Every result is compared bit for bit with the host upload of the same pixels (psm_set_images / _u8 through DispEst) on a
context of the same kind: the channel planes and the gradient, raw and filtered cost slices, and both maps.  The ordering
tests hold the context's streams back behind a bounded spin (psm_wait_stream on a torch stream running
torch.cuda._sleep, as tests/test_gpu_stream_order.py does with psm_set_stream) and assert the spin is still running when
the call that could race has been issued."""
import ctypes as C

import numpy as np
import pytest

import image_cases as IC
from primestereomatch_b200 import DispEst, capi
from test_gpu_parity import assert_same

torch = pytest.importorskip("torch")

from primestereomatch_b200.torch_stereo import TorchStereo, frame_layout  # noqa: E402

pytestmark = pytest.mark.gpu

D = 64
HOLD_MS = 250.0
CAL_CYCLES = 50_000_000
L = None


@pytest.fixture(scope="module", autouse=True)
def lib():
    global L
    L = capi.lib()


def bits(a):
    """float arrays compared by bit pattern (NaN payloads and -0 included)"""
    return a.view(np.uint32) if a.dtype == np.float32 else a


# -- layouts of a BGR numpy frame as device tensors -------------------------------------------------------------------
def as_layout(img, layout, seed=0):
    """-> (tensor, channels): the BGR frame `img` (H, W, 3) on the device in one of the header's layouts"""
    t = torch.from_numpy(np.ascontiguousarray(img)).cuda()
    H, W, _ = img.shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    junk = lambda *shape: (torch.randint(0, 256, shape, generator=g, device="cuda").to(t.dtype)  # noqa: E731
                           if t.dtype == torch.uint8 else torch.rand(shape, generator=g, device="cuda") * 7 - 3)
    if layout == "hwc_bgr":
        return t, "bgr"
    if layout == "hwc_rgb":
        return t.flip(2).contiguous(), "rgb"
    if layout == "chw_rgb":
        return t.flip(2).permute(2, 0, 1).contiguous(), "rgb"
    if layout == "bgra":
        return torch.cat([t, junk(H, W, 1)], 2).contiguous(), "bgr"
    if layout == "hwc_view":      # a window of a larger 4-channel tensor: padded row step, column offset
        big = junk(H + 3, W + 7, 4)
        v = big[1:1 + H, 3:3 + W, :3]
        v.copy_(t)
        return v, "bgr"
    if layout == "chw_view":      # planes of a larger planar tensor, RGB order
        big = junk(3, H + 2, W + 9)
        v = big[:, 2:, 5:5 + W]
        v.copy_(t.flip(2).permute(2, 0, 1))
        return v, "rgb"
    raise ValueError(layout)


LAYOUTS = ["hwc_bgr", "hwc_rgb", "chw_rgb", "bgra", "hwc_view", "chw_view"]


def set_planes(handle, lt, rt, channels, hw):
    pix, lf, row, col, _ = frame_layout(lt, *hw, channels)
    _, rf, row2, col2, _ = frame_layout(rt, *hw, channels)
    assert (row, col) == (row2, col2)
    capi.check(L.psm_set_images_device_planes(handle, pix, (C.c_void_p * 3)(*lf[0]), (C.c_void_p * 3)(*rf[0]), row, col),
               handle)


def host_and_device(l, r, d, layout, kw=None, seed=0, setup=None):
    """(host DispEst, device DispEst): the same context twice, one fed by psm_set_images[_u8], one by the planes call"""
    kw = kw or {}
    host, dev = DispEst(l, r, d, **kw), DispEst(l, r, d, **kw)
    for de in (host, dev):
        if setup:
            setup(de)
    lt, ch = as_layout(l, layout, seed)
    rt, _ = as_layout(r, layout, seed + 1)
    host.CostConst_GPU()
    set_planes(dev.handle, lt, rt, ch, l.shape[:2])
    capi.check(L.psm_cost_const(dev.handle), dev.handle)
    torch.cuda.synchronize()
    return host, dev


def compare_planes(host, dev, what):
    for view in (0, 1):
        for plane in (0, 1, 2, 12):
            assert_same(bits(dev.read_guide_plane(view, plane)), bits(host.read_guide_plane(view, plane)),
                        f"{what} view {view} plane {plane}")


def compare_slices(host, dev, what, ds, views=(0, 1)):
    for view in views:
        for d in ds:
            assert_same(bits(dev.read_cost_slice(view, d)), bits(host.read_cost_slice(view, d)), f"{what} view {view} d {d}")


def compare_maps(host, dev, what, filt=None):
    for de in (host, dev):
        (filt or (lambda e: e.CostFilter_GPU()))(de)
        de.DispSelect_GPU()
    assert_same(dev.lDisMap, host.lDisMap, f"{what} lDisMap")
    if host.rDisMap is not None:
        assert_same(dev.rDisMap, host.rDisMap, f"{what} rDisMap")


# -- every layout, both scenes, both sample types ---------------------------------------------------------------------
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("kind", ["u8", "f32"])
@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_layouts_equal_the_host_upload(scene, kind, layout, scenes):
    l8, r8, lf, rf = scenes[scene]
    l, r = (l8, r8) if kind == "u8" else (lf, rf)
    host, dev = host_and_device(l, r, D, layout)
    with host, dev:
        what = f"{scene} {kind} {layout}"
        compare_planes(host, dev, what)
        compare_slices(host, dev, what + " raw", (0, 1, 31, 63))
        for de in (host, dev):
            de.CostFilter_GPU()
        compare_slices(host, dev, what + " filtered", (0, 1, 31, 63))
        for de in (host, dev):
            de.DispSelect_GPU()
        assert_same(dev.lDisMap, host.lDisMap, what + " lDisMap")
        assert_same(dev.rDisMap, host.rDisMap, what + " rDisMap")


@pytest.mark.parametrize("hw", [(1, 1), (5, 3), (13, 37), (7, 18)])
@pytest.mark.parametrize("kind", ["u8", "f32"])
@pytest.mark.parametrize("layout", ["hwc_bgr", "chw_view", "bgra"])
def test_small_and_ragged_sizes(hw, kind, layout):
    H, W = hw
    rng = np.random.default_rng([H, W])
    l8, r8 = (rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for _ in range(2))
    l, r = (l8, r8) if kind == "u8" else (l8.astype(np.float32) / 255, r8.astype(np.float32) / 255)
    host, dev = host_and_device(l, r, 4, layout)
    with host, dev:
        what = f"{H}x{W} {kind} {layout}"
        compare_planes(host, dev, what)
        compare_slices(host, dev, what + " raw", range(4))
        compare_maps(host, dev, what)


@pytest.mark.parametrize("kind", IC.KINDS)
@pytest.mark.parametrize("layout", ["hwc_bgr", "chw_rgb"])
def test_float_image_kinds_take_the_host_route(kind, layout):
    """negative, -0, inf, NaN, >= 2^61 and the unflagged inexact kinds: the same planes, flags (so the same filter
    route) and results as the interleaved float upload"""
    W, H, d = 64, 40, 16
    l, r = IC.frame(kind, W, H, d)
    host, dev = host_and_device(l, r, d, layout)
    with host, dev:
        compare_planes(host, dev, kind)
        for de in (host, dev):
            de.CostFilter_GPU()
        compare_slices(host, dev, kind + " filtered", range(d))
        for de in (host, dev):
            de.DispSelect_GPU()
        assert_same(dev.lDisMap, host.lDisMap, kind + " lDisMap")
        assert_same(dev.rDisMap, host.rDisMap, kind + " rDisMap")


# -- every kind of context ---------------------------------------------------------------------------------------------
CONTEXTS = {
    "blocked_ragged": (D, dict(block_slices=24), None),
    "u16_d300": (300, dict(map_bits=16), None),
    "left_only": (D, {}, lambda de: de.setViews("left")),
    "multi2": (D, dict(devices=[0, 0]), None),
    "multi3": (D, dict(devices=[0, 0, 0]), None),
    "multi2_blocked": (D, dict(devices=[0, 0], block_slices=20), None),
    "multi3_blocked": (D, dict(devices=[0, 0, 0], block_slices=7), None),
}


@pytest.mark.parametrize("name", list(CONTEXTS))
@pytest.mark.parametrize("kind", ["u8", "f32"])
def test_context_kinds(name, kind, scenes):
    d, kw, setup = CONTEXTS[name]
    l8, r8, lf, rf = scenes["Cones"]
    l, r = (l8, r8) if kind == "u8" else (lf, rf)
    for layout in ("hwc_bgr", "chw_rgb"):
        host, dev = host_and_device(l, r, d, layout, kw, setup=setup)
        with host, dev:
            what = f"{name} {kind} {layout}"
            compare_planes(host, dev, what)
            compare_maps(host, dev, what)
            for de in (host, dev):
                de.PostProcess_GPU()
            assert_same(dev.lDisMap, host.lDisMap, what + " post-processed lDisMap")
            if host.rDisMap is not None:
                assert_same(dev.rDisMap, host.rDisMap, what + " post-processed rDisMap")


# -- TorchStereo -------------------------------------------------------------------------------------------------------
SETTINGS = {
    "default": lambda e: None,
    "window_cost": lambda e: (e.setGuidedFilter(5, 1e-3), e.setMatchingCost(0.7, 0.05, 0.02)),
    "post_filter": lambda e: e.setPostFilter(5, 12.0, 2, "iv1"),
    "lr_fill_wmf": lambda e: e.setLRCheck(capi.PSM_LR_FILL_WMF),
    "lr_fill": lambda e: e.setLRCheck(capi.PSM_LR_FILL),
    "left_only": lambda e: e.setViews("left"),
}


@pytest.mark.parametrize("fgf", [False, True])
@pytest.mark.parametrize("setting", list(SETTINGS))
def test_torch_stereo_equals_dispest(setting, fgf, scenes):
    l8, r8, _, _ = scenes["Teddy"]
    H, W, _ = l8.shape
    pp = setting in ("post_filter", "lr_fill_wmf", "lr_fill")
    with DispEst(l8, r8, D) as de, TorchStereo(W, H, D) as ts:
        for e in (de, ts):
            SETTINGS[setting](e)
            e.setSubsampleRate(2)
        de.CostConst_GPU()
        de.CostFilter_FGF_GPU() if fgf else de.CostFilter_GPU()
        de.DispSelect_GPU()
        if pp:
            de.PostProcess_GPU()
        lt = torch.from_numpy(l8).cuda().flip(2).permute(2, 0, 1).contiguous()   # torchvision's CHW RGB
        rt = torch.from_numpy(r8).cuda().flip(2).permute(2, 0, 1).contiguous()
        lm, rm = ts.match(lt, rt, channels="rgb", fgf=fgf, post_process=pp)
        assert lm.dtype == torch.uint8 and lm.shape == (H, W) and lm.device == ts.device
        assert_same(lm.cpu().numpy(), de.lDisMap, f"{setting} fgf={fgf} lmap")
        if setting == "left_only":
            assert rm is None
        else:
            assert_same(rm.cpu().numpy(), de.rDisMap, f"{setting} fgf={fgf} rmap")


@pytest.mark.parametrize("kw", [dict(), dict(map_bits=16), dict(block_slices=24), dict(devices=[0, 0])])
def test_torch_stereo_batches_and_contexts(kw, scenes):
    """a (B, H, W, 3) u8 batch and a (B, 3, H, W) float batch, one frame after another on one context"""
    names = ["Cones", "Teddy", "Cones"]
    H, W, _ = scenes["Cones"][0].shape
    want = {}
    for s in ("Cones", "Teddy"):
        with DispEst(scenes[s][0], scenes[s][1], D, **kw) as de:
            de.CostConst_GPU()
            de.CostFilter_GPU()
            de.DispSelect_GPU()
            want[s] = (de.lDisMap.copy(), de.rDisMap.copy())
    with TorchStereo(W, H, D, **kw) as ts:
        mdt = torch.uint16 if kw.get("map_bits") == 16 else torch.uint8
        batch = lambda v: torch.stack([torch.from_numpy(scenes[s][v]) for s in names]).cuda()  # noqa: E731
        hwc_u8 = (batch(0), batch(1))
        chw_f32 = tuple(batch(v).permute(0, 3, 1, 2).contiguous() for v in (2, 3))
        for k, (lb, rb) in enumerate((hwc_u8, chw_f32)):
            lm, rm = ts.match(lb, rb)
            assert lm.shape == (3, H, W) and lm.dtype == mdt
            for b, s in enumerate(names):
                got_l, got_r = lm[b].cpu().numpy(), rm[b].cpu().numpy()
                assert_same(got_l, want[s][0].astype(got_l.dtype), f"{kw} batch {k} frame {b} lmap")
                assert_same(got_r, want[s][1].astype(got_r.dtype), f"{kw} batch {k} frame {b} rmap")


# -- ordering ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cycles_per_ms():
    s = torch.cuda.Stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(s):
        torch.cuda._sleep(1_000_000)
        e0.record(s)
        torch.cuda._sleep(CAL_CYCLES)
        e1.record(s)
    e1.synchronize()
    return CAL_CYCLES / e0.elapsed_time(e1)


def hold(ts, cycles_per_ms, ms=HOLD_MS):
    """every stream of the context waits behind a spin of about `ms` on a side stream -> its end event"""
    s, done = torch.cuda.Stream(), torch.cuda.Event()
    with torch.cuda.stream(s):
        torch.cuda._sleep(int(ms * cycles_per_ms))
        done.record(s)
    capi.check(L.psm_wait_stream(ts.handle, C.c_void_p(s.cuda_stream)), ts.handle)
    return done


def still_held(done, what):
    assert not done.query(), f"the hold ended before {what} was issued: the sequence did not race the context"


@pytest.fixture(scope="module")
def scene_maps(scenes):
    out = {}
    for s in ("Cones", "Teddy"):
        with DispEst(scenes[s][0], scenes[s][1], D) as de:
            de.CostConst_GPU()
            de.CostFilter_GPU()
            de.DispSelect_GPU()
            out[s] = (de.lDisMap.copy(), de.rDisMap.copy())
    for v in (0, 1):
        assert not np.array_equal(out["Cones"][v], out["Teddy"][v])
    return out


def dev_frame(scenes, s):
    return torch.from_numpy(scenes[s][0]).cuda(), torch.from_numpy(scenes[s][1]).cuda()


def check_maps(lm, rm, want, what):
    assert_same(lm.cpu().numpy(), want[0], what + " lmap")
    assert_same(rm.cpu().numpy(), want[1], what + " rmap")


KINDS = {"single": {}, "multi2": dict(devices=[0, 0])}


@pytest.mark.parametrize("ctx_kind", list(KINDS))
def test_frame_written_on_a_side_stream(ctx_kind, scenes, scene_maps, cycles_per_ms):
    """The frame is written by a torch kernel on a side stream that runs after the context's hold has ended; match on
    that stream must wait for it (psm_wait_stream), not read the frame's earlier pixels."""
    H, W, _ = scenes["Cones"][0].shape
    with TorchStereo(W, H, D, **KINDS[ctx_kind]) as ts:
        l, r = dev_frame(scenes, "Teddy")
        ts.match(l, r)                                     # first use outside the hold
        new_l, new_r = dev_frame(scenes, "Cones")
        torch.cuda.synchronize()
        side = torch.cuda.Stream()
        done = hold(ts, cycles_per_ms)
        with torch.cuda.stream(side):
            torch.cuda._sleep(int(2 * HOLD_MS * cycles_per_ms))   # the write lands after the context's hold
            l.copy_(new_l)
            r.copy_(new_r)
            lm, rm = ts.match(l, r)
        still_held(done, "match")
        torch.cuda.synchronize()
        check_maps(lm, rm, scene_maps["Cones"], f"{ctx_kind} side-stream frame")


@pytest.mark.parametrize("ctx_kind", list(KINDS))
def test_input_overwritten_right_after_match(ctx_kind, scenes, scene_maps, cycles_per_ms):
    """The caller overwrites its input tensors on its stream as soon as match returns, with the context held: the
    maps are still those of the original frame (psm_signal_stream orders the overwrite after the reads)."""
    H, W, _ = scenes["Cones"][0].shape
    with TorchStereo(W, H, D, **KINDS[ctx_kind]) as ts:
        l, r = dev_frame(scenes, "Cones")
        ts.match(l, r)
        other_l, other_r = dev_frame(scenes, "Teddy")
        torch.cuda.synchronize()
        done = hold(ts, cycles_per_ms)
        lm, rm = ts.match(l, r)
        l.copy_(other_l)
        r.copy_(other_r)
        still_held(done, "the overwrite")
        torch.cuda.synchronize()
        check_maps(lm, rm, scene_maps["Cones"], f"{ctx_kind} overwritten input")


@pytest.mark.parametrize("post_process", [False, True])
@pytest.mark.parametrize("ctx_kind", list(KINDS))
def test_consumer_reads_complete_maps(ctx_kind, post_process, scenes, scene_maps, cycles_per_ms):
    """A consumer on torch's stream reads the maps right after match: it sees complete maps, twice in a row."""
    H, W, _ = scenes["Cones"][0].shape
    with DispEst(scenes["Teddy"][0], scenes["Teddy"][1], D) as de:
        de.CostConst_GPU()
        de.CostFilter_GPU()
        de.DispSelect_GPU()
        if post_process:
            de.PostProcess_GPU()
        teddy = (de.lDisMap.copy(), de.rDisMap.copy())
    with TorchStereo(W, H, D, **KINDS[ctx_kind]) as ts:
        l, r = dev_frame(scenes, "Teddy")
        ts.match(l, r, post_process=post_process)
        torch.cuda.synchronize()
        done = hold(ts, cycles_per_ms)
        outs = []
        for _ in range(2):
            lm, rm = ts.match(l, r, post_process=post_process)
            outs.append((lm.clone(), rm.clone()))          # on torch's stream, right after the signal
            del lm, rm                                      # freed on the stream: the next match may reuse them
        still_held(done, "the consumers")
        torch.cuda.synchronize()
        for k, (lm, rm) in enumerate(outs):
            check_maps(lm, rm, teddy, f"{ctx_kind} consumer {k}")


# -- launches, rejected calls, state rules -----------------------------------------------------------------------------
def launches(de):
    return de.launch_count()


@pytest.mark.parametrize("kw", [dict(), dict(devices=[0, 0])])
def test_launch_counts(kw, scenes):
    l8, r8, lf, rf = scenes["Cones"]
    with DispEst(l8, r8, D, **kw) as de:
        n0 = launches(de)
        capi.check(L.psm_set_images_u8(de.handle, l8.ctypes.data, l8.strides[0], r8.ctypes.data, r8.strides[0]), de.handle)
        n1 = launches(de)
        dl, dr = torch.from_numpy(lf).cuda(), torch.from_numpy(rf).cuda()
        capi.check(L.psm_set_images_device(de.handle, dl.data_ptr(), W3(lf), dr.data_ptr(), W3(rf)), de.handle)
        n2 = launches(de)
        lt, ch = as_layout(l8, "chw_rgb")
        rt, _ = as_layout(r8, "chw_rgb")
        set_planes(de.handle, lt, rt, ch, l8.shape[:2])
        n3 = launches(de)
        shards = len(kw.get("devices", [0]))
        assert n1 - n0 == 4 * shards and n2 - n1 == 4 * shards     # unchanged: ingest + halo pass per view and shard
        assert n3 - n2 == 4                                          # one ingest_kernel + halo pass per view
        de.sync()


def W3(img):
    return img.shape[1] * 3 * img.itemsize


def test_rejected_arguments_change_nothing(scenes):
    l8, r8, _, _ = scenes["Cones"]
    H, W, _ = l8.shape
    with DispEst(l8, r8, D) as de:
        h = de.handle
        lt, _ = as_layout(l8, "hwc_bgr")
        ft = torch.zeros(H, W, 3, device="cuda")
        p, f = lt.data_ptr(), ft.data_ptr()
        ok = (C.c_void_p * 3)(p, p + 1, p + 2)
        okf = (C.c_void_p * 3)(f, f + 4, f + 8)
        n0 = launches(de)
        cases = [
            (capi.PSM_PIX_U8, None, ok, 3 * W, 3, "null channel pointer array"),
            (capi.PSM_PIX_U8, ok, (C.c_void_p * 3)(p, None, p + 2), 3 * W, 3, "null pointer for channel 1"),
            (0, ok, ok, 3 * W, 3, "unknown pixel type"),
            (3, ok, ok, 3 * W, 3, "unknown pixel type"),
            (capi.PSM_PIX_U8, ok, ok, 3 * W, 0, "col_step"),
            (capi.PSM_PIX_F32, okf, okf, 12 * W, 3, "col_step"),
            (capi.PSM_PIX_U8, ok, ok, 3 * (W - 1), 3, "row_step"),    # one byte short of (W - 1) * 3 + 1
            (capi.PSM_PIX_U8, ok, ok, 3 * W, 1 << 62, "row_step"),
            (capi.PSM_PIX_F32, okf, (C.c_void_p * 3)(f + 2, f + 4, f + 8), 12 * W, 12, "aligned"),
            (capi.PSM_PIX_F32, okf, okf, 12 * W + 2, 12, "multiples"),
        ]
        for pix, lp, rp, row, col, text in cases:
            assert L.psm_set_images_device_planes(h, pix, lp, rp, row, col) == capi.PSM_EINVAL, text
            assert text.encode() in L.psm_last_error(h), (text, L.psm_last_error(h))
        for lp, step in [(f + 2, 12 * W), (f, 12 * W + 2)]:   # interleaved float frames: the same 4-byte rule
            assert L.psm_set_images_device(h, lp, step, f, 12 * W) == capi.PSM_EINVAL, (lp - f, step)
            assert b"not a multiple of the 4 bytes" in L.psm_last_error(h), L.psm_last_error(h)
        hf = np.zeros((H, W, 3), np.float32)
        assert L.psm_set_images_async(h, hf.ctypes.data, 12 * W, None, 12 * W) == capi.PSM_EINVAL
        assert b"view 1" in L.psm_last_error(h), L.psm_last_error(h)
        assert L.psm_set_images_commit(h) == capi.PSM_ESTATE   # nothing was uploaded
        assert L.psm_cost_const(h) == capi.PSM_ESTATE      # no frame was taken
        m = torch.zeros(H, W, dtype=torch.uint8, device="cuda")
        for args, code in [((2, m.data_ptr(), W, m.data_ptr(), W), capi.PSM_EINVAL),
                           ((0, None, W, m.data_ptr(), W), capi.PSM_EINVAL),
                           ((0, m.data_ptr(), W - 1, m.data_ptr(), W), capi.PSM_EINVAL),
                           ((0, m.data_ptr(), W, None, W), capi.PSM_EINVAL),
                           ((0, m.data_ptr(), W, m.data_ptr(), W - 1), capi.PSM_EINVAL),
                           ((0, m.data_ptr(), W, m.data_ptr(), W), capi.PSM_ESTATE),   # no selection yet
                           ((1, m.data_ptr(), W, m.data_ptr(), W), capi.PSM_ESTATE)]:  # no post-process yet
            assert L.psm_copy_maps_device(h, *args) == code, args
        assert launches(de) == n0
        de.sync()


@pytest.mark.parametrize("kw", [dict(), dict(devices=[0, 0]), dict(map_bits=16)])
def test_copy_maps_state_rules(kw, scenes):
    l8, r8, _, _ = scenes["Cones"]
    H, W, _ = l8.shape
    with DispEst(l8, r8, D, **kw) as de:
        h = de.handle
        wide = kw.get("map_bits") == 16
        step = W * (2 if wide else 1)
        m = [torch.full((H, step), 7, dtype=torch.uint8, device="cuda") for _ in range(2)]
        ptrs = lambda: (m[0].data_ptr(), step, m[1].data_ptr(), step)  # noqa: E731
        host = lambda k: m[k].cpu().numpy().view(np.uint16) if wide else m[k].cpu().numpy()  # noqa: E731
        de.CostConst_GPU()
        de.CostFilter_GPU()
        assert L.psm_copy_maps_device(h, 0, *ptrs()) == capi.PSM_ESTATE
        de.DispSelect_GPU()
        capi.check(L.psm_copy_maps_device(h, 0, *ptrs()), h)
        torch.cuda.synchronize()
        assert_same(host(0), de.lDisMap, "selection lmap")
        assert_same(host(1), de.rDisMap, "selection rmap")
        assert L.psm_copy_maps_device(h, 1, *ptrs()) == capi.PSM_ESTATE
        de.PostProcess_GPU()
        capi.check(L.psm_copy_maps_device(h, 1, *ptrs()), h)
        torch.cuda.synchronize()
        assert_same(host(0), de.lDisMap, "post-processed lmap")
        assert_same(host(1), de.rDisMap, "post-processed rmap")
        de.setViews("left")       # resets the frame: nothing to copy until a selection / post-process has run again
        for which in (0, 1):
            assert L.psm_copy_maps_device(h, which, m[0].data_ptr(), step, None, 0) == capi.PSM_ESTATE
            assert L.psm_copy_maps_device(h, which, *ptrs()) == capi.PSM_EINVAL    # d_right on a left-only context
        de.CostConst_GPU()
        de.CostFilter_GPU()
        de.DispSelect_GPU()
        capi.check(L.psm_copy_maps_device(h, 0, m[0].data_ptr(), step, None, 0), h)
        assert L.psm_copy_maps_device(h, 1, m[0].data_ptr(), step, None, 0) == capi.PSM_ESTATE
        torch.cuda.synchronize()
        assert_same(host(0), de.lDisMap, "left-only lmap")


def test_wait_and_signal_on_the_default_stream(scenes, scene_maps):
    """NULL is the legacy default stream; a context bound with psm_set_stream keeps its binding"""
    l8, r8, _, _ = scenes["Cones"]
    with DispEst(l8, r8, D) as de:
        s = torch.cuda.Stream()
        capi.check(L.psm_set_stream(de.handle, C.c_void_p(s.cuda_stream)), de.handle)
        dl, dr = dev_frame(scenes, "Cones")
        capi.check(L.psm_wait_stream(de.handle, None), de.handle)
        set_planes(de.handle, dl, dr, "bgr", l8.shape[:2])
        for call in (L.psm_cost_const, L.psm_cost_filter, L.psm_disp_select_device):
            capi.check(call(de.handle), de.handle)
        m = [torch.empty_like(dl[..., 0]) for _ in range(2)]
        W = dl.shape[1]
        capi.check(L.psm_copy_maps_device(de.handle, 0, m[0].data_ptr(), W, m[1].data_ptr(), W), de.handle)
        capi.check(L.psm_signal_stream(de.handle, None), de.handle)
        torch.cuda.synchronize()
        check_maps(m[0], m[1], scene_maps["Cones"], "bound stream")
        capi.check(L.psm_set_stream(de.handle, None), de.handle)
