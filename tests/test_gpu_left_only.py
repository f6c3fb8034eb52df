"""GPU: left-only frames (PSM_OPT_VIEWS = PSM_VIEWS_LEFT).  A left-only frame skips every right-view stage after ingest.
Its left map must equal the two-view context's left map bit for bit, and the C oracle's where the repository has one; the
right view's buffers must keep their contents; switching back must not expose a right-view result of an earlier frame."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import image_cases as IC
from conftest import ROOT
from oracle import oracle as O
from primestereomatch_b200 import DispEst, capi, synth

pytestmark = pytest.mark.gpu


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def assert_same(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, f"{what}: {a.shape} {a.dtype} vs {b.shape} {b.dtype}"
    if not np.array_equal(a, b):
        bad = np.argwhere(a != b)
        i = tuple(bad[0])
        raise AssertionError(f"{what}: {len(bad)} of {a.size} differ, first at {list(i)}: {a[i]!r} vs {b[i]!r}")


def frame(de, fgf=None, post=False):
    de.CostConst_GPU()
    if fgf:
        de.setSubsampleRate(fgf)
        de.CostFilter_FGF_GPU()
    else:
        de.CostFilter_GPU()
    de.DispSelect_GPU()
    if post:
        de.PostProcess_GPU()
    return de.lDisMap.copy(), None if de.rDisMap is None else de.rDisMap.copy()


def both_and_left(l, r, D, setup=None, **kw):
    """one frame in a two-view context and in a left-only one -> (two-view maps, left-only left map)"""
    run_kw = {k: kw.pop(k) for k in ("fgf", "post") if k in kw}
    with DispEst(l, r, D, **kw) as de:
        if setup:
            setup(de)
        want = frame(de, **run_kw)
    with DispEst(l, r, D, **kw) as de:
        de.setViews("left")
        if setup:
            setup(de)
        got = frame(de, **run_kw)
        assert got[1] is None and de.rDisMap is None
    assert_same(got[0], want[0], "left-only vs two-view left map")
    return want, got[0]


# ---- 1. the scenes, both input formats ------------------------------------------------------------------------------
@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
@pytest.mark.parametrize("u8", [False, True])
def test_scenes(scene, u8, scenes, oracle_scene_results):
    l8, r8, l, r = scenes[scene]
    _, got = both_and_left(*((l8, r8) if u8 else (l, r)), 64)
    assert_same(got, oracle_scene_results[scene]["ld"], f"{scene} left-only vs oracle")


def test_u16_maps_at_d300():
    D, W = 300, 364
    k = next(k for k in range(1, 200) if 1 + (k * 17) % (D - 2) > 255)
    l8, r8, _ = synth.stereo_pair_u8(W, 40 * k + 48, D, seed=D)
    l, r = synth.to_f32(l8[40 * k - 8:]), synth.to_f32(r8[40 * k - 8:])
    _, got = both_and_left(l, r, D)
    lf, _ = O.cost_filter(l, r, *O.cost_const(l, r, D)[2:])
    assert_same(got, O.wta(lf, np.uint16), "D=300 left-only vs oracle")
    assert got.dtype == np.uint16 and int(got.max()) > 255


# ---- 2. a sharded context's keys -------------------------------------------------------------------------------------
def test_sharded_keys_uint64(scenes, oracle_scene_results):
    torch = pytest.importorskip("torch")
    _, _, l, r = scenes["Teddy"]
    H, W, _ = l.shape
    L = capi.lib()
    want = torch.zeros((2, 2, H * W), dtype=torch.int64, device="cuda")   # [view][rank][pix], two-view shards
    got = torch.zeros((2, H * W), dtype=torch.int64, device="cuda")       # [rank][pix], left-only shards
    for views, keys in (("both", want), ("left", got)):
        shards = [DispEst(l, r, 64, d_begin=0, d_count=27), DispEst(l, r, 64, d_begin=27, d_count=37)]
        try:
            for rank, de in enumerate(shards):
                de.setViews(views)
                de.CostConst_GPU(); de.CostFilter_GPU()
                right = keys[1, rank].data_ptr() if views == "both" else None
                capi.check(L.psm_disp_select_keys(de.handle, (keys[0, rank] if views == "both" else keys[rank]).data_ptr(),
                                                  right), de.handle)
                de.sync()
            if views == "left":
                ld = np.zeros((H, W), np.uint8)
                capi.check(L.psm_disp_reduce_keys(shards[0].handle, keys.data_ptr(), None, 2, ptr(ld), W, None, 0),
                           shards[0].handle)
                assert_same(ld, oracle_scene_results["Teddy"]["ld"], "reduced left-only keys vs oracle")
        finally:
            for de in shards:
                de.close()
    assert_same(got.cpu().numpy().view(np.uint64), want[0].cpu().numpy().view(np.uint64), "left keys (uint64)")


# ---- 3. blocked and multi-device contexts ----------------------------------------------------------------------------
@pytest.mark.parametrize("block", [1, 7, 64])
def test_blocked(block):
    W, H, D = 227, 61, 64
    l, r, _ = synth.stereo_pair_f32(W, H, D, seed=5)
    _, got = both_and_left(l, r, D, block_slices=block)
    assert_same(got, O.pipeline(l, r, D)["lDis"], f"blocked {block} left-only vs oracle")


@pytest.mark.parametrize("devices", [[0, 0], [0, 0, 0]])
@pytest.mark.parametrize("block", [None, 7])
def test_multi_device(devices, block):
    W, H, D = 227, 61, 64
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=11)
    _, got = both_and_left(l8, r8, D, devices=devices, block_slices=block)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    assert_same(got, O.pipeline(l, r, D)["lDis"], f"{devices} block {block} left-only vs oracle")


# ---- 4. every filter path --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", [1, 2, 4, 8])
def test_fgf(s):
    W, H, D = 227, 61, 48
    l, r, _ = synth.stereo_pair_f32(W, H, D, seed=s)
    _, got = both_and_left(l, r, D, fgf=s)
    lf, _ = O.cost_filter_fgf(l, r, *O.cost_const(l, r, D)[2:], s=s)
    assert_same(got, O.wta(lf), f"FGF s={s} left-only vs oracle")


@pytest.mark.parametrize("window", [5, 16])
def test_window(window):
    W, H, D = 227, 61, 48
    l, r, _ = synth.stereo_pair_f32(W, H, D, seed=window)
    _, got = both_and_left(l, r, D, setup=lambda de: de.setGuidedFilter(window, 1e-3))
    assert_same(got, O.pipeline(l, r, D, window=window, eps=1e-3)["lDis"], f"window {window} left-only vs oracle")


def test_matching_cost():
    W, H, D = 227, 61, 48
    l, r, _ = synth.stereo_pair_f32(W, H, D, seed=3)
    _, got = both_and_left(l, r, D, setup=lambda de: de.setMatchingCost(0.6, 0.2, 0.05))
    assert_same(got, O.pipeline(l, r, D, alpha=0.6, tau_color=0.2, tau_grad=0.05)["lDis"], "cost setting vs oracle")


@pytest.mark.parametrize("mode", [capi.PSM_CVF_MIXED, capi.PSM_CVF_NAIVE])
def test_mixed_and_naive(mode):
    W, H, D = 227, 61, 48
    l, r, _ = synth.stereo_pair_f32(W, H, D, seed=21)
    _, got = both_and_left(l, r, D, setup=lambda de: de.set_option(capi.PSM_OPT_CVF_MODE, mode))
    if mode == capi.PSM_CVF_NAIVE:
        assert_same(got, O.pipeline(l, r, D)["lDis"], "NAIVE left-only vs oracle")


@pytest.mark.parametrize("kind", ["negative", "above1", "nan"])
def test_reference_order_pass(kind):
    """float frames outside the integer domain take the reference-order pass for the flagged view"""
    W, H, D = 96, 40, 24
    l, r = IC.frame(kind, W, H, D)
    _, got = both_and_left(l, r, D)
    if kind in IC.FLAGGED:   # flagged views run in OpenCV's order: bit for bit with the oracle
        with np.errstate(all="ignore"):
            lf, _ = O.cost_filter(l, r, *O.cost_const(l, r, D)[2:])
        assert_same(got, O.wta(lf), f"{kind} left-only vs oracle")


# ---- 5. the post-filter ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("generic", [False, True])
def test_post_filter(generic):
    W, H, D = 227, 61, 48
    l, r, _ = synth.stereo_pair_f32(W, H, D, seed=8)
    setup = (lambda de: de.setPostFilter(5, 12.0, 2, "iv1")) if generic else None
    _, got = both_and_left(l, r, D, setup=setup, post=True)
    pp = dict(r=5, sigma=12.0, iterations=2, weight="iv1") if generic else {}
    assert_same(got, O.post_process(l, O.pipeline(l, r, D)["lDis"], **pp), "post-filtered left-only vs oracle")


# ---- 6. geometry edges -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W,H,D", [(227, 61, 40), (13, 11, 8), (30, 9, 12)])
def test_geometry(W, H, D):
    l, r, _ = synth.stereo_pair_f32(W, H, D, seed=W)
    _, got = both_and_left(l, r, D)
    assert_same(got, O.pipeline(l, r, D)["lDis"], f"{W}x{H}x{D} left-only vs oracle")


# ---- 7. the right view is not touched; launch counts -----------------------------------------------------------------
class DeviceArray:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 3}


def device_bytes(torch, de, what, n):
    p, pitch = C.c_void_p(), C.c_size_t()
    capi.check(capi.lib().psm_device_ptr(de.handle, what, C.byref(p), C.byref(pitch)), de.handle)
    return p.value, torch.as_tensor(DeviceArray(p.value, n), device="cuda")


def test_right_view_untouched(scenes):
    torch = pytest.importorskip("torch")
    l8, r8, _, _ = scenes["Cones"]
    H, W, _ = l8.shape
    D = 64
    Wp = None
    with DispEst(l8, r8, D) as de:
        frame(de, post=True)   # allocates the post-filtered maps
        de.sync()
        pitch = C.c_size_t()
        capi.check(capi.lib().psm_device_ptr(de.handle, 1, C.byref(C.c_void_p()), C.byref(pitch)), de.handle)
        Wp = pitch.value
        sizes = {1: D * H * Wp * 4, 3: H * W, 5: H * W}
        bufs = {w: device_bytes(torch, de, w, n) for w, n in sizes.items()}
        de.setViews("left")
        pattern = torch.arange(max(sizes.values()), device="cuda", dtype=torch.int64).remainder(251).to(torch.uint8)
        for w, (_, t) in bufs.items():
            t.copy_(pattern[:t.numel()])
        torch.cuda.synchronize()
        for _ in range(2):
            frame(de, post=True)
        de.sync()
        for w, (addr, t) in bufs.items():
            assert device_bytes(torch, de, w, 1)[0] == addr, f"psm_device_ptr {w} moved"
            assert torch.equal(t, pattern[:t.numel()]), f"psm_device_ptr {w}: a left-only frame wrote the right view"


def stage_counts(de, post=True):
    L = capi.lib()
    h = de.handle
    l, r = np.ascontiguousarray(de._lImg), np.ascontiguousarray(de._rImg)
    steps = [lambda: capi.check(L.psm_set_images_u8(h, ptr(l), l.strides[0], ptr(r), r.strides[0]), h),
             lambda: capi.check(L.psm_cost_const(h), h),
             lambda: capi.check(L.psm_cost_filter(h), h),
             lambda: de.DispSelect_GPU()]
    if post:
        steps.append(lambda: de.PostProcess_GPU())
    out = []
    for s in steps:
        n = de.launch_count()
        s()
        out.append(de.launch_count() - n)
    return out


@pytest.mark.parametrize("block", [None, 16])
def test_launch_counts(block):
    W, H, D = 227, 61, 64
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=2)
    with DispEst(l8, r8, D, block_slices=block) as de:
        both = stage_counts(de, post=block is None)
        de.setViews("left")
        left = stage_counts(de, post=block is None)
    if block is None:
        # ingest: ingest + halo per view; CVC: one launch for the views it builds; filter: guide + streaming kernel;
        # selection: one WTA per view; post-filter: pack + filter per view
        assert both == [4, 1, 2, 2, 4] and left == [4, 1, 2, 1, 2], (both, left)
    else:
        nb = D // block   # filter: guide, then per block (CVC after the first) the streaming kernel and the fold
        assert both == [4, 1, 1 + 2 * nb + nb - 1, 2] and left == [4, 1, 1 + 2 * nb + nb - 1, 1], (both, left)


# ---- 8. switching back, rejected calls, the async upload pair, the C++ demo ------------------------------------------
def test_switch_back_no_stale_right(scenes):
    """frame A with both views, frame B left-only, then both views on frame B without a new upload"""
    _, _, la, ra = scenes["Cones"]
    _, _, lb, rb = scenes["Teddy"]
    D = 64
    ref_b = O.pipeline(lb, rb, D)
    L = capi.lib()
    with DispEst(la, ra, D) as de:
        frame(de)
        de.setInputImages(lb, rb)
        de.setViews("left")
        got_l, _ = frame(de)
        assert_same(got_l, ref_b["lDis"], "frame B left-only")
        de.setViews("both")
        h = de.handle
        capi.check(L.psm_cost_const(h), h)
        capi.check(L.psm_cost_filter(h), h)
        de.DispSelect_GPU()
        assert_same(de.lDisMap, ref_b["lDis"], "frame B both views, left")
        assert_same(de.rDisMap, ref_b["rDis"], "frame B both views, right (a stale right guide would differ)")


def expect(rc, code, de, *words):
    text = capi.lib().psm_last_error(de.handle).decode()
    assert rc == code, (rc, text)
    for w in words:
        assert w in text, (w, text)


def test_rejected_calls():
    W, H, D = 96, 40, 24
    l, r, _ = synth.stereo_pair_f32(W, H, D, seed=4)
    L = capi.lib()
    ld, rd = np.zeros((H, W), np.uint8), np.zeros((H, W), np.uint8)
    plane = np.zeros((H, W), np.float32)
    a3, b = np.zeros((3, H, W), np.float32), np.zeros((H, W), np.float32)
    with DispEst(l, r, D) as de:
        h = de.handle
        frame(de)
        for bad in (0, 3, -1):
            expect(L.psm_set_option(h, capi.PSM_OPT_VIEWS, bad), capi.PSM_EINVAL, de, "PSM_OPT_VIEWS")
        capi.check(L.psm_disp_select(h, ptr(ld), W, ptr(rd), W), h)   # unchanged: still both views, still selectable
        capi.check(L.psm_set_option(h, capi.PSM_OPT_VIEWS, capi.PSM_VIEWS_LEFT), h)
        # the stage state is reset: the next stage must be psm_cost_const
        expect(L.psm_cost_filter(h), capi.PSM_ESTATE, de, "PSM_OPT_VIEWS")
        expect(L.psm_cost_filter_fgf(h, 4), capi.PSM_ESTATE, de, "PSM_OPT_VIEWS")
        expect(L.psm_disp_select_device(h), capi.PSM_ESTATE, de)
        expect(L.psm_post_process(h, ptr(ld), W, None, 0), capi.PSM_ESTATE, de, "PSM_OPT_VIEWS")
        capi.check(L.psm_cost_const(h), h)
        capi.check(L.psm_cost_filter(h), h)
        expect(L.psm_disp_select(h, ptr(ld), W, ptr(rd), W), capi.PSM_EINVAL, de, "PSM_OPT_VIEWS", "NULL")
        expect(L.psm_disp_select_async(h, ptr(ld), W, ptr(rd), W), capi.PSM_EINVAL, de, "PSM_OPT_VIEWS")
        expect(L.psm_disp_select_keys(h, ptr(np.zeros(1, np.uint64)), ptr(np.zeros(1, np.uint64))), capi.PSM_EINVAL, de,
               "PSM_OPT_VIEWS")
        capi.check(L.psm_disp_select(h, ptr(ld), W, None, 0), h)
        for mode in (capi.PSM_LR_FILL_WMF, capi.PSM_LR_FILL):
            de.setLRCheck(mode)
            expect(L.psm_post_process(h, ptr(ld), W, None, 0), capi.PSM_ESTATE, de, "psm_set_lr_check", "PSM_OPT_VIEWS")
        de.setLRCheck(capi.PSM_LR_OFF)
        expect(L.psm_post_process(h, ptr(ld), W, ptr(rd), W), capi.PSM_EINVAL, de, "PSM_OPT_VIEWS")
        capi.check(L.psm_post_process(h, ptr(ld), W, None, 0), h)
        R = capi.PSM_RIGHT
        expect(L.psm_read_cost_slice(h, R, 3, ptr(plane), W * 4), capi.PSM_ESTATE, de, "PSM_OPT_VIEWS")
        expect(L.psm_read_ab_slice(h, R, 3, ptr(a3), ptr(b)), capi.PSM_ESTATE, de, "PSM_OPT_VIEWS")
        for p in range(3, 12):
            expect(L.psm_read_guide_plane(h, R, p, ptr(plane), W * 4), capi.PSM_ESTATE, de, "PSM_OPT_VIEWS")
        for p in (0, 1, 2, 12):
            capi.check(L.psm_read_guide_plane(h, R, p, ptr(plane), W * 4), h)
        for v in (capi.PSM_LEFT, R):
            expect(L.psm_read_valid_mask(h, v, ptr(ld), W), capi.PSM_ESTATE, de, "PSM_OPT_VIEWS")
        capi.check(L.psm_read_cost_slice(h, capi.PSM_LEFT, 3, ptr(plane), W * 4), h)
        # back to both views: the right view is stale until psm_cost_const
        capi.check(L.psm_set_option(h, capi.PSM_OPT_VIEWS, capi.PSM_VIEWS_BOTH), h)
        expect(L.psm_read_cost_slice(h, R, 3, ptr(plane), W * 4), capi.PSM_ESTATE, de, "PSM_OPT_VIEWS")
        expect(L.psm_disp_select(h, ptr(ld), W, ptr(rd), W), capi.PSM_ESTATE, de)


def test_python_facade_views():
    W, H, D = 96, 40, 24
    l, r, _ = synth.stereo_pair_f32(W, H, D, seed=6)
    with DispEst(l, r, D) as de:
        for bad in ("right", "LEFT", 1, None):
            with pytest.raises(ValueError):
                de.setViews(bad)
        assert de.rDisMap is not None
        de.setViews("left")
        frame(de)
        assert de.rDisMap is None
        de.setLRCheck(capi.PSM_LR_FILL)
        with pytest.raises(capi.PsmError):
            de.PostProcess_GPU()
        de.setLRCheck(capi.PSM_LR_OFF)
        de.setViews("both")
        assert de.rDisMap is not None and not de.rDisMap.any()
        ld, rd = frame(de)
        ref = O.pipeline(l, r, D)
        assert_same(ld, ref["lDis"], "left after switching back")
        assert_same(rd, ref["rDis"], "right after switching back")


def test_async_upload_pair_alternating(scenes, oracle_scene_results):
    L = capi.lib()
    seq = ["Cones", "Teddy", "Cones", "Teddy"]
    l8, r8, _, _ = scenes["Cones"]
    H, W, _ = l8.shape
    with DispEst(l8, r8, 64) as de:
        de.setViews("left")
        h = de.handle

        def upload(name):
            l, r = scenes[name][0], scenes[name][1]
            capi.check(L.psm_set_images_u8_async(h, ptr(l), l.strides[0], ptr(r), r.strides[0]), h)

        upload(seq[0])
        capi.check(L.psm_set_images_commit(h), h)
        for k, name in enumerate(seq):
            capi.check(L.psm_cost_const(h), h)
            capi.check(L.psm_cost_filter(h), h)
            if k + 1 < len(seq):
                upload(seq[k + 1])   # the next frame's copy overlaps this frame's filter
            ld = np.zeros((H, W), np.uint8)
            capi.check(L.psm_disp_select(h, ptr(ld), W, None, 0), h)
            assert_same(ld, oracle_scene_results[name]["ld"], f"frame {k} ({name})")
            if k + 1 < len(seq):
                capi.check(L.psm_set_images_commit(h), h)


def test_cpp_demo_left_only(tmp_path, scenes, oracle, oracle_scene_results):
    exe = os.path.join(ROOT, "primestereomatch_b200", "host", "dispest_demo")
    if not os.path.exists(exe):
        pytest.skip("dispest_demo not built")
    _, _, l, r = scenes["Teddy"]
    H, W, _ = l.shape
    l.tofile(tmp_path / "l.f32"); r.tofile(tmp_path / "r.f32")
    maps = {}
    for flag in ([], ["--left-only"]):
        tag = "lo" if flag else "both"
        out = subprocess.run([exe, *flag, str(W), str(H), "64", str(tmp_path / "l.f32"), str(tmp_path / "r.f32"),
                              str(tmp_path / f"l_{tag}.u8"), str(tmp_path / f"r_{tag}.u8")],
                             capture_output=True, text=True, timeout=120)
        assert out.returncode == 0, out.stderr
        maps[tag] = np.fromfile(tmp_path / f"l_{tag}.u8", np.uint8).reshape(H, W)
    assert not (tmp_path / "r_lo.u8").exists()
    assert_same(maps["lo"], maps["both"], "demo --left-only left map")
    assert_same(maps["lo"], oracle.post_process(l, oracle_scene_results["Teddy"]["ld"]), "demo --left-only vs oracle")


# ---- 9. switching back on contexts with an exchange block ------------------------------------------------------------
@pytest.mark.parametrize("block", [None, 7])
def test_multi_device_switch_back(block):
    """two co-located shards: two-view, left-only, two-view, two-view frames on one context, selection and post-filter
    after each; the post-filter is refused only while the exchanged right map is older than the left one"""
    W, H, D = 227, 61, 64
    pairs = [synth.stereo_pair_f32(W, H, D, seed=30 + k)[:2] for k in range(2)]
    refs = [O.pipeline(l, r, D) for l, r in pairs]
    L = capi.lib()
    with DispEst(*pairs[0], D, devices=[0, 0], block_slices=block) as de:
        plan = [("both", 0), ("left", 1), ("both", 1), ("both", 0), ("left", 0), ("both", 1)]
        for k, (views, p) in enumerate(plan):
            l, r = pairs[p]
            de.setViews(views)
            de.setInputImages(l, r)
            if views == "both" and k > 0 and plan[k - 1][0] == "left":
                de.CostConst_GPU()   # the right map in the exchange blocks is from an earlier frame until a selection
                expect(L.psm_post_process(de.handle, ptr(np.zeros((H, W), np.uint8)), W, ptr(np.zeros((H, W), np.uint8)), W),
                       capi.PSM_ESTATE, de, "left-only")
            ld, rd = frame(de)
            what = f"frame {k} ({views}, block {block})"
            assert_same(ld, refs[p]["lDis"], f"{what} left")
            if views == "both":
                assert_same(rd, refs[p]["rDis"], f"{what} right")
            de.PostProcess_GPU()
            assert_same(de.lDisMap, O.post_process(l, refs[p]["lDis"]), f"{what} post-filtered left")
            if views == "both":
                assert_same(de.rDisMap, O.post_process(r, refs[p]["rDis"]), f"{what} post-filtered right")


def test_fused_exchange_switch_back(scenes, oracle_scene_results):
    """two ranks in one process on the flag-synchronised fused exchange (PSM_OPT_P2P_SYNC = 1): two-view, left-only,
    left-only, two-view and two-view frames, each fetched; the device-side waits must follow the per-view frame counts"""
    L = capi.lib()
    names = ["Teddy", "Cones", "Teddy", "Cones", "Teddy"]
    views = ["both", "left", "left", "both", "both"]
    l0, r0 = scenes["Teddy"][2:]
    H, W, _ = l0.shape
    shards = [DispEst(l0, r0, 64, d_begin=0, d_count=40), DispEst(l0, r0, 64, d_begin=40, d_count=24)]
    try:
        bufs = (C.c_void_p * 2)()
        for k, de in enumerate(shards):
            p = C.c_void_p()
            capi.check(L.psm_p2p_create_buffer(de.handle, 2, C.byref(p)), de.handle)
            bufs[k] = p.value
        for k, de in enumerate(shards):
            capi.check(L.psm_p2p_set_peers(de.handle, bufs, 2, k), de.handle)
        for f, (name, v) in enumerate(zip(names, views)):
            l, r = scenes[name][2:]
            for de in shards:
                de.setViews(v)
                de.setInputImages(l, r)
                de.CostConst_GPU()
                if v == "both" and f > 0 and views[f - 1] == "left":
                    expect(L.psm_disp_fetch_p2p(de.handle, ptr(np.zeros((H, W), np.uint8)), W,
                                                ptr(np.zeros((H, W), np.uint8)), W), capi.PSM_ESTATE, de, "left-only")
                de.CostFilter_GPU()
                capi.check(L.psm_disp_select_keys_p2p(de.handle), de.handle)
            for de in shards:
                de.sync()                                   # stands in for the cross-rank barrier
            for de in shards:
                capi.check(L.psm_disp_reduce_p2p(de.handle), de.handle)
            for de in shards:
                de.sync()
            for rank, de in enumerate(shards):
                ld, rd = np.zeros((H, W), np.uint8), np.zeros((H, W), np.uint8)
                right = ptr(rd) if v == "both" else None
                capi.check(L.psm_disp_fetch_p2p(de.handle, ptr(ld), W, right, W), de.handle)
                what = f"frame {f} ({name}, {v}) rank {rank}"
                assert_same(ld, oracle_scene_results[name]["ld"], f"{what} left")
                if v == "both":
                    assert_same(rd, oracle_scene_results[name]["rd"], f"{what} right")
    finally:
        for de in shards:
            de.close()
