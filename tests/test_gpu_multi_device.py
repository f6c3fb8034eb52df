"""GPU: multi-device contexts (psm_create_multi).  One context drives several shards through the fused exchange, ordered
by CUDA events.  Its maps must equal a single-device context's of the same geometry bit for bit, and the CPU oracle's
where the repository has one.  On one H100 the shards are co-located on device 0: every code path runs except real
peer stores.  The same parity cases run on [0, 1] and on every visible device when there are two or more GPUs."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import pp_chain as PP
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


def run(l, r, D, setup=None, fgf=None, post=False, **kw):
    """one frame through a context -> (left map, right map[, left mask, right mask])"""
    with DispEst(l, r, D, **kw) as de:
        if setup:
            setup(de)
        de.CostConst_GPU()
        if fgf:
            de.setSubsampleRate(fgf)
            de.CostFilter_FGF_GPU()
        else:
            de.CostFilter_GPU()
        de.DispSelect_GPU()
        if post:
            de.PostProcess_GPU()
            if de.lr_mode:
                return de.lDisMap.copy(), de.rDisMap.copy(), de.lValid.copy(), de.rValid.copy()
        return de.lDisMap.copy(), de.rDisMap.copy()


def same_maps(got, want, what):
    for k, (g, w) in enumerate(zip(got, want)):
        assert_same(g, w, f"{what} [{k}]")


def ngpu():
    return capi.lib().psm_device_count()


def device_lists():
    """co-located shards on device 0; [0, 1] and every visible device where there are two or more"""
    out = [[0, 0], [0, 0, 0]]
    if ngpu() >= 2:
        out += [[0, 1], list(range(min(ngpu(), 8)))]
    return out


def distinct(devs):
    if len(set(devs)) > 1 and ngpu() < 2:
        pytest.skip("needs >= 2 GPUs")


# ---- 1. shard counts with uneven remainders, both map formats, against the single-device context and the oracle -------
@pytest.mark.parametrize("D,n", [(64, 2), (64, 3), (64, 8), (61, 8)])
@pytest.mark.parametrize("u8", [False, True])
def test_shard_counts_match_single_device_and_oracle(D, n, u8):
    W, H = 227, 61
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=D + n)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    li, ri = (l8, r8) if u8 else (l, r)
    want = run(li, ri, D)
    ref = O.pipeline(l, r, D)
    same_maps(want, (ref["lDis"], ref["rDis"]), "single vs oracle")
    same_maps(run(li, ri, D, devices=[0] * n), want, f"n={n}")
    assert want[0].any()


@pytest.mark.parametrize("devices", [[0, 0, 0], [0, 1], "all"])
def test_u16_maps_at_d300(devices):
    if devices == "all":
        devices = list(range(min(max(ngpu(), 1), 8)))
        if len(devices) < 2:
            pytest.skip("needs >= 2 GPUs")
    distinct(devices)
    D, W = 300, 364
    k = next(k for k in range(1, 200) if 1 + (k * 17) % (D - 2) > 255)
    l8, r8, _ = synth.stereo_pair_u8(W, 40 * k + 48, D, seed=D)
    l, r = synth.to_f32(l8[40 * k - 8:]), synth.to_f32(r8[40 * k - 8:])
    want = run(l, r, D)
    got = run(l, r, D, devices=devices)
    same_maps(got, want, f"D=300 on {devices}")
    lf, rf = O.cost_filter(l, r, *O.cost_const(l, r, D)[2:])
    assert_same(got[0], O.wta(lf, np.uint16), "D=300 left vs oracle")
    assert int(got[0].max()) > 255


# ---- 2. blocked shards (ragged last blocks) next to unblocked ones ----------------------------------------------------
@pytest.mark.parametrize("devices", device_lists())
@pytest.mark.parametrize("block", [7, 16])
def test_blocked_shards(devices, block):
    distinct(devices)
    W, H, D = 227, 61, 64
    l, r, _ = synth.stereo_pair_f32(W, H, D, seed=9)
    want = run(l, r, D)
    same_maps(run(l, r, D, block_slices=block), want, "single blocked")
    same_maps(run(l, r, D, devices=devices, block_slices=block), want, f"{devices} blocked {block}")
    same_maps(run(l, r, D, devices=devices), want, f"{devices} unblocked")


def test_blocked_u16_at_d1024():
    W, H, D, B = 1090, 24, 1024, 100
    l8, r8, _ = synth.stereo_pair_u8(W, 48 + 40 * 16, 1024, seed=3)
    k = next(k for k in range(1, 40) if 1 + (k * 17) % (D - 2) > 255)
    l, r = synth.to_f32(l8[40 * k - 8:40 * k - 8 + H]), synth.to_f32(r8[40 * k - 8:40 * k - 8 + H])
    want = run(l, r, D, block_slices=B, map_bits=16)
    got = run(l, r, D, devices=[0, 0, 0], block_slices=B, map_bits=16)
    same_maps(got, want, "D=1024 blocked shards")
    lf, rf = O.cost_filter(l, r, *O.cost_const(l, r, D)[2:])
    assert_same(got[1], O.wta(rf, np.uint16), "D=1024 right vs oracle")
    assert int(got[0].max()) > 255


# ---- 3. filter paths and settings -------------------------------------------------------------------------------------
SETTINGS = {
    "fgf4": dict(fgf=4),
    "fgf2_blocked": dict(fgf=2, block_slices=9),
    "window5": dict(setup=lambda de: de.setGuidedFilter(5, 1e-3)),
    "cost": dict(setup=lambda de: de.setMatchingCost(0.11, 0.21, 0.008)),
    "post": dict(setup=lambda de: de.setPostFilter(4, 10.0, 2, "iv1"), post=True),
    "mixed": dict(setup=lambda de: de.set_option(capi.PSM_OPT_CVF_MODE, capi.PSM_CVF_MIXED)),
}


@pytest.mark.parametrize("name", list(SETTINGS))
def test_settings(name):
    W, H, D = 227, 61, 40
    l, r, _ = synth.stereo_pair_f32(W, H, D, seed=5)
    kw = SETTINGS[name]
    want = run(l, r, D, **kw)
    same_maps(run(l, r, D, devices=[0, 0, 0], **kw), want, name)
    assert want[0].any()
    if name == "post":
        ref = O.pipeline(l, r, D)
        same_maps(want, PP.chain(l, r, ref["lDis"], ref["rDis"], setting=(4, 10.0, 2, "iv1"))[:2], "post vs oracle")


@pytest.mark.parametrize("mode", [capi.PSM_LR_FILL_WMF, capi.PSM_LR_FILL])
@pytest.mark.parametrize("devices", device_lists())
def test_lr_check_and_valid_masks(mode, devices, scenes):
    distinct(devices)
    l8, r8, _, _ = scenes["Cones"]
    l8, r8 = np.ascontiguousarray(l8[100:196, 80:336]), np.ascontiguousarray(r8[100:196, 80:336])
    l, r = synth.to_f32(l8), synth.to_f32(r8)

    def setup(de):
        de.setLRCheck(mode)

    want = run(l8, r8, 64, setup=setup, post=True)
    got = run(l8, r8, 64, setup=setup, post=True, devices=devices)
    same_maps(got, want, f"lr {mode} on {devices}")
    ref = O.pipeline(l, r, 64)
    pl, pr, (lv, rv) = PP.chain(l, r, ref["lDis"], ref["rDis"], lr=mode)
    assert_same(got[2], lv, "left mask vs oracle"); assert_same(got[3], rv, "right mask vs oracle")
    same_maps(got[:2], (pl, pr), "post-processed vs oracle")


# ---- 4. frames in a row: host (float, u8) and device frames, no host wait between frames ------------------------------
def _frames(n, W, H, D):
    out = []
    for f in range(n):
        l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=100 + f)
        out.append((l8, r8))
    return out


@pytest.mark.parametrize("kind", ["f32", "u8", "device"])
@pytest.mark.parametrize("devices", device_lists())
def test_consecutive_frames(kind, devices):
    """three frames with different images, each: upload, CVC, CVF, asynchronous selection into its own page-locked
    buffers, post-filter on the device; one host wait at the end.  A setter changes before the third frame."""
    import torch
    distinct(devices)
    W, H, D = 301, 53, 48
    frames = _frames(3, W, H, D)
    L = capi.lib()
    want = []
    with DispEst(frames[0][0], frames[0][1], D) as ref:
        for f, (l8, r8) in enumerate(frames):
            if f == 2:
                ref.setGuidedFilter(5, 1e-3); ref.setPostFilter(3, 25.5, 1, "exp")
            li, ri = (l8, r8) if kind == "u8" else (synth.to_f32(l8), synth.to_f32(r8))
            ref.setInputImages(li, ri)
            ref.CostConst_GPU(); ref.CostFilter_GPU(); ref.DispSelect_GPU()
            sel = (ref.lDisMap.copy(), ref.rDisMap.copy())
            ref.PostProcess_GPU()
            want.append((sel, (ref.lDisMap.copy(), ref.rDisMap.copy())))
    dev_imgs = [[torch.from_numpy(synth.to_f32(x)).to("cuda:%d" % devices[0]) for x in fr] for fr in frames]
    torch.cuda.synchronize()
    pinned = [[torch.zeros((H, W), dtype=torch.uint8).pin_memory() for _ in range(2)] for _ in frames]
    with DispEst(frames[0][0], frames[0][1], D, devices=devices) as de:
        h = de.handle
        for f, (l8, r8) in enumerate(frames):
            if f == 2:
                de.setGuidedFilter(5, 1e-3); de.setPostFilter(3, 25.5, 1, "exp")
            if kind == "u8":
                capi.check(L.psm_set_images_u8(h, ptr(l8), 3 * W, ptr(r8), 3 * W), h)
            elif kind == "f32":
                lf, rf = synth.to_f32(l8), synth.to_f32(r8)
                capi.check(L.psm_set_images(h, ptr(lf), 12 * W, ptr(rf), 12 * W), h)
            else:
                li, ri = dev_imgs[f]
                capi.check(L.psm_set_images_device(h, li.data_ptr(), 12 * W, ri.data_ptr(), 12 * W), h)
            capi.check(L.psm_cost_const(h), h)
            capi.check(L.psm_cost_filter(h), h)
            pl, pr = pinned[f]
            capi.check(L.psm_disp_select_async(h, pl.data_ptr(), W, pr.data_ptr(), W), h)
            capi.check(L.psm_post_process_device(h), h)
        de.sync()
        for f in range(3):
            same_maps([p.numpy() for p in pinned[f]], want[f][0], f"{kind} frame {f} selection on {devices}")
        # the context's device maps after psm_sync: selectors 2 / 3 the last selection, 4 / 5 its post-filter
        dev = [read_device_map(L, h, what, H, W) for what in (2, 3, 4, 5)]
        same_maps(dev[:2], want[2][0], f"{kind} last frame device maps on {devices}")
        same_maps(dev[2:], want[2][1], f"{kind} last frame post-filter on {devices}")


def read_device_map(L, h, what, H, W):
    p, pitch = C.c_void_p(), C.c_size_t()
    capi.check(L.psm_device_ptr(h, what, C.byref(p), C.byref(pitch)), h)
    assert p.value and pitch.value == W
    m = np.empty((H, W), np.uint8)
    rt = C.CDLL("libcudart.so.12")
    rt.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
    assert rt.cudaMemcpy(ptr(m), p, H * W, 4) == 0   # cudaMemcpyDefault
    return m


# ---- 5. per-slice reads routed to the owning shard, errors, launches ---------------------------------------------------
def test_cost_slices_are_routed_to_their_shard():
    W, H, D = 130, 40, 64
    l, r, _ = synth.stereo_pair_f32(W, H, D, seed=12)
    with DispEst(l, r, D) as one, DispEst(l, r, D, devices=[0, 0, 0]) as de:   # shards [0, 21), [21, 42), [42, 64)
        one.CostConst_GPU(); de.CostConst_GPU()
        for d in (0, 20, 21, 41, 42, 63):
            assert_same(de.read_cost_slice(1, d), one.read_cost_slice(1, d), f"raw slice {d}")
        a, b = de.read_ab_slice(0, 50)
        a0, b0 = one.read_ab_slice(0, 50)
        assert_same(a, a0, "a of slice 50"); assert_same(b, b0, "b of slice 50")
        for plane in (0, 4, 12):
            assert_same(de.read_guide_plane(1, plane), one.read_guide_plane(1, plane), f"guide plane {plane}")
        sl = one.read_cost_slice(0, 30) * 0.5
        de.write_cost_slice(0, 30, sl); one.write_cost_slice(0, 30, sl)
        one.CostFilter_GPU(); de.CostFilter_GPU()
        assert_same(de.read_cost_volume(0), one.read_cost_volume(0), "filtered left volume")
        one.DispSelect_GPU(); de.DispSelect_GPU()
        same_maps((de.lDisMap, de.rDisMap), (one.lDisMap, one.rDisMap), "maps after a written slice")
        with pytest.raises(capi.PsmError) as e:
            de.read_cost_slice(0, D)
        assert e.value.code == capi.PSM_EINVAL


def test_errors_and_state():
    L = capi.lib()
    W, H, D = 64, 24, 40
    l, r, _ = synth.stereo_pair_f32(W, H, D, seed=2)
    u8 = np.zeros((H, W), np.uint8)
    ctx = C.c_void_p()
    assert L.psm_create_multi(C.byref(ctx), W, H, D, (C.c_int * 2)(0, ngpu()), 2, 0, 8) == capi.PSM_EINVAL
    assert not ctx and b"not available" in L.psm_last_error(None)
    with DispEst(l, r, D, devices=[0, 0]) as de:
        h = de.handle
        assert L.psm_cost_const(h) == capi.PSM_ESTATE
        de.CostConst_GPU()
        assert L.psm_disp_select(h, ptr(u8), W, ptr(u8), W) == capi.PSM_ESTATE
        assert L.psm_disp_select_u16(h, ptr(u8), 2 * W, ptr(u8), 2 * W) == capi.PSM_EINVAL
        # a setter value the shards reject leaves the context as it was
        with pytest.raises(capi.PsmError):
            de.setGuidedFilter(0, 1e-4)
        with pytest.raises(capi.PsmError):
            de.setLRCheck(7)
        keys = (C.c_void_p * 2)()
        p, pitch = C.c_void_p(), C.c_size_t()
        hs = C.create_string_buffer(64)
        calls = {
            "psm_set_stream": lambda: L.psm_set_stream(h, None),
            "psm_set_images_async": lambda: L.psm_set_images_async(h, ptr(l), 12 * W, ptr(r), 12 * W),
            "psm_set_images_u8_async": lambda: L.psm_set_images_u8_async(h, ptr(u8), 3 * W, ptr(u8), 3 * W),
            "psm_set_images_commit": lambda: L.psm_set_images_commit(h),
            "psm_device_ptr 0": lambda: L.psm_device_ptr(h, 0, C.byref(p), C.byref(pitch)),
            "psm_device_ptr 1": lambda: L.psm_device_ptr(h, 1, C.byref(p), C.byref(pitch)),
            "psm_disp_select_keys": lambda: L.psm_disp_select_keys(h, keys[0], keys[1]),
            "psm_disp_reduce_keys": lambda: L.psm_disp_reduce_keys(h, keys[0], keys[1], 2, None, 0, None, 0),
            "psm_disp_reduce_keys_u16": lambda: L.psm_disp_reduce_keys_u16(h, keys[0], keys[1], 2, None, 0, None, 0),
            "psm_p2p_create_buffer": lambda: L.psm_p2p_create_buffer(h, 2, C.byref(p)),
            "psm_ipc_export": lambda: L.psm_ipc_export(h, p, hs),
            "psm_ipc_import": lambda: L.psm_ipc_import(h, hs.raw, C.byref(p)),
            "psm_p2p_set_peers": lambda: L.psm_p2p_set_peers(h, keys, 2, 0),
            "psm_disp_select_keys_p2p": lambda: L.psm_disp_select_keys_p2p(h),
            "psm_disp_reduce_p2p": lambda: L.psm_disp_reduce_p2p(h),
            "psm_disp_fetch_p2p": lambda: L.psm_disp_fetch_p2p(h, ptr(u8), W, ptr(u8), W),
            "psm_disp_fetch_p2p_u16": lambda: L.psm_disp_fetch_p2p_u16(h, ptr(u8), 2 * W, ptr(u8), 2 * W),
            "PSM_OPT_P2P_SYNC": lambda: L.psm_set_option(h, capi.PSM_OPT_P2P_SYNC, 1),
        }
        for name, call in calls.items():
            assert call() == capi.PSM_EINVAL, name
            assert b"multi-device" in L.psm_last_error(h), name
        # still computes what a single-device context computes, at the default settings
        de.CostFilter_GPU(); de.DispSelect_GPU()
        same_maps((de.lDisMap, de.rDisMap), run(l, r, D), "after the rejected calls")
        ms = C.c_float()
        assert L.psm_read_valid_mask(h, 0, ptr(u8), W) == capi.PSM_ESTATE
        assert L.psm_stage_ms(h, 5, C.byref(ms)) == capi.PSM_ESTATE
        for stage in (0, 1, 2, 3, 4):
            assert de.stage_ms(stage) > 0, stage


def test_launch_counts():
    """a multi-device context counts its shards' launches: per shard what a shard context launches, plus the exchange"""
    W, H, D, n = 200, 40, 48, 3
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=4)
    with DispEst(l8, r8, D) as one, DispEst(l8, r8, D, devices=[0] * n) as de:
        c = {}
        for name, ctx in (("one", one), ("multi", de)):
            c[name] = []
            for stage in (ctx.CostConst_GPU, ctx.CostFilter_GPU, ctx.DispSelect_GPU):
                k = ctx.launch_count(); stage(); c[name].append(ctx.launch_count() - k)
        # ingest + CVC and the filter on every shard; selection: a scatter and a reduce per view and shard
        assert c["multi"] == [n * c["one"][0], n * c["one"][1], n * 4], c
        same_maps((de.lDisMap, de.rDisMap), (one.lDisMap, one.rDisMap), "maps")


# ---- 6. the C++ facade ------------------------------------------------------------------------------------------------
def test_cpp_demo_with_device_list(tmp_path):
    exe = os.path.join(ROOT, "primestereomatch_b200", "host", "dispest_demo")
    if not os.path.exists(exe):
        pytest.skip("dispest_demo not built")
    W, H, D = 300, 48, 64
    l, r, _ = synth.stereo_pair_f32(W, H, D, seed=8)
    l.tofile(tmp_path / "l.f32"); r.tofile(tmp_path / "r.f32")
    maps = {}
    devs = "0,1" if ngpu() >= 2 else "0,0,0"
    for pre in ([], ["--devices", devs], ["--devices", devs, "--block-slices", "10"]):
        out = subprocess.run([exe, *pre, str(W), str(H), str(D), str(tmp_path / "l.f32"), str(tmp_path / "r.f32"),
                              str(tmp_path / "l.u8"), str(tmp_path / "r.u8")], capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stderr
        maps[" ".join(pre)] = (np.fromfile(tmp_path / "l.u8", np.uint8), np.fromfile(tmp_path / "r.u8", np.uint8))
    for k, m in maps.items():
        same_maps(m, maps[""], f"C++ demo {k!r}")
    assert maps[""][0].any()
