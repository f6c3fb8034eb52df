"""GPU: blocked contexts (psm_create_blocked), which hold a few disparity slices at a time and fold each block's
winner-take-all into running keys.  Their maps equal the unblocked context's and the CPU oracle's bit for bit on every
filter path, at ragged block sizes, sharded, after post-processing, and at a depth no card could hold unblocked."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import image_cases as IC
from conftest import ROOT
from oracle import oracle as O
from primestereomatch_b200 import DispEst, capi, synth
from primestereomatch_b200.sharding import shard_range

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


def run(l, r, D, block=None, setup=None, fgf=None, post=False, **kw):
    """one frame through a context -> (left map, right map)"""
    with DispEst(l, r, D, block_slices=block, **kw) as de:
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
        return de.lDisMap.copy(), de.rDisMap.copy()


def oracle_maps(l, r, D):
    _, _, lraw, rraw = O.cost_const(l, r, D)
    lf, rf = O.cost_filter(l, r, lraw, rraw)
    return O.wta(lf, np.uint16), O.wta(rf, np.uint16)


# ---- 1. the scenes: block holding only d = 0, 3- and 4-slice CTA shapes, ragged last blocks, one block ---------------
@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
@pytest.mark.parametrize("u8", [False, True])
def test_scenes_match_oracle_and_unblocked(scene, u8, scenes, oracle_scene_results):
    l8, r8, l, r = scenes[scene]
    li, ri = (l8, r8) if u8 else (l, r)
    ref = oracle_scene_results[scene]
    want = run(li, ri, 64)
    assert_same(want[0], ref["ld"], "unblocked left vs oracle")
    for block in (1, 3, 4, 7, 12, 63, 64):
        got = run(li, ri, 64, block)
        assert_same(got[0], ref["ld"], f"block {block} left vs oracle")
        assert_same(got[1], ref["rd"], f"block {block} right vs oracle")
        assert_same(got[1], want[1], f"block {block} right vs unblocked")


# ---- 2. every filter path on one ragged size --------------------------------------------------------------------------
PW, PH, PD, PB = 227, 61, 40, 7


def _path_frame(path):
    if path in ("negative", "above1"):   # outside the integer domain: the reference-order pass for the flagged view
        return IC.frame(path, PW, PH, PD)
    l, r, _ = synth.stereo_pair_f32(PW, PH, PD, seed=5)
    return l, r


PATHS = {
    "exact": {},
    "mixed": dict(setup=lambda de: de.set_option(capi.PSM_OPT_CVF_MODE, capi.PSM_CVF_MIXED)),
    "naive": dict(setup=lambda de: de.set_option(capi.PSM_OPT_CVF_MODE, capi.PSM_CVF_NAIVE)),
    "window5": dict(setup=lambda de: de.setGuidedFilter(5, 1e-3)),
    "window16": dict(setup=lambda de: de.setGuidedFilter(16, 1e-4)),
    "cost": dict(setup=lambda de: de.setMatchingCost(0.11, 0.21, 0.008)),
    "fgf1": dict(fgf=1), "fgf2": dict(fgf=2), "fgf4": dict(fgf=4), "fgf8": dict(fgf=8),
    "negative": {}, "above1": {},
}


@pytest.mark.parametrize("path", list(PATHS))
def test_every_filter_path(path):
    l, r = _path_frame(path)
    want = run(l, r, PD, **PATHS[path])
    got = run(l, r, PD, PB, **PATHS[path])
    assert_same(got[0], want[0], f"{path} left"); assert_same(got[1], want[1], f"{path} right")
    assert want[0].any()


# ---- 3. 16-bit maps over a wide range ---------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [300, 600])
def test_u16_wide_range_against_oracle(D):
    W = D + 64
    # rows around the first 40-row band of the synthetic pair whose disparity exceeds 255
    k = next(k for k in range(1, 200) if 1 + (k * 17) % (D - 2) > 255)
    l8, r8, _ = synth.stereo_pair_u8(W, 40 * k + 48, D, seed=D)
    l, r = synth.to_f32(l8[40 * k - 8:]), synth.to_f32(r8[40 * k - 8:])
    ld, rd = oracle_maps(l, r, D)
    got = run(l, r, D, 64, map_bits=16)
    assert_same(got[0], ld, f"D={D} left"); assert_same(got[1], rd, f"D={D} right")
    assert int(ld.max()) > 255


# ---- 4. sharded: blocked shards emit the unblocked shards' keys -------------------------------------------------------
def test_sharded_blocked_keys():
    import torch
    W, H, D, G, B = 300, 40, 200, 2, 13
    l, r, _ = synth.stereo_pair_f32(W, H, D, seed=11)
    L = capi.lib()
    want = run(l, r, D)
    keys = {}
    for block in (None, B):
        keys[block] = []
        for k in range(G):
            b, n = shard_range(D, G, k)
            with DispEst(l, r, D, d_begin=b, d_count=n, block_slices=block) as de:
                de.CostConst_GPU(); de.CostFilter_GPU()
                kk = torch.empty((2, W * H), dtype=torch.int64, device="cuda")
                capi.check(L.psm_disp_select_keys(de.handle, kk[0].data_ptr(), kk[1].data_ptr()), de.handle)
                de.sync()
                keys[block].append(kk)
    for k in range(G):
        assert torch.equal(keys[B][k], keys[None][k]), f"shard {k}: blocked keys differ"
    gathered = torch.stack(keys[B], 1).contiguous()
    ld = np.zeros((H, W), np.uint8); rd = np.zeros((H, W), np.uint8)
    with DispEst(l, r, D, d_begin=0, d_count=D // 2, block_slices=B) as de:
        capi.check(L.psm_disp_reduce_keys(de.handle, gathered[0].data_ptr(), gathered[1].data_ptr(), G,
                                          ptr(ld), W, ptr(rd), W), de.handle)
    assert_same(ld, want[0], "reduced left"); assert_same(rd, want[1], "reduced right")


# ---- 5. post-filter and left-right check consume the maps -------------------------------------------------------------
@pytest.mark.parametrize("lr", [capi.PSM_LR_OFF, capi.PSM_LR_FILL_WMF, capi.PSM_LR_FILL])
def test_post_processing(lr, scenes):
    l8, r8, _, _ = scenes["Cones"]
    l, r = np.ascontiguousarray(l8[100:228, 80:336]), np.ascontiguousarray(r8[100:228, 80:336])

    def setup(de):
        de.setLRCheck(lr)

    want = run(l, r, 64, setup=setup, post=True)
    got = run(l, r, 64, 12, setup=setup, post=True)
    assert_same(got[0], want[0], f"lr {lr} left"); assert_same(got[1], want[1], f"lr {lr} right")


# ---- 6. a depth no card can hold unblocked ----------------------------------------------------------------------------
def test_full_hd_at_d2560():
    import torch
    W, H, D, B, BAND, CROP = 1920, 1080, 2560, 128, 16, 32
    Wp = 1984
    free, total = torch.cuda.mem_get_info()
    assert 4 * D * H * Wp * 4 > total, "the unblocked volumes would fit on this card"
    if free < 6 * 2 ** 30:
        pytest.skip(f"needs about 5 GiB of device memory, {free / 2**30:.1f} GiB free")
    l8, r8, _ = synth.stereo_pair_u8(W, H, 256, seed=D)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    with DispEst(l, r, D, map_bits=16, block_slices=B) as de:
        de.CostConst_GPU(); de.CostFilter_GPU(); de.DispSelect_GPU()
        got_l, got_r = de.lDisMap[:BAND].copy(), de.rDisMap[:BAND].copy()
    ld, rd = oracle_maps(np.ascontiguousarray(l[:CROP]), np.ascontiguousarray(r[:CROP]), D)
    assert_same(got_l, ld[:BAND], "D=2560 top band left"); assert_same(got_r, rd[:BAND], "D=2560 top band right")


# ---- 7. errors and state ----------------------------------------------------------------------------------------------
def _check_resident(de, full, lo, hi):
    """de's slice reads accept exactly the slices [lo, hi) and return full's there; every other slice is not resident
    where de owns it and not owned elsewhere"""
    for d in range(de.d_begin - 1, de.d_begin + de.d_count + 1):
        for view in (0, 1):
            if lo <= d < hi:
                assert_same(de.read_cost_slice(view, d), full.read_cost_slice(view, d), f"view {view} slice {d}")
                (a, b), (a0, b0) = de.read_ab_slice(view, d), full.read_ab_slice(view, d)
                assert_same(a, a0, f"a of view {view} slice {d}"); assert_same(b, b0, f"b of view {view} slice {d}")
                continue
            why = "not resident" if de.d_begin <= d < de.d_begin + de.d_count else "not owned"
            for read in (de.read_cost_slice, de.read_ab_slice):
                with pytest.raises(capi.PsmError) as e:
                    read(view, d)
                assert e.value.code == capi.PSM_EINVAL and why in str(e.value), (view, d, str(e.value))


def _walk(de, full, B, fgf):
    """one frame's CVC and filter stage through a blocked context and an unblocked one of the same range: the first block
    is resident after CVC and the last after the filter; stage 4 is not recorded on the blocked context"""
    L, ms = capi.lib(), C.c_float()
    end = de.d_begin + de.d_count
    last = de.d_begin + (de.d_count - 1) // B * B
    full.CostConst_GPU(); de.CostConst_GPU()
    _check_resident(de, full, de.d_begin, min(de.d_begin + B, end))
    assert L.psm_stage_ms(de.handle, 4, C.byref(ms)) == capi.PSM_ESTATE
    for ctx in (full, de):
        (ctx.CostFilter_FGF_GPU if fgf else ctx.CostFilter_GPU)()
    _check_resident(de, full, last, end)
    assert L.psm_stage_ms(de.handle, 4, C.byref(ms)) == capi.PSM_ESTATE


def test_errors_and_state():
    L = capi.lib()
    W, H, D, B = 64, 24, 40, 16
    l, r, _ = synth.stereo_pair_f32(W, H, D, seed=2)
    ctx = C.c_void_p()
    for args in ((W, H, D, 0, D, 0, 8), (W, H, D, 0, D, D + 1, 8), (W, H, D, 0, D, -1, 8), (W, H, D, 0, D, B, 12),
                 (W, H, 300, 0, 300, B, 8), (W, H, 5000, 0, 5000, B, 16), (W, H, D, 30, 20, B, 8)):
        assert L.psm_create_blocked(C.byref(ctx), *args, 0) == capi.PSM_EINVAL, args
        assert not ctx and L.psm_last_error(None)
    with pytest.raises(capi.PsmError):
        DispEst(l, r, D, block_slices=0)
    u8 = np.zeros((H, W), np.uint8)
    sl = np.zeros((H, W), np.float32)
    with DispEst(l, r, D) as full, DispEst(l, r, D, block_slices=B) as de:
        h = de.handle
        # stages out of order
        assert L.psm_cost_filter(h) == capi.PSM_ESTATE and b"psm_cost_filter before" in L.psm_last_error(h)
        assert L.psm_cost_filter_fgf(h, 4) == capi.PSM_ESTATE and b"psm_cost_filter_fgf before" in L.psm_last_error(h)
        assert L.psm_disp_select(h, ptr(u8), W, ptr(u8), W) == capi.PSM_ESTATE
        _check_resident(de, full, 0, 0)   # nothing resident yet
        # the last block (40 = 16 + 16 + 8) holds filtered costs; psm_device_ptr 0 / 1 point at it
        _walk(de, full, B, fgf=False)
        with pytest.raises(capi.PsmError) as e:
            de.write_cost_slice(0, 1, sl)
        assert e.value.code == capi.PSM_EINVAL and "blocked" in str(e.value)
        with pytest.raises(RuntimeError):
            de.read_cost_volume(0)
        p, pitch = C.c_void_p(), C.c_size_t()
        capi.check(L.psm_device_ptr(h, 0, C.byref(p), C.byref(pitch)), h)
        assert p.value and pitch.value >= W
        assert L.psm_disp_select_keys_p2p(h) == capi.PSM_EINVAL and b"blocked" in L.psm_last_error(h)
        # stage 4 is not recorded on a blocked context; stages 1 and 2 are
        assert de.stage_ms(1) > 0 and de.stage_ms(2) > 0 and full.stage_ms(4) > 0
        full.DispSelect_GPU(); de.DispSelect_GPU()
        assert_same(de.lDisMap, full.lDisMap, "left"); assert_same(de.rDisMap, full.rDisMap, "right")
        assert de.stage_ms(3) > 0
        _walk(de, full, B, fgf=True)
        full.DispSelect_GPU(); de.DispSelect_GPU()
        assert_same(de.lDisMap, full.lDisMap, "FGF left"); assert_same(de.rDisMap, full.rDisMap, "FGF right")
    # a shard off its block grid: blocks [7,15) .. [31,39), then [39,40)
    with DispEst(l, r, D, d_begin=7, d_count=33) as full, DispEst(l, r, D, d_begin=7, d_count=33, block_slices=8) as de:
        _check_resident(de, full, 7, 7)
        for fgf in (False, True):
            _walk(de, full, 8, fgf)


# Filter-stage launches (unblocked, at B = 16) on 200 x 40 x 50, whose blocks are 16 + 16 + 16 + 2 slices.  A blocked stage
# launches its guide kernels once, then per block its filter, the block's CVC after the first block and one fold:
# guide + 4 x filter + 3 + 4.
FILTER_LAUNCHES = {
    "exact": (2, 12),      # guide, streaming filter
    "mixed": (2, 12),
    "naive": (2, 12),      # guide, every slice in the reference order
    "window5": (3, 16),    # generic-window guide; generic-window filter, then the reference-order pass
    "window16": (3, 16),
    "cost": (2, 12),
    # per view: low-resolution guide, low-resolution filter, up-sampling; blocked: both guides, then 4 x 2 views x 2
    "fgf1": (6, 25), "fgf2": (6, 25), "fgf4": (6, 25), "fgf8": (6, 25),
    "negative": (4, 17),   # float frames: guide and its reference-order pass; filter and the reference-order pass
    "above1": (4, 17),
    "left": (2, 12),       # left-only: the one-view guide and filter
}


def test_launch_counts():
    """unblocked contexts launch what they did before the blocked path existed; a blocked filter stage launches its guide
    once, then per block its CVC (after the first), its filter and one fold.  Every filter path and a left-only context
    is run; the mismatches of all of them are reported together."""
    W, H, D, B = 200, 40, 50, 16
    u8 = synth.stereo_pair_u8(W, H, D, seed=4)[:2]
    bad = []
    for path, counts in FILTER_LAUNCHES.items():
        l, r = IC.frame(path, W, H, D) if path in ("negative", "above1") else u8
        kw = dict(setup=lambda de: de.setViews("left")) if path == "left" else PATHS[path]
        views = 1 if path == "left" else 2
        for block, cvf in zip((None, B), counts):
            with DispEst(l, r, D, block_slices=block) as de:
                if "setup" in kw:
                    kw["setup"](de)
                if "fgf" in kw:
                    de.setSubsampleRate(kw["fgf"])
                c = []
                for stage in (de.CostConst_GPU, de.CostFilter_FGF_GPU if "fgf" in kw else de.CostFilter_GPU,
                              de.DispSelect_GPU):
                    n = de.launch_count(); stage(); c.append(de.launch_count() - n)
                # CostConst_GPU: ingest (2 views x ingest + halo) and one CVC launch; selection: one kernel per view
                if c != [5, cvf, views]:
                    bad.append((path, block, c, [5, cvf, views]))
    assert not bad, bad


# ---- 8. the C++ facade ------------------------------------------------------------------------------------------------
def test_cpp_demo_blocked(tmp_path):
    exe = os.path.join(ROOT, "primestereomatch_b200", "host", "dispest_demo")
    if not os.path.exists(exe):
        pytest.skip("dispest_demo not built")
    W, H, D = 300, 48, 64
    l, r, _ = synth.stereo_pair_f32(W, H, D, seed=8)
    l.tofile(tmp_path / "l.f32"); r.tofile(tmp_path / "r.f32")
    maps = {}
    for block in (None, 12):
        pre = ["--block-slices", str(block)] if block else []
        out = subprocess.run([exe, *pre, str(W), str(H), str(D), str(tmp_path / "l.f32"), str(tmp_path / "r.f32"),
                              str(tmp_path / "l.u8"), str(tmp_path / "r.u8")], capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stderr
        maps[block] = (np.fromfile(tmp_path / "l.u8", np.uint8), np.fromfile(tmp_path / "r.u8", np.uint8))
    assert_same(maps[12][0], maps[None][0], "C++ blocked left"); assert_same(maps[12][1], maps[None][1], "C++ blocked right")
    assert maps[None][0].any()
