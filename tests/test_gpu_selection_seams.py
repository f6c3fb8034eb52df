"""GPU: disparity selection of blocked (psm_create_blocked) and multi-device (psm_create_multi) contexts where a block or
shard seam could change the answer.  Every frame runs through an unblocked context, blocked contexts at B = 1, 2, 3, a
ragged B and B = D, and multi-device contexts of 2, 3 and 8 shards co-located on device 0, unblocked and blocked.  Their
maps are compared with the oracle's arg-min (O.wta) of the oracle's filtered volumes, and the packed (cost, d) keys of
the single-device contexts (psm_disp_select_keys) with the key model of selection_cases.py, as uint64, bit for bit.
Blocked shards owning [d_begin, d_begin + d_count) (d_begin not a multiple of their B) are compared with the model on
their own slices.

The frames: the flagged image kinds (costs +-inf, NaN, FLT_MAX) under the exact filter and the FGF, the 16-bit
wide frame at D = 300, whose winners above 255 lie in the third 128-slice block, MIXED, the inexact kinds (against the unblocked
context), frames built so that exact ties straddle the seams (each case asserts that they do), images below 16 pixels,
fewer pixels than shards, D = 2 with one-slice blocks, and a 1920 x 1080 frame at D = 2560 whose winners lie in blocks
2 to 11."""
import os

import numpy as np
import pytest

import image_cases as IC
import mixed_model as MM
import selection_cases as S
from gif_cases import assert_same
from oracle import oracle as O
from primestereomatch_b200 import DispEst, capi, synth

pytestmark = pytest.mark.gpu

U8, U16 = np.uint8, np.uint16


# ---- running a frame --------------------------------------------------------------------------------------------------
def select(l, r, D, dtype, *, keys=True, maps=True, setup=None, fgf=None, **kw):
    """one frame through a context -> (left map, right map, left keys, right keys); keys are None unless asked for"""
    import torch
    H, W = l.shape[:2]
    with DispEst(l, r, D, map_bits=8 * np.dtype(dtype).itemsize, **kw) as de:
        if setup:
            setup(de)
        assert de.CostConst_GPU() == 0
        if fgf:
            de.setSubsampleRate(fgf)
            assert de.CostFilter_FGF_GPU() == 0
        else:
            assert de.CostFilter_GPU() == 0
        lk = rk = None
        if keys:
            kk = torch.empty((2, H * W), dtype=torch.int64, device="cuda:0")
            capi.check(capi.lib().psm_disp_select_keys(de.handle, kk[0].data_ptr(), kk[1].data_ptr()), de.handle)
            de.sync()
            lk, rk = kk.cpu().numpy().view(np.uint64).reshape(2, H, W)
        lm = rm = None
        if maps:
            assert de.DispSelect_GPU() == 0
            lm, rm = de.lDisMap.copy(), de.rDisMap.copy()
    return lm, rm, lk, rk


def contexts(D, blocks=None, shards=(2, 3, 8), shard_block=3):
    """-> [(name, DispEst keywords, the slice ranges whose keys it reduces)]"""
    if blocks is None:
        blocks = (1, 2, 3, max(1, 2 * D // 3), D)
    out = [("unblocked", {}, [(0, D)])]
    for B in sorted(set(b for b in blocks if 1 <= b <= D)):
        out.append((f"B={B}", dict(block_slices=B), S.block_ranges(0, D, B)))
    for n in shards:
        if n <= D:
            out.append((f"{n} shards", dict(devices=[0] * n), S.multi_ranges(D, n)))
            out.append((f"{n} shards B={shard_block}", dict(devices=[0] * n, block_slices=shard_block),
                        S.multi_ranges(D, n, shard_block)))
    return out


def check_frame(l, r, D, dtype, want_maps, want_keys, what, cases=None, vols=None, ties=False, **kw):
    """every context's maps equal want_maps; the single-device contexts' keys equal want_keys; blocked shards' keys equal
    the model on their slices (vols given) or the unblocked shards' keys.  ties: every context with a seam has pixels
    whose winner ties across it."""
    cases = contexts(D) if cases is None else cases
    for name, ctx, ranges in cases:
        multi = "devices" in ctx
        lm, rm, lk, rk = select(l, r, D, dtype, keys=not multi, **ctx, **kw)
        assert_same(lm, want_maps[0], f"{what}, {name}: left map")
        assert_same(rm, want_maps[1], f"{what}, {name}: right map")
        if not multi:
            assert_same(lk, want_keys[0], f"{what}, {name}: left keys")
            assert_same(rk, want_keys[1], f"{what}, {name}: right keys")
        if ties and vols is not None and len(ranges) > 1:
            n = sum(S.seam_ties(v, k, ranges) for v, k in zip(vols, want_keys))
            assert n > 0, f"{what}, {name}: no winner ties across a seam"
    # blocked shards, the middle one starting off its block grid
    n = min(3, D)
    for k in range(n):
        b, c = S.shard_range(D, n, k)
        B = min(2, c)
        _, _, lk, rk = select(l, r, D, dtype, maps=False, d_begin=b, d_count=c, block_slices=B, **kw)
        if vols is not None:
            want = [S.fold(v, S.block_ranges(b, c, B)) for v in vols]
        else:
            want = select(l, r, D, dtype, maps=False, d_begin=b, d_count=c, **kw)[2:]
        assert_same(lk, want[0], f"{what}, shard [{b}, {b + c}) B={B}: left keys")
        assert_same(rk, want[1], f"{what}, shard [{b}, {b + c}) B={B}: right keys")


def oracle_check(l, r, D, dtype, vols, what, **kw):
    """maps against O.wta of the volumes, keys against the model of the volumes"""
    keys = [S.scan_keys(v) for v in vols]
    maps = [O.wta(v, dtype) for v in vols]
    for v in range(2):
        assert_same(S.disparity(keys[v], dtype), maps[v], f"{what}: the model's view {v} vs O.wta")
    check_frame(l, r, D, dtype, maps, keys, what, vols=vols, **kw)
    return maps


def filtered(l, r, D, fgf=None):
    with np.errstate(all="ignore"):
        _, _, lraw, rraw = O.cost_const(l, r, D)
        if fgf:
            return O.cost_filter_fgf(l, r, lraw, rraw, s=fgf)
        return O.cost_filter(l, r, lraw, rraw)


# ---- 1. flagged kinds: costs +-inf, NaN and FLT_MAX cross every seam --------------------------------------------------
@pytest.mark.parametrize("kind", IC.FLAGGED)
def test_flagged_exact(kind):
    W, H, D = IC.MAIN
    l, r = IC.frame(kind, W, H, D)
    oracle_check(l, r, D, U8, filtered(l, r, D), f"{kind} exact")


@pytest.mark.parametrize("s", [2, 4])
@pytest.mark.parametrize("kind", IC.FLAGGED)
def test_flagged_fgf(kind, s):
    W, H, D = IC.MAIN
    l, r = IC.frame(kind, W, H, D)
    oracle_check(l, r, D, U8, filtered(l, r, D, fgf=s), f"{kind} FGF s={s}", fgf=s)


@pytest.mark.parametrize("kind", IC.FLAGGED)
def test_flagged_wide_u16(kind):
    """D = 300: the left winners above 255 lie in the third block at B = 128 and past the 36th at B = 7"""
    l, r = IC.wide_frame(kind)
    W, H, D = IC.WIDE
    cases = contexts(D, blocks=(7, 128, 200, D), shard_block=7)
    maps = oracle_check(l, r, D, U16, filtered(l, r, D), f"{kind} D=300", cases=cases)
    assert int(maps[0].max()) > 255


# ---- 2. MIXED on in-domain frames, against its CPU model --------------------------------------------------------------
def test_mixed():
    W, H, D = 227, 61, 40
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=5)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    _, _, lraw, rraw = O.cost_const(l, r, D)
    vols = (MM.cost_filter_mixed(O, l, lraw), MM.cost_filter_mixed(O, r, rraw))
    oracle_check(l, r, D, U8, vols, "MIXED",
                 setup=lambda de: de.set_option(capi.PSM_OPT_CVF_MODE, capi.PSM_CVF_MIXED))


# ---- 3. inexact kinds: the tuned order differs from OpenCV's within the carried bound: against the unblocked context ---
@pytest.mark.parametrize("kind", IC.INEXACT)
def test_inexact_against_unblocked(kind):
    W, H, D = IC.MAIN
    l, r = IC.frame(kind, W, H, D)
    lm, rm, lk, rk = select(l, r, D, U8)
    assert_same(S.disparity(lk, U8), lm, f"{kind}: unblocked keys vs maps")
    check_frame(l, r, D, U8, (lm, rm), (lk, rk), f"{kind}", cases=contexts(D)[1:])


# ---- 4. exact ties across the seams -----------------------------------------------------------------------------------
def periodic_pair(p, s, W, H, seed=0):
    """u8 views of period p, the right one the left shifted by s: raw slices d and d + p are identical wherever both
    match inside the image, so their filtered costs tie bit for bit"""
    rng = np.random.default_rng([seed, p, s])
    pat = rng.integers(0, 256, (H, p, 3), dtype=U8)
    x = np.arange(W)
    return np.ascontiguousarray(pat[:, x % p]), np.ascontiguousarray(pat[:, (x + s) % p])


def white_vs_noise(W, H, seed=0):
    """D > W: every slice d > x of pixel x is the same border cost, so whole blocks tie"""
    rng = np.random.default_rng([seed, W, H])
    return np.full((H, W, 3), 255, U8), rng.integers(0, 256, (H, W, 3), dtype=U8)


TIES = {
    "periodic5": (lambda: periodic_pair(5, 2, 160, 24), 24, U8),
    "periodic7": (lambda: periodic_pair(7, 3, 160, 24), 24, U8),
    "white50_d120": (lambda: white_vs_noise(50, 24), 120, U8),
    "white300_d600": (lambda: white_vs_noise(300, 16), 600, U16),
    "constant": (lambda: (np.full((20, 64, 3), 128, U8),) * 2, 32, U8),
}


@pytest.mark.parametrize("name", list(TIES))
def test_ties_across_seams(name):
    make, D, dtype = TIES[name]
    l8, r8 = make()
    vols = filtered(O.u8_to_f32(l8), O.u8_to_f32(r8), D)
    maps = oracle_check(l8, r8, D, dtype, vols, name, ties=True)
    if dtype == U16:
        assert int(maps[0].max()) > 255
    assert maps[0].any()


# ---- 5. geometry edges: below 16 pixels (the reference-order pass for every block), fewer pixels than shards, ----------
#         W not a multiple of 4, H not a multiple of kScatterRows, D = 2 with one-slice blocks
GEOMETRIES = [(1, 1, 9), (2, 1, 5), (2, 3, 6), (5, 40, 12), (40, 7, 24), (43, 13, 20), (30, 18, 2)]


@pytest.mark.parametrize("W,H,D", GEOMETRIES)
def test_geometry_edges(W, H, D):
    rng = np.random.default_rng([W, H, D])
    base = rng.integers(0, 256, (H, W + 2, 3), dtype=U8)
    l8, r8 = np.ascontiguousarray(base[:, 2:]), np.ascontiguousarray(base[:, :W])
    vols = filtered(O.u8_to_f32(l8), O.u8_to_f32(r8), D)
    oracle_check(l8, r8, D, U8, vols, f"{W}x{H} D={D}", cases=contexts(D, shard_block=1 if D == 2 else 3))


# ---- 6. shards on distinct devices --------------------------------------------------------------------------------------
def ngpu():
    return capi.lib().psm_device_count()


def distinct(devs):
    if len(set(devs)) > 1 and ngpu() < 2:
        pytest.skip("needs >= 2 GPUs")


@pytest.mark.parametrize("devices", [[0, 1], "all"])
def test_distinct_devices(devices):
    if devices == "all":
        devices = list(range(min(max(ngpu(), 1), 8)))
        if len(devices) < 2:
            pytest.skip("needs >= 2 GPUs")
    distinct(devices)
    for what, (l, r, D, vols) in {
        "periodic5": (*periodic_pair(5, 2, 160, 24), 24, None),
        "nan": (*IC.frame("nan", *IC.MAIN), IC.MAIN[2], None),
    }.items():
        li, ri = (O.u8_to_f32(l), O.u8_to_f32(r)) if l.dtype == U8 else (l, r)
        want = [O.wta(v) for v in filtered(li, ri, D)]
        for block in (None, 2):
            lm, rm, _, _ = select(l, r, D, U8, keys=False, devices=devices, block_slices=block)
            assert_same(lm, want[0], f"{what} on {devices} B={block}: left")
            assert_same(rm, want[1], f"{what} on {devices} B={block}: right")


# ---- 7. full HD at D = 2560: the winners lie in blocks 2 to 11 ---------------------------------------------------------
def test_full_hd_late_blocks():
    import torch
    W, H, D, B, CROP = 1920, 1080, 2560, 128, 32
    free, _ = torch.cuda.mem_get_info()
    if free < 12 * 2 ** 30:
        pytest.skip(f"needs about 10 GiB of device memory, {free / 2**30:.1f} GiB free")
    l8, _, _ = synth.stereo_pair_u8(W, H, 256, seed=D)
    dgt = np.array([300, 700, 1100, 1500])[(np.arange(H) // 40) % 4]
    r8 = np.take_along_axis(l8, ((np.arange(W)[None, :] + dgt[:, None]) % W)[:, :, None].repeat(3, 2), 1)
    l, r = synth.to_f32(l8), synth.to_f32(r8)
    got = select(l, r, D, U16, keys=False, block_slices=B)[:2]
    # two interior bands (disparity 1500 and 700) and the bottom one (1100): 16 rows each with an 8-row margin in
    # their 32-row crops where the crop edge is not the image's (the filter reaches 8 rows up and 7 down)
    for y0 in (7 * 40, 13 * 40, H - 24):
        c0 = y0 - 8
        with np.errstate(all="ignore"):
            _, _, lraw, rraw = O.cost_const(l[c0:c0 + CROP], r[c0:c0 + CROP], D, threads=os.cpu_count())
            lf, rf = O.cost_filter(l[c0:c0 + CROP], r[c0:c0 + CROP], lraw, rraw, threads=os.cpu_count())
        del lraw, rraw
        rows = slice(y0 - c0, CROP if c0 + CROP == H else 24)
        want = O.wta(lf, U16)[rows], O.wta(rf, U16)[rows]
        del lf, rf
        ys = slice(y0, y0 + want[0].shape[0])
        assert_same(got[0][ys], want[0], f"rows {ys} left"); assert_same(got[1][ys], want[1], f"rows {ys} right")
        d = int(dgt[y0])
        assert (want[0][:, d:] > 255).mean() > 0.5 and (want[1][:, :W - d] > 255).mean() > 0.5, d
    multi = select(l, r, D, U16, keys=False, devices=[0, 0], block_slices=B)[:2]
    assert_same(multi[0], got[0], "[0, 0] blocked left"); assert_same(multi[1], got[1], "[0, 0] blocked right")
