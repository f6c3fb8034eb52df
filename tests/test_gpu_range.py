"""GPU: range contexts over [min_disp, max_disp) (psm_create_range, DispEst / TorchStereo min_disp).  Every kind of
context (unblocked with 8- and 16-bit maps, blocked at B = 1, a B that does not divide the slice count and a B above it,
multi-device with co-located shards, unblocked and blocked, left-only frames) holds, after psm_cost_const and after each
filter path (exact, MIXED, a non-default window, the Fast Guided Filter at s = 2 and 4), the raw and filtered slices of a
[0, max_disp) context bit for bit, and its maps, cost triples and runner-up equal range_cases.definition applied to that
context's filtered volume: on Cones and Teddy (u8 and float), at min_disp 1, 2, 17, 40 and 63, on volumes written with
psm_write_cost_slice (NaN, +inf, ties at the seam).  Then min_disp = 0 against the existing creation calls, the
left-right check and post-filter on range maps, the debug reads, TorchStereo with a held-back stream, and the
multi-process path: two shards of the range reduced through keys."""
import ctypes as C

import numpy as np
import pytest

import image_cases as IC
import lr_oracle as LR
import pp_chain as PP
import range_cases as RC
import selection_cases as S
from oracle import oracle as O
from primestereomatch_b200 import DispEst, capi, synth

pytestmark = pytest.mark.gpu

U8, U16, U32 = np.uint8, np.uint16, np.uint32
D = 64

KINDS = [("unblocked", {}), ("B=1", dict(block_slices=1)), ("B=7", dict(block_slices=7)), ("B=64", dict(block_slices=64)),
         ("2 shards", dict(devices=[0, 0])), ("3 shards B=5", dict(devices=[0, 0, 0], block_slices=5))]


def window(de):
    de.setGuidedFilter(5, 1e-3)


def mixed(de):
    de.set_option(capi.PSM_OPT_CVF_MODE, capi.PSM_CVF_MIXED)


PATHS = {"exact": (None, None), "mixed": (mixed, None), "window": (window, None), "fgf2": (None, 2), "fgf4": (None, 4)}


def assert_bits(got, want, what):
    got = np.ascontiguousarray(got)
    got = got.view(U32) if got.dtype == np.float32 else got
    want = np.ascontiguousarray(want)
    want = want.view(U32) if want.dtype == np.float32 else want
    assert got.shape == want.shape, f"{what}: shape {got.shape} vs {want.shape}"
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{what}: {len(bad)} of {got.size} entries differ, first at {tuple(bad[0])}: " \
                          f"{got[tuple(bad[0])]:#x} vs {want[tuple(bad[0])]:#x}"


def resident(lo, hi, kw, last):
    """the slices a context of kind kw over [lo, hi) holds: all of them unblocked, else each shard's first block after
    psm_cost_const (last False) or its last block after a filter stage"""
    n = len(kw.get("devices") or [0])
    B = kw.get("block_slices")
    out = []
    for b, c in RC.shard_ranges(lo, hi, n):
        if not B:
            out += range(b, b + c)
        else:
            blocks = S.block_ranges(b, c, min(B, c))
            bb, bc = blocks[-1] if last else blocks[0]
            out += range(bb, bb + bc)
    return out


def run(l, r, hi, lo, dtype=U8, *, setup=None, fgf=None, left_only=False, writes=(), slices=True, **kw):
    """one frame on a context over [lo, hi) with costs and runner-up on -> dict: maps, costs, runner, and with slices the
    raw slices it holds after psm_cost_const and the filtered ones after the filter ({(view, d): slice})"""
    views = (0,) if left_only else (0, 1)
    with DispEst(l, r, hi, map_bits=8 * np.dtype(dtype).itemsize, min_disp=lo, **kw) as de:
        if setup:
            setup(de)
        if left_only:
            de.setViews("left")
        de.setCostOutput(True)
        de.setRunnerUpOutput(True)
        assert de.CostConst_GPU() == 0
        for v, d, src in writes:
            if lo <= d < hi:
                de.write_cost_slice(v, d, src)
        raw = {(v, d): de.read_cost_slice(v, d) for v in views for d in resident(lo, hi, kw, False)} if slices else {}
        if fgf:
            de.setSubsampleRate(fgf)
            assert de.CostFilter_FGF_GPU() == 0
        else:
            assert de.CostFilter_GPU() == 0
        filt = {(v, d): de.read_cost_slice(v, d) for v in views for d in resident(lo, hi, kw, True)} if slices else {}
        assert de.DispSelect_GPU() == 0
        return dict(maps=[de.lDisMap.copy(), None if de.rDisMap is None else de.rDisMap.copy()],
                    costs=[de.lCosts, de.rCosts], runner=[de.lRunnerUp, de.rRunnerUp], raw=raw, filt=filt)


def check(l, r, hi, los, kinds, what, dtype=U8, left_only=False, writes=(), **kw):
    """the full [0, hi) context's volumes, then every (min_disp, kind): the slices it holds equal the full context's, its
    outputs equal range_cases.definition on the full context's filtered volume"""
    full = run(l, r, hi, 0, dtype, writes=writes, **kw)
    views = (0,) if left_only else (0, 1)
    fvol = [np.stack([full["filt"][(v, d)] for d in range(hi)]) for v in views]
    for lo in los:
        want = [RC.definition(fvol[v], lo) for v in views]
        for name, ctx in kinds:
            n = len(ctx.get("devices") or [0])
            if n > hi - lo:
                continue
            tag = f"{what}, [{lo}, {hi}) {name}"
            got = run(l, r, hi, lo, dtype, left_only=left_only, writes=writes, **ctx, **kw)
            for key, s in got["raw"].items():
                assert_bits(s, full["raw"][key], f"{tag}: raw slice {key}")
            for key, s in got["filt"].items():
                assert_bits(s, full["filt"][key], f"{tag}: filtered slice {key}")
            if left_only:
                assert got["maps"][1] is None and got["costs"][1] is None and got["runner"][1] is None
            for v in views:
                assert_bits(got["maps"][v].astype(np.int64), want[v][0], f"{tag}: view {v} map")
                assert_bits(got["costs"][v], want[v][1], f"{tag}: view {v} costs")
                assert_bits(got["runner"][v], want[v][2], f"{tag}: view {v} runner-up")
    return fvol


# ---- the same slices, every filter path; the scenes ------------------------------------------------------------------------
@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("u8", [True, False])
@pytest.mark.parametrize("scene", ["Cones", "Teddy"])
def test_scenes_every_path(scene, u8, path, scenes):
    l8, r8, l, r = scenes[scene]
    setup, fgf = PATHS[path]
    frame = (l8, r8) if u8 else (l, r)
    check(*frame, D, (17,), KINDS, f"{scene} u8={u8} {path}", setup=setup, fgf=fgf)


# ---- selection outputs at every start ------------------------------------------------------------------------------------
def test_selection_every_start():
    l8, r8, _ = synth.stereo_pair_u8(227, 61, D, seed=21)
    fvol = check(l8, r8, D, (1, 2, 17, 40, 63), KINDS, "synthetic")
    assert (fvol[0] > 0).any()


@pytest.mark.parametrize("kind", ["nan", "posinf", "fltmax"])
def test_flagged_frames(kind):
    W, H, DD = IC.MAIN
    l, r = IC.frame(kind, W, H, DD)
    check(l, r, DD, (1, 5), KINDS[:3] + KINDS[4:5], f"{kind}")


def test_written_volumes():
    """raw slices written with psm_write_cost_slice on both contexts (unblocked kinds only): NaN, +inf, and one cost at
    min_disp - 1, min_disp and min_disp + 1 (a tie across the seam that a full-range arg-min gives to min_disp - 1)"""
    W, H = 96, 24
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=4)
    rng = np.random.default_rng(5)
    writes = []
    for lo in (17, 40):
        for v in (0, 1):
            tie = rng.random((H, W)).astype(np.float32) * 0.01   # one slice three times: filtered, it ties exactly
            for d, fill in ((lo - 1, None), (lo, None), (lo + 1, None), (lo + 5, np.nan), (lo + 6, np.inf)):
                s = tie if fill is None else rng.random((H, W)).astype(np.float32) + 1.0
                if fill is not None:
                    s[:, ::3] = fill
                writes.append((v, d, s))
    kinds = [KINDS[0], KINDS[4]]
    fvol = check(l8, r8, D, (17, 40), kinds, "written", writes=writes)
    assert np.array_equal(fvol[0][16], fvol[0][17]) and np.array_equal(fvol[0][17], fvol[0][18])
    assert np.isnan(fvol[0][22]).any() and not np.isfinite(fvol[0][23]).all()


def test_left_only():
    l8, r8, _ = synth.stereo_pair_u8(160, 48, D, seed=8)
    check(l8, r8, D, (17, 40), KINDS, "left-only", left_only=True)


def test_wide_u16():
    l, r = IC.wide_frame("nan")
    W, H, DD = IC.WIDE
    kinds = [KINDS[0], ("B=7", dict(block_slices=7)), ("B=128", dict(block_slices=128)), KINDS[4],
             ("2 shards B=7", dict(devices=[0, 0], block_slices=7))]
    fvol = check(l, r, DD, (129, 280), kinds, "nan D=300", U16)
    assert int(RC.definition(fvol[0], 129)[0].max()) > 255


# ---- min_disp = 0 is the existing context ------------------------------------------------------------------------------------
def frame_counts(de):
    c = []
    for stage in (de.CostConst_GPU, de.CostFilter_GPU, de.DispSelect_GPU):
        n = de.launch_count(); stage(); c.append(de.launch_count() - n)
    return c


@pytest.mark.parametrize("bits,kw", [(8, {}), (16, {}), (8, dict(block_slices=7)), (16, dict(block_slices=64)),
                                     (8, dict(devices=[0, 0])), (8, dict(devices=[0, 0, 0], block_slices=5))])
def test_zero_start_is_the_existing_context(bits, kw):
    """psm_create_range(min_disp = 0) against psm_create_sharded / _u16 / _blocked / _multi: maps, costs, runner-up and
    launch counts, options off and on"""
    l8, r8, _ = synth.stereo_pair_u8(160, 48, D, seed=13)
    L = capi.lib()
    out = []
    for via_range in (False, True):
        with DispEst(l8, r8, D, map_bits=bits, **kw) as de:
            if via_range:
                devs = kw.get("devices") or [0]
                ctx = C.c_void_p()
                capi.check(L.psm_create_range(C.byref(ctx), 160, 48, 0, D, (C.c_int * len(devs))(*devs), len(devs),
                                              kw.get("block_slices", 0), bits))
                L.psm_destroy(de._ctx)
                de._ctx = ctx
            res = [frame_counts(de), de.lDisMap.copy(), de.rDisMap.copy()]
            de.setCostOutput(True)
            de.setRunnerUpOutput(True)
            res += [frame_counts(de), de.lDisMap.copy(), de.lCosts, de.rCosts, de.lRunnerUp, de.rRunnerUp]
            out.append(res)
    for k, (a, b) in enumerate(zip(*out)):
        assert_bits(np.asarray(a), np.asarray(b), f"output {k}")


# ---- left-right check and post-filter on range maps ---------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [{}, dict(devices=[0, 0])])
def test_lr_check_and_post_filter(kw):
    W, H, lo = 128, 40, 17
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=31)
    l, r = O.u8_to_f32(l8), O.u8_to_f32(r8)
    for mode in (0, 1, 2):
        with DispEst(l8, r8, D, min_disp=lo, **kw) as de:
            de.setLRCheck(mode)
            assert de.CostConst_GPU() == 0 and de.CostFilter_GPU() == 0 and de.DispSelect_GPU() == 0
            ld, rd = de.lDisMap.copy(), de.rDisMap.copy()
            assert ((ld == 0) | (ld >= lo)).all() and (ld >= lo).mean() > 0.9
            assert de.PostProcess_GPU() == 0
            want = PP.chain(l, r, ld, rd, lr=mode)
            assert_bits(de.lDisMap, want[0], f"mode {mode} left")
            assert_bits(de.rDisMap, want[1], f"mode {mode} right")
            if mode:
                masks = LR.lr_check(ld, rd)
                assert_bits(de.lValid, masks[0], f"mode {mode} left mask")
                assert_bits(de.rValid, masks[1], f"mode {mode} right mask")


# ---- debug reads and device pointers ----------------------------------------------------------------------------------------
class _Dev:
    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = dict(shape=shape, typestr="<f4", data=(ptr, False), version=2)


def test_debug_reads_and_device_ptr():
    import torch
    W, H, lo = 96, 24, 17
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=2)
    L = capi.lib()
    with DispEst(l8, r8, D, min_disp=lo) as de:
        assert de.CostConst_GPU() == 0 and de.CostFilter_GPU() == 0
        dst = np.empty((H, W), np.float32)
        a3, b = np.empty((3, H, W), np.float32), np.empty((H, W), np.float32)
        for d in (lo - 1, 0, D):
            assert L.psm_read_cost_slice(de.handle, 0, d, dst.ctypes.data, dst.strides[0]) == capi.PSM_EINVAL
            assert L.psm_write_cost_slice(de.handle, 0, d, dst.ctypes.data, dst.strides[0]) == capi.PSM_EINVAL
            assert L.psm_read_ab_slice(de.handle, 0, d, a3.ctypes.data, b.ctypes.data) == capi.PSM_EINVAL
        a, b = de.read_ab_slice(0, lo)
        assert np.isfinite(a).all()
        ptr, pitch = C.c_void_p(), C.c_size_t()
        de.sync()
        for v in (0, 1):
            capi.check(L.psm_device_ptr(de.handle, v, C.byref(ptr), C.byref(pitch)), de.handle)
            vol = torch.as_tensor(_Dev(ptr.value, (D - lo, H, pitch.value)), device="cuda:0")[:, :, :W].cpu().numpy()
            for d in (lo, lo + 1, 40, D - 1):
                assert_bits(vol[d - lo], de.read_cost_slice(v, d), f"view {v} slice {d} at offset {d - lo}")


# ---- TorchStereo ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [{}, dict(block_slices=5), dict(devices=[0, 0])])
def test_torch_held_back_stream(kw):
    import torch
    from primestereomatch_b200.torch_stereo import TorchStereo
    W, H, DD, lo = 160, 48, 24, 9
    frames = [synth.stereo_pair_u8(W, H, DD, seed=s)[:2] for s in (11, 12)]
    want = []
    for l, r in frames:
        o = run(l, r, DD, lo, slices=False, **kw)
        want.append(o["maps"] + o["costs"] + o["runner"])
    lsrc = torch.from_numpy(np.stack([f[0] for f in frames])).to("cuda:0")
    rsrc = torch.from_numpy(np.stack([f[1] for f in frames])).to("cuda:0")
    torch.cuda.synchronize()
    with TorchStereo(W, H, DD, min_disp=lo, **kw) as ts:
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            lt, rt = torch.zeros_like(lsrc), torch.zeros_like(rsrc)
            torch.cuda._sleep(200_000_000)   # the frames are written only after the held-back work, on the same stream
            lt.copy_(lsrc)
            rt.copy_(rsrc)
            out = ts.match(lt, rt, costs=True, runner_up=True)
            plain = ts.match(lt[1], rt[1])
        s.synchronize()
    assert len(out) == 6 and len(plain) == 2
    for b in range(2):
        for k in range(6):
            assert_bits(out[k][b].cpu().numpy(), want[b][k], f"batch frame {b} output {k}")
    assert_bits(plain[0].cpu().numpy(), want[1][0], "costs and runner-up off again: left map")


# ---- the multi-process path on one card: shards of the range through keys ---------------------------------------------------
@pytest.mark.parametrize("lo", [17, 40])
def test_shards_through_keys(lo):
    """two psm_create_u16 shards splitting [lo, D) (sharding.shard_range(..., min_disp=lo)), psm_disp_select_keys on each
    and psm_disp_reduce_keys_u16 over both give the range context's maps"""
    import torch
    from primestereomatch_b200.sharding import shard_range
    W, H = 128, 40
    l8, r8, _ = synth.stereo_pair_u8(W, H, D, seed=17)
    want = run(l8, r8, D, lo, U16, slices=False)["maps"]
    L = capi.lib()
    gathered = torch.empty((2, 2, H * W), dtype=torch.int64, device="cuda:0")
    shards = [DispEst(l8, r8, D, map_bits=16, d_begin=b, d_count=c) for b, c in (shard_range(D, 2, k, lo) for k in range(2))]
    try:
        for k, de in enumerate(shards):
            assert de.CostConst_GPU() == 0 and de.CostFilter_GPU() == 0
            capi.check(L.psm_disp_select_keys(de.handle, gathered[0, k].data_ptr(), gathered[1, k].data_ptr()), de.handle)
            de.sync()
        lm, rm = np.zeros((H, W), U16), np.zeros((H, W), U16)
        de = shards[0]
        capi.check(L.psm_disp_reduce_keys_u16(de.handle, gathered[0].data_ptr(), gathered[1].data_ptr(), 2,
                                              lm.ctypes.data, 2 * W, rm.ctypes.data, 2 * W), de.handle)
    finally:
        for de in shards:
            de.close()
    assert_bits(lm, want[0], "left map")
    assert_bits(rm, want[1], "right map")
