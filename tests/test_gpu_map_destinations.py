"""GPU: the map calls that copy maps out of a context (psm_disp_select*, psm_disp_reduce_keys*, psm_disp_fetch_p2p*,
psm_post_process*) check their destinations before their first launch.  A null left map or a step below a row returns
PSM_EINVAL with nothing enqueued, and the next valid call gives the maps a fresh context gives."""
import ctypes as C

import numpy as np
import pytest
import torch

from primestereomatch_b200 import DispEst, capi, synth

pytestmark = pytest.mark.gpu

W, H, D = 61, 23, 24
SPLIT = 13   # the fused exchange's two ranks own [0, SPLIT) and [SPLIT, D)

# the calls each kind of context takes; "fused" is two ranks of the flag-synchronised fused exchange in one process
CALLS = ("select", "select_async", "reduce_keys", "post_process")
COMBOS = [(kind, call) for kind in ("unblocked", "blocked") for call in CALLS]
COMBOS += [("multi", call) for call in ("select", "select_async", "post_process")]
COMBOS += [("fused", "fetch"), ("fused", "post_process")]


@pytest.fixture(scope="module")
def pair():
    return synth.stereo_pair_f32(W, H, D, seed=11)[:2]


def check(rc, de):
    capi.check(rc, de.handle)


def make(kind, bits, views, pair):
    """-> the context (a list of one, or the fused exchange's two ranks) for a frame of `pair` with `views`"""
    l, r = pair
    kw = dict(map_bits=bits)
    if kind == "fused":
        des = [DispEst(l, r, D, d_begin=0, d_count=SPLIT, **kw), DispEst(l, r, D, d_begin=SPLIT, d_count=D - SPLIT, **kw)]
        L = capi.lib()
        bufs = (C.c_void_p * 2)()
        for k, de in enumerate(des):
            p = C.c_void_p()
            check(L.psm_p2p_create_buffer(de.handle, 2, C.byref(p)), de)
            bufs[k] = p.value
        for k, de in enumerate(des):
            check(L.psm_p2p_set_peers(de.handle, bufs, 2, k), de)
    else:
        kw.update(dict(block_slices=7) if kind == "blocked" else dict(devices=[0, 0]) if kind == "multi" else {})
        des = [DispEst(l, r, D, **kw)]
    for de in des:
        de.setViews(views)
    return des


def prepare(des, kind, call, keys):
    """every stage in front of `call`, on every rank"""
    L = capi.lib()
    for de in des:
        de.CostConst_GPU()
        de.CostFilter_GPU()
    de = des[0]
    if kind == "fused":
        for s in des:
            check(L.psm_disp_select_keys_p2p(s.handle), s)
        for s in des:
            s.sync()   # stands in for the cross-rank barrier
        for s in des:
            check(L.psm_disp_reduce_p2p(s.handle), s)
        for s in des:
            s.sync()
    elif call == "post_process":
        check(L.psm_disp_select_device(de.handle), de)
    elif call == "reduce_keys":
        check(L.psm_disp_select_keys(de.handle, keys[0].data_ptr(), keys[1].data_ptr() if de.rDisMap is not None else None),
              de)
    de.sync()


def call_maps(des, call, bits, keys, left, left_step, right, right_step):
    L, de = capi.lib(), des[0]
    u16 = bits == 16
    if call == "reduce_keys":
        fn = L.psm_disp_reduce_keys_u16 if u16 else L.psm_disp_reduce_keys
        kr = keys[1].data_ptr() if de.rDisMap is not None else None
        return fn(de.handle, keys[0].data_ptr(), kr, 1, left, left_step, right, right_step)
    fn = {"select": L.psm_disp_select_u16 if u16 else L.psm_disp_select,
          "select_async": L.psm_disp_select_u16_async if u16 else L.psm_disp_select_async,
          "fetch": L.psm_disp_fetch_p2p_u16 if u16 else L.psm_disp_fetch_p2p,
          "post_process": L.psm_post_process_u16 if u16 else L.psm_post_process}[call]
    rc = fn(de.handle, left, left_step, right, right_step)
    if call == "select_async" and rc == capi.PSM_OK:
        de.sync()
    return rc


def valid_maps(des, call, bits, keys):
    dt = np.uint16 if bits == 16 else np.uint8
    maps = [np.full((H, W), 7, dt) for _ in range(2)]
    both = des[0].rDisMap is not None
    right = (maps[1].ctypes.data, maps[1].strides[0]) if both else (None, 0)
    check(call_maps(des, call, bits, keys, maps[0].ctypes.data, maps[0].strides[0], *right), des[0])
    return maps if both else maps[:1]


def bad_destinations(call, views, bits, buf):
    """-> {case: destination arguments} over the host buffers `buf`, each large enough for a map of either format"""
    row = W * bits // 8
    left, right = buf[0].ctypes.data, buf[1].ctypes.data
    rargs = (right, row) if views == "both" else (None, 0)
    cases = {"short left step": (left, row - 1, *rargs)}
    if call != "reduce_keys":   # psm_disp_reduce_keys: a null left map means "no host copy"
        cases["null left map"] = (None, row, *rargs)
    if views == "both":
        cases["short right step"] = (left, row, right, row - 1)
    return cases


def close(des):
    for de in des:
        de.close()


@pytest.mark.parametrize("views", ["both", "left"])
@pytest.mark.parametrize("bits", [8, 16])
@pytest.mark.parametrize("kind, call", COMBOS)
def test_bad_destination_enqueues_nothing(kind, call, bits, views, pair):
    keys = [torch.zeros(H * W, dtype=torch.int64, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()
    fresh = make(kind, bits, views, pair)
    try:
        prepare(fresh, kind, call, keys)
        want = valid_maps(fresh, call, bits, keys)
    finally:
        close(fresh)
    des = make(kind, bits, views, pair)
    try:
        buf = [np.zeros((H, W), np.uint16) for _ in range(2)]
        for what, args in bad_destinations(call, views, bits, buf).items():
            prepare(des, kind, call, keys)
            n = des[0].launch_count()
            rc = call_maps(des, call, bits, keys, *args)
            text = capi.lib().psm_last_error(des[0].handle).decode()
            assert rc == capi.PSM_EINVAL, (what, rc, text)
            assert "bad disparity map pointer/step" in text, (what, text)
            assert des[0].launch_count() == n, f"{what}: {des[0].launch_count() - n} launches before PSM_EINVAL"
            got = valid_maps(des, call, bits, keys)
            for v, (g, w) in enumerate(zip(got, want)):
                assert np.array_equal(g, w), f"{what}: view {v} differs from a fresh context's in {np.count_nonzero(g != w)}"
    finally:
        close(des)
