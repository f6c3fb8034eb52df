"""Checks shared by the GPU tests of the selection's per-pixel outputs (PSM_OPT_COSTS, PSM_OPT_RUNNER_UP): bit-pattern
comparison of float planes, error codes and messages of the C-ABI, and the launch counts of one frame."""
import ctypes as C

import numpy as np

from primestereomatch_b200 import capi

U32 = np.uint32


def assert_bits(got, want, what, nan_any=False):
    """equal bit patterns; nan_any: a NaN equals a NaN of any sign and payload (the oracle's volume has the host's NaNs)"""
    got = np.ascontiguousarray(got)
    got = got.view(U32) if got.dtype == np.float32 else got
    want = np.ascontiguousarray(want)
    want = want.view(U32) if want.dtype == np.float32 else want
    diff = got != want
    if nan_any:
        diff &= ~(((got & 0x7FFFFFFF) > 0x7F800000) & ((want & 0x7FFFFFFF) > 0x7F800000))
    bad = np.argwhere(diff)
    assert bad.size == 0, f"{what}: {len(bad)} of {got.size} entries differ, first at {tuple(bad[0])}: " \
                          f"{got[tuple(bad[0])]:#010x} vs {want[tuple(bad[0])]:#010x}"


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def expect(rc, code, de, *words):
    """rc is the error code `code`, and the context's last error names every one of words"""
    text = capi.lib().psm_last_error(de.handle).decode()
    assert rc == code, (rc, code, text)
    for w in words:
        assert w in text, (w, text)


def frame_counts(de):
    """launch counts of CostConst_GPU, the filter and DispSelect_GPU, and the maps"""
    c = []
    for stage in (de.CostConst_GPU, de.CostFilter_GPU, de.DispSelect_GPU):
        n = de.launch_count(); stage(); c.append(de.launch_count() - n)
    return c, de.lDisMap.copy(), None if de.rDisMap is None else de.rDisMap.copy()
