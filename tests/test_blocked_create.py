"""CPU: psm_create_blocked validates geometry, block size and map bits before it touches CUDA, so these calls return
PSM_EINVAL on a machine without a device."""
import ctypes as C

import pytest

from primestereomatch_b200 import capi


@pytest.mark.parametrize("args", [
    (0, 8, 64, 0, 64, 8, 8),        # width
    (8, 0, 64, 0, 64, 8, 8),        # height
    (8, 8, 1, 0, 1, 1, 8),          # max_disp below 2
    (8, 8, 257, 0, 257, 8, 8),      # above 256 with 8-bit maps
    (8, 8, 4097, 0, 4097, 8, 16),   # above 4096
    (8, 8, 64, -1, 10, 8, 8),       # shard outside [0, max_disp)
    (8, 8, 64, 60, 10, 8, 8),
    (8, 8, 64, 0, 0, 1, 8),
    (8, 8, 64, 0, 64, 0, 8),        # block_slices outside 1..d_count
    (8, 8, 64, 0, 64, -3, 8),
    (8, 8, 64, 0, 64, 65, 8),
    (8, 8, 64, 16, 16, 17, 16),
    (8, 8, 64, 0, 64, 8, 0),        # map bits
    (8, 8, 64, 0, 64, 8, 12),
    (8, 8, 64, 0, 64, 8, 32),
])
def test_bad_arguments_are_rejected_before_cuda(args):
    L = capi.lib()
    ctx = C.c_void_p()
    assert L.psm_create_blocked(C.byref(ctx), *args, 0) == capi.PSM_EINVAL
    assert not ctx
    assert L.psm_last_error(None)


def test_null_out():
    assert capi.lib().psm_create_blocked(None, 8, 8, 64, 0, 64, 8, 8, 0) == capi.PSM_EINVAL


def test_symbol_is_listed():
    assert "psm_create_blocked" in capi.SYMBOLS
