"""CPU: psm_create_multi validates geometry, the device list, block size and map bits before it touches CUDA, so these
calls return PSM_EINVAL on a machine without a device; a device id the machine does not have is PSM_EINVAL too."""
import ctypes as C

import numpy as np
import pytest

from primestereomatch_b200 import DispEst, capi


def create(W, H, D, devices, block, bits, n=None):
    ctx = C.c_void_p()
    arr = None if devices is None else (C.c_int * max(1, len(devices)))(*devices)
    rc = capi.lib().psm_create_multi(C.byref(ctx), W, H, D, arr, len(devices or []) if n is None else n, block, bits)
    return rc, ctx


@pytest.mark.parametrize("args", [
    (0, 8, 64, [0, 0], 0, 8),              # width
    (8, 0, 64, [0, 0], 0, 8),              # height
    (8, 8, 1, [0], 0, 8),                  # max_disp below 2
    (8, 8, 257, [0, 0], 0, 8),             # above 256 with 8-bit maps
    (8, 8, 4097, [0, 0], 0, 16),           # above 4096
    (8, 8, 64, [0, 0], 0, 0),              # map bits
    (8, 8, 64, [0, 0], 0, 12),
    (8, 8, 64, [0, 0], 0, 32),
    (8, 8, 64, [], 0, 8),                  # no device
    (8, 8, 64, [0] * 9, 0, 8),             # more shards than the exchange has ranks
    (8, 8, 3, [0, 0, 0, 0], 0, 8),         # more shards than slices
    (8, 8, 64, [0, 0], -1, 8),             # negative block size
    (8, 8, 64, [0, -1], 0, 8),             # negative device id
    (8, 8, 64, [0, 4096], 0, 8),           # a device id no machine has
])
def test_bad_arguments_are_rejected(args):
    rc, ctx = create(*args)
    assert rc == capi.PSM_EINVAL
    assert not ctx
    assert capi.lib().psm_last_error(None)


def test_null_devices_and_out():
    L = capi.lib()
    rc, ctx = create(8, 8, 64, None, 0, 8, n=2)
    assert rc == capi.PSM_EINVAL and not ctx and b"devices" in L.psm_last_error(None)
    devs = (C.c_int * 2)(0, 0)
    assert L.psm_create_multi(None, 8, 8, 64, devs, 2, 0, 8) == capi.PSM_EINVAL


def test_facade_rejects_a_shard_range_with_devices():
    l = np.zeros((8, 8, 3), np.uint8)
    for kw in (dict(d_begin=8), dict(d_count=32)):
        with pytest.raises(ValueError):
            DispEst(l, l, 64, devices=[0, 0], **kw)


def test_symbol_is_listed():
    assert "psm_create_multi" in capi.SYMBOLS
