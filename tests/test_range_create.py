"""CPU: psm_create_range validates its arguments before it touches CUDA, so these calls return PSM_EINVAL on a machine
without a device.  Then the declaration, and the Python keyword rules of min_disp, which need no device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT
from primestereomatch_b200 import DispEst, capi
from primestereomatch_b200.dispest import create_context
from primestereomatch_b200.sharding import shard_range


def create(w, h, lo, hi, devices, n, block, bits):
    L = capi.lib()
    ctx = C.c_void_p()
    arr = None if devices is None else (C.c_int * max(1, len(devices)))(*devices)
    rc = L.psm_create_range(C.byref(ctx), w, h, lo, hi, arr, n, block, bits)
    return rc, ctx


@pytest.mark.parametrize("args,words", [
    ((0, 8, 0, 64, [0], 1, 0, 8), b"geometry"),          # width
    ((8, 0, 0, 64, [0], 1, 0, 8), b"geometry"),          # height
    ((8, 8, -1, 64, [0], 1, 0, 8), b"negative"),         # min_disp < 0
    ((8, 8, 0, 1, [0], 1, 0, 8), b"below 2"),            # max_disp < 2
    ((8, 8, -3, 1, [0], 1, 0, 8), b"negative"),
    ((8, 8, 64, 64, [0], 1, 0, 8), b"not below"),        # min_disp >= max_disp
    ((8, 8, 70, 64, [0], 1, 0, 8), b"not below"),
    ((8, 8, 0, 64, [0], 1, 0, 12), b"map_bits"),         # map bits
    ((8, 8, 0, 64, [0], 1, 0, 0), b"map_bits"),
    ((8, 8, 128, 257, [0], 1, 0, 8), b"above 256"),      # max_disp, not n, bounds 8-bit maps
    ((8, 8, 4000, 4097, [0], 1, 0, 16), b"above 4096"),
    ((8, 8, 0, 64, [0], 0, 0, 8), b"n_devices"),         # n_devices outside 1..min(8, n)
    ((8, 8, 0, 64, [0] * 9, 9, 0, 8), b"n_devices"),
    ((8, 8, 60, 64, [0] * 5, 5, 0, 8), b"n_devices"),
    ((8, 8, 63, 64, [0, 0], 2, 0, 8), b"n_devices"),
    ((8, 8, 16, 64, [0], 1, -1, 8), b"negative"),        # block_slices < 0
    ((8, 8, 16, 64, [0, 0], 2, -5, 16), b"negative"),
    ((8, 8, 16, 64, None, 1, 0, 8), b"devices is null"),
    ((8, 8, 16, 64, None, 3, 4, 8), b"devices is null"),
    ((8, 8, 16, 64, [-1], 1, 0, 8), b"negative"),        # a negative device id
    ((8, 8, 16, 64, [0, -2], 2, 0, 8), b"negative"),
])
def test_bad_arguments_are_rejected_before_cuda(args, words):
    rc, ctx = create(*args)
    assert rc == capi.PSM_EINVAL
    assert not ctx
    assert words in capi.lib().psm_last_error(None)


def test_null_out():
    devs = (C.c_int * 1)(0)
    assert capi.lib().psm_create_range(None, 8, 8, 16, 64, devs, 1, 0, 8) == capi.PSM_EINVAL


def test_symbol_is_declared_and_listed():
    with open(os.path.join(ROOT, "include", "prime_stereo_b200.h")) as f:
        header = f.read()
    assert re.search(r"int psm_create_range\(psm_ctx\*\* out, int width, int height, int min_disp, int max_disp,\s*"
                     r"const int\* devices, int n_devices, int block_slices, int map_bits\);", header)
    assert "psm_create_range" in capi.SYMBOLS
    assert hasattr(capi.lib(), "psm_create_range")


@pytest.mark.parametrize("kw", [dict(d_begin=8), dict(d_count=32), dict(d_begin=0, d_count=64)])
def test_min_disp_is_not_a_shard(kw):
    """min_disp > 0 together with d_begin / d_count: ValueError before any context exists"""
    with pytest.raises(ValueError, match="min_disp"):
        create_context(8, 8, 64, 8, min_disp=16, **kw)
    img = np.zeros((8, 8, 3), np.uint8)
    with pytest.raises(ValueError, match="min_disp"):
        DispEst(img, img, 64, min_disp=16, **kw)


def test_shard_range_of_a_range():
    for D in (2, 13, 64, 300):
        for lo in sorted({0, 1, D // 2, D - 1}):
            for world in range(1, min(8, D - lo) + 1):
                parts = [shard_range(D, world, k, min_disp=lo) for k in range(world)]
                assert parts[0][0] == lo and sum(c for _, c in parts) == D - lo
                assert all(b + c == nb for (b, c), (nb, _) in zip(parts, parts[1:]))
                assert all(c == (D - lo) // world for _, c in parts[:-1])
                if lo == 0:
                    assert parts == [shard_range(D, world, k) for k in range(world)]
    for bad in ((64, 1, 0, -1), (64, 1, 0, 64), (64, 5, 0, 60), (64, 2, 2, 0)):
        with pytest.raises(ValueError):
            shard_range(*bad[:3], min_disp=bad[3])
