"""CPU: the device-frame calls (psm_set_images_device_planes, psm_wait_stream, psm_signal_stream, psm_copy_maps_device)
are declared and bound, their constants equal the header's, a null context is PSM_EINVAL before any CUDA call, and
TorchStereo's frame checks (frame_layout) reject CPU tensors, wrong dtypes, shapes and strides without a device.  The same
calls' argument checks on a live context are in tests/test_gpu_device_frames.py."""
import ctypes as C
import os
import re

import pytest

from conftest import ROOT
from primestereomatch_b200 import capi

torch = pytest.importorskip("torch")

from primestereomatch_b200.torch_stereo import frame_layout  # noqa: E402

NEW = ["psm_set_images_device_planes", "psm_wait_stream", "psm_signal_stream", "psm_copy_maps_device"]


def test_symbols_are_declared_bound_and_exported():
    text = open(os.path.join(ROOT, "include", "prime_stereo_b200.h")).read()
    L = capi.lib()
    for name in NEW:
        assert re.search(rf"\bint {name}\(", text), name
        assert name in capi.SYMBOLS
        assert getattr(L, name).argtypes, name


def test_pixel_types_match_the_header():
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "prime_stereo_b200.h")).read(), flags=re.S)
    h = {k: int(v) for k, v in re.findall(r"\b(PSM_PIX_[A-Z0-9_]+)\s*=\s*(\d+)", text)}
    assert h == {"PSM_PIX_U8": capi.PSM_PIX_U8, "PSM_PIX_F32": capi.PSM_PIX_F32} == {"PSM_PIX_U8": 1, "PSM_PIX_F32": 2}


def test_null_context_is_rejected_first():
    L = capi.lib()
    buf = (C.c_uint8 * 64)()
    p = C.cast(buf, C.c_void_p).value
    planes = (C.c_void_p * 3)(p, p + 1, p + 2)
    assert L.psm_set_images_device_planes(None, capi.PSM_PIX_U8, planes, planes, 64, 3) == capi.PSM_EINVAL
    assert L.psm_set_images_device_planes(None, 7, None, None, 0, 0) == capi.PSM_EINVAL
    assert L.psm_wait_stream(None, None) == capi.PSM_EINVAL
    assert L.psm_signal_stream(None, None) == capi.PSM_EINVAL
    assert L.psm_copy_maps_device(None, 0, p, 64, p, 64) == capi.PSM_EINVAL
    assert L.psm_copy_maps_device(None, 5, None, 0, None, 0) == capi.PSM_EINVAL
    assert b"null context" in L.psm_last_error(None)


H, W = 6, 10


def test_layouts_give_the_table_of_the_header():
    hwc = torch.zeros(H, W, 3, dtype=torch.uint8)
    pix, frames, row, col, batched = frame_layout(hwc, H, W)
    p = hwc.data_ptr()
    assert (pix, frames, row, col, batched) == (capi.PSM_PIX_U8, [(p, p + 1, p + 2)], 3 * W, 3, False)
    assert frame_layout(hwc, H, W, "rgb")[1] == [(p + 2, p + 1, p)]
    chw = torch.zeros(3, H, W)
    q, plane = chw.data_ptr(), H * W * 4
    assert frame_layout(chw, H, W, "rgb")[1:4] == ([(q + 2 * plane, q + plane, q)], 4 * W, 4)
    bgra = torch.zeros(H, W, 4)
    assert frame_layout(bgra, H, W)[2:4] == (16 * W, 16)
    batch = torch.zeros(2, H, W, 3, dtype=torch.uint8)
    pix, frames, _, _, batched = frame_layout(batch, H, W)
    assert batched and frames[1][0] - frames[0][0] == H * W * 3
    padded = torch.zeros(H, W + 5, 3, dtype=torch.uint8)[:, 2:2 + W]   # a padded row step and a column offset
    assert frame_layout(padded, H, W)[1:4] == ([tuple(padded.data_ptr() + k for k in range(3))], 3 * (W + 5), 3)


@pytest.mark.parametrize("bad, err", [
    (lambda: torch.zeros(H, W, 3, dtype=torch.float64), TypeError),
    (lambda: torch.zeros(H, W, 3, dtype=torch.int16), TypeError),
    (lambda: torch.zeros(H, W, 3, dtype=torch.float16), TypeError),
    (lambda: torch.zeros(H, W, 2, dtype=torch.uint8), ValueError),          # channel count
    (lambda: torch.zeros(4, H, W, dtype=torch.uint8), ValueError),          # CHW with 4 planes
    (lambda: torch.zeros(H + 1, W, 3, dtype=torch.uint8), ValueError),      # size
    (lambda: torch.zeros(H, W, dtype=torch.uint8), ValueError),             # gray
    (lambda: torch.zeros(1, 1, H, W, 3, dtype=torch.uint8), ValueError),    # rank
    (lambda: torch.zeros(0, H, W, 3, dtype=torch.uint8), ValueError),       # empty batch
    (lambda: torch.zeros(H, 1, 3, dtype=torch.uint8).expand(H, W, 3), ValueError),              # column stride 0
    (lambda: torch.zeros(W, H, 3, dtype=torch.uint8).transpose(0, 1), ValueError),              # rows overlap
    (lambda: torch.zeros(3, W, H).transpose(1, 2), ValueError),                                  # planar, transposed
    (lambda: torch.zeros(H, W, 3, dtype=torch.uint8).numpy(), TypeError),                       # not a tensor
])
def test_bad_frames_are_rejected(bad, err):
    with pytest.raises(err):
        frame_layout(bad(), H, W)


def test_bad_channel_order_is_rejected():
    for bad in ("BGR", "rgba", "", None):
        with pytest.raises(ValueError):
            frame_layout(torch.zeros(H, W, 3, dtype=torch.uint8), H, W, bad)


def test_cpu_tensors_are_rejected_without_a_device():
    """TorchStereo.match checks both frames in full before any device work; a CPU frame of a valid layout fails on its
    device (the context's device, here a cuda device that need not exist)."""
    from primestereomatch_b200.torch_stereo import TorchStereo
    ts = TorchStereo.__new__(TorchStereo)   # the checks need the geometry and device alone, not a context
    ts.width, ts.height, ts.device = W, H, torch.device("cuda", 0)
    ok = torch.zeros(H, W, 3, dtype=torch.uint8)
    with pytest.raises(ValueError, match="CUDA tensors"):
        ts._layout(ok, ok, "bgr")
    with pytest.raises(ValueError, match="same shape, dtype and strides"):
        ts._layout(ok, torch.zeros(H, W + 2, 3, dtype=torch.uint8)[:, :W], "bgr")
    with pytest.raises(ValueError, match="same shape, dtype and strides"):
        ts._layout(ok, torch.zeros(H, W, 3), "bgr")
    with pytest.raises(TypeError):
        ts._layout(ok, torch.zeros(H, W, 3, dtype=torch.int32), "bgr")
