"""primestereomatch_b200 -- H100-native (sm_90a) STEREO_GIF hot path: CVC -> CVF -> WTA.

The product is the CUDA library `libprime_stereo_b200.so` (sources in csrc/, C-ABI in
include/prime_stereo_b200.h).  `DispEst` mirrors the reference facade over that C-ABI.
"""
from .dispest import DispEst, device_count, MAX_CPU_THREADS, OCV_DE, OCL_DE  # noqa: F401
from . import capi, synth  # noqa: F401

__all__ = ["DispEst", "device_count", "capi", "synth"]


def __getattr__(name):
    # TorchStereo imports torch: only on first use, so the numpy facade never pays for it
    if name == "TorchStereo":
        from .torch_stereo import TorchStereo
        return TorchStereo
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
