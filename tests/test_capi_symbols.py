"""CPU-only: the in-tree CUDA library loads and exports every symbol the C-ABI header declares.
No compute call is made (there is no GPU in the build container)."""
import ctypes
import os
import re

import pytest

from conftest import ROOT
from primestereomatch_b200 import capi


def header_symbols():
    text = open(os.path.join(ROOT, "include", "prime_stereo_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(psm_[a-z0-9_]+)\s*\(", text)))


def test_header_and_binding_agree():
    assert header_symbols() == sorted(capi.SYMBOLS)


def test_library_exports_every_declared_symbol():
    assert os.path.exists(capi.LIB_PATH), "build with `make -C primestereomatch_b200/csrc`"
    L = ctypes.CDLL(capi.LIB_PATH)
    for name in header_symbols():
        assert hasattr(L, name), f"{name} missing from libprime_stereo_b200.so"


def test_build_info_and_error_paths_without_gpu():
    L = capi.lib()
    info = L.psm_build_info().decode()
    assert "sm_90a" in info
    n = L.psm_device_count()
    assert n >= 0
    ctx = ctypes.c_void_p()
    # invalid geometry is rejected before any CUDA call
    assert L.psm_create(ctypes.byref(ctx), 0, 10, 64, 0) == capi.PSM_EINVAL
    assert L.psm_create(ctypes.byref(ctx), 64, 64, 300, 0) == capi.PSM_EINVAL
    assert L.psm_create_sharded(ctypes.byref(ctx), 64, 64, 64, 60, 8, 0) == capi.PSM_EINVAL
    assert b"bad" in L.psm_last_error(None)
    if n == 0:
        # no device: creation must fail loudly (no CPU fallback exists)
        assert L.psm_create(ctypes.byref(ctx), 64, 64, 64, 0) == capi.PSM_ECUDA
        assert not ctx


def test_product_never_imports_the_oracle():
    """The oracle is test infrastructure: nothing under primestereomatch_b200/ may reference it."""
    pkg = os.path.join(ROOT, "primestereomatch_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp", "Makefile")):
                text = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "stereo_oracle" not in text and "from oracle" not in text and "import oracle" not in text, f
