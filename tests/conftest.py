import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    # the built artefacts are git-ignored: on a fresh checkout compile them once (nvcc cross-compiles
    # sm_90a without a GPU; the oracle is plain gcc)
    lib = os.path.join(ROOT, "primestereomatch_b200", "libprime_stereo_b200.so")
    orc = os.path.join(ROOT, "oracle", "libstereo_oracle.so")
    if not (os.path.exists(lib) and os.path.exists(orc)):
        import __graft_entry__
        __graft_entry__.build()


def read_png(path, gray=False):
    """PNG reader: cv2 when importable (it is in this image), else PIL."""
    try:
        import cv2
        return cv2.imread(path, cv2.IMREAD_GRAYSCALE if gray else cv2.IMREAD_UNCHANGED)
    except ImportError:  # pragma: no cover
        from PIL import Image
        a = np.array(Image.open(path).convert("L") if gray else Image.open(path))
        return a[:, :, ::-1].copy() if a.ndim == 3 else a


@pytest.fixture(scope="session")
def golden():
    with open(os.path.join(GOLDEN, "golden.json")) as f:
        return json.load(f)


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as O
    O.lib()
    return O


@pytest.fixture(scope="session")
def scenes(oracle):
    """{'Cones': (l_u8, r_u8, l_f32, r_f32), 'Teddy': ...} -- BGR as cv::imread gives."""
    out = {}
    for name in ("Cones", "Teddy"):
        s = name.lower()
        l8 = read_png(os.path.join(GOLDEN, f"{s}_im2.png"))
        r8 = read_png(os.path.join(GOLDEN, f"{s}_im6.png"))
        out[name] = (l8, r8, oracle.u8_to_f32(l8), oracle.u8_to_f32(r8))
    return out


@pytest.fixture(scope="session")
def oracle_scene_results(oracle, scenes):
    """Oracle intermediates for both scenes, D=64 (computed once per session, ~1 s each)."""
    res = {}
    for name, (_, _, l, r) in scenes.items():
        lg, rg, lraw, rraw = oracle.cost_const(l, r, 64)
        lf, rf = oracle.cost_filter(l, r, lraw, rraw)
        ld, rd = oracle.disp_select(lf, rf)
        res[name] = dict(lg=lg, rg=rg, lraw=lraw, rraw=rraw, lf=lf, rf=rf, ld=ld, rd=rd)
    return res
