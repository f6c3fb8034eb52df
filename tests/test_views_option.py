"""CPU-only: the left-only option (PSM_OPT_VIEWS).  The Python constants equal the header's, psm_cvf_plan keeps its
two-view answer, and the facade rejects bad values before it needs a device."""
import os
import re

import numpy as np
import pytest

from conftest import ROOT
from primestereomatch_b200 import DispEst, capi


def header_constants():
    text = open(os.path.join(ROOT, "include", "prime_stereo_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return {k: int(v) for k, v in re.findall(r"\b(PSM_[A-Z0-9_]+)\s*=\s*(-?\d+)", text)}


def test_constants_match_the_header():
    h = header_constants()
    for name in ("PSM_OPT_VIEWS", "PSM_VIEWS_LEFT", "PSM_VIEWS_BOTH", "PSM_OPT_CVF_MODE", "PSM_OPT_P2P_SYNC",
                 "PSM_LEFT", "PSM_RIGHT", "PSM_LR_OFF", "PSM_LR_FILL_WMF", "PSM_LR_FILL"):
        assert getattr(capi, name) == h[name], name
    assert (capi.PSM_OPT_VIEWS, capi.PSM_VIEWS_LEFT, capi.PSM_VIEWS_BOTH) == (5, 1, 2)


def test_public_plan_keeps_its_two_view_grid():
    q = capi.cvf_plan(1920, 1080, 128)
    per_view = q["nseg"] * (q["nstrips"] * q["ndgroups"] + q["pack_ndg"])
    assert q["grid"] == 2 * per_view and q["pack_first"] == 2 * q["nseg"] * q["nstrips"] * q["ndgroups"]


def test_facade_argument_checks_without_a_device():
    l = np.zeros((8, 8, 3), np.float32)
    de = DispEst(l, l, 4, ocl=False)
    for bad in ("right", "Left", "", 1, 2, None, b"left"):
        with pytest.raises(ValueError):
            de.setViews(bad)
    for good in ("left", "both"):   # valid values reach the device check
        with pytest.raises(RuntimeError):
            de.setViews(good)
    assert de.rDisMap is not None
