"""GPU: the all-pairs sweep (tests/config_sweep.py) on live contexts, every output bit for bit against the oracle
composition.

One context per creation group runs its configurations in order, a new seeded frame per step, through the public
setters (DispEst, and the C-ABI for device planes).  Between steps only the settings whose level changes are set, so an
option the next configuration does not use is turned back off, as a caller reconfiguring a context would.  Each step
compares the selection maps (read before PostProcess_GPU overwrites lDisMap), costs, runner-up, post-processed maps,
valid masks and points.  A failing configuration is run again on a fresh context, and the message says which: a
failure only after the previous step is state that step left behind, one on a fresh context is an interaction."""
import ctypes as C

import numpy as np
import pytest

import config_sweep as S
import reproject_oracle as RP
from oracle import oracle as O
from primestereomatch_b200 import DispEst, capi

torch = pytest.importorskip("torch")

from primestereomatch_b200.torch_stereo import frame_layout  # noqa: E402

pytestmark = pytest.mark.gpu

CONFIGS, GROUPS = S.generate()
INDEX = {(c["group"], c["step"]): i for i, c in enumerate(CONFIGS)}
POST_OFF = ((capi.PSM_DCHECK_OFF, 1), (capi.PSM_SPECKLE_OFF, 0, 0), capi.PSM_LR_OFF, S.DEFAULT_WMF)


def post_settings(level):
    return POST_OFF if S.POSTS[level] is None else S.POSTS[level]


def configure(de, prev, c):
    """the setters of every per-frame setting whose level differs from prev's (prev None: a fresh context, at the
    defaults)"""
    prev = prev or S.DEFAULT
    if c["views"] != prev["views"]:
        de.setViews(c["views"])
    if c["cost"] != prev["cost"]:
        de.setMatchingCost(*S.COSTS[c["cost"]])
    mode, window, eps, s = S.FILTERS[c["filter"]]
    pmode, pwindow, peps, _ = S.FILTERS[prev["filter"]]
    if (window, eps) != (pwindow, peps):
        de.setGuidedFilter(window, eps)
    if mode != pmode:
        de.set_option(capi.PSM_OPT_CVF_MODE, capi.PSM_CVF_MIXED if mode == "mixed" else capi.PSM_CVF_EXACT)
    if s is not None:
        de.setSubsampleRate(s)
    costs, runner = S.OUTPUTS[c["outputs"]]
    pcosts, prunner = S.OUTPUTS[prev["outputs"]]
    if costs != pcosts:
        de.setCostOutput(costs)
    if runner != prunner:
        de.setRunnerUpOutput(runner)
    new, old = post_settings(c["post"]), post_settings(prev["post"])
    for setter, a, b in ((de.setDisparityCheck, new[0], old[0]), (de.setSpeckleFilter, new[1], old[1])):
        if a != b:
            setter(*a)
    if new[2] != old[2]:
        de.setLRCheck(new[2])
    if new[3] != old[3]:
        de.setPostFilter(*new[3])
    rectify, was = S.ENTRIES[c["entry"]][0] == "rectify", S.ENTRIES[prev["entry"]][0] == "rectify"
    if was and not rectify:
        de.setRectify(None, None, None)


def set_planes(de, lt, rt, channels, hw):
    pix, lf, row, col, _ = frame_layout(lt, *hw, channels)
    _, rf, row2, col2, _ = frame_layout(rt, *hw, channels)
    assert (row, col) == (row2, col2)
    capi.check(capi.lib().psm_set_images_device_planes(de.handle, pix, (C.c_void_p * 3)(*lf[0]), (C.c_void_p * 3)(*rf[0]),
                                                       row, col), de.handle)


def feed(de, c, fr):
    """the step's frames into de through the configuration's entry, then the cost stage"""
    path, pix = S.ENTRIES[c["entry"]]
    l8, r8 = fr["src"]
    if path == "rectify":
        de.setRectify(fr["maps"][0], fr["maps"][1], fr["src_size"])
    if path in ("host", "rectify"):
        de.setInputImages(*((l8, r8) if pix == "u8" else (O.u8_to_f32(l8), O.u8_to_f32(r8))))
        de.CostConst_GPU()
        return
    if pix == "u8":   # interleaved BGR bytes
        lt, rt, ch = torch.from_numpy(l8).cuda(), torch.from_numpy(r8).cuda(), "bgr"
    else:             # planar RGB floats
        lt, rt = (torch.from_numpy(O.u8_to_f32(x)).cuda().flip(2).permute(2, 0, 1).contiguous() for x in (l8, r8))
        ch = "rgb"
    torch.cuda.synchronize()
    set_planes(de, lt, rt, ch, l8.shape[:2])
    capi.check(capi.lib().psm_cost_const(de.handle), de.handle)
    de.sync()


def run_step(de, prev, c, fr):
    """one frame of configuration c on de (whose last frame ran prev) -> the outputs c enables, keyed as expect's"""
    configure(de, prev, c)
    feed(de, c, fr)
    s = S.FILTERS[c["filter"]][3]
    assert (de.CostFilter_FGF_GPU() if s is not None else de.CostFilter_GPU()) == 0
    assert de.DispSelect_GPU() == 0
    views = (0,) if c["views"] == "left" else (0, 1)
    names = ("left", "right")
    got = {}
    for v in views:
        got["selection", v] = (de.lDisMap, de.rDisMap)[v].copy()
        if de.cost_output:
            got["costs", v] = (de.lCosts, de.rCosts)[v].view(np.uint32).copy()
        if de.runner_up_output:
            got["runner_up", v] = (de.lRunnerUp, de.rRunnerUp)[v].view(np.uint32).copy()
        if c["reproject"] == "selection":
            got["points_selection", v] = de.reproject(S.Q, names[v], "selection")
    if S.POSTS[c["post"]] is not None:
        assert de.PostProcess_GPU() == 0
        dcheck, speckle, lr, _ = S.POSTS[c["post"]]
        masked = lr != 0 and dcheck[0] != capi.PSM_DCHECK_ONLY and speckle[0] != capi.PSM_SPECKLE_ONLY
        for v in views:
            got["post", v] = (de.lDisMap, de.rDisMap)[v].copy()
            if masked:
                got["valid", v] = (de.lValid, de.rValid)[v].copy()
            if c["reproject"] == "post":
                got["points_post", v] = de.reproject(S.Q, names[v], "post", handle_missing=True)
    return got


def mismatches(got, want):
    """-> one line per output that differs"""
    out = []
    if sorted(got) != sorted(want):
        out.append(f"outputs {sorted(got)} vs expected {sorted(want)}")
    for key in sorted(set(got) & set(want)):
        what = f"{key[0]} {('left', 'right')[key[1]]}"
        g, w = got[key], want[key]
        if key[0].startswith("points"):
            try:
                RP.assert_points_equal(g, w, what)
            except AssertionError as e:
                out.append(str(e))
            continue
        if g.shape != w.shape or g.dtype != w.dtype:
            out.append(f"{what}: {g.dtype} {g.shape} vs {w.dtype} {w.shape}")
        elif not np.array_equal(g, w):
            bad = np.argwhere(g != w)
            i = tuple(bad[0])
            out.append(f"{what}: {len(bad)} of {g.size} differ, first at {list(i)}: {g[i]!r} vs {w[i]!r}")
    return out


def run_sequence(seq):
    """seq's configurations in order on one new context -> [(index, config, previous config or None, [lines])] of the
    steps that failed"""
    W, H, D, bits = S.geometry(seq[0])
    blank = np.zeros((H, W, 3), np.uint8)
    failures = []
    with DispEst(blank, blank, D, map_bits=bits, **S.KINDS[seq[0]["kind"]]) as de:
        prev = None
        for c in seq:
            fr = S.frames(c, S.step_seed(c))
            try:
                lines = mismatches(run_step(de, prev, c, fr), S.expect(c, fr))
            except (capi.PsmError, AssertionError) as e:
                lines = [f"raised {type(e).__name__}: {e}"]
            if lines:
                failures.append((INDEX[c["group"], c["step"]], c, prev, lines))
            prev = c
    return failures


def report(failures):
    """the failures of a context's sequence, each with the result of its configuration on a fresh context"""
    text = []
    for idx, c, prev, lines in failures:
        fresh = run_sequence([c]) if prev is not None else []
        verdict = ("first step of the context" if prev is None else
                   "also fails on a fresh context: an interaction of its settings" if fresh else
                   "passes on a fresh context: state left by the previous step")
        text.append(f"configuration {idx} (context {c['group']}, step {c['step']}): {S.describe(c)}\n"
                    f"  previous step on this context: {'none' if prev is None else S.describe(prev)}\n"
                    f"  {verdict}\n" + "\n".join("    " + ln for ln in lines))
    return "\n".join(text)


@pytest.mark.parametrize("gi", range(len(GROUPS)),
                         ids=[f"{gi}-{g['kind']}-{g['format']}-{g['shape']}" for gi, g in enumerate(GROUPS)])
def test_context_sequence(gi):
    failures = run_sequence([c for c in CONFIGS if c["group"] == gi])
    if failures:
        pytest.fail(report(failures), pytrace=False)
