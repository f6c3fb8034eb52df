"""All-pairs sweep of a context's settings (test_config_sweep.py on the CPU, test_gpu_config_sweep.py on the device).

Every feature's own tests hold its setting to the oracle with the other settings mostly at their defaults.  This module
describes the settings as factors with a few levels each, generates a list of configurations in which every allowed pair
of levels of every two factors occurs at least once, and composes the oracle's existing pieces into the outputs each
configuration enables (`expect`).  It adds no numerics of its own.

Factors.  The creation-time ones (`CREATION`: context kind, map format and shape) fix a context; the per-frame ones
(`PER_FRAME`) are the setters a caller may change between frames.  Shapes are stated relative to the format's D so that
they keep their meaning at D = 300:
  - "140x48"  W = D + 92: every disparity-check column range non-empty;
  - "113x37"  W = 112 k + 1 > D: one column past the exact guided filter's 112-column strips;
  - "61x15"   W = D + 13, H = 15 < 16: the default-window filter runs in OpenCV's order (the cvf_ref path), MIXED included;
  - "narrow"  W = D - 8: W <= D, so no column takes part in the disparity check.

Constraints are predicates over partial configurations (`CONSTRAINTS`); each returns True when the factors it judges
are not all assigned yet.  Each judges two factors (dcheck_columns_take_part also reads the format, which the shapes
satisfy by construction), and each factor has a level every constraint allows, so every pair they allow has a valid
completion.

The generator is a deterministic greedy all-pairs construction: it covers the creation pairs with as few creation groups
as it can, then builds per-frame configurations for the groups in rounds (at least three per group, so every context
is reconfigured at least twice), each the best of a few candidates drawn with a constant seed, until no allowed pair is
left uncovered."""
import itertools
import os
import random

import numpy as np

import cost_triple_cases as CT
import mixed_model as MM
import pp_chain as PP
import range_cases as RC
import rectify_oracle as RO
import reproject_oracle as RP
import runner_up_cases as RU
from oracle import oracle as O
from primestereomatch_b200 import synth

SEED = 20261018
MIN_STEPS = 3            # configurations per context at least
CANDIDATES = 12          # candidate configurations drawn per step; the one covering the most uncovered pairs is kept
INF = float("inf")

# ---- factors and levels -------------------------------------------------------------------------------------------------
KINDS = {   # DispEst keyword arguments
    "unblocked": {},
    "blocked7": {"block_slices": 7},                       # ragged last block at D = 48 and D = 300
    "blocked1": {"block_slices": 1},
    "range9": {"min_disp": 9},
    "range9_blocked7": {"min_disp": 9, "block_slices": 7},
    "multi2": {"devices": [0, 0]},
    "multi3_blocked5": {"devices": [0, 0, 0], "block_slices": 5},
}
FORMATS = {"u8": (48, None), "u16_d48": (48, 16), "u16_d300": (300, None)}   # (D, map_bits)
SHAPES = {
    "140x48": lambda D: (D + 92, 48),
    "113x37": lambda D: (112 * (D // 112 + 1) + 1, 37),
    "61x15": lambda D: (D + 13, 15),
    "narrow": lambda D: (D - 8, 20),
}
VIEWS = ("both", "left")
ENTRIES = {   # (path, pixel type): host upload, device planes (one interleaved, one planar layout) or rectification
    "host_f32": ("host", "f32"), "host_u8": ("host", "u8"), "planes_hwc_u8": ("planes", "u8"),
    "planes_chw_f32": ("planes", "f32"), "rectify": ("rectify", "u8"),
}
COSTS = {"default": (0.9, INF, INF), "custom": (0.11, 0.21, 0.008)}   # (alpha, tau_color, tau_grad)
FILTERS = {   # (mode, window, eps, FGF sub-sampling rate or None)
    "exact": ("exact", 8, 1e-4, None),
    "window5": ("exact", 5, 1e-3, None),
    "window16": ("exact", 16, 1e-4, None),
    "mixed": ("mixed", 8, 1e-4, None),
    "fgf2": ("exact", 8, 1e-4, 2),
    "fgf4": ("exact", 8, 1e-4, 4),
}
OUTPUTS = {"none": (False, False), "costs": (True, False), "runner_up": (False, True), "both": (True, True)}
DEFAULT_WMF = (9, 25.5, 1, "exp")
GENERIC_WMF = (3, 25.5, 2, "iv1")
POSTS = {   # (dcheck (mode, max_diff), speckle (mode, max_size, max_diff), lr mode, post-filter setting); None: not run
    "off": None,
    "chain": ((1, 1), (1, 20, 1), 1, DEFAULT_WMF),     # dcheck FIRST + speckle FIRST + LR 1 + the default WMF
    "lr2": ((0, 1), (0, 0, 0), 2, DEFAULT_WMF),
    "speckle_only": ((0, 1), (2, 20, 1), 0, DEFAULT_WMF),
    "dcheck_only": ((2, 0), (0, 0, 0), 0, DEFAULT_WMF),
    "generic_wmf_lr1": ((0, 1), (0, 0, 0), 1, GENERIC_WMF),
}
REPROJECTS = ("none", "selection", "post")

FACTORS = {
    "kind": tuple(KINDS), "format": tuple(FORMATS), "shape": tuple(SHAPES),
    "views": VIEWS, "entry": tuple(ENTRIES), "cost": tuple(COSTS), "filter": tuple(FILTERS), "outputs": tuple(OUTPUTS),
    "post": tuple(POSTS), "reproject": REPROJECTS,
}
NAMES = tuple(FACTORS)
CREATION = ("kind", "format", "shape")
PER_FRAME = tuple(f for f in NAMES if f not in CREATION)
DEFAULT = {"kind": "unblocked", "format": "u8", "shape": "140x48", "views": "both", "entry": "host_f32", "cost": "default",
           "filter": "exact", "outputs": "none", "post": "off", "reproject": "none"}


def geometry(config):
    """-> (W, H, D, map_bits) of a configuration's creation levels"""
    D, bits = FORMATS[config["format"]]
    W, H = SHAPES[config["shape"]](D)
    return W, H, D, (16 if D > 256 else 8) if bits is None else bits


# ---- constraints ----------------------------------------------------------------------------------------------------------
def _has(config, *names):
    return all(n in config for n in names)


def mixed_at_default_window(c):
    """PSM_CVF_MIXED exists for the default guided filter alone"""
    if not _has(c, "filter"):
        return True
    mode, window, eps, _ = FILTERS[c["filter"]]
    return mode != "mixed" or (window, eps) == (8, 1e-4)


def rectify_takes_u8(c):
    """rectification reads u8 camera frames"""
    return not _has(c, "entry") or ENTRIES[c["entry"]] != ("rectify", "f32")


def dcheck_needs_costs(c):
    """the disparity check reads plane 1 of the selection's costs"""
    if not _has(c, "post", "outputs") or POSTS[c["post"]] is None:
        return True
    return POSTS[c["post"]][0][0] == 0 or OUTPUTS[c["outputs"]][0]


def left_only_checks_one_view(c):
    """a left-only context has no right outputs: its left-right check is the disparity check's fill"""
    if not _has(c, "views", "post") or c["views"] != "left" or POSTS[c["post"]] is None:
        return True
    dcheck, _, lr, _ = POSTS[c["post"]]
    return lr == 0 or dcheck[0] == 1


def dcheck_columns_take_part(c):
    """the disparity check has columns x >= D to check, except on the shape made to have none"""
    if not _has(c, "post", "format", "shape") or POSTS[c["post"]] is None or POSTS[c["post"]][0][0] == 0:
        return True
    W, _, D, _ = geometry(c)
    return W > D or c["shape"] == "narrow"


def reproject_post_needs_post(c):
    """the post-processed map exists only after the post-process stage"""
    return not _has(c, "reproject", "post") or c["reproject"] != "post" or POSTS[c["post"]] is not None


CONSTRAINTS = (mixed_at_default_window, rectify_takes_u8, dcheck_needs_costs, left_only_checks_one_view,
               dcheck_columns_take_part, reproject_post_needs_post)


def valid(config):
    return all(p(config) for p in CONSTRAINTS)


# ---- pairs and the generator ----------------------------------------------------------------------------------------------
def pairs_of(config):
    """the level pairs ((f1, a), (f2, b)), f1 before f2 in NAMES, of the factors config assigns"""
    fs = [f for f in NAMES if f in config]
    return {((f1, config[f1]), (f2, config[f2])) for f1, f2 in itertools.combinations(fs, 2)}


def allowed_pairs():
    """every pair of levels of two factors that no constraint rules out"""
    out = set()
    for f1, f2 in itertools.combinations(NAMES, 2):
        for a in FACTORS[f1]:
            for b in FACTORS[f2]:
                if valid({f1: a, f2: b}):
                    out.add(((f1, a), (f2, b)))
    return out


def _creation_groups(uncovered, rng):
    want = {p for p in uncovered if p[0][0] in CREATION and p[1][0] in CREATION}
    cands = [dict(zip(CREATION, t)) for t in itertools.product(*(FACTORS[f] for f in CREATION))]
    rng.shuffle(cands)
    groups = []
    while want:
        best = max(cands, key=lambda g: len(pairs_of(g) & want))
        groups.append(best)
        want -= pairs_of(best)
    return groups


def _candidate(group, uncovered, rng):
    """one per-frame completion of a creation group: factors in a random order, each at the valid level that covers the
    most uncovered pairs with the factors already assigned (ties at random)"""
    c = dict(group)
    order = list(PER_FRAME)
    rng.shuffle(order)
    for f in order:
        options = [lv for lv in FACTORS[f] if valid({**c, f: lv})]
        assert options, (c, f)
        scored = [(len(pairs_of({**c, f: lv}) & uncovered), rng.random(), lv) for lv in options]
        c[f] = max(scored)[2]
    assert valid(c), c
    return {f: c[f] for f in NAMES}


def _best(group, uncovered, rng):
    cands = [_candidate(group, uncovered, rng) for _ in range(CANDIDATES)]
    return max(cands, key=lambda c: len(pairs_of(c) & uncovered))


def generate():
    """-> (configurations, groups): the configurations in running order, each a dict factor -> level with 'group' and
    'step' added (its context and its place in that context's sequence); groups = the creation levels of each context"""
    rng = random.Random(SEED)
    uncovered = allowed_pairs()
    groups = _creation_groups(uncovered, rng)
    steps = [[] for _ in groups]

    def add(gi, c):
        steps[gi].append(c)
        uncovered.difference_update(pairs_of(c))

    for _ in range(MIN_STEPS):
        for gi, g in enumerate(groups):
            add(gi, _best(g, uncovered, rng))
    while uncovered:
        progress = False
        for gi, g in enumerate(groups):
            c = _best(g, uncovered, rng)
            if pairs_of(c) & uncovered:
                add(gi, c)
                progress = True
        assert progress, f"{len(uncovered)} pairs no configuration covers"
    configs = []
    for gi, seq in enumerate(steps):
        for si, c in enumerate(seq):
            configs.append({**c, "group": gi, "step": si})
    return configs, groups


def describe(config):
    return ", ".join(f"{f}={config[f]}" for f in NAMES)


# ---- frames -------------------------------------------------------------------------------------------------------------
RECTIFY_MARGIN = (12, 6)   # source frames this much larger than the output on each side


def _pair(W, H, seed):
    """a synthetic u8 pair with noise on the right view, so the maps hold mismatches for the checks to find"""
    l8, r8, _ = synth.stereo_pair_u8(W, H, 48, seed=seed)
    rng = np.random.default_rng(seed)
    r8 = np.clip(r8.astype(np.int16) + rng.integers(-24, 25, r8.shape), 0, 255).astype(np.uint8)
    return l8, r8


def frames(config, seed):
    """the frame pair of one step: {'src': (left, right) u8 as they enter the context, 'maps': None or each view's
    rectification maps (xy, a), 'src_size': (SW, SH)}"""
    W, H, _, _ = geometry(config)
    if ENTRIES[config["entry"]][0] != "rectify":
        return {"src": _pair(W, H, seed), "maps": None, "src_size": (W, H)}
    SW, SH = W + 2 * RECTIFY_MARGIN[0], H + 2 * RECTIFY_MARGIN[1]
    maps = tuple(synth.rectify_maps(W, H, SW, SH, view=v) for v in range(2))
    return {"src": _pair(SW, SH, seed), "maps": maps, "src_size": (SW, SH)}


def step_seed(config):
    return SEED + 1000 * config["group"] + config["step"]


def ingested(fr):
    """the u8 pair the cost stages see: the frames, or their rectified crops"""
    if fr["maps"] is None:
        return fr["src"]
    return tuple(RO.remap(s, *m) for s, m in zip(fr["src"], fr["maps"]))


Q = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reproject_cases.npz"))["q_rectify_shift"]


# ---- the oracle composition ---------------------------------------------------------------------------------------------
def filtered(config, l, r, lraw, rraw):
    """both views' filtered volumes of the whole range [0, D), as the configuration's filter computes them"""
    mode, window, eps, s = FILTERS[config["filter"]]
    H, W = l.shape[:2]
    if s is not None:
        return O.cost_filter_fgf(l, r, lraw, rraw, s, window=window, eps=eps)
    if mode == "mixed" and W >= 16 and H >= 16:   # below one strip every mode runs in OpenCV's order
        return MM.cost_filter_mixed(O, l, lraw), MM.cost_filter_mixed(O, r, rraw)
    return O.cost_filter(l, r, lraw, rraw, window=window, eps=eps)


def expect(config, fr, D=None):
    """every output the configuration enables, from the oracle's pieces -> dict keyed (output, view), view 0 left / 1
    right: 'selection' (the maps DispSelect_GPU returns), 'costs' and 'runner_up' (uint32 bit patterns), 'post' (the
    maps PostProcess_GPU returns), 'valid' (lValid / rValid where the left-right check ran), 'points_selection' /
    'points_post' (reprojectImageTo3D of those maps, the post ones with handle_missing).  D: the format's unless given."""
    _, _, D0, bits = geometry(config)
    D = D0 if D is None else D
    lo = KINDS[config["kind"]].get("min_disp", 0)
    views = (0,) if config["views"] == "left" else (0, 1)
    l8, r8 = ingested(fr)
    l, r = O.u8_to_f32(l8), O.u8_to_f32(r8)
    alpha, tau_color, tau_grad = COSTS[config["cost"]]
    _, _, lraw, rraw = O.cost_const(l, r, D, alpha=alpha, tau_color=tau_color, tau_grad=tau_grad)
    vols = filtered(config, l, r, lraw, rraw)
    dtype = np.uint16 if bits == 16 else np.uint8
    out = {}
    costs = [None, None]
    for v in views:
        if lo:
            m, c, ru = RC.definition(vols[v], lo)
        else:
            m = O.wta(vols[v], np.uint16).astype(np.int64)
            c, ru = CT.gather(vols[v], m), RU.definition(vols[v], m)
        out["selection", v] = m.astype(dtype)
        costs[v] = c
        with_costs, with_runner = OUTPUTS[config["outputs"]]
        if with_costs:
            out["costs", v] = c
        if with_runner:
            out["runner_up", v] = ru
    post = POSTS[config["post"]]
    if post is not None:
        dcheck, speckle, lr, setting = post
        q = [None if c is None else c[1].view(np.float32) for c in costs]
        ld, rd, masks = PP.chain(l, r, out["selection", 0], out.get(("selection", 1)), dcheck=dcheck, costs=q, D=D,
                                 speckle=speckle, lr=lr, setting=setting)
        for v, m in zip(views, (ld, rd)):
            out["post", v] = m
            if masks is not None:
                out["valid", v] = masks[v]
    if config["reproject"] != "none":
        which = config["reproject"]
        for v in views:
            out["points_" + which, v] = RP.reproject(out[which, v], Q, handle_missing=which == "post")
    return out

