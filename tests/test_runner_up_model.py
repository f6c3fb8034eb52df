"""CPU-only: the runner-up away from the winner (PSM_OPT_RUNNER_UP).  The decomposed forms of runner_up_cases.py (the
single-scan four-lowest list, blocked folds of it at every block size, shard picks reduced through slots for 1-8 shards,
blocked and not) equal the definition (a direct scan given the map), as uint32 bit patterns, on volumes with NaN of both
signs and with payloads, +-inf, -0 beside +0, FLT_MAX, denormals, exact ties across every seam, winners at 1 and D - 1,
pixels whose every cost is NaN, and D = 2 and 3, where no runner-up exists.  Then the declarations."""
import os
import re

import numpy as np
import pytest

import cost_triple_cases as CT
import runner_up_cases as RU
import selection_cases as S
from conftest import ROOT
from primestereomatch_b200 import capi

DS = (2, 3, 4, 5, 9, 13)


def assert_bits(got, want, what):
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{what}: {len(bad)} entries differ, first {tuple(bad[0])}: " \
                          f"{got[tuple(bad[0])]:#010x} vs {want[tuple(bad[0])]:#010x}"


def volume(D, seed=0):
    """CT.volume with more exact ties: half its columns hold only three distinct costs, so ties sit across every seam"""
    v = CT.volume(D, seed=seed)
    rng = np.random.default_rng([seed, D, 7])
    few = np.array([0x3E800000, 0x80000000, 0x00000000], np.uint32).view(np.float32)
    v[:, :, 24:] = few[rng.integers(0, 3, v[:, :, 24:].shape)]
    return v


@pytest.mark.parametrize("D", DS)
def test_definition_by_hand(D):
    v = volume(D)
    m = CT.winners(S.scan_keys(v))
    got = RU.definition(v, m)
    f, b = v, CT.bits(v)
    H, W = m.shape
    for y in range(H):
        for x in range(W):
            cands = [d for d in range(1, D) if f[d, y, x] < np.inf]
            cands.sort(key=lambda d: (float(f[d, y, x]), d))   # -0 == +0 as Python floats
            away = [d for d in cands if abs(d - m[y, x]) >= 2]
            r = away[0] if away else 0
            assert got[0, y, x] == np.float32(r).view(np.uint32), (y, x)
            assert got[1, y, x] == (b[r, y, x] if r else 0x7FC00000), (y, x)
    if D <= 3:
        assert (got[0] == 0).all() and (got[1] == 0x7FC00000).all()
    assert (m[:, 0] == 0).all() and (got[0][:, 0] == 0).all()          # every cost NaN: no runner-up
    assert (m[:, 1] == 1).all() and (m[:, 2] == D - 1).all()         # winners at 1 and at D - 1


@pytest.mark.parametrize("D", DS)
def test_volumes_cover_the_edge_cases(D):
    v = volume(D)
    b = CT.bits(v)
    for pattern in (0x80000000, 0, 0xFFC00000, 0x7FC00123, 0x7F800000, 0xFF800000, 0x7F7FFFFF, 0x00000001):
        assert (b == pattern).any(), hex(pattern)
    if D > 4:
        m = CT.winners(S.scan_keys(v))
        r = RU.definition(v, m)[0].view(np.float32)
        assert (r > 0).mean() > 0.5


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("D", DS)
def test_single_scan_list(D, seed):
    v = volume(D, seed)
    lc, ld = RU.scan_list(v)
    keys = S.scan_keys(v)
    assert np.array_equal(RU.head_key(lc, ld), keys), "the list's head is the arg-min's key"
    m, got = RU.single(v)
    assert np.array_equal(m, CT.winners(keys))
    assert_bits(got, RU.definition(v, m), f"D={D} single scan")


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("D", DS)
def test_blocked_fold_every_block_size(D, seed):
    v = volume(D, seed)
    keys = S.scan_keys(v)
    want = RU.definition(v, CT.winners(keys))
    for B in range(1, D + 1):
        lc, ld = RU.fold(v, S.block_ranges(0, D, B))
        assert np.array_equal(RU.head_key(lc, ld), keys), f"B={B}: head"
        m, got = RU.single(v, B)
        assert_bits(got, want, f"D={D} B={B}")


@pytest.mark.parametrize("blocked", [False, True])
@pytest.mark.parametrize("D", DS)
def test_shards_through_slots(D, blocked):
    v = volume(D, seed=3)
    keys = S.scan_keys(v)
    want = RU.definition(v, CT.winners(keys))
    for n in range(1, min(8, D) + 1):
        for B in ((1, 2, 3) if blocked else (None,)):
            m, got = RU.multi(v, n, B)
            assert np.array_equal(m, CT.winners(keys)), (n, B)
            assert_bits(got, want, f"D={D} n={n} B={B}")


def test_seam_ties_are_exercised():
    """the runner-up decided by the lowest-d rule between entries on opposite sides of a block or shard seam"""
    D = 13
    v = volume(D)
    m = CT.winners(S.scan_keys(v))
    r = RU.definition(v, m)
    rd = r[0].view(np.float32).astype(np.int64)
    f = v
    qr = np.take_along_axis(f, rd[None], 0)[0]
    tie_later = np.zeros(m.shape, bool)
    for d in range(1, D):
        tie_later |= (rd > 0) & (d > rd) & (np.abs(d - m) >= 2) & (f[d] == qr)
    assert tie_later.sum() > 10


def test_uniqueness_equivalence():
    """the caller-side uniqueness test from the planes equals the brute-force one on the volume, at ratios 5, 10, 15"""
    for D in (5, 9, 13):
        for seed in (0, 1):
            v = CT.volume(D, seed=seed)
            v[~np.isfinite(v)] = 1.0   # the test is defined on finite costs
            m = CT.winners(S.scan_keys(v))
            runner = RU.definition(v, m).view(np.float32)
            qm = np.take_along_axis(v, m[None], 0)[0]
            for u in (5, 10, 15):
                assert np.array_equal(RU.uniqueness_from_planes(runner, qm, u), RU.uniqueness_brute(v, m, u)), (D, seed, u)


def test_header_and_capi_constant():
    with open(os.path.join(ROOT, "include", "prime_stereo_b200.h")) as f:
        header = f.read()
    assert int(re.search(r"PSM_OPT_RUNNER_UP\s*=\s*(\d+)", header).group(1)) == capi.PSM_OPT_RUNNER_UP == 7
    for sym in ("psm_copy_runner_up_device", "psm_read_runner_up"):
        assert re.search(rf"int {sym}\(psm_ctx\* ctx", header), sym
        assert sym in capi.SYMBOLS
