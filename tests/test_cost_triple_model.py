"""CPU-only: the costs beside each winner (PSM_OPT_COSTS).  The decomposed tracking of cost_triple_cases.py (blocked walks,
shard ownership) equals the definition (a gather from the volume at the selection map), as uint32 bit patterns, on volumes
with NaN of both signs and with payloads, +-inf, -0 beside +0, FLT_MAX, denormals and exact ties across every seam.  Then
the declarations and the facades' argument checks, which need no device."""
import os
import re

import numpy as np
import pytest

import cost_triple_cases as CT
import selection_cases as S
from conftest import ROOT
from primestereomatch_b200 import DispEst, capi

DS = (2, 3, 5, 9, 13)


def assert_bits(got, want, what):
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{what}: {len(bad)} entries differ, first {tuple(bad[0])}: " \
                          f"{got[tuple(bad[0])]:#010x} vs {want[tuple(bad[0])]:#010x}"


@pytest.mark.parametrize("D", DS)
def test_volumes_cover_the_edge_cases(D):
    v = CT.volume(D)
    m = CT.winners(S.scan_keys(v))
    assert (m[:, 0] == 0).all() and (m[:, 1] == 1).all()
    assert (m[:, 2] == D - 1).all() and (m[:, 3] == 1).all()
    assert (m > 0).mean() > 0.5
    b = CT.bits(v)
    assert (b == 0x80000000).any() and (b == 0).any() and (b == 0xFFC00000).any() and (b == 0x7F7FFFFF).any()


@pytest.mark.parametrize("D", DS)
def test_gather_is_the_definition(D):
    v = CT.volume(D)
    m = CT.winners(S.scan_keys(v))
    got = CT.gather(v, m)
    b = CT.bits(v)
    H, W = m.shape
    for y in range(H):
        for x in range(W):
            for k in range(3):
                d = m[y, x] + k - 1
                want = b[d, y, x] if 0 <= d < D else 0x7FC00000
                assert got[k, y, x] == want, (y, x, k)
    assert (got[0][m == 0] == 0x7FC00000).all() and (got[1][m == 0] == b[0][m == 0]).all()


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("D", DS)
def test_blocked_walk_equals_the_gather(D, seed):
    v = CT.volume(D, seed=seed)
    keys = S.scan_keys(v)
    want = CT.gather(v, CT.winners(keys))
    for B in range(1, D + 1):
        blocks = S.block_ranges(0, D, B)
        k, planes = CT.track(v, blocks)
        assert (k == keys).all(), f"D={D} B={B}: keys"
        assert_bits(planes[:3], want, f"D={D} B={B}")
        assert_bits(planes[3], CT.bits(v)[blocks[-1][0] + blocks[-1][1] - 1], f"D={D} B={B}: last slice")
        assert_bits(planes[4], CT.bits(v)[0], f"D={D} B={B}: first slice")


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("D", DS)
def test_shards_equal_the_gather(D, seed):
    v = CT.volume(D, seed=seed)
    keys = S.scan_keys(v)
    m_want = CT.winners(keys)
    want = CT.gather(v, m_want)
    seams = 0
    for n in range(1, min(8, D) + 1):
        for B in (None, 1, 2, 3):
            m, got, writers = CT.multi(v, n, B)
            what = f"D={D} {n} shards B={B}"
            assert (m == m_want).all(), f"{what}: map"
            assert (writers == 1).all(), f"{what}: entries without exactly one writer"
            assert_bits(got, want, what)
            if n > 1:
                seams += S.seam_ties(v, keys, S.multi_ranges(D, n, B))
    assert D == 2 or seams > 0, "no winner ties across a shard or block seam"


def test_ties_and_seam_winners_are_exercised():
    """across the volumes, winners sit on the first and the last slice of some block and of some shard"""
    first = last = 0
    for D in DS[2:]:
        m = CT.winners(S.scan_keys(CT.volume(D)))
        for B in (2, 3):
            for b, c in S.block_ranges(0, D, B)[1:]:
                first += (m == b).sum()
                last += (m == b + c - 1).sum()
        for b, c in S.shard_ranges(D, 3)[1:]:
            first += (m == b).sum()
            last += (m == b - 1).sum()
    assert first > 0 and last > 0


# ---- declarations and facades ------------------------------------------------------------------------------------------
def header():
    return open(os.path.join(ROOT, "include", "prime_stereo_b200.h")).read()


def test_declarations():
    text = re.sub(r"/\*.*?\*/", "", header(), flags=re.S)
    consts = {k: int(v) for k, v in re.findall(r"\b(PSM_[A-Z0-9_]+)\s*=\s*(-?\d+)", text)}
    assert consts["PSM_OPT_COSTS"] == capi.PSM_OPT_COSTS == 6
    assert re.search(r"int psm_copy_costs_device\(psm_ctx\* ctx, float\* d_left, float\* d_right, size_t row_step\);", text)
    assert re.search(r"int psm_read_costs\(psm_ctx\* ctx, int view, float\* dst, size_t row_step\);", text)
    for name in ("psm_copy_costs_device", "psm_read_costs"):
        assert name in capi.SYMBOLS
    L = capi.lib()
    assert len(L.psm_copy_costs_device.argtypes) == 4 and len(L.psm_read_costs.argtypes) == 4
    assert "psm_set_option(PSM_OPT_COSTS, 1)" in header()   # listed among the calls that may wait for the device


def test_dispest_argument_checks_without_a_device():
    l = np.zeros((8, 8, 3), np.float32)
    de = DispEst(l, l, 4, ocl=False)
    for bad in (1, 0, "on", None, np.bool_(True)):
        with pytest.raises(TypeError):
            de.setCostOutput(bad)
    for good in (True, False):   # valid values reach the device check
        with pytest.raises(RuntimeError):
            de.setCostOutput(good)
    assert de.cost_output is False and de.lCosts is None and de.rCosts is None


def test_torch_match_checks_costs_first():
    torch = pytest.importorskip("torch")
    from primestereomatch_b200.torch_stereo import TorchStereo
    ts = object.__new__(TorchStereo)   # no context: the check comes before any device work
    t = torch.zeros((8, 8, 3), dtype=torch.uint8)
    for bad in (1, "yes", None):
        with pytest.raises(TypeError):
            ts.match(t, t, costs=bad)
