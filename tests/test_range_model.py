"""CPU-only: a range context over [min_disp, max_disp) (psm_create_range).  The decomposed forms of range_cases.py (one
scan, block folds from min_disp at every block size 1..n, 1-8 shards of the range with cost ownership and runner-up slots,
blocked and not) read only the range's slices and equal the definition, a direct scan of the full volume restricted to
the range, as uint32 bit patterns.  min_disp covers 0, 1, 2, 3, D / 2 and D - 1 on volumes with NaN of both signs, +-inf,
-0 beside +0, exact ties across the min_disp seam and every other seam, a full-range winner below min_disp and pixels
whose every cost in the range is NaN.  At min_disp = 0 the definition is the existing selection, cost triple and
runner-up."""
import numpy as np
import pytest

import cost_triple_cases as CT
import range_cases as RC
import runner_up_cases as RU
import selection_cases as S

DS = (2, 3, 4, 5, 9, 13)
CASES = [(D, lo) for D in DS for lo in RC.min_disps(D)]


def assert_bits(got, want, what):
    bad = np.argwhere(got != want)
    assert bad.size == 0, f"{what}: {len(bad)} entries differ, first {tuple(bad[0])}: " \
                          f"{got[tuple(bad[0])]:#010x} vs {want[tuple(bad[0])]:#010x}"


def check(v, lo, n, B, want, what):
    m, costs, runner, writers = RC.context(v, lo, n, B)
    assert np.array_equal(m, want[0]), f"{what}: map"
    assert (writers == 1).all(), f"{what}: cost entries without exactly one writer"
    assert_bits(costs, want[1], f"{what}: costs")
    assert_bits(runner, want[2], f"{what}: runner-up")


@pytest.mark.parametrize("D,lo", CASES)
def test_definition_by_hand(D, lo):
    v = RC.volume(D, lo)
    m, costs, runner = RC.definition(v, lo)
    b = CT.bits(v)
    H, W = m.shape
    for y in range(H):
        for x in range(W):
            cands = [d for d in range(max(1, lo), D) if v[d, y, x] < np.inf]
            cands.sort(key=lambda d: (float(v[d, y, x]), d))   # -0 == +0 as Python floats
            mm = cands[0] if cands else 0
            assert m[y, x] == mm, (y, x)
            for k in range(3):
                d = mm + k - 1
                assert costs[k, y, x] == (b[d, y, x] if lo <= d < D else 0x7FC00000), (y, x, k)
            away = [d for d in cands if abs(d - mm) >= 2]
            r = away[0] if away else 0
            assert runner[0, y, x] == np.float32(r).view(np.uint32) and \
                runner[1, y, x] == (b[r, y, x] if r else 0x7FC00000), (y, x)


@pytest.mark.parametrize("D", DS)
def test_zero_start_is_the_existing_definition(D):
    v = RC.volume(D, 0)
    m, costs, runner = RC.definition(v, 0)
    assert np.array_equal(m, CT.winners(S.scan_keys(v)))
    assert_bits(costs, CT.gather(v, m), "costs")
    assert_bits(runner, RU.definition(v, m), "runner-up")
    for n in range(1, min(8, D) + 1):
        for B in (None, 1, 2, 3):
            got = RC.context(v, 0, n, B)
            m_ct, c_ct, w_ct = CT.multi(v, n, B)
            m_ru, r_ru = RU.multi(v, n, B)
            assert np.array_equal(got[0], m_ct) and np.array_equal(got[0], m_ru)
            assert_bits(got[1], c_ct, f"n={n} B={B}: the existing shard ownership")
            assert np.array_equal(got[3], w_ct)
            assert_bits(got[2], r_ru, f"n={n} B={B}: the existing slots")


@pytest.mark.parametrize("D,lo", CASES)
def test_volumes_cover_the_edge_cases(D, lo):
    v = RC.volume(D, lo)
    m, costs, runner = RC.definition(v, lo)
    full = CT.winners(S.scan_keys(v))
    if lo >= 2:
        assert (full[:, 4] == lo - 1).all(), "a full-range winner below min_disp"
        assert (m[:, 4] != lo - 1).all()
        assert (m[:, 6] == 0).all() and (costs[:, :, 6] == 0x7FC00000).all(), "no winner: every entry NaN"
    if lo >= 1:
        assert (m[:, 5] == lo).all(), "the lowest d of the tie across the seam that lies in the range"
        assert (m[:, 6] == 0).all() and (costs[0][:, 6] == 0x7FC00000).all()
    assert (m[:, 7] == max(lo, 1)).all() or lo == 0
    b = CT.bits(v[lo:])
    for pattern in (0x80000000, 0, 0x7F800000, 0xFFC00000):
        assert (b == pattern).any(), hex(pattern)


@pytest.mark.parametrize("seed", [0, 1])
@pytest.mark.parametrize("D,lo", CASES)
def test_single_scan_and_every_block_size(D, lo, seed):
    v = RC.volume(D, lo, seed)
    want = RC.definition(v, lo)
    check(v, lo, None, None, want, f"D={D} lo={lo} unblocked")
    for B in range(1, D - lo + 1):
        check(v, lo, None, B, want, f"D={D} lo={lo} B={B}")


@pytest.mark.parametrize("blocked", [False, True])
@pytest.mark.parametrize("D,lo", CASES)
def test_shards_of_the_range(D, lo, blocked):
    v = RC.volume(D, lo, seed=3)
    want = RC.definition(v, lo)
    for n in range(1, min(8, D - lo) + 1):
        for B in ((1, 2, 3) if blocked else (None,)):
            check(v, lo, n, B, want, f"D={D} lo={lo} n={n} B={B}")


def test_only_the_range_is_read():
    """changing every slice below min_disp changes nothing the decomposed forms return"""
    D, lo = 13, 6
    v = RC.volume(D, lo)
    w = v.copy()
    w[:lo] = -np.inf
    for n, B in ((None, None), (None, 4), (3, None), (3, 2)):
        a, b = RC.context(v, lo, n, B), RC.context(w, lo, n, B)
        for x, y in zip(a, b):
            assert np.array_equal(x, y)


def test_seam_ties_are_exercised():
    """pixels whose winner ties, bit for bit up to the sign of zero, with a cost across a block or shard seam"""
    D, lo = 13, 3
    v = RC.volume(D, lo)
    m = RC.definition(v, lo)[0]
    keys = S.scan_keys(v[lo:], lo)
    assert np.array_equal(CT.winners(keys), m)
    assert S.seam_ties(v[lo:], keys, S.block_ranges(lo, D - lo, 2), lo) > 10
    assert S.seam_ties(v[lo:], keys, RC.shard_ranges(lo, D, 3), lo) > 10
