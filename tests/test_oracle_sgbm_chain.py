"""CPU: sgbm_chain.chain, the post-process chain with the uniqueness test and the median, is pp_chain.chain with both
off, and puts the two steps where StereoSGBM runs them: uniqueness before the disparity check, the median between the
check and speckle removal."""
import numpy as np
import pytest

import dcheck_oracle as DC
import median_oracle as MD
import pp_chain as PP
import runner_up_cases as RU
import sgbm_chain as SC
import speckle_oracle as SP
import unique_oracle as UN


@pytest.fixture(scope="module")
def cones(scenes, oracle_scene_results):
    _, _, l, r = scenes["Cones"]
    ref = oracle_scene_results["Cones"]
    vols = (ref["lf"], ref["rf"])
    maps = (ref["ld"], ref["rd"])
    qm = tuple(DC.winner_costs(v, m) for v, m in zip(vols, maps))
    qr = tuple(RU.definition(v, m)[1].view(np.float32) for v, m in zip(vols, maps))
    return l, r, maps, qm, qr


@pytest.mark.parametrize("dcheck,speckle,lr", [((0, 1), (0, 0, 0), 2), ((1, 1), (1, 100, 32), 2), ((2, 0), (0, 0, 0), 0),
                                               ((0, 1), (2, 50, 1), 0), ((1, 1), (0, 0, 0), 1)])
def test_with_both_off_it_is_the_existing_chain(cones, dcheck, speckle, lr):
    l, r, (ld, rd), qm, qr = cones
    got = SC.chain(l, r, ld, rd, dcheck=dcheck, costs=qm, D=64, speckle=speckle, lr=lr)
    want = PP.chain(l, r, ld, rd, dcheck=dcheck, costs=qm, D=64, speckle=speckle, lr=lr)
    for a, b in zip(got[:2], want[:2]):
        assert np.array_equal(a, b)
    assert (got[2] is None) == (want[2] is None)
    if want[2] is not None:
        assert all(np.array_equal(a, b) for a, b in zip(got[2], want[2]))


def test_step_order_and_only_modes(cones):
    l, r, (ld, rd), qm, qr = cones
    u = UN.check(ld, qm[0], qr[0], 10), UN.check(rd, qm[1], qr[1], 10)
    c = DC.check(u[0], qm[0], 64, 1), DC.check(u[1], qm[1], 64, 1, view=1)
    m = MD.median(c[0], 3), MD.median(c[1], 3)
    kw = dict(costs=qm, runner=qr, D=64)
    assert all(np.array_equal(a, b) for a, b in zip(SC.chain(l, r, ld, rd, uniqueness=(2, 10), **kw)[:2], u))
    assert all(np.array_equal(a, b)
               for a, b in zip(SC.chain(l, r, ld, rd, uniqueness=(1, 10), dcheck=(2, 1), **kw)[:2], c))
    assert all(np.array_equal(a, b)
               for a, b in zip(SC.chain(l, r, ld, rd, uniqueness=(1, 10), dcheck=(1, 1), median=(2, 3), **kw)[:2], m))
    full = SC.chain(l, r, ld, rd, uniqueness=(1, 10), dcheck=(1, 1), median=(1, 3), speckle=(2, 100, 32), **kw)
    assert np.array_equal(full[0], SP.filter_speckles(m[0], 100, 32)) and full[2] is None
    # the median alone sits in front of speckle removal and the left-right step
    alone = SC.chain(l, r, ld, rd, median=(1, 5), lr=2, **kw)
    assert all(np.array_equal(a, b) for a, b in zip(alone, PP.chain(l, r, MD.median(ld, 5), MD.median(rd, 5), lr=2)))
    # the left-only form fills from its own map
    left = SC.chain(l, None, ld, None, uniqueness=(1, 10), lr=2, **kw)
    assert left[1] is None and np.array_equal(left[2][0], (u[0] >= 2).astype(np.uint8))
