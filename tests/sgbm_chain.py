"""What psm_post_process computes with the uniqueness test and the median in the chain: StereoSGBM's order,
uniqueness -> disparity check -> median -> speckle removal -> left-right check / fill -> post-filter, each step the CPU
restatement the tests pin to its own reference (unique_oracle, dcheck_oracle, median_oracle, then pp_chain.chain for
the rest).  Test infrastructure.
"""
import dcheck_oracle as DC
import median_oracle as MD
import pp_chain as PP
import unique_oracle as UN


def chain(l_img, r_img, ld, rd, *, uniqueness=(0, 0), runner=(None, None), dcheck=(0, 1), costs=(None, None), D=None,
          median=(0, 0), speckle=(0, 0, 0), lr=0, setting=(9, 25.5, 1, "exp")):
    """psm_post_process with psm_set_uniqueness_check(uniqueness = (mode, ratio)) over the winners' costs (costs = q(m)
    of left, right) and the runner-up's (runner = q(r) of left, right), psm_set_disparity_check(dcheck = (mode,
    max_diff)) at max_disp D, psm_set_median_blur(median = (mode, ksize)), then pp_chain.chain's speckle removal,
    left-right check / fill and post-filter -> (left, right, (lValid, rValid) or None); right None when rd is None (a
    left-only context, which fills with valid = v >= 2).  With uniqueness and median off this is pp_chain.chain."""
    mode, ratio = uniqueness
    if mode:
        ld = UN.check(ld, costs[0], runner[0], ratio)
        rd = None if rd is None else UN.check(rd, costs[1], runner[1], ratio)
        if mode == 2:
            return ld, rd, None
    mode, diff = dcheck
    if mode:
        ld = DC.check(ld, costs[0], D, diff)
        rd = None if rd is None else DC.check(rd, costs[1], D, diff, view=1)
        if mode == 2:
            return ld, rd, None
    mode, ksize = median
    if mode:
        ld = MD.median(ld, ksize)
        rd = None if rd is None else MD.median(rd, ksize)
        if mode == 2:
            return ld, rd, None
    return PP.chain(l_img, r_img, ld, rd, speckle=speckle, lr=lr, setting=setting)
