"""What psm_post_process computes: the post-process stage's steps in their order, each one the CPU restatement the tests
pin to its own reference (dcheck_oracle, speckle_oracle, lr_oracle and the oracle's post-filter).  Test infrastructure.
"""
import numpy as np

import dcheck_oracle as DC
import lr_oracle as LR
import speckle_oracle as SP
from oracle import oracle as O


def chain(l_img, r_img, ld, rd, *, dcheck=(0, 1), costs=(None, None), D=None, speckle=(0, 0, 0), lr=0,
          setting=(9, 25.5, 1, "exp")):
    """psm_post_process with psm_set_disparity_check(dcheck = (mode, max_diff)) over the winners' costs (left, right)
    at max_disp D, psm_set_speckle_filter(speckle = (mode, max_size, max_diff)), psm_set_lr_check(lr) and post-filter
    `setting` -> (left, right, (lValid, rValid) or None); right None when rd is None (a left-only context, which fills
    with valid = v >= 2)."""
    mode, diff = dcheck
    if mode:
        ld = DC.check(ld, costs[0], D, diff)
        rd = None if rd is None else DC.check(rd, costs[1], D, diff, view=1)
        if mode == 2:
            return ld, rd, None
    if speckle[0]:
        ld = SP.filter_speckles(ld, *speckle[1:])
        rd = None if rd is None else SP.filter_speckles(rd, *speckle[1:])
        if speckle[0] == 2:
            return ld, rd, None
    masks = None
    if lr:
        if rd is None:
            lv = (ld >= 2).astype(np.uint8)
            ld, masks = LR.fill(ld, lv), (lv, None)
        else:
            lv, rv, ld, rd = LR.lr_check_fill(ld, rd)
            masks = (lv, rv)
        if lr == 2:
            return ld, rd, masks
    return O.post_process(l_img, ld, *setting), None if rd is None else O.post_process(r_img, rd, *setting), masks
