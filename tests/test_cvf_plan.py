"""CPU-only: the streaming guided-filter kernel's work decomposition (psm_cvf_plan, pure host logic of
primestereomatch_b200/csrc/psm_capi.cu) restated from the column / row bookkeeping documented at the top of
psm_cvf_stream.cuh: every output column of every slice is stored exactly once, every image row belongs to exactly one
segment, and the packed remainder's lane groups are aligned and end at the image edge."""
import pytest

from primestereomatch_b200 import capi

STRIP = 112


def stored_columns(plan, W):
    """(strip or 'packed', first stored column, one past the last) for every column range the kernel stores"""
    out = []
    for s in range(plan["nstrips"]):
        lo = s * STRIP
        shifted = plan["pack_gl"] == 0 and s == plan["nstrips"] - 1 and s > 0
        x0 = ((W - STRIP + 3) & ~3) if shifted else lo
        cols = [x0 + 4 * lane + j for lane in range(28) for j in range(4)          # lanes 0..27 store 4 columns each
                if lo <= x0 + 4 * lane < W and x0 + 4 * lane + j < W]
        out.append((s, cols))
    if plan["pack_gl"]:
        gl, x0, lo = plan["pack_gl"], plan["pack_x0"], plan["nstrips"] * STRIP
        cols = [x0 + 4 * lane + j for lane in range(gl - 4) for j in range(4)
                if lo <= x0 + 4 * lane < W and x0 + 4 * lane + j < W]
        out.append(("packed", cols))
    return out


@pytest.mark.parametrize("W", [16, 17, 64, 112, 113, 128, 129, 130, 160, 161, 224, 225, 227, 240, 260, 300, 340, 450, 451,
                               1280, 1920, 1921, 2047, 3840])
@pytest.mark.parametrize("no_pack", [False, True])
def test_every_column_is_stored_exactly_once(W, no_pack):
    plan = capi.cvf_plan(W, 375, 64, no_pack=no_pack)
    seen = [0] * W
    for _, cols in stored_columns(plan, W):
        for x in cols:
            seen[x] += 1
    assert seen == [1] * W, (plan, [x for x, n in enumerate(seen) if n != 1][:8])
    if no_pack:
        assert plan["pack_gl"] == 0 and plan["nstrips"] == (W + STRIP - 1) // STRIP


@pytest.mark.parametrize("W", [113, 128, 129, 160, 240, 450, 1280, 1920])
def test_packed_remainder_geometry(W):
    plan = capi.cvf_plan(W, 100, 37)
    gl, x0 = plan["pack_gl"], plan["pack_x0"]
    assert gl in (8, 16) and x0 % 4 == 0
    rem = W - plan["nstrips"] * STRIP
    assert 0 < rem <= 4 * (gl - 4)                               # the remainder fits the group's output lanes
    assert x0 <= plan["nstrips"] * STRIP and x0 + 4 * (gl - 4) >= W   # ... which start inside the last full strip and reach the edge
    assert x0 + 4 * gl - 9 <= W + 10                             # input columns stay inside the row's mirrored halo
    wpc = plan["threads"] // 32
    assert plan["pack_ndg"] * wpc * (32 // gl) >= 37             # every slice has a lane group
    assert plan["grid"] == plan["pack_first"] + 2 * plan["nseg"] * plan["pack_ndg"]


@pytest.mark.parametrize("H", [16, 23, 64, 300, 375, 720, 1080, 2160])
@pytest.mark.parametrize("d_count", [3, 16, 32, 64, 128, 256])
def test_row_segments_partition_the_image(H, d_count):
    plan = capi.cvf_plan(1920, H, d_count)
    ns, rows = plan["nseg"], plan["seg_rows"]
    assert rows % 8 == 0 and ns >= 1
    assert (ns - 1) * rows < H <= ns * rows                      # segments [k*rows, min(H, (k+1)*rows)) cover the rows once
    if ns > 1:
        assert rows >= 16 and H - (ns - 1) * rows >= 8           # only the first / last segment ever sees a reflected row
    wpc = plan["threads"] // 32
    assert wpc in (3, 4) and plan["ndgroups"] * wpc >= d_count > (plan["ndgroups"] - 1) * wpc
    assert plan["pack_first"] == 2 * ns * plan["nstrips"] * plan["ndgroups"]


def test_measured_plans():
    """The segment counts the planner picks for a 132-SM H100.  A/B of the CVF kernel over forced segment counts on an
    H100 80GB HBM3 (700 W): each pick was the fastest count or within 1.5 % of it."""
    assert capi.cvf_plan(1920, 1080, 128)["nseg"] == 5           # C4
    assert capi.cvf_plan(1280, 720, 64)["nseg"] == 6             # C3
    assert capi.cvf_plan(1920, 1080, 16)["nseg"] == 8            # C4 on 8 GPUs
    assert capi.cvf_plan(1920, 1080, 32)["nseg"] == 10           # C5 on 8 GPUs
    assert capi.cvf_plan(1920, 1080, 16)["threads"] == 128       # 4 x 4 slices, no idle warp slot


def test_bad_arguments():
    with pytest.raises(capi.PsmError):
        capi.cvf_plan(0, 10, 4)
    with pytest.raises(capi.PsmError):
        capi.cvf_plan(10, 10, 0)
