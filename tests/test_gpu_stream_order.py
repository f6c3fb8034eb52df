"""GPU tests of the ordering between the context's streams: the synchronous and pipelined uploads
(psm_set_images[_u8], psm_set_images[_u8]_async + psm_set_images_commit), psm_disp_select[_u16]_async and the
device-side calls, each issued while the compute stream is held back.

An idle H100 finishes every frame long before the host issues the next call, so a missing event between the copy
stream and the compute stream, or a call that returns before it has read the caller's buffer, gives the right maps
anyway.  Here the stream the context is bound to (psm_set_stream) first runs a bounded spin of about HOLD_MS
(torch.cuda._sleep, calibrated once per module with CUDA events); everything the test issues queues behind it.  Each
test asserts that the spin is still running right after the call that could race has been issued, so a host too slow
to get there in time fails the test instead of passing it vacuously.  Every frame's maps are then compared with the
oracle maps of its own scene: Cones and Teddy at D = 64 (450 x 375), whose maps differ, so a frame computed from the
other frame's pixels is always detected.
"""
import ctypes as C

import numpy as np
import pytest

from primestereomatch_b200 import DispEst, capi
from test_gpu_parity import assert_same

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

D = 64
HOLD_MS = 250.0            # long enough for the host to issue a whole test sequence behind it
CAL_CYCLES = 50_000_000    # about 25 ms of spin for the calibration


@pytest.fixture(scope="module")
def cycles_per_ms():
    """torch.cuda._sleep cycles per millisecond on this device, timed with CUDA events."""
    s = torch.cuda.Stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(s):
        torch.cuda._sleep(1_000_000)   # first launch outside the measurement
        e0.record(s)
        torch.cuda._sleep(CAL_CYCLES)
        e1.record(s)
    e1.synchronize()
    return CAL_CYCLES / e0.elapsed_time(e1)


def hold(stream, cycles_per_ms):
    """Spin `stream` for about HOLD_MS -> an event that completes when the spin ends."""
    done = torch.cuda.Event()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(int(HOLD_MS * cycles_per_ms))
        done.record(stream)
    return done


def still_held(done, what):
    assert not done.query(), f"the hold ended before {what} was issued: the sequence did not race the compute stream"


@pytest.fixture(scope="module")
def want(oracle_scene_results):
    """Oracle maps of both scenes (u8 frames give the same maps as float frames)."""
    for k in ("ld", "rd"):
        assert not np.array_equal(oracle_scene_results["Cones"][k], oracle_scene_results["Teddy"][k])
    return oracle_scene_results


@pytest.fixture
def make_ctx(scenes):
    """make_ctx(map_bits) -> (DispEst at D = 64, the torch stream it is bound to).  Teardown waits for both."""
    made = []

    def make(map_bits=8):
        _, _, l, r = scenes["Cones"]
        de = DispEst(l, r, D, map_bits=map_bits)
        made.append(de)
        stream = torch.cuda.Stream()
        capi.check(capi.lib().psm_set_stream(de.handle, C.c_void_p(stream.cuda_stream)), de.handle)
        return de, stream

    yield make
    try:
        for de in made:
            de.sync()
    finally:
        torch.cuda.synchronize()
        for de in made:
            de.close()


def pinned(scenes, scene, kind):
    """A new pinned copy of a scene's left and right image, float (kind "f32") or 8-bit (kind "u8")."""
    l8, r8, l, r = scenes[scene]
    a, b = (l8, r8) if kind == "u8" else (l, r)
    return torch.from_numpy(a).pin_memory(), torch.from_numpy(b).pin_memory()


def refill(frame, scenes, scene):
    """Overwrite a pinned frame in place with another scene's pixels."""
    l8, r8, l, r = scenes[scene]
    u8 = frame[0].dtype == torch.uint8
    frame[0].copy_(torch.from_numpy(l8 if u8 else l))
    frame[1].copy_(torch.from_numpy(r8 if u8 else r))


def upload(de, frame, how):
    """psm_set_images[_u8] (how "sync") or psm_set_images[_u8]_async (how "async") of a pinned frame."""
    L = capi.lib()
    l, r = frame
    u8 = l.dtype == torch.uint8
    fn = {("sync", False): L.psm_set_images, ("sync", True): L.psm_set_images_u8,
          ("async", False): L.psm_set_images_async, ("async", True): L.psm_set_images_u8_async}[how, u8]
    step = l.shape[1] * 3 * l.element_size()
    capi.check(fn(de.handle, l.data_ptr(), step, r.data_ptr(), step), de.handle)


def commit(de):
    capi.check(capi.lib().psm_set_images_commit(de.handle), de.handle)


def new_maps(de):
    """Two pinned host maps in the context's format, filled with a value no selection writes at this shape."""
    H, W = de.hei, de.wid
    nbytes = 2 if de.map_bits == 16 else 1
    return tuple(torch.full((H, W * nbytes), 255, dtype=torch.uint8).pin_memory() for _ in range(2))


def select_async(de, maps):
    L = capi.lib()
    fn = L.psm_disp_select_u16_async if de.map_bits == 16 else L.psm_disp_select_async
    step = maps[0].shape[1]
    capi.check(fn(de.handle, maps[0].data_ptr(), step, maps[1].data_ptr(), step), de.handle)


def stages(de, maps):
    """Cost volume, guided filter and the selection into pinned host maps, all asynchronous."""
    L = capi.lib()
    capi.check(L.psm_cost_const(de.handle), de.handle)
    capi.check(L.psm_cost_filter(de.handle), de.handle)
    select_async(de, maps)


def check(de, maps, ref, what):
    for m, key, view in ((maps[0], "ld", "lDisMap"), (maps[1], "rd", "rDisMap")):
        got = m.numpy().view(np.uint16) if de.map_bits == 16 else m.numpy()
        assert_same(got, ref[key].astype(got.dtype), f"{what} {view}")


def warm_up(de, frame):
    """One pipelined frame outside the hold: the first asynchronous upload allocates the second staging set and the
    first float frame the guided filter's scratch, and either may synchronise."""
    upload(de, frame, "async")
    commit(de)
    stages(de, new_maps(de))
    de.sync()
    torch.cuda.synchronize()


@pytest.mark.parametrize("kind", ["f32", "u8"])
def test_synchronous_first_frame_then_pipeline(kind, make_ctx, scenes, want, cycles_per_ms):
    """psm_set_images[_u8] for the first frame, then the two-deep pipeline: the third frame's upload goes into the
    staging set the synchronous frame was copied into, and must wait until that frame's ingest has read it."""
    de, stream = make_ctx()
    warm_up(de, pinned(scenes, "Teddy", kind))
    order = ["Cones", "Teddy", "Teddy", "Cones"]   # frame 2 shares its staging set with frame 0: different scenes
    frames = [pinned(scenes, s, kind) for s in order]
    maps = [new_maps(de) for _ in order]
    done = hold(stream, cycles_per_ms)
    upload(de, frames[0], "sync")
    for k in range(len(order)):
        if k + 1 < len(order):
            upload(de, frames[k + 1], "async")
            if k + 1 == 2:
                still_held(done, "the upload into the synchronous frame's staging set")
        stages(de, maps[k])
        if k + 1 < len(order):
            commit(de)
    de.sync()
    for k, s in enumerate(order):
        check(de, maps[k], want[s], f"frame {k} ({s}, {kind})")


@pytest.mark.parametrize("kind", ["f32", "u8"])
def test_async_upload_into_the_set_of_a_synchronous_frame(kind, make_ctx, scenes, want, cycles_per_ms):
    """async -> commit -> psm_set_images[_u8] -> async -> commit -> async: the last upload targets the staging set the
    synchronous frame used while that frame's ingest is still held back."""
    de, stream = make_ctx()
    warm_up(de, pinned(scenes, "Teddy", kind))
    order = ["Cones", "Teddy", "Cones", "Cones"]    # frame 3 shares its staging set with frame 1: different scenes
    frames = [pinned(scenes, s, kind) for s in order]
    maps = [new_maps(de) for _ in order]
    upload(de, frames[0], "async")
    commit(de)
    stages(de, maps[0])
    done = hold(stream, cycles_per_ms)             # frame 0 has been ingested in front of the hold
    upload(de, frames[1], "sync")
    stages(de, maps[1])
    upload(de, frames[2], "async")
    commit(de)
    stages(de, maps[2])
    upload(de, frames[3], "async")
    still_held(done, "the upload into the synchronous frame's staging set")
    commit(de)
    stages(de, maps[3])
    de.sync()
    for k, s in enumerate(order):
        check(de, maps[k], want[s], f"frame {k} ({s}, {kind})")


@pytest.mark.parametrize("kind", ["f32", "u8"])
def test_host_buffers_reusable_after_commit(kind, make_ctx, scenes, want, cycles_per_ms):
    """The caller refills its pinned frame as soon as psm_set_images_commit has returned, while the upload of that frame
    is still waiting for the frame before last to leave its staging set: the committed frame keeps its pixels."""
    de, stream = make_ctx()
    warm_up(de, pinned(scenes, "Teddy", kind))
    order = ["Cones", "Teddy", "Cones"]
    frames = [pinned(scenes, s, kind) for s in order]
    maps = [new_maps(de) for _ in order]
    done = hold(stream, cycles_per_ms)
    for k in range(2):
        upload(de, frames[k], "async")
        commit(de)
        stages(de, maps[k])
    upload(de, frames[2], "async")                 # frame 0's staging set: this copy waits for the held ingest
    still_held(done, "the upload of the frame to be refilled")
    commit(de)
    refill(frames[2], scenes, "Teddy")
    stages(de, maps[2])
    de.sync()
    for k, s in enumerate(order):
        check(de, maps[k], want[s], f"frame {k} ({s}, {kind})")


@pytest.mark.parametrize("kind", ["f32", "u8"])
def test_host_buffers_reusable_after_synchronous_upload(kind, make_ctx, scenes, want, cycles_per_ms):
    """The caller refills its pinned frame as soon as psm_set_images[_u8] has returned, with the compute stream held:
    the frame keeps its pixels."""
    de, stream = make_ctx()
    warm_up(de, pinned(scenes, "Teddy", kind))
    frame = pinned(scenes, "Cones", kind)
    maps = new_maps(de)
    done = hold(stream, cycles_per_ms)
    upload(de, frame, "sync")
    still_held(done, "the refill")
    refill(frame, scenes, "Teddy")
    stages(de, maps)
    de.sync()
    check(de, maps, want["Cones"], f"Cones ({kind})")


@pytest.mark.parametrize("map_bits", [8, 16])
def test_async_selection_into_distinct_buffers(map_bits, make_ctx, scenes, want, cycles_per_ms):
    """Four frames of psm_disp_select[_u16]_async into four pinned map pairs, all issued behind the hold: each pair
    holds its own frame's maps after psm_sync."""
    de, stream = make_ctx(map_bits)
    dev = {s: (torch.from_numpy(scenes[s][2]).cuda(), torch.from_numpy(scenes[s][3]).cuda()) for s in ("Cones", "Teddy")}
    step = de.wid * 3 * 4
    L = capi.lib()

    def set_device(s):
        capi.check(L.psm_set_images_device(de.handle, dev[s][0].data_ptr(), step, dev[s][1].data_ptr(), step), de.handle)

    set_device("Teddy")
    stages(de, new_maps(de))
    de.sync()
    torch.cuda.synchronize()
    order = ["Cones", "Teddy", "Cones", "Teddy"]
    maps = [new_maps(de) for _ in order]
    done = hold(stream, cycles_per_ms)
    for k, s in enumerate(order):
        set_device(s)
        stages(de, maps[k])
    still_held(done, "the last selection")
    de.sync()
    for k, s in enumerate(order):
        check(de, maps[k], want[s], f"frame {k} ({s}, {map_bits}-bit maps)")


class _DeviceMap:
    """A context's device map as a __cuda_array_interface__ object (torch.as_tensor wraps it without a copy)."""

    def __init__(self, de, what):
        p, pitch = C.c_void_p(), C.c_size_t()
        capi.check(capi.lib().psm_device_ptr(de.handle, what, C.byref(p), C.byref(pitch)), de.handle)
        assert p.value and pitch.value == de.wid
        self.__cuda_array_interface__ = {"shape": (de.hei, de.wid), "typestr": "|u1", "data": (p.value, False),
                                         "version": 2, "strides": None}


def test_steady_state_device_frame_does_not_synchronise(make_ctx, scenes, oracle, want, cycles_per_ms):
    """A frame through psm_set_images_device, psm_cost_const, psm_cost_filter in EXACT, MIXED and NAIVE,
    psm_cost_filter_fgf at an unchanged rate, psm_disp_select_device and psm_post_process_device at unchanged settings
    returns with the hold still running: none of these calls waits on the host once its first use is behind it.  Each
    stage's maps (copied on the held stream as they are made) equal the oracle's."""
    de, stream = make_ctx()
    _, _, l, r = scenes["Cones"]
    ref = want["Cones"]
    fl, fr = oracle.cost_filter_fgf(l, r, ref["lraw"], ref["rraw"], s=4)
    fgf = dict(zip(("ld", "rd"), oracle.disp_select(fl, fr)))
    pp = {"ld": oracle.post_process(l, fgf["ld"]), "rd": oracle.post_process(r, fgf["rd"])}
    dl, dr = torch.from_numpy(l).cuda(), torch.from_numpy(r).cuda()
    step = de.wid * 3 * 4
    L = capi.lib()
    modes = [("EXACT", capi.PSM_CVF_EXACT), ("MIXED", capi.PSM_CVF_MIXED), ("NAIVE", capi.PSM_CVF_NAIVE)]

    def frame(copy_maps):
        capi.check(L.psm_set_images_device(de.handle, dl.data_ptr(), step, dr.data_ptr(), step), de.handle)
        for name, mode in modes:
            de.set_option(capi.PSM_OPT_CVF_MODE, mode)
            capi.check(L.psm_cost_const(de.handle), de.handle)
            capi.check(L.psm_cost_filter(de.handle), de.handle)
            capi.check(L.psm_disp_select_device(de.handle), de.handle)
            copy_maps(name, 2)
        de.set_option(capi.PSM_OPT_CVF_MODE, capi.PSM_CVF_EXACT)
        capi.check(L.psm_cost_const(de.handle), de.handle)
        capi.check(L.psm_cost_filter_fgf(de.handle, 4), de.handle)
        capi.check(L.psm_disp_select_device(de.handle), de.handle)
        copy_maps("FGF", 2)
        capi.check(L.psm_post_process_device(de.handle), de.handle)
        copy_maps("post-processed", 4)

    frame(lambda name, first: None)   # first use: scratch, FGF buffers, weight table
    de.sync()
    torch.cuda.synchronize()
    names = [m[0] for m in modes] + ["FGF", "post-processed"]
    out = {n: tuple(torch.full((de.hei, de.wid), 255, dtype=torch.uint8, device="cuda") for _ in range(2)) for n in names}
    src = {first: tuple(torch.as_tensor(_DeviceMap(de, first + v), device="cuda") for v in range(2)) for first in (2, 4)}
    torch.cuda.synchronize()

    def copy_maps(name, first):
        with torch.cuda.stream(stream):
            for v in range(2):
                out[name][v].copy_(src[first][v])

    done = hold(stream, cycles_per_ms)
    frame(copy_maps)
    still_held(done, "the end of the frame")
    de.sync()
    torch.cuda.synchronize()
    for name in names:
        expect = pp if name == "post-processed" else (fgf if name == "FGF" else ref)
        assert_same(out[name][0].cpu().numpy(), expect["ld"], f"{name} lDisMap")
        assert_same(out[name][1].cpu().numpy(), expect["rd"], f"{name} rDisMap")


def test_switching_to_the_own_stream_mid_frame(make_ctx, scenes, want, cycles_per_ms):
    """psm_set_stream(NULL) between the cost volume and the filter of a frame ingested on the held stream, with the
    next frame's upload pending: that frame and the two after it, on the context's own stream, keep their maps."""
    de, stream = make_ctx()
    warm_up(de, pinned(scenes, "Teddy", "f32"))
    order = ["Cones", "Teddy", "Cones"]
    frames = [pinned(scenes, s, "f32") for s in order]
    maps = [new_maps(de) for _ in order]
    L = capi.lib()
    done = hold(stream, cycles_per_ms)
    upload(de, frames[0], "async")
    commit(de)
    capi.check(L.psm_cost_const(de.handle), de.handle)
    upload(de, frames[1], "async")
    still_held(done, "the stream switch")
    capi.check(L.psm_set_stream(de.handle, None), de.handle)
    capi.check(L.psm_cost_filter(de.handle), de.handle)
    select_async(de, maps[0])
    commit(de)
    upload(de, frames[2], "async")                 # frame 0's staging set: its ingest was recorded on the held stream
    stages(de, maps[1])
    commit(de)
    stages(de, maps[2])
    de.sync()
    for k, s in enumerate(order):
        check(de, maps[k], want[s], f"frame {k} ({s})")
