"""ctypes binding of the C-ABI (include/prime_stereo_b200.h -> libprime_stereo_b200.so).

This is the thinnest possible layer: it loads the in-tree shared library and declares the
argument types of every exported symbol.  There is NO fallback: if the library is missing or
fails to load, importing this module's `lib()` raises -- the product never computes on the CPU.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libprime_stereo_b200.so")

# every symbol include/prime_stereo_b200.h declares (tests assert the .so exports them all)
SYMBOLS = [
    "psm_device_count", "psm_create", "psm_create_sharded", "psm_destroy", "psm_set_option",
    "psm_set_stream", "psm_set_images", "psm_set_images_u8", "psm_set_images_device",
    "psm_set_images_async", "psm_set_images_u8_async", "psm_set_images_commit", "psm_disp_select_async",
    "psm_cost_const", "psm_cost_filter", "psm_disp_select", "psm_disp_select_device",
    "psm_post_process", "psm_post_process_device", "psm_cost_filter_fgf", "psm_disp_select_keys", "psm_disp_reduce_keys", "psm_p2p_create_buffer", "psm_ipc_export", "psm_ipc_import",
    "psm_p2p_set_peers", "psm_disp_select_keys_p2p", "psm_disp_reduce_p2p", "psm_disp_fetch_p2p", "psm_read_cost_slice", "psm_write_cost_slice",
    "psm_read_guide_plane", "psm_read_ab_slice", "psm_device_ptr", "psm_stage_ms",
    "psm_launch_count", "psm_sync", "psm_last_error", "psm_build_info", "psm_cvf_plan", "psm_set_guided_filter",
    "psm_set_matching_cost", "psm_set_post_filter", "psm_create_u16", "psm_disp_select_u16", "psm_disp_select_u16_async",
    "psm_disp_reduce_keys_u16", "psm_disp_fetch_p2p_u16", "psm_post_process_u16", "psm_set_lr_check", "psm_read_valid_mask",
    "psm_create_blocked", "psm_create_multi", "psm_set_images_device_planes", "psm_wait_stream", "psm_signal_stream",
    "psm_copy_maps_device", "psm_copy_costs_device", "psm_read_costs", "psm_copy_runner_up_device", "psm_read_runner_up",
    "psm_create_range", "psm_set_speckle_filter", "psm_set_disparity_check", "psm_reproject_device", "psm_read_points", "psm_set_rectify",
    "psm_set_images_device_yuv", "psm_set_images_yuv", "psm_set_images_yuv_async",
    "psm_set_images_device_bayer", "psm_set_images_bayer", "psm_set_images_bayer_async",
    "psm_set_uniqueness_check", "psm_set_median_blur",
]

PSM_OK, PSM_EINVAL, PSM_ECUDA, PSM_ESTATE, PSM_ENOMEM = 0, 1, 2, 3, 4
PSM_LEFT, PSM_RIGHT = 0, 1
PSM_OPT_CVF_MODE, PSM_OPT_GRAY_MODE, PSM_OPT_TIMING, PSM_OPT_P2P_SYNC, PSM_OPT_VARIANT = 1, 2, 3, 4, 100
PSM_OPT_VIEWS = 5
PSM_OPT_COSTS = 6
PSM_OPT_RUNNER_UP = 7
PSM_VIEWS_LEFT, PSM_VIEWS_BOTH = 1, 2
PSM_CVF_EXACT, PSM_CVF_MIXED, PSM_CVF_NAIVE = 0, 1, 2
PSM_WMF_EXP, PSM_WMF_IV1, PSM_WMF_IV2, PSM_WMF_OFF = 0, 1, 2, 5
PSM_LR_OFF, PSM_LR_FILL_WMF, PSM_LR_FILL = 0, 1, 2
PSM_SPECKLE_OFF, PSM_SPECKLE_FIRST, PSM_SPECKLE_ONLY = 0, 1, 2
PSM_DCHECK_OFF, PSM_DCHECK_FIRST, PSM_DCHECK_ONLY = 0, 1, 2
PSM_UNIQUE_OFF, PSM_UNIQUE_FIRST, PSM_UNIQUE_ONLY = 0, 1, 2
PSM_MEDIAN_OFF, PSM_MEDIAN_FIRST, PSM_MEDIAN_ONLY = 0, 1, 2
PSM_PIX_U8, PSM_PIX_F32 = 1, 2
PSM_YUV_420, PSM_YUV_422 = 1, 2
PSM_YUV_NV12, PSM_YUV_NV21, PSM_YUV_I420, PSM_YUV_YV12, PSM_YUV_YUYV, PSM_YUV_UYVY, PSM_YUV_YVYU = 1, 2, 3, 4, 5, 6, 7
# the YUV formats by cv2's name (COLOR_YUV2BGR_<name>), and which are 4:2:0
YUV_FORMATS = {"nv12": PSM_YUV_NV12, "nv21": PSM_YUV_NV21, "i420": PSM_YUV_I420, "yv12": PSM_YUV_YV12,
               "yuyv": PSM_YUV_YUYV, "uyvy": PSM_YUV_UYVY, "yvyu": PSM_YUV_YVYU}
YUV_420 = ("nv12", "nv21", "i420", "yv12")
PSM_BAYER_RGGB, PSM_BAYER_BGGR, PSM_BAYER_GRBG, PSM_BAYER_GBRG = 1, 2, 3, 4
PSM_DEMOSAIC_BILINEAR, PSM_DEMOSAIC_EA = 1, 2
# the Bayer patterns by the colours of the 2 x 2 cell at (0, 0) in reading order, and the demosaicing methods
BAYER_PATTERNS = {"rggb": PSM_BAYER_RGGB, "bggr": PSM_BAYER_BGGR, "grbg": PSM_BAYER_GRBG, "gbrg": PSM_BAYER_GBRG}
DEMOSAIC_METHODS = {"bilinear": PSM_DEMOSAIC_BILINEAR, "ea": PSM_DEMOSAIC_EA}

_lib = None


class PsmError(RuntimeError):
    def __init__(self, code, text):
        super().__init__(f"prime_stereo_b200 error {code}: {text}")
        self.code = code


def lib():
    """Load the CUDA library (once). Raises OSError if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise OSError(
            f"{LIB_PATH} not found: build it with `make -C primestereomatch_b200/csrc` "
            "(or __graft_entry__.build()); there is no CPU fallback")
    L = C.CDLL(LIB_PATH)
    vp, sz, i, u8p, fp = C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p
    L.psm_device_count.argtypes = []
    L.psm_cvf_plan.argtypes = [i, i, i, i, i, C.POINTER(C.c_int), i]
    L.psm_create.argtypes = [C.POINTER(vp), i, i, i, i]
    L.psm_create_sharded.argtypes = [C.POINTER(vp), i, i, i, i, i, i]
    L.psm_create_u16.argtypes = [C.POINTER(vp), i, i, i, i, i, i]
    L.psm_create_blocked.argtypes = [C.POINTER(vp), i, i, i, i, i, i, i, i]
    L.psm_create_multi.argtypes = [C.POINTER(vp), i, i, i, C.POINTER(C.c_int), i, i, i]
    L.psm_create_range.argtypes = [C.POINTER(vp), i, i, i, i, C.POINTER(C.c_int), i, i, i]
    L.psm_disp_select_u16.argtypes = [vp, vp, sz, vp, sz]
    L.psm_disp_select_u16_async.argtypes = [vp, vp, sz, vp, sz]
    L.psm_disp_reduce_keys_u16.argtypes = [vp, vp, vp, i, vp, sz, vp, sz]
    L.psm_disp_fetch_p2p_u16.argtypes = [vp, vp, sz, vp, sz]
    L.psm_post_process_u16.argtypes = [vp, vp, sz, vp, sz]
    L.psm_destroy.argtypes = [vp]
    L.psm_set_option.argtypes = [vp, i, i]
    L.psm_set_guided_filter.argtypes = [vp, i, C.c_float]
    L.psm_set_matching_cost.argtypes = [vp, C.c_float, C.c_float, C.c_float]
    L.psm_set_post_filter.argtypes = [vp, i, C.c_float, i, i]
    L.psm_set_lr_check.argtypes = [vp, i]
    L.psm_set_speckle_filter.argtypes = [vp, i, i, i]
    L.psm_set_disparity_check.argtypes = [vp, i, i]
    L.psm_set_uniqueness_check.argtypes = [vp, i, i]
    L.psm_set_median_blur.argtypes = [vp, i, i]
    L.psm_set_rectify.argtypes = [vp, i, i, vp, sz, vp, sz, vp, sz, vp, sz]
    L.psm_read_valid_mask.argtypes = [vp, i, u8p, sz]
    L.psm_set_stream.argtypes = [vp, vp]
    L.psm_set_images.argtypes = [vp, fp, sz, fp, sz]
    L.psm_set_images_u8.argtypes = [vp, u8p, sz, u8p, sz]
    L.psm_set_images_device.argtypes = [vp, fp, sz, fp, sz]
    L.psm_set_images_device_planes.argtypes = [vp, i, C.POINTER(vp), C.POINTER(vp), sz, sz]
    L.psm_set_images_device_yuv.argtypes = [vp, i, C.POINTER(vp), C.POINTER(vp), sz, sz, sz, sz]
    L.psm_set_images_yuv.argtypes = [vp, i, u8p, sz, u8p, sz]
    L.psm_set_images_yuv_async.argtypes = [vp, i, u8p, sz, u8p, sz]
    L.psm_set_images_device_bayer.argtypes = [vp, i, i, vp, vp, sz, sz]
    L.psm_set_images_bayer.argtypes = [vp, i, i, u8p, sz, u8p, sz]
    L.psm_set_images_bayer_async.argtypes = [vp, i, i, u8p, sz, u8p, sz]
    L.psm_wait_stream.argtypes = [vp, vp]
    L.psm_signal_stream.argtypes = [vp, vp]
    L.psm_copy_maps_device.argtypes = [vp, i, vp, sz, vp, sz]
    L.psm_copy_costs_device.argtypes = [vp, fp, fp, sz]
    L.psm_read_costs.argtypes = [vp, i, fp, sz]
    L.psm_copy_runner_up_device.argtypes = [vp, fp, fp, sz]
    L.psm_read_runner_up.argtypes = [vp, i, fp, sz]
    L.psm_reproject_device.argtypes = [vp, i, vp, vp, i, fp, fp, sz]
    L.psm_read_points.argtypes = [vp, i, i, vp, i, fp, sz]
    L.psm_set_images_async.argtypes = [vp, fp, sz, fp, sz]
    L.psm_set_images_u8_async.argtypes = [vp, u8p, sz, u8p, sz]
    L.psm_set_images_commit.argtypes = [vp]
    L.psm_disp_select_async.argtypes = [vp, u8p, sz, u8p, sz]
    L.psm_cost_filter_fgf.argtypes = [vp, i]
    L.psm_post_process.argtypes = [vp, u8p, sz, u8p, sz]
    L.psm_post_process_device.argtypes = [vp]
    L.psm_cost_const.argtypes = [vp]
    L.psm_cost_filter.argtypes = [vp]
    L.psm_disp_select.argtypes = [vp, u8p, sz, u8p, sz]
    L.psm_disp_select_device.argtypes = [vp]
    L.psm_disp_select_keys.argtypes = [vp, vp, vp]
    L.psm_disp_reduce_keys.argtypes = [vp, vp, vp, i, u8p, sz, u8p, sz]
    L.psm_p2p_create_buffer.argtypes = [vp, i, C.POINTER(vp)]
    L.psm_ipc_export.argtypes = [vp, vp, C.c_char_p]
    L.psm_ipc_import.argtypes = [vp, C.c_char_p, C.POINTER(vp)]
    L.psm_p2p_set_peers.argtypes = [vp, C.POINTER(vp), i, i]
    L.psm_disp_select_keys_p2p.argtypes = [vp]
    L.psm_disp_reduce_p2p.argtypes = [vp]
    L.psm_disp_fetch_p2p.argtypes = [vp, u8p, sz, u8p, sz]
    L.psm_read_cost_slice.argtypes = [vp, i, i, fp, sz]
    L.psm_write_cost_slice.argtypes = [vp, i, i, fp, sz]
    L.psm_read_guide_plane.argtypes = [vp, i, i, fp, sz]
    L.psm_read_ab_slice.argtypes = [vp, i, i, fp, fp]
    L.psm_device_ptr.argtypes = [vp, i, C.POINTER(vp), C.POINTER(sz)]
    L.psm_stage_ms.argtypes = [vp, i, C.POINTER(C.c_float)]
    L.psm_launch_count.argtypes = [vp, C.POINTER(C.c_uint64)]
    L.psm_sync.argtypes = [vp]
    L.psm_last_error.argtypes = [vp]
    L.psm_last_error.restype = C.c_char_p
    L.psm_build_info.argtypes = []
    L.psm_build_info.restype = C.c_char_p
    for name in SYMBOLS:
        if name not in ("psm_last_error", "psm_build_info"):
            getattr(L, name).restype = C.c_int
    _lib = L
    return L


def check(rc, ctx=None):
    if rc != 0:
        text = lib().psm_last_error(ctx)
        raise PsmError(rc, text.decode() if text else "?")


PLAN_FIELDS = ("threads", "nstrips", "ndgroups", "nseg", "seg_rows", "pack_gl", "pack_x0", "pack_ndg", "pack_first", "grid")


def cvf_plan(width, height, d_count, sm_count=132, no_pack=False):
    """psm_cvf_plan as a dict (needs no device)."""
    out = (C.c_int * 10)()
    rc = lib().psm_cvf_plan(width, height, d_count, sm_count, 1 if no_pack else 0, out, 10)
    if rc != PSM_OK:
        raise PsmError(rc, "psm_cvf_plan: bad arguments")
    return dict(zip(PLAN_FIELDS, list(out)))
