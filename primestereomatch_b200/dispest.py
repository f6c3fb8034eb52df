"""Host-side mirror of the reference's `DispEst` facade for the GPU compute mode.

Mirrors /root/reference/include/DispEst.h:21-109 (same method names, argument meaning and
return conventions: stage methods return 0 on success) with numpy arrays standing in for
cv::Mat.  Only the `_GPU` stage methods -- the path behind the `m` toggle -- are implemented,
and they are thin calls into the C-ABI (include/prime_stereo_b200.h); the CPU stage methods are
out of scope for this package (SURVEY.md section 8) and raise NotImplementedError.

The C++ twin that a maintainer links into the reference application is
primestereomatch_b200/host/DispEstB200.{h,cpp}; see INTEGRATION.md.
"""
import ctypes as C

import numpy as np

from . import capi

MAX_CPU_THREADS = 8  # reference include/ComFunc.h:52
OCV_DE, OCL_DE = 0, 1  # reference include/ComFunc.h:46-47


def device_count():
    """Role of openCLdevicepoll() (reference src/main.cpp:29): gates the `m` toggle."""
    return capi.lib().psm_device_count()


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def resolve_map_bits(max_disp, map_bits):
    """map_bits None -> 8-bit maps for max_disp <= 256, 16-bit above; 8 and 16 stay.  Raises ValueError otherwise."""
    if map_bits not in (None, 8, 16):
        raise ValueError(f"map_bits must be None, 8 or 16 (got {map_bits!r})")
    return map_bits if map_bits is not None else (16 if max_disp > 256 else 8)


def create_context(width, height, max_disp, map_bits, *, device=0, d_begin=0, d_count=None, block_slices=None,
                   devices=None, min_disp=0):
    """The context DispEst and TorchStereo run on, as a c_void_p handle (psm_destroy frees it): a multi-device context
    over `devices` (psm_create_multi, block_slices blocks every shard), a blocked context (psm_create_blocked), or one of
    [d_begin, d_begin + d_count) on `device` with map_bits-bit maps (psm_create_u16 / psm_create_sharded).  min_disp > 0:
    a range context over [min_disp, max_disp) of the same kind (psm_create_range); it is not a shard, so d_begin /
    d_count raise ValueError with it."""
    L = capi.lib()
    ctx = C.c_void_p()
    dc = max_disp - d_begin if d_count is None else d_count
    if min_disp:
        if d_begin != 0 or d_count is not None:
            raise ValueError("min_disp (a range context over [min_disp, max_disp)) excludes d_begin / d_count")
        devs = [int(device)] if devices is None else [int(x) for x in devices]
        arr = (C.c_int * max(1, len(devs)))(*devs)
        capi.check(L.psm_create_range(C.byref(ctx), width, height, int(min_disp), max_disp, arr, len(devs),
                                      int(block_slices or 0), map_bits))
    elif devices is not None:
        devs = [int(x) for x in devices]
        arr = (C.c_int * max(1, len(devs)))(*devs)
        capi.check(L.psm_create_multi(C.byref(ctx), width, height, max_disp, arr, len(devs), int(block_slices or 0),
                                      map_bits))
    elif block_slices is not None:
        capi.check(L.psm_create_blocked(C.byref(ctx), width, height, max_disp, int(d_begin), int(dc), int(block_slices),
                                        map_bits, int(device)))
    else:
        create = L.psm_create_u16 if map_bits == 16 else L.psm_create_sharded
        capi.check(create(C.byref(ctx), width, height, max_disp, int(d_begin), int(dc), int(device)))
    return ctx


def rectify_args(left_maps, right_maps, src_size, width, height):
    """The psm_set_rectify arguments after the context's size and ctx: (args, arrays) -- args = (SW, SH, then a pointer
    and a byte row step for each of xy_left, a_left, xy_right, a_right), arrays = the numpy arrays they point into (keep
    them alive for the call).  left_maps / right_maps: (xy, a), xy int16 (H, W, 2) (initUndistortRectifyMap's map[0],
    CV_16SC2), a uint16 (H, W) (map[1], CV_16UC1), both already cropped to the context's W x H; rows may lie any step
    apart (a cropped view of the full map is taken as it is).  src_size: (SW, SH), the size of the camera frames.  All
    three None: rectification off (0 x 0, null maps).  Raises TypeError or ValueError before any device work."""
    if left_maps is None and right_maps is None and src_size is None:
        return (0, 0, None, 0, None, 0, None, 0, None, 0), ()
    if left_maps is None or right_maps is None or src_size is None:
        raise ValueError("setRectify takes both views' maps and the source size, or None for all three (off)")
    try:
        sw, sh = (int(v) for v in src_size)
    except (TypeError, ValueError):
        raise TypeError(f"src_size must be (width, height) (got {src_size!r})") from None
    if not (1 <= sw <= 32767 and 1 <= sh <= 32767):
        raise ValueError(f"source size {sw} x {sh}: each side must lie in 1..32767 (the int16 map coordinates)")
    args, arrays = [sw, sh], []
    for name, maps in (("left", left_maps), ("right", right_maps)):
        if not isinstance(maps, (tuple, list)) or len(maps) != 2:
            raise TypeError(f"{name} maps must be a pair (xy, a)")
        for what, m, dtype, shape, inner in (("xy", maps[0], np.int16, (height, width, 2), (4, 2)),
                                             ("a", maps[1], np.uint16, (height, width), (2,))):
            m = np.asarray(m)
            if m.dtype != dtype or m.shape != shape:
                raise ValueError(f"{name} {what} map must be {np.dtype(dtype).name} of shape {shape} (the maps cropped to the "
                                 f"context's {width} x {height}; got {m.dtype} {m.shape})")
            if m.strides[1:] != inner or m.strides[0] < 0:
                m = np.ascontiguousarray(m)   # each row is read as a dense run of entries
            arrays.append(m)
            args += [_ptr(m), m.strides[0]]
    return tuple(args), tuple(arrays)


def yuv_format(format):
    """PSM_YUV_* of a format name ("nv12", "nv21", "i420", "yv12", "yuyv", "uyvy" or "yvyu", cv2's COLOR_YUV2BGR_<NAME>)
    -> (format code, True for 4:2:0); ValueError on any other value"""
    name = format.lower() if isinstance(format, str) else format
    if name not in capi.YUV_FORMATS:
        raise ValueError(f"unknown YUV format {format!r}: one of {', '.join(capi.YUV_FORMATS)}")
    return capi.YUV_FORMATS[name], name in capi.YUV_420


def yuv_shape(format, width, height):
    """the shape of a YUV frame of width x height in cv2's layout: (H * 3 / 2, W) for 4:2:0, (H, W, 2) for 4:2:2.
    ValueError on an unknown format, an odd width or (4:2:0) an odd height."""
    _, is420 = yuv_format(format)
    if width % 2 or (is420 and height % 2):
        raise ValueError(f"YUV frames of {width} x {height}: the width must be even, and the height too for 4:2:0")
    return (height * 3 // 2, width) if is420 else (height, width, 2)


def bayer_kind(pattern, method="bilinear"):
    """(PSM_BAYER_*, PSM_DEMOSAIC_*) of a pattern name ("rggb", "bggr", "grbg" or "gbrg": the colours of the 2 x 2 cell at
    (0, 0) in reading order) and a method name ("bilinear" or "ea", cv2's COLOR_Bayer<PATTERN>2BGR and _EA); ValueError on
    any other value"""
    names = []
    for value, table, what in ((pattern, capi.BAYER_PATTERNS, "Bayer pattern"),
                               (method, capi.DEMOSAIC_METHODS, "demosaicing method")):
        name = value.lower() if isinstance(value, str) else value
        if name not in table:
            raise ValueError(f"unknown {what} {value!r}: one of {', '.join(table)}")
        names.append(table[name])
    return tuple(names)


class _Context:
    """The settings and lifetime DispEst and TorchStereo share.  A subclass sets _lib (the library, or None when it was
    constructed without the GPU path: every setter then raises RuntimeError), _ctx (the context's handle) and _map_size
    (the maps' (W, H)).  Each setter passes its values to the C-ABI, which judges them (PsmError), and returns 0.  The
    docstrings name DispEst's stages; TorchStereo.match runs the same ones."""

    src_size = None   # setRectify: (SW, SH) of the camera frames the frame calls take; None = frames of the maps' size
    # setLRCheck's last accepted mode, for callers that read it; PostProcess_GPU asks the context whether the check ran
    lr_mode = capi.PSM_LR_OFF

    # -- lifetime ---------------------------------------------------------------------------
    def close(self):
        if self._lib is not None and self._ctx:
            self._lib.psm_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    @property
    def handle(self):
        return self._ctx

    def _check(self, rc):
        capi.check(rc, self._ctx)

    def _need_gpu(self):
        if self._lib is None:
            raise RuntimeError("DispEst was constructed with ocl=False: the GPU stages are unavailable")

    # -- settings ---------------------------------------------------------------------------
    def setGuidedFilter(self, window, eps):
        """Guided-filter window and regulariser (the reference's compile-time GIF_R_WIN and GIF_EPS, include/ComFunc.h:49-50)
        for every later CostFilter_GPU / CostFilter_FGF_GPU call; default (8, 1e-4).  Raises PsmError on values outside
        1 <= window <= 32, 0 < eps < inf."""
        self._need_gpu()
        self._check(self._lib.psm_set_guided_filter(self._ctx, int(window), float(eps)))
        return 0

    def setMatchingCost(self, alpha, tau_color, tau_grad):
        """Matching-cost weight and truncation thresholds (the reference's compile-time ALPHA_32F, TAU_1_32F and TAU_2_32F,
        include/CVC.h:18-23, with the truncation of src/CVC.cpp:24-25,36-37 applied) for every later CostConst_GPU call;
        default (0.9, inf, inf), the reference as shipped.  Raises PsmError unless 0 <= alpha <= 1 and each tau is >= 0 or
        inf (no truncation)."""
        self._need_gpu()
        self._check(self._lib.psm_set_matching_cost(self._ctx, float(alpha), float(tau_color), float(tau_grad)))
        return 0

    _WMF_WEIGHTS = {"exp": capi.PSM_WMF_EXP, "iv1": capi.PSM_WMF_IV1, "iv2": capi.PSM_WMF_IV2, "off": capi.PSM_WMF_OFF}

    def setPostFilter(self, radius, sigma=25.5, iterations=1, weight="exp"):
        """Joint weighted-median post-filter (JointWMF::filter's r, sigma, iter and weightType; the reference's PP::processDM
        passes MED_SZ/2 = 9 and the defaults) for every later PostProcess_GPU call; default (9, 25.5, 1, "exp").  weight is
        "exp", "iv1", "iv2" or "off".  Raises PsmError unless 1 <= radius <= 32, 2^-16 <= sigma <= 2^16 and
        1 <= iterations <= 16, and on any other weight name."""
        self._need_gpu()
        wt = self._WMF_WEIGHTS.get(weight, -1) if isinstance(weight, str) else -1
        self._check(self._lib.psm_set_post_filter(self._ctx, int(radius), float(sigma), int(iterations), wt))
        return 0

    def setLRCheck(self, mode):
        """Left-right consistency check and occlusion fill (the reference's lrCheck / fillInv, commented out in
        PP::processDM, src/PP.cpp:405-406) for every later PostProcess_GPU call: 0 off (default), 1 check + fill + the
        post-filter (processDM with those lines restored), 2 check + fill only.  With mode 1 or 2 PostProcess_GPU also
        fills lValid / rValid (0/1).  Raises PsmError on any other mode."""
        self._need_gpu()
        self._check(self._lib.psm_set_lr_check(self._ctx, int(mode)))
        self.lr_mode = int(mode)
        return 0

    def setSpeckleFilter(self, mode, max_size=0, max_diff=0):
        """Speckle removal (OpenCV's filterSpeckles(map, 0, max_size, max_diff)) for every later PostProcess_GPU call:
        0 off (default), 1 first (then the check and / or post-filter of setLRCheck / setPostFilter on its result), 2 only
        (its maps are the result; lValid / rValid are not read).  Every 4-connected blob of non-zero pixels whose
        neighbours differ by at most max_diff, of at most max_size pixels, becomes 0 (invalid).  Raises PsmError on any
        other mode, or unless max_size >= 1 and max_diff >= 0 with the filter on."""
        self._need_gpu()
        self._check(self._lib.psm_set_speckle_filter(self._ctx, int(mode), int(max_size), int(max_diff)))
        return 0

    def setDisparityCheck(self, mode, max_diff=1):
        """One-view disparity check (OpenCV's validateDisparity, StereoSGBM's disp12MaxDiff) for every later
        PostProcess_GPU call: 0 off (default), 1 first (then setSpeckleFilter's removal and the check and / or post-filter
        of setLRCheck / setPostFilter on its result), 2 only (its maps are the result; lValid / rValid are not read).  In
        each row, the pixels at x >= maxDis claim the other view's column their disparity points at, the lowest cost of
        setCostOutput's centre plane winning; a pixel whose disparity differs from its column's winner's by more than
        max_diff becomes 0 (invalid).  Needs setCostOutput(True) for the selection it checks.  On a left-only context,
        mode 1 with setLRCheck 1 or 2 fills the left map where it is below 2 and fills lValid.  Raises PsmError on any
        other mode, on max_diff outside [0, 4095], or on a context that owns part of the range with the check on."""
        self._need_gpu()
        self._check(self._lib.psm_set_disparity_check(self._ctx, int(mode), int(max_diff)))
        return 0

    def setUniquenessCheck(self, mode, ratio=10):
        """Uniqueness test (OpenCV StereoSGBM's uniquenessRatio) for every later PostProcess_GPU call: 0 off (default),
        1 first (then the rest of the chain -- setDisparityCheck, setMedianBlur, setSpeckleFilter, setLRCheck,
        setPostFilter -- on its result), 2 only (its maps are the result; lValid / rValid are not read).  A pixel with
        m != 0 becomes 0 (invalid) when its runner-up's cost q(r) (setRunnerUpOutput's plane 1) is within ratio percent
        of its winner's cost q(m) (setCostOutput's centre plane): q(r) * (100 - ratio) < q(m) * 100, exactly.  Needs
        setCostOutput(True) and setRunnerUpOutput(True) for the selection it tests.  On a left-only context, mode 1 with
        setLRCheck 1 or 2 fills the left map where it is below 2 and fills lValid.  Raises PsmError on any other mode, on
        ratio outside [0, 100], or on a context that owns part of the range with the test on."""
        self._need_gpu()
        self._check(self._lib.psm_set_uniqueness_check(self._ctx, int(mode), int(ratio)))
        return 0

    def setMedianBlur(self, mode, ksize=3):
        """ksize x ksize median (OpenCV's medianBlur, StereoSGBM's fixed medianBlur(disp, 3)) for every later
        PostProcess_GPU call, after the uniqueness test and the disparity check: 0 off (default), 1 first (then
        setSpeckleFilter's removal and the check and / or post-filter on its result), 2 only (the chain up to the median;
        its maps are the result; lValid / rValid are not read).  Equals cv2.medianBlur(map, ksize) on the u8 or u16 map,
        zeros included as values.  Raises PsmError on any other mode or on ksize other than 3 or 5."""
        self._need_gpu()
        self._check(self._lib.psm_set_median_blur(self._ctx, int(mode), int(ksize)))
        return 0

    def setRectify(self, left_maps, right_maps, src_size):
        """Rectify every later frame on the device (psm_set_rectify): the reference's video-mode remap(frame, rec,
        map[0], map[1], INTER_LINEAR) and crop, bit for bit.  left_maps / right_maps: (xy, a) of each view as
        initUndistortRectifyMap(..., CV_16SC2) returns them, cropped to the maps' W x H (xy int16 (H, W, 2), a uint16
        (H, W)); src_size: (SW, SH) of the camera frames.  setInputImages then takes uint8 frames of SH x SW x 3, and
        TorchStereo.match uint8 frames of (SH, SW) in any layout frame_layout reads (the two halves of one side-by-side
        tensor included); float frames raise PsmError (DispEst) or ValueError (TorchStereo).  None for all three turns it
        off.  Raises TypeError / ValueError on malformed maps before any device work."""
        args, _keep = rectify_args(left_maps, right_maps, src_size, *self._map_size)
        self._need_gpu()
        self._check(self._lib.psm_set_rectify(self._ctx, *args))
        self.src_size = None if src_size is None else (args[0], args[1])
        return 0

    _VIEWS = {"left": capi.PSM_VIEWS_LEFT, "both": capi.PSM_VIEWS_BOTH}   # the values of each class's own setViews

    # -- measurement helpers ----------------------------------------------------------------
    def stage_ms(self, stage):
        ms = C.c_float()
        self._check(self._lib.psm_stage_ms(self._ctx, stage, C.byref(ms)))
        return ms.value

    def launch_count(self):
        n = C.c_uint64()
        self._check(self._lib.psm_launch_count(self._ctx, C.byref(n)))
        return n.value


class DispEst(_Context):
    """DispEst(l, r, d, t, ocl) -- reference src/DispEst.cpp:10-143.

    l, r : HxWx3 images, both float32 in [0,1] (CV_32FC3) or both uint8 (CV_8UC3), BGR order.
    d    : maxDis.   t : CPU threads (kept for API compatibility).   ocl : use the GPU path.
    map_bits : None (8-bit maps for d <= 256, 16-bit above), 8 or 16 (16-bit maps at any d, d <= 4096).  With 16 bits
    lDisMap / rDisMap are uint16 (CV_16UC1) and the context comes from psm_create_u16; their low byte is the
    reference's uchar map.
    block_slices : None (the volumes hold every owned slice) or the number of slices a blocked context
    (psm_create_blocked) holds at once: the filter stages walk the owned range in blocks of that many, so device memory
    depends on it instead of on d.  The maps are the same either way; read_cost_volume is not available.
    devices : None (one device, `device`) or a list of CUDA device ids: a multi-device context (psm_create_multi) whose
    shard k runs on devices[k] and owns the k-th contiguous part of [0, d); ids may repeat.  The maps equal a
    single-device context's.  Not combinable with d_begin / d_count; block_slices blocks every shard.
    min_disp : 0 (default) or the first disparity of a range context over [min_disp, d) (psm_create_range), of the kind
    the other arguments select: it holds d - min_disp slices, its maps hold absolute disparities and its costs and
    runner-up are NaN / 0 outside the range.  Not combinable with d_begin / d_count (ValueError).
    """

    def __init__(self, l, r, d, t=MAX_CPU_THREADS, ocl=True, device=0, d_begin=0, d_count=None, map_bits=None,
                 block_slices=None, devices=None, min_disp=0):
        l, r = np.asarray(l), np.asarray(r)
        if l.dtype != r.dtype or l.shape != r.shape:
            # reference: "DE: Error - Left & Right images are of different types." then exit(1)
            raise ValueError("DE: Error - Left & Right images are of different types.")
        if l.ndim != 3 or l.shape[2] != 3 or l.dtype not in (np.float32, np.uint8):
            raise ValueError("DispEst expects HxWx3 float32 or uint8 images")
        self.hei, self.wid = int(l.shape[0]), int(l.shape[1])
        self._map_size = (self.wid, self.hei)
        self.maxDis = int(d)
        self.map_bits = resolve_map_bits(self.maxDis, map_bits)
        mdt = np.uint16 if self.map_bits == 16 else np.uint8
        self.threads = int(t)
        self.useOCL = bool(ocl)
        self.subsample_rate = 4
        self.lDisMap = np.zeros((self.hei, self.wid), mdt)  # DispEst.cpp:46-47
        self.rDisMap = np.zeros((self.hei, self.wid), mdt)
        self.lValid = np.zeros((self.hei, self.wid), np.uint8)  # DispEst.cpp:48-49
        self.rValid = np.zeros((self.hei, self.wid), np.uint8)
        self.cost_output = False
        self.lCosts = self.rCosts = None   # setCostOutput(True): DispSelect_GPU's (3, H, W) float32 costs
        self.runner_up_output = False
        self.lRunnerUp = self.rRunnerUp = None   # setRunnerUpOutput(True): DispSelect_GPU's (2, H, W) float32 runner-up
        if devices is not None and (d_begin != 0 or d_count is not None):
            raise ValueError("devices (a multi-device context over the whole range) excludes d_begin / d_count")
        if min_disp and (d_begin != 0 or d_count is not None):
            raise ValueError("min_disp (a range context over [min_disp, max_disp)) excludes d_begin / d_count")
        self.min_disp = int(min_disp)
        self._lImg, self._rImg = l, r
        self._yuv = None   # setInputImagesYUV's format code while its frames are the input
        self._bayer = None   # setInputImagesBayer's (pattern, method) codes while its frames are the input
        self._ctx = C.c_void_p()
        self._lib = None
        if self.useOCL:
            self._lib = capi.lib()
            self._ctx = create_context(self.wid, self.hei, self.maxDis, self.map_bits, device=device, d_begin=d_begin,
                                       d_count=d_count, block_slices=block_slices, devices=devices, min_disp=min_disp)
        if self.min_disp:
            d_begin = self.min_disp
        self.d_begin, self.d_count = d_begin, (self.maxDis - d_begin if d_count is None else d_count)
        self.block_slices = None if devices is not None and not block_slices else block_slices   # 0: unblocked shards
        self.devices = None if devices is None else list(devices)

    # -- reference public methods -----------------------------------------------------------
    def setInputImages(self, leftImg, rightImg):
        """DispEst.cpp:164-170 (asserts equal types, keeps the headers)."""
        leftImg, rightImg = np.asarray(leftImg), np.asarray(rightImg)
        assert leftImg.dtype == rightImg.dtype
        self._lImg, self._rImg = leftImg, rightImg
        self._yuv = self._bayer = None
        return 0

    def setInputImagesYUV(self, left, right, format):
        """YUV frames as input (psm_set_images_yuv): uint8 numpy arrays in cv2's shapes, (H * 3 / 2, W) for the 4:2:0
        formats "nv12", "nv21", "i420", "yv12" and (H, W, 2) for the 4:2:2 formats "yuyv", "uyvy", "yvyu", of the
        constructor's size or setRectify's source size.  CostConst_GPU converts them to BGR on the device as
        cv2.cvtColor(frame, COLOR_YUV2BGR_<FORMAT>) does, bit for bit.  Raises ValueError on an unknown format and TypeError
        on frames that are not uint8; CostConst_GPU checks the shape."""
        code, _ = yuv_format(format)
        left, right = np.asarray(left), np.asarray(right)
        if left.dtype != np.uint8 or right.dtype != np.uint8:
            raise TypeError(f"YUV frames must be uint8 (got {left.dtype}, {right.dtype})")
        self._lImg, self._rImg = left, right
        self._yuv = (code, format)
        self._bayer = None
        return 0

    def setInputImagesBayer(self, left, right, pattern, method="bilinear"):
        """Bayer raw frames as input (psm_set_images_bayer): uint8 numpy arrays (H, W) of the constructor's size or
        setRectify's source size, whose pixel (0, 0) starts the pattern ("rggb", "bggr", "grbg" or "gbrg").  CostConst_GPU
        demosaics them on the device as cv2.cvtColor(frame, COLOR_Bayer<PATTERN>2BGR) (method "bilinear") or _EA ("ea")
        does, bit for bit.  Raises ValueError on an unknown pattern or method and TypeError on frames that are not uint8;
        CostConst_GPU checks the shape."""
        codes = bayer_kind(pattern, method)
        left, right = np.asarray(left), np.asarray(right)
        if left.dtype != np.uint8 or right.dtype != np.uint8:
            raise TypeError(f"Bayer frames must be uint8 (got {left.dtype}, {right.dtype})")
        self._lImg, self._rImg = left, right
        self._yuv = None
        self._bayer = codes
        return 0

    def setThreads(self, newThreads):
        """DispEst.cpp:172-179."""
        if newThreads > MAX_CPU_THREADS:
            return -1
        self.threads = int(newThreads)
        return 0

    def setSubsampleRate(self, newRate):
        self.subsample_rate = int(newRate)

    def setViews(self, views):
        """Which disparity maps the later frames compute (PSM_OPT_VIEWS): "both" (default) or "left".  "left" skips every
        right-view stage after ingest; DispSelect_GPU and PostProcess_GPU then fill lDisMap alone, rDisMap is None, and
        setLRCheck modes 1 and 2 make PostProcess_GPU raise.  Changing it restarts the frame at CostConst_GPU.  Raises
        ValueError on any other value."""
        if not isinstance(views, str) or views not in self._VIEWS:
            raise ValueError(f'setViews takes "left" or "both" (got {views!r})')
        self._need_gpu()
        capi.check(self._lib.psm_set_option(self._ctx, capi.PSM_OPT_VIEWS, self._VIEWS[views]), self._ctx)
        if views == "left":
            self.rDisMap = None
        elif self.rDisMap is None:
            self.rDisMap = np.zeros_like(self.lDisMap)
        return 0

    def setCostOutput(self, on):
        """Whether DispSelect_GPU also fills lCosts / rCosts (PSM_OPT_COSTS): numpy float32 (3, H, W) whose plane k holds
        the filtered cost at disparity m + k - 1, m the selection map, bit for bit as the filter left it; the quiet NaN
        0x7FC00000 where m + k - 1 lies outside [0, maxDis).  rCosts is None on left-only frames.  Changing it restarts
        the frame at CostConst_GPU.  Raises TypeError unless on is a bool, PsmError on a context that owns part of the
        disparity range (d_begin / d_count)."""
        self.cost_output = self._set_output("setCostOutput", capi.PSM_OPT_COSTS, on)
        self.lCosts = self.rCosts = None
        return 0

    def setRunnerUpOutput(self, on):
        """Whether DispSelect_GPU also fills lRunnerUp / rRunnerUp (PSM_OPT_RUNNER_UP): numpy float32 (2, H, W), plane 0
        the runner-up r (the lowest-cost disparity d >= 1 with |d - m| >= 2, m the selection map; 0 where none exists),
        plane 1 its filtered cost bit for bit (the quiet NaN 0x7FC00000 where r = 0).  rRunnerUp is None on left-only
        frames.  Changing it restarts the frame at CostConst_GPU.  Raises TypeError unless on is a bool, PsmError on a
        context that owns part of the disparity range (d_begin / d_count)."""
        self.runner_up_output = self._set_output("setRunnerUpOutput", capi.PSM_OPT_RUNNER_UP, on)
        self.lRunnerUp = self.rRunnerUp = None
        return 0

    def _set_output(self, name, key, on):
        """the option `key` of a per-pixel output = on (a bool), through the setter `name` -> on"""
        if not isinstance(on, bool):
            raise TypeError(f"{name} takes True or False (got {on!r})")
        self._need_gpu()
        capi.check(self._lib.psm_set_option(self._ctx, key, int(on)), self._ctx)
        return on

    def _read_output(self, read, n):
        """both views' n result planes of a per-pixel output (read: psm_read_costs or psm_read_runner_up) -> (left,
        right), right None on left-only frames"""
        out = [None, None]
        for view in (capi.PSM_LEFT,) if self.rDisMap is None else (capi.PSM_LEFT, capi.PSM_RIGHT):
            out[view] = np.empty((n, self.hei, self.wid), np.float32)
            capi.check(read(self._ctx, view, _ptr(out[view]), out[view].strides[1]), self._ctx)
        return tuple(out)

    @staticmethod
    def _map_arg(m):
        return (None, 0) if m is None else (_ptr(m), m.strides[0])

    def set_option(self, key, value):
        capi.check(self._lib.psm_set_option(self._ctx, int(key), int(value)), self._ctx)

    def CostConst_GPU(self):
        """DispEst.cpp:272-276: upload both images, build both raw cost volumes on the device."""
        self._need_gpu()
        l = np.ascontiguousarray(self._lImg)
        r = np.ascontiguousarray(self._rImg)
        w, h = self.src_size or (self.wid, self.hei)
        if self._yuv is not None:
            code, name = self._yuv
            shape = yuv_shape(name, w, h)
            if l.shape != shape or r.shape != shape:
                raise ValueError(f"{name} frames must be {shape}: the size DispEst was constructed with, or the source size "
                                 f"of setRectify (got {l.shape}, {r.shape})")
            capi.check(self._lib.psm_set_images_yuv(self._ctx, code, _ptr(l), l.strides[0], _ptr(r), r.strides[0]),
                       self._ctx)
            capi.check(self._lib.psm_cost_const(self._ctx), self._ctx)
            return 0
        if self._bayer is not None:
            if l.shape != (h, w) or r.shape != (h, w):
                raise ValueError(f"Bayer frames must be {(h, w)}: the size DispEst was constructed with, or the source size "
                                 f"of setRectify (got {l.shape}, {r.shape})")
            capi.check(self._lib.psm_set_images_bayer(self._ctx, *self._bayer, _ptr(l), l.strides[0], _ptr(r),
                                                      r.strides[0]), self._ctx)
            capi.check(self._lib.psm_cost_const(self._ctx), self._ctx)
            return 0
        if l.shape != (h, w, 3) or r.shape != l.shape:
            raise ValueError(f"input images must be {h} x {w} x 3: the size DispEst was constructed with, or the source "
                             "size of setRectify")
        if l.dtype == np.uint8:
            capi.check(self._lib.psm_set_images_u8(self._ctx, _ptr(l), l.strides[0], _ptr(r), r.strides[0]), self._ctx)
        else:
            capi.check(self._lib.psm_set_images(self._ctx, _ptr(l), l.strides[0], _ptr(r), r.strides[0]), self._ctx)
        capi.check(self._lib.psm_cost_const(self._ctx), self._ctx)
        return 0

    def CostFilter_GPU(self):
        """DispEst.cpp:299-308."""
        self._need_gpu()
        capi.check(self._lib.psm_cost_filter(self._ctx), self._ctx)
        return 0

    def CostFilter_FGF_GPU(self):
        """Device twin of DispEst::CostFilter_FGF (DispEst.cpp:281-296): Fast Guided Filter at the sub-sampling rate
        set by setSubsampleRate (default 4, like StereoMatch.cpp:33)."""
        self._need_gpu()
        capi.check(self._lib.psm_cost_filter_fgf(self._ctx, int(self.subsample_rate)), self._ctx)
        return 0

    def DispSelect_GPU(self):
        """DispEst.cpp:323-328: WTA, results land in lDisMap / rDisMap."""
        self._need_gpu()
        sel = self._lib.psm_disp_select_u16 if self.map_bits == 16 else self._lib.psm_disp_select
        capi.check(sel(self._ctx, _ptr(self.lDisMap), self.lDisMap.strides[0], *self._map_arg(self.rDisMap)), self._ctx)
        if self.cost_output:
            self.lCosts, self.rCosts = self._read_output(self._lib.psm_read_costs, 3)
        if self.runner_up_output:
            self.lRunnerUp, self.rRunnerUp = self._read_output(self._lib.psm_read_runner_up, 2)
        return 0

    def PostProcess_GPU(self):
        """DispEst.cpp:338-344 -> PP::processDM (PP.cpp:402-425): joint weighted-median filter of both maps (after the
        left-right check and fill, or instead of the filter, as setLRCheck selects); the reference runs it on the CPU even
        in GPU mode, here it is a device stage.  The uniqueness test, the disparity check, the median and speckle
        removal run first, in that order, or end the chain, as setUniquenessCheck, setDisparityCheck, setMedianBlur and
        setSpeckleFilter select.  Results replace lDisMap / rDisMap."""
        self._need_gpu()
        pp = self._lib.psm_post_process_u16 if self.map_bits == 16 else self._lib.psm_post_process
        capi.check(pp(self._ctx, _ptr(self.lDisMap), self.lDisMap.strides[0], *self._map_arg(self.rDisMap)), self._ctx)
        masks = ((capi.PSM_LEFT, self.lValid),) + (((capi.PSM_RIGHT, self.rValid),) if self.rDisMap is not None else ())
        for view, mask in masks:
            rc = self._lib.psm_read_valid_mask(self._ctx, view, _ptr(mask), mask.strides[0])
            if rc == capi.PSM_ESTATE:   # the check did not run (a left-only fill masks the left view alone)
                break
            capi.check(rc, self._ctx)
        return 0

    _VIEW = {"left": capi.PSM_LEFT, "right": capi.PSM_RIGHT}
    _WHICH = {"selection": 0, "post": 1}

    def reproject(self, Q, view="left", which="post", handle_missing=False):
        """OpenCV's reprojectImageTo3D(map, xyz, Q, handleMissingValues) of one view's map on the device
        (psm_read_points) -> (H, W, 3) float32 X, Y, Z, bit for bit as cv2 computes them (NaN payloads aside).  Q: the
        rig's 4 x 4 reprojection matrix (stereoRectify's Q); view: "left" or "right"; which: "post" (the maps of the
        last PostProcess_GPU) or "selection" (those of the last DispSelect_GPU); handle_missing: Z = 10000 wherever the
        map holds its minimum.  Raises PsmError (PSM_ESTATE) before the stage that makes the maps has run."""
        self._need_gpu()
        q = np.ascontiguousarray(np.asarray(Q, np.float64).reshape(4, 4))
        if not isinstance(handle_missing, bool):
            raise TypeError(f"handle_missing must be True or False (got {handle_missing!r})")
        view_id = self._VIEW.get(view, -1) if isinstance(view, str) else -1
        which_id = self._WHICH.get(which, -1) if isinstance(which, str) else -1
        out = np.empty((self.hei, self.wid, 3), np.float32)
        capi.check(self._lib.psm_read_points(self._ctx, which_id, view_id, _ptr(q), int(handle_missing), _ptr(out),
                                             out.strides[0]), self._ctx)
        return out

    def CostConst(self):
        raise NotImplementedError("CPU stage (reference src/CVC.cpp) is not part of this package")

    CostConst_CPU = CostFilter = CostFilter_CPU = CostFilter_FGF = DispSelect_CPU = PostProcess_CPU = CostConst

    # -- parity / debugging helpers (role of DispEst::printCV, DispEst.cpp:181-194) ------------
    def read_cost_slice(self, view, d):
        out = np.empty((self.hei, self.wid), np.float32)
        capi.check(self._lib.psm_read_cost_slice(self._ctx, view, d, _ptr(out), out.strides[0]), self._ctx)
        return out

    def read_cost_volume(self, view):
        if self.block_slices is not None:
            raise RuntimeError("read_cost_volume on a blocked context: it holds one block of slices at a time "
                               "(read_cost_slice reads a slice of the resident block)")
        return np.stack([self.read_cost_slice(view, d) for d in range(self.d_begin, self.d_begin + self.d_count)])

    def write_cost_slice(self, view, d, src):
        src = np.ascontiguousarray(src, np.float32)
        capi.check(self._lib.psm_write_cost_slice(self._ctx, view, d, _ptr(src), src.strides[0]), self._ctx)

    def read_guide_plane(self, view, plane):
        out = np.empty((self.hei, self.wid), np.float32)
        capi.check(self._lib.psm_read_guide_plane(self._ctx, view, plane, _ptr(out), out.strides[0]), self._ctx)
        return out

    def read_ab_slice(self, view, d):
        a = np.empty((3, self.hei, self.wid), np.float32)
        b = np.empty((self.hei, self.wid), np.float32)
        capi.check(self._lib.psm_read_ab_slice(self._ctx, view, d, _ptr(a), _ptr(b)), self._ctx)
        return a, b

    def sync(self):
        capi.check(self._lib.psm_sync(self._ctx), self._ctx)
