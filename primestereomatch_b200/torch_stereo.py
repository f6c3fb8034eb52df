"""PyTorch interface: stereo frames that are already CUDA tensors in, disparity maps as CUDA tensors out.

`TorchStereo` runs the same contexts as `DispEst` (one device, blocked, or several devices) on frames in GPU memory --
NVDEC / nvJPEG output, `torchvision.io.decode_jpeg(..., device="cuda")`, another model's tensor -- in any of the layouts
`psm_set_images_device_planes` reads in place: HWC BGR / RGB, BGRA / RGBA and planar CHW, 8-bit or float, any row
stride.  `match` orders itself against torch's current stream with events (psm_wait_stream / psm_signal_stream) and
never waits on the host, so the frames and maps stay in the caller's stream order.  The maps equal, bit for bit, those of
the host upload of the same pixels.  Importing this module imports torch; the package imports it only on first use.
"""
import ctypes as C

import numpy as np
import torch

from . import capi
from .dispest import _Context, bayer_kind, create_context, resolve_map_bits, yuv_format, yuv_shape

_PIX = {torch.uint8: capi.PSM_PIX_U8, torch.float32: capi.PSM_PIX_F32}
_ORDER = {"bgr": (0, 1, 2), "rgb": (2, 1, 0)}   # the tensor channel that holds B, G and R
# the per-pixel outputs of match, in their return order: argument (and attribute) name, option, planes, device copy-out
_OUTPUTS = (("costs", capi.PSM_OPT_COSTS, 3, "psm_copy_costs_device"),
            ("runner_up", capi.PSM_OPT_RUNNER_UP, 2, "psm_copy_runner_up_device"))


def frame_layout(t, height, width, channels="bgr"):
    """The psm_set_images_device_planes arguments of a frame tensor, or of each frame of a batch.

    t: uint8 or float32, shaped (H, W, C) with C = 3 or 4 (the fourth channel, alpha, is not read), (3, H, W), or either
    with a leading batch dimension; (H, W, C) is taken when both fit.  channels: "bgr" or "rgb", the order of the first
    three channels.  -> (pix_type, [(B, G, R) byte addresses] per frame, row_step, col_step, batched).  Raises TypeError
    or ValueError on anything the layout cannot express (a column stride of 0, rows that overlap, other shapes); the
    tensor's device is not looked at."""
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"expected a torch.Tensor (got {type(t).__name__})")
    if t.dtype not in _PIX:
        raise TypeError(f"frames must be uint8 or float32 tensors (got {t.dtype})")
    if channels not in _ORDER:
        raise ValueError(f'channels must be "bgr" or "rgb" (got {channels!r})')
    if t.dim() not in (3, 4):
        raise ValueError(f"frames must be (H, W, C), (3, H, W) or batches of them (got shape {tuple(t.shape)})")
    shape, strides = tuple(t.shape[-3:]), tuple(t.stride()[-3:])
    if shape[:2] == (height, width) and shape[2] in (3, 4):
        sr, sc, sch = strides
    elif shape == (3, height, width):
        sch, sr, sc = strides
    else:
        raise ValueError(f"frames must be ({height}, {width}, 3 or 4) or (3, {height}, {width}), optionally with a leading "
                         f"batch dimension (got shape {tuple(t.shape)})")
    elem = t.element_size()
    row_step, col_step = sr * elem, sc * elem
    if sc < 1:
        raise ValueError(f"the column stride is {sc} elements: pixels of a row must not share samples")
    if row_step < (width - 1) * col_step + elem:
        raise ValueError(f"the row stride ({sr} elements) is shorter than a row ({width} pixels {sc} elements apart)")
    batched = t.dim() == 4
    n, bstride = (t.shape[0], t.stride(0) * elem) if batched else (1, 0)
    if n < 1:
        raise ValueError("empty batch")
    base = t.data_ptr()
    order = _ORDER[channels]
    frames = [tuple(base + b * bstride + order[c] * sch * elem for c in range(3)) for b in range(n)]
    return _PIX[t.dtype], frames, row_step, col_step, batched


def yuv_layout(t, height, width, format):
    """The psm_set_images_device_yuv arguments of a YUV frame tensor, or of each frame of a batch.

    t: uint8, in cv2's shape for the format -- (H * 3 / 2, W) for "nv12", "nv21", "i420", "yv12", (H, W, 2) for "yuyv",
    "uyvy", "yvyu" -- optionally with a leading batch dimension, any strides (the halves of one side-by-side frame
    included), except that I420 / YV12 frames, whose chroma planes are packed rows of W / 2 samples, must be contiguous.
    -> (sampling, [(Y, U, V) byte addresses] per frame, y_row_step, y_col_step, c_row_step, c_col_step, batched).  Raises
    TypeError or ValueError on anything the layout cannot express; the tensor's device is not looked at."""
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"expected a torch.Tensor (got {type(t).__name__})")
    if t.dtype != torch.uint8:
        raise TypeError(f"YUV frames must be uint8 tensors (got {t.dtype})")
    code, is420 = yuv_format(format)
    shape = yuv_shape(format, width, height)
    if t.dim() not in (len(shape), len(shape) + 1) or tuple(t.shape[-len(shape):]) != shape:
        raise ValueError(f"{format} frames must be {shape}, optionally with a leading batch dimension "
                         f"(got shape {tuple(t.shape)})")
    s = t.stride()[-len(shape):]
    sr, sc = s[0], s[1]
    if sc < 1:
        raise ValueError(f"the column stride is {sc} elements: pixels of a row must not share samples")
    if sr < (width - 1) * sc + 1:
        raise ValueError(f"the row stride ({sr} elements) is shorter than a row ({width} pixels {sc} elements apart)")
    name = format.lower()
    if is420:
        uv = height * sr   # the chroma rows follow the luma rows
        if name in ("i420", "yv12"):
            if (sr, sc) != (width, 1):
                raise ValueError(f"{name} frames must be contiguous: their chroma planes are packed rows of {width // 2} "
                                 f"samples (got strides {tuple(s)})")
            q = (width // 2) * (height // 2)
            u, v = (uv, uv + q) if name == "i420" else (uv + q, uv)
            offsets, steps = (0, u, v), (sr, 1, width // 2, 1)
        else:
            u, v = (uv, uv + sc) if name == "nv12" else (uv + sc, uv)
            offsets, steps = (0, u, v), (sr, sc, sr, 2 * sc)
    else:
        sch = s[2]   # (H, W, 2): sample k of pixel x; the chroma pair (U, V or V, U) spans pixels 2i and 2i + 1
        offsets = {"yuyv": (0, sch, sc + sch), "uyvy": (sch, 0, sc), "yvyu": (0, sc + sch, sch)}[name]
        steps = (sr, sc, sr, 2 * sc)
    sampling = capi.PSM_YUV_420 if is420 else capi.PSM_YUV_422
    batched = t.dim() == len(shape) + 1
    n, bstride = (t.shape[0], t.stride(0)) if batched else (1, 0)
    if n < 1:
        raise ValueError("empty batch")
    base = t.data_ptr()
    frames = [tuple(base + b * bstride + o for o in offsets) for b in range(n)]
    return (sampling, frames) + steps + (batched,)


def bayer_layout(t, height, width, pattern, method="bilinear"):
    """The psm_set_images_device_bayer arguments of a Bayer frame tensor, or of each frame of a batch.

    t: uint8 (H, W), optionally with a leading batch dimension, any strides (the halves of one side-by-side (H, 2W) frame
    included; each half is demosaiced as a frame of its own, and pattern names its own pixel (0, 0)).  -> (pattern code,
    method code, [byte address] per frame, row_step, col_step, batched).  Raises TypeError or ValueError on anything the
    layout cannot express; the tensor's device is not looked at."""
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"expected a torch.Tensor (got {type(t).__name__})")
    if t.dtype != torch.uint8:
        raise TypeError(f"Bayer frames must be uint8 tensors (got {t.dtype})")
    codes = bayer_kind(pattern, method)
    if t.dim() not in (2, 3) or tuple(t.shape[-2:]) != (height, width):
        raise ValueError(f"Bayer frames must be ({height}, {width}), optionally with a leading batch dimension "
                         f"(got shape {tuple(t.shape)})")
    sr, sc = t.stride()[-2:]
    if sc < 1:
        raise ValueError(f"the column stride is {sc} elements: pixels of a row must not share samples")
    if sr < (width - 1) * sc + 1:
        raise ValueError(f"the row stride ({sr} elements) is shorter than a row ({width} pixels {sc} elements apart)")
    batched = t.dim() == 3
    n, bstride = (t.shape[0], t.stride(0)) if batched else (1, 0)
    if n < 1:
        raise ValueError("empty batch")
    base = t.data_ptr()
    return codes + ([base + b * bstride for b in range(n)], sr, sc, batched)


def _pointers(frame):
    """the C argument of one frame's addresses: three channel or plane pointers, or one frame pointer"""
    return C.c_void_p(frame) if isinstance(frame, int) else (C.c_void_p * 3)(*frame)


class TorchStereo(_Context):
    """TorchStereo(width, height, max_disp, *, device=None, map_bits=None, block_slices=None, devices=None, min_disp=0)

    The context `DispEst` creates for the same arguments: `device` (an index, "cuda:k" or torch.device; None = the
    current device), `map_bits` (None: 8-bit maps up to max_disp 256, 16-bit above), `block_slices` (a blocked context),
    `devices` (a multi-device context whose frames and maps live on devices[0]), `min_disp` (a range context over
    [min_disp, max_disp), psm_create_range).  The setters pass their values straight to the C-ABI, which rejects bad ones
    with PsmError."""

    def __init__(self, width, height, max_disp, *, device=None, map_bits=None, block_slices=None, devices=None, min_disp=0):
        self.width, self.height, self.max_disp = int(width), int(height), int(max_disp)
        self._map_size = (self.width, self.height)
        self.min_disp = int(min_disp)
        self.map_bits = resolve_map_bits(self.max_disp, map_bits)
        if devices is not None:
            index = int(devices[0]) if len(devices) else 0
        else:
            dev = torch.device("cuda", device) if isinstance(device, int) else torch.device(device or "cuda")
            index = dev.index if dev.index is not None else torch.cuda.current_device()
        self.device = torch.device("cuda", index)
        self.subsample_rate = 4
        self.views = capi.PSM_VIEWS_BOTH
        self.costs = False   # PSM_OPT_COSTS as match() last set it
        self.runner_up = False   # PSM_OPT_RUNNER_UP as match() last set it
        self.dcheck = capi.PSM_DCHECK_OFF   # setDisparityCheck's mode
        self.unique = capi.PSM_UNIQUE_OFF   # setUniquenessCheck's mode
        self._lib = capi.lib()
        self._ctx = C.c_void_p()
        self._ctx = create_context(self.width, self.height, self.max_disp, self.map_bits, device=index,
                                   block_slices=block_slices, devices=devices, min_disp=self.min_disp)

    # -- settings (the C-ABI judges every value) ---------------------------------------------
    def setDisparityCheck(self, mode, max_diff=1):
        """DispEst.setDisparityCheck.  match(post_process=True) then turns PSM_OPT_COSTS on itself, since the check reads
        the winners' costs; it returns them only with costs=True."""
        super().setDisparityCheck(mode, max_diff)
        self.dcheck = int(mode)
        return 0

    def setUniquenessCheck(self, mode, ratio=10):
        """DispEst.setUniquenessCheck.  match(post_process=True) then turns PSM_OPT_COSTS and PSM_OPT_RUNNER_UP on
        itself, since the test reads both; it returns them only with costs=True / runner_up=True."""
        super().setUniquenessCheck(mode, ratio)
        self.unique = int(mode)
        return 0

    def setViews(self, views):
        value = self._VIEWS.get(views, -1) if isinstance(views, str) else -1
        self._check(self._lib.psm_set_option(self._ctx, capi.PSM_OPT_VIEWS, value))
        self.views = value

    def setSubsampleRate(self, rate):
        """The Fast Guided Filter's sub-sampling rate for match(..., fgf=True); psm_cost_filter_fgf judges it."""
        self.subsample_rate = int(rate)

    # -- frames -------------------------------------------------------------------------------
    def _layout(self, left, right, channels, yuv=None, bayer=None, demosaic="bilinear"):
        """Both frames' layout, checked in full before any device work: (H, W) frames, or uint8 frames of the source
        size while setRectify is on -> (the C-ABI call that takes them, its arguments before the pointers, left frames,
        right frames, its steps, batched)"""
        w, h = self.src_size or (self.width, self.height)
        if yuv is not None and bayer is not None:
            raise ValueError("yuv and bayer: a frame is one or the other")
        if bayer is not None:
            pattern, method, lf, row_step, col_step, batched = bayer_layout(left, h, w, bayer, demosaic)
            other = bayer_layout(right, h, w, bayer, demosaic)
            if left.shape != right.shape or (row_step, col_step) != other[3:5]:
                raise ValueError("left and right must have the same shape and strides")
            self._check_devices(left, right)
            return "psm_set_images_device_bayer", (pattern, method), lf, other[2], (row_step, col_step), batched
        if yuv is not None:
            sampling, lf, *steps, batched = yuv_layout(left, h, w, yuv)
            other = yuv_layout(right, h, w, yuv)
            if left.shape != right.shape or tuple(steps) != tuple(other[2:6]):
                raise ValueError("left and right must have the same shape and strides")
            self._check_devices(left, right)
            return "psm_set_images_device_yuv", (sampling,), lf, other[1], tuple(steps), batched
        pix, lf, row_step, col_step, batched = frame_layout(left, h, w, channels)
        other = frame_layout(right, h, w, channels)
        if self.src_size is not None and pix != capi.PSM_PIX_U8:
            raise ValueError("setRectify is on: rectification reads uint8 camera frames only (got float32)")
        if left.shape != right.shape or left.dtype != right.dtype or (pix, row_step, col_step) != (other[0], other[2], other[3]):
            raise ValueError("left and right must have the same shape, dtype and strides")
        self._check_devices(left, right)
        return "psm_set_images_device_planes", (pix,), lf, other[1], (row_step, col_step), batched

    def _check_devices(self, left, right):
        for name, t in (("left", left), ("right", right)):
            if t.device != self.device:
                raise ValueError(f"{name} is on {t.device}: frames must be CUDA tensors on the context's device {self.device}")

    def match(self, left, right, *, channels="bgr", yuv=None, bayer=None, demosaic="bilinear", fgf=False,
              post_process=False, costs=False, runner_up=False, points=None, handle_missing=False):
        """Disparity maps of one frame pair or a batch -> (lmap, rmap): new uint8 / uint16 tensors of shape (H, W) or
        (B, H, W) on the context's device; rmap is None on a left-only context.

        yuv="nv12" (or "nv21", "i420", "yv12", "yuyv", "uyvy", "yvyu"): the frames are uint8 YUV tensors in cv2's shapes
        (yuv_layout; the halves of one side-by-side frame included), converted to BGR on the device as
        cv2.cvtColor(frame, COLOR_YUV2BGR_<FORMAT>) does (psm_set_images_device_yuv); channels is not read.

        bayer="rggb" (or "bggr", "grbg", "gbrg"): the frames are uint8 Bayer tensors (H, W) (bayer_layout; the halves of
        one side-by-side frame included, each demosaiced as a frame of its own), demosaiced on the device as
        cv2.cvtColor(frame, COLOR_Bayer<PATTERN>2BGR) does with demosaic="bilinear", or _EA with demosaic="ea"
        (psm_set_images_device_bayer); channels is not read.

        costs=True -> (lmap, rmap, lcosts, rcosts): also the filtered costs beside each winner of the selection maps
        (PSM_OPT_COSTS, psm_copy_costs_device), new float32 tensors (3, H, W) or (B, 3, H, W) whose plane k holds the cost
        at disparity m + k - 1, bit for bit (the quiet NaN 0x7FC00000 outside [min_disp, max_disp)); rcosts is None on a
        left-only context.  The option is set when it differs from the last call's, which restarts the frame; with
        setDisparityCheck or setUniquenessCheck on and post_process=True it is on whatever costs says.

        runner_up=True -> also (lrunner, rrunner), appended after any costs: each pixel's runner-up away from the winner
        (PSM_OPT_RUNNER_UP, psm_copy_runner_up_device), new float32 tensors (2, H, W) or (B, 2, H, W): plane 0 the
        disparity r (0 where none exists), plane 1 its filtered cost bit for bit (the quiet NaN 0x7FC00000 where r = 0);
        rrunner is None on a left-only context.  The option is set when it differs from the last call's; with
        setUniquenessCheck on and post_process=True it is on whatever runner_up says.

        points=(Q_left, Q_right) -> also (lpts, rpts), appended last: OpenCV's reprojectImageTo3D of the maps this call
        returns (post-processed or selection) with each view's 4 x 4 reprojection matrix (psm_reproject_device), new
        float32 tensors (H, W, 3) or (B, H, W, 3) of X, Y, Z; either Q may be None, and its tensor is then None.
        handle_missing=True sets Z = 10000 wherever a map holds its minimum.

        After psm_wait_stream on torch's current stream: psm_set_images_device_planes (or _device_yuv, _device_bayer), psm_cost_const, the guided filter
        (the Fast Guided Filter at setSubsampleRate's rate with fgf=True), psm_disp_select_device, psm_post_process_device
        with post_process=True (the chain setUniquenessCheck, setDisparityCheck, setMedianBlur, setSpeckleFilter,
        setLRCheck and setPostFilter configure),
        psm_copy_maps_device and, with points, psm_reproject_device of each frame of a batch in turn; then
        psm_signal_stream.  No host synchronisation: the inputs may be overwritten or freed, and the maps read, on that stream at once."""
        wanted = (costs, runner_up)
        for (name, *_), on in zip(_OUTPUTS, wanted):
            if not isinstance(on, bool):
                raise TypeError(f"{name} must be True or False (got {on!r})")
        if not isinstance(handle_missing, bool):
            raise TypeError(f"handle_missing must be True or False (got {handle_missing!r})")
        qs = None
        if points is not None:
            if not isinstance(points, (tuple, list)) or len(points) != 2:
                raise TypeError("points must be a pair (Q_left, Q_right), either of them None")
            qs = [None if q is None else (C.c_double * 16)(*np.asarray(q, np.float64).reshape(4, 4).ravel())
                  for q in points]
            if qs[1] is not None and self.views != capi.PSM_VIEWS_BOTH:
                raise ValueError("points: a right Q on a left-only context (setViews('left'))")
            if qs[0] is None and qs[1] is None:
                raise ValueError("points: give a Q for at least one view")
        set_images, lead, lf, rf, steps, batched = self._layout(left, right, channels, yuv, bayer, demosaic)
        L, ctx = self._lib, self._ctx
        H, W = self.height, self.width
        mdt = torch.uint16 if self.map_bits == 16 else torch.uint8
        shape = (len(lf), H, W) if batched else (H, W)
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        lmap = torch.empty(shape, dtype=mdt, device=self.device)
        rmap = torch.empty(shape, dtype=mdt, device=self.device) if self.views == capi.PSM_VIEWS_BOTH else None
        row = W * lmap.element_size()
        outs = []   # (copy-out call, left planes, right planes) of each output asked for
        for (name, key, n, copy), on in zip(_OUTPUTS, wanted):
            # the disparity check of the post-process reads the costs, the uniqueness test the costs and the runner-up
            needed = self.unique != capi.PSM_UNIQUE_OFF or (key == capi.PSM_OPT_COSTS and self.dcheck != capi.PSM_DCHECK_OFF)
            option = on or (post_process and needed)
            if option != getattr(self, name):
                self._check(L.psm_set_option(ctx, key, int(option)))
                setattr(self, name, option)
            if on:
                oshape = (len(lf), n, H, W) if batched else (n, H, W)
                outs.append((getattr(L, copy), torch.empty(oshape, dtype=torch.float32, device=self.device),
                             None if rmap is None else torch.empty(oshape, dtype=torch.float32, device=self.device)))
        pts = [None, None]
        if qs is not None:
            pshape = (len(lf), H, W, 3) if batched else (H, W, 3)
            pts = [None if q is None else torch.empty(pshape, dtype=torch.float32, device=self.device) for q in qs]
        self._check(L.psm_wait_stream(ctx, stream))
        for b in range(len(lf)):
            self._check(getattr(L, set_images)(ctx, *lead, _pointers(lf[b]), _pointers(rf[b]), *steps))
            self._check(L.psm_cost_const(ctx))
            self._check(L.psm_cost_filter_fgf(ctx, self.subsample_rate) if fgf else L.psm_cost_filter(ctx))
            self._check(L.psm_disp_select_device(ctx))
            if post_process:
                self._check(L.psm_post_process_device(ctx))
            lm = lmap[b] if batched else lmap
            rm = None if rmap is None else (rmap[b] if batched else rmap)
            self._check(L.psm_copy_maps_device(ctx, 1 if post_process else 0, lm.data_ptr(), row,
                                               None if rm is None else rm.data_ptr(), row))
            for copy, lo, ro in outs:
                lo = lo[b] if batched else lo
                ro = None if ro is None else (ro[b] if batched else ro)
                self._check(copy(ctx, lo.data_ptr(), None if ro is None else ro.data_ptr(), W * 4))
            if qs is not None:
                lp, rp = ((None if p is None else (p[b] if batched else p).data_ptr()) for p in pts)
                self._check(L.psm_reproject_device(ctx, 1 if post_process else 0, qs[0], qs[1], int(handle_missing),
                                                   lp, rp, W * 12))
        self._check(L.psm_signal_stream(ctx, stream))
        return (lmap, rmap) + tuple(t for _, lo, ro in outs for t in (lo, ro)) + \
            (tuple(pts) if qs is not None else ())
