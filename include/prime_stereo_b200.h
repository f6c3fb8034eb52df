/*
 * prime_stereo_b200.h -- C-ABI of the H100-native (sm_90a) STEREO_GIF hot path
 * (cost-volume construction -> guided-image-filter cost aggregation -> WTA).
 *
 * This is the drop-in boundary that sits under the reference's DispEst "_GPU" stage
 * methods (the `m`-toggle compute mode).  Plain C linkage, plain pointers and sizes,
 * no C++/torch/OpenCV types.  Every entry point returns 0 on success and a non-zero
 * PSM_E* code on failure (the reference's stage methods are `int`, 0 = success:
 * /root/reference/src/DispEst.cpp:275,307,327); psm_last_error() gives the text.
 *
 * Reference interfaces replaced (paths relative to /root/reference):
 *   psm_device_count      <-> openCLdevicepoll()                 src/main.cpp:29, src/oclUtil.cpp:18
 *   psm_create / destroy  <-> DispEst::DispEst(..., ocl=true) OpenCL part / ~DispEst
 *                                                                 src/DispEst.cpp:57-140, :145-162
 *   psm_set_images        <-> DispEst::setInputImages + H2D in CVC_cl::buildCV
 *                                                                 src/DispEst.cpp:164-170, src/CVC_cl.cpp:93-160
 *   psm_cost_const        <-> DispEst::CostConst_GPU             src/DispEst.cpp:272-276
 *   psm_cost_filter       <-> DispEst::CostFilter_GPU            src/DispEst.cpp:299-308
 *   psm_cost_filter_fgf   <-> DispEst::CostFilter_FGF -> FastGuidedFilter   src/DispEst.cpp:281-296, src/fastguidedfilter.cpp
 *   psm_disp_select       <-> DispEst::DispSelect_GPU + D2H in DispSel_cl::CVSelect
 *                                                                 src/DispEst.cpp:323-328, src/DispSel_cl.cpp:123-134
 *   psm_post_process      <-> DispEst::PostProcess_GPU -> PP::processDM -> JointWMF::filter
 *                                                                 src/DispEst.cpp:338-344, src/PP.cpp:402-425
 *   psm_set_lr_check      <-> PP::processDM's lrCheck + fillInv (commented out there)  src/PP.cpp:17-143, :405-406
 *   psm_set_speckle_filter <-> cv::filterSpeckles, as the reference's StereoSGBM matcher configures it (speckleWindowSize,
 *                             speckleRange)                       src/StereoMatch.cpp:654-655
 *   psm_set_disparity_check <-> cv::validateDisparity, the same matcher's disp12MaxDiff = 1  src/StereoMatch.cpp:651
 *   psm_set_uniqueness_check <-> StereoSGBM's uniqueness test, the same matcher's uniquenessRatio = 10
 *                                                                 src/StereoMatch.cpp:653
 *   psm_set_median_blur   <-> cv::medianBlur(disp, 3), which StereoSGBM::compute runs on every map it returns
 *   psm_reproject_device  <-> cv::reprojectImageTo3D with the rig's Q (camProps.Q, computed and never read there)
 *                                                                 src/StereoMatch.cpp:456-457
 *   psm_read_cost_slice   <-> DispEst::printCV (cost-slice dump) src/DispEst.cpp:181-194
 *   psm_stage_ms          <-> cvc_time/cvf_time/dispsel_time     src/StereoMatch.cpp:209-241
 *
 * Numerics contract: results equal the reference's CPU building blocks src/CVC.cpp, src/CVF.cpp (GuidedFilter_cv, the
 * full-resolution guided filter) and src/DispSel.cpp bit for bit -- NOT the divergent OpenCL kernels (SURVEY.md section
 * 2.1), and NOT what the reference binary's CPU mode runs today: StereoMatch::compute calls CostFilter_FGF (the
 * sub-sampled Fast Guided Filter) because the CostFilter_CPU that would call GuidedFilter_cv is declared but never
 * defined; that branch is psm_cost_filter_fgf.  "Bit for bit" for the box filters: cv::boxFilter keeps running fp64
 * sums along every row and down every column, so a rounding error, an inf or a NaN that enters one stays in it for the
 * rest of the row or column.  The tuned kernels sum in other orders and equal the reference while every fp64 sum is
 * exact.  Outside that domain, in OpenCV's order and bit for bit: every slice psm_write_cost_slice received with a
 * negative, -0, inf, NaN or >= 2^63 cost, every slice of a view whose image holds a negative, -0, inf, NaN or >= 2^61
 * value or whose solve terms are not finite, the guide of a view with a nonzero channel value outside [2^-12, 1], and
 * everything in PSM_CVF_NAIVE.  That pass is slow (one thread per row, then per column) and needs 48 bytes of scratch
 * per pixel, allocated on first use; u8 frames at the default window never take or allocate it.  Costs written
 * directly into the device volumes (psm_device_ptr) are not inspected.  Finite, non-negative costs whose window sums
 * are not exact (a magnitude range of more than ~2^29 in one row or column, such as a band of 1e15 above costs near
 * 1e-3) keep the tuned order: there q differs from the reference by up to the fp64 rounding the running sums carry,
 * which can be far more than one ulp of a small mean.  PSM_CVF_MIXED trades the bit-exact q for speed inside the tolerance
 * the task states (a, b bit-exact, |dq| <= 4e-6 on O(1) costs).  See DESIGN.md.
 *
 * Threading: one psm_ctx must not be used concurrently; it may be used from different
 * host threads over its life (every call binds its CUDA device first), matching how the
 * reference constructs DispEst on the HCI thread and runs stages on the worker thread.
 * Distinct contexts may be used concurrently from different host threads, on one device or
 * several: a kernel's dynamic shared-memory limit, which the CUDA runtime keeps once per
 * process and device, is only ever raised, so no context's setting can make another's launch
 * fail (DESIGN.md section 29).  psm_last_error(NULL) reports the calling thread's own last
 * failed creation.
 *
 * Host synchronisation: the calls documented as asynchronous only enqueue work once their first use is behind them.
 * On first use, or on the first call after a setting change, these may wait for the device (allocations, cudaFree,
 * blocking uploads): psm_set_images_async / _u8_async (the second staging set), psm_cost_filter and psm_read_ab_slice
 * (the scratch of the reference-order pass: float frames, a non-default guided filter, PSM_CVF_NAIVE, flagged slices),
 * psm_cost_filter_fgf (buffers and up-sampling plan, rebuilt for every new sub-sampling rate), psm_post_process_device
 * (its buffers and, after a change of sigma or weight type, the weight table; with psm_set_speckle_filter on, the
 * labels and counts, 8 * W * H bytes per view; with psm_set_disparity_check on rows over 6144 columns, its claim words;
 * with two or more of the uniqueness, check, median, removal and left-right steps, one map per computed view between
 * them),
 * psm_set_option(PSM_OPT_COSTS, 1) (the
 * cost planes), psm_set_option(PSM_OPT_RUNNER_UP, 1) (the runner-up planes, lists and slots), psm_reproject_device with
 * handle_missing (8 bytes of scratch).  Run them once before a
 * latency-critical
 * loop.  psm_set_stream always waits for the stream it leaves.
 */
#ifndef PRIME_STEREO_B200_H
#define PRIME_STEREO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct psm_ctx psm_ctx;

enum {
    PSM_OK = 0,
    PSM_EINVAL = 1,   /* bad argument */
    PSM_ECUDA = 2,    /* CUDA runtime error (text in psm_last_error) */
    PSM_ESTATE = 3,   /* stage called out of order (images not set, ...) */
    PSM_ENOMEM = 4
};

/* Views */
enum { PSM_LEFT = 0, PSM_RIGHT = 1 };

/* psm_set_option keys */
enum {
    PSM_OPT_CVF_MODE = 1,  /* PSM_CVF_* below; default PSM_CVF_EXACT */
    PSM_OPT_GRAY_MODE = 2, /* 0: fma(c2,.114,fma(c0,.299,c1*.587)) (OpenCV SIMD/IPP builds, default)
                              1: (c0*.299+c1*.587)+c2*.114 (non-FMA OpenCV builds) */
    PSM_OPT_TIMING = 3,    /* 1: record cudaEvents around each stage (default 1) */
    PSM_OPT_P2P_SYNC = 4,  /* fused multi-GPU exchange: 1 (default) = the kernels synchronise across ranks by
                              device-side flags in the exchange blocks (no library collective, no host barrier);
                              0 = the caller separates select / reduce / fetch by its own cross-rank barriers */
    PSM_OPT_VIEWS = 5,     /* PSM_VIEWS_BOTH (default) or PSM_VIEWS_LEFT: which disparity maps a frame computes; see
                              "Left-only frames" below */
    PSM_OPT_COSTS = 6,     /* 0 (default) or 1: the selection stages also keep the filtered costs beside each winner;
                              see psm_copy_costs_device */
    PSM_OPT_RUNNER_UP = 7  /* 0 (default) or 1: the selection stages also keep each pixel's runner-up disparity away
                              from the winner and its filtered cost; see psm_copy_runner_up_device */
    /* keys 100..106 are kernel tuning knobs used by bench.py experiments (variant, rows per segment, extra
       shared memory, threads per CTA, block remap, packed remainder strips off, CVC build); they never
       change results */
};
/* Values of PSM_OPT_VIEWS */
enum { PSM_VIEWS_LEFT = 1, PSM_VIEWS_BOTH = 2 };

/* Left-only frames (PSM_OPT_VIEWS = PSM_VIEWS_LEFT), for callers that consume the left map alone: about half of a
 * frame's device work computes the right view, which only the right map and the left-right check use.
 *   - Any value other than PSM_VIEWS_LEFT / PSM_VIEWS_BOTH returns PSM_EINVAL and changes nothing.  Changing the value
 *     keeps the current images and resets the frame's stages: the next stage must be psm_cost_const (every other stage
 *     returns PSM_ESTATE until then), and the earlier maps, masks, volumes and right-view guide are stale.
 *   - Ingest (psm_set_images*) is unchanged: both images are uploaded and ingested, because the left costs read the
 *     right image and its gradient (the right view's ingest planes 0-2 and 12 stay readable).
 *   - psm_cost_const builds the left raw volume; psm_cost_filter / psm_cost_filter_fgf compute the left guide and
 *     filter the left volume (every mode, window and rate; blocked contexts fold the left running keys only).
 *   - Selection writes the left map (and the left keys) only.  The right map pointer of psm_disp_select*,
 *     psm_disp_fetch_p2p* and psm_post_process* and the right key / gathered-key pointers of psm_disp_select_keys and
 *     psm_disp_reduce_keys* must be NULL: a non-NULL one returns PSM_EINVAL.  The fused exchange moves and reduces the
 *     left keys only; every rank must use the same setting.  Multi-device contexts forward the option to every shard.
 *   - psm_post_process* filters the left map only.  With a left-right check mode (psm_set_lr_check 1 or 2) it returns
 *     PSM_ESTATE: the check needs both maps; psm_set_disparity_check(PSM_DCHECK_FIRST) or
 *     psm_set_uniqueness_check(PSM_UNIQUE_FIRST) replaces it with the one-view tests and fills the left map.
 *     psm_set_lr_check itself may be called at any time.
 *   - PSM_ESTATE: psm_read_cost_slice, psm_read_ab_slice and psm_read_guide_plane planes 3-11 of the right view, and
 *     psm_read_valid_mask (of the left view too, unless the last post-process filled after the one-view tests).
 *   - Nothing else is written: the right volume, the right map, the right post-filtered map and the right mask keep
 *     their contents.  psm_device_ptr returns the same addresses, and no device memory is freed or allocated.
 *     psm_stage_ms reports the left view's work, psm_launch_count the kernels that ran. */

enum {
    PSM_CVF_EXACT = 0, /* streaming fused kernel, every box sum accumulated in fp64: bit-exact q */
    PSM_CVF_MIXED = 1, /* the tolerance mode north_star allows for fp32: first box stage fp64 (a, b bit-exact), second
                          box stage fp32 with a fixed summation tree: q within ~3e-6 of EXACT, deterministic
                          (tests/mixed_model.py restates it on the CPU); same maps as EXACT on every tested frame */
    PSM_CVF_NAIVE = 2  /* every slice in OpenCV's own summation order (psm_cvf_ref.cuh): slow device-side reference */
};

/* Diagnostic, needs no device: the work decomposition the streaming guided-filter kernel would use for a W x H x d_count
 * problem on a GPU with sm_count SMs (no reference counterpart; the reference's unit of parallel work is the slice,
 * src/DispEst.cpp:235-268).  out[0..9] = threads per CTA, full 112-column strips, slice groups, row segments, rows per
 * segment, lanes per slice of the packed remainder (0 = none), first output-aligned column of the packed remainder,
 * packed slice groups, first packed CTA, grid size.  The CPU tests check its invariants (every column and row of every
 * slice is produced exactly once). */
int psm_cvf_plan(int width, int height, int d_count, int sm_count, int no_pack, int* out, int n);

/* Number of usable CUDA devices (0 if none / no driver): gates the `m` toggle. */
int psm_device_count(void);

/* Create a context for W x H images and disparities [0, max_disp) on CUDA device `device`.
 * Allocates all device state (planar images, gradients, guide planes, both cost volumes,
 * disparity maps).  max_disp <= 256 (u8 disparity maps; psm_create_u16 for up to 4096). */
int psm_create(psm_ctx** out, int width, int height, int max_disp, int device);

/* Disparity-sharded context (multi-GPU, one context per GPU): this context owns the global
 * slices [d_begin, d_begin + d_count) of a max_disp-deep problem.  psm_create == shard [0,max_disp). */
int psm_create_sharded(psm_ctx** out, int width, int height, int max_disp,
                       int d_begin, int d_count, int device);

/* Context with 16-bit disparity maps (uint16_t), for 2 <= max_disp <= 4096, owning the global slices
 * [d_begin, d_begin + d_count) ([0, max_disp) = unsharded).  Holds at any D, D <= 256 included; geometry is validated
 * before any CUDA call (PSM_EINVAL), allocation failure returns PSM_ENOMEM.  The map format is fixed at creation:
 *   - format-neutral calls work on both kinds of context and write maps in the context's format: psm_disp_select_device,
 *     psm_disp_select_keys, psm_disp_select_keys_p2p, psm_disp_reduce_p2p, psm_post_process_device and every setter;
 *   - the map calls with host copies have a _u16 twin (psm_disp_select_u16, psm_disp_select_u16_async,
 *     psm_disp_reduce_keys_u16, psm_disp_fetch_p2p_u16, psm_post_process_u16); a u8 call on a u16 context, or a _u16
 *     call on a u8 context, returns PSM_EINVAL and names the right call;
 *   - psm_device_ptr selectors 2-5 return the 16-bit maps (pitch_elems = W);
 *   - the exchange block of psm_p2p_create_buffer holds 2-byte maps.
 * The selection is DispSel::CVSelect's arg-min kept as an int: the low byte of a 16-bit map is the reference's uchar map.
 * The post-filter is the same weighted median on the wider value range (JointWMF::filter on the map as CV_32F with
 * nI = max_disp).  4096 keeps a 12-bit disparity and the 18 colour bits in one packed u32; memory is the practical limit
 * below that (four W x H x d_count float volumes: about 35 GB at 1920 x 1080 x 1024).  See DESIGN.md section 14. */
int psm_create_u16(psm_ctx** out, int width, int height, int max_disp,
                   int d_begin, int d_count, int device);

/* Blocked context: owns the global slices [d_begin, d_begin + d_count) of a max_disp-deep problem like psm_create_u16,
 * but holds only `block_slices` of them at a time (1 <= block_slices <= d_count), so its device memory depends on the
 * block size instead of on d_count.  map_bits 8 (max_disp <= 256, the u8 map calls) or 16 (max_disp <= 4096, the _u16
 * calls).  Geometry, block size and map bits are validated before any CUDA call (PSM_EINVAL); allocation failure
 * returns PSM_ENOMEM.  Every map equals the one an unblocked context with the same arguments gives, bit for bit.
 * Device memory, with Wp = psm's row pitch (W rounded up to 4, plus 44 columns of halo, rounded up to 32 floats; at
 * least 160) and B = block_slices:
 *     4 * B * H * Wp * 4 bytes    the four volumes (two views, raw and filtered)
 *   + 16 * H * W                  two running-key planes (uint64)
 *   + about 2 * 20 * H * Wp * 4 + 2 * H * W * (3 * 4 + map_bits / 8)   guide planes, staging, maps
 * plus what the stages allocate on first use (post-filter; reference-order scratch: 48 bytes per pixel; FGF: 16 * B
 * bytes of coefficient means per low-resolution pixel).  At 1920 x 1080 (Wp = 1984) one slice of volume is 32.7 MiB: B = 128 takes about 4.3 GiB.
 * Stages on a blocked context:
 *   - psm_cost_const builds the raw costs of the first block (stage 1 times it);
 *   - psm_cost_filter / psm_cost_filter_fgf compute the guide once, then filter every block (building its raw costs
 *     first, for every block after the first) and fold its winner-take-all into the running keys.  Stage 2 covers the
 *     whole walk; stage 4 is not recorded (psm_stage_ms(4) returns PSM_ESTATE);
 *   - psm_disp_select* reduce the running keys to the maps (stage 3); psm_disp_select_keys copies them to the caller's
 *     buffers, so blocked shards feed psm_disp_reduce_keys as unblocked ones do.  Post-filter and left-right check as usual;
 *   - PSM_EINVAL, with the reason in psm_last_error: psm_write_cost_slice, psm_disp_select_keys_p2p, and
 *     psm_read_cost_slice / psm_read_ab_slice of a slice that is not resident (the first block after psm_cost_const,
 *     filtered costs of the last block after a filter stage);
 *   - psm_device_ptr selectors 0 / 1 return the resident block (slice d at offset d - its first slice).
 * See DESIGN.md section 16. */
int psm_create_blocked(psm_ctx** out, int width, int height, int max_disp,
                       int d_begin, int d_count, int block_slices, int map_bits, int device);

/* Multi-device context: one context over n_devices shards in this process, shard k on CUDA device devices[k] owning the
 * contiguous slices sharding.py's shard_range gives (max_disp / n_devices each, the last shard takes the remainder).
 * Devices may repeat: several shards on one device is a legal configuration.  block_slices 0 gives unblocked shards,
 * otherwise every shard is blocked (psm_create_blocked) with min(block_slices, its slice count).  map_bits 8
 * (max_disp <= 256, the u8 map calls) or 16 (max_disp <= 4096, the _u16 calls).  Every map equals the one a single-device
 * context of the same geometry gives, bit for bit.
 *   - PSM_EINVAL before any CUDA call: bad geometry or map bits, n_devices outside 1..min(8, max_disp), a null `devices`,
 *     a negative device id or block_slices < 0.  Then PSM_EINVAL for a device id at or above the device count, or for a
 *     pair of distinct devices without peer access (the message names the pair).  Peer access is enabled between every
 *     pair of distinct devices ("already enabled" is success) and never disabled: it is process-wide.  Allocation
 *     failure returns PSM_ENOMEM and frees what was built.
 *   - Every setter, psm_set_option (except PSM_OPT_P2P_SYNC), psm_cost_const, psm_cost_filter and psm_cost_filter_fgf
 *     go to every shard; a setter value one shard rejects leaves the context unchanged.
 *   - psm_set_images / _u8: the first shard uploads the frame once, as a single-device context does (host buffers are
 *     reusable on return); every other shard receives it from the first shard's device memory, device to device, and
 *     ingests it itself.  psm_set_images_device takes images resident on the first device, ordered against the work the
 *     context enqueues as for a single-device context (psm_sync, or the caller's own synchronisation).
 *   - psm_disp_select* and _u16: every shard scatters its minima (blocked shards: their running keys) into the
 *     reducers' exchange blocks, then every shard reduces its pixel chunk into every shard's maps; the kernels are
 *     ordered by CUDA events across the shards' streams and never wait on a flag.  The first shard's maps are the
 *     context's: psm_device_ptr selectors 2 / 3 (complete once psm_sync returns after psm_disp_select_device), the
 *     post-process (psm_post_process, _u16, _device, psm_read_valid_mask, selectors 4-7) runs on the first shard.
 *   - psm_read_cost_slice, psm_read_ab_slice and psm_write_cost_slice (unblocked shards only) go to the shard that owns
 *     global slice d; psm_read_guide_plane reads the first shard's planes.
 *   - psm_stage_ms: stages 0-2 and 4 are the longest of the shards' own times (stage 0 of the other shards covers the
 *     device-to-device copy; stage 4 is not recorded on blocked shards); stage 3 is timed on the first shard's stream
 *     from before its scatter to its maps being complete, so it includes the waits for the other shards; stage 5 is the
 *     first shard's.  psm_launch_count is the sum over the shards, psm_sync waits for every shard.
 *   - PSM_EINVAL, with the reason in psm_last_error: psm_set_stream (a stream belongs to one device), the asynchronous
 *     upload pair psm_set_images_async / _u8_async / _commit, psm_device_ptr selectors 0 / 1 (the volumes are split),
 *     psm_disp_select_keys, psm_disp_reduce_keys*, every psm_p2p_* / psm_ipc_* / *_p2p call, PSM_OPT_P2P_SYNC.
 * Device memory per shard: the shard's context (psm_create_u16 or psm_create_blocked of its slices) plus its exchange
 * block, about 16 * H * W + 2 * H * W * map_bits / 8 bytes.  See DESIGN.md section 17. */
int psm_create_multi(psm_ctx** out, int width, int height, int max_disp,
                     const int* devices, int n_devices, int block_slices, int map_bits);

/* Range context: solves the problem over disparities [min_disp, max_disp), 0 <= min_disp < max_disp, and holds its
 * n = max_disp - min_disp slices (or blocks of them), so memory and time follow n rather than max_disp.  A rig that never
 * sees anything beyond a known depth (a bin, a conveyor, a wall) has no disparity below some minimum; this is OpenCV's
 * minDisparity of StereoBM / StereoSGBM.
 *   - What it creates: n_devices == 1 with block_slices == 0 an unblocked context on devices[0], with block_slices > 0 a
 *     blocked one (psm_create_blocked) holding min(block_slices, n) slices; n_devices >= 2 a multi-device context
 *     (psm_create_multi) whose shards split [min_disp, max_disp) as psm_create_multi splits [0, max_disp).  min_disp = 0
 *     gives exactly the context psm_create_u16 (psm_create_sharded for 8-bit maps) / psm_create_blocked /
 *     psm_create_multi give over [0, max_disp).
 *   - PSM_EINVAL before any CUDA call: W or H below 1, min_disp < 0, max_disp < 2, min_disp >= max_disp, map_bits other
 *     than 8 (max_disp <= 256) or 16 (max_disp <= 4096), n_devices outside 1..min(8, n), block_slices < 0, a null
 *     `devices` or a negative device id.  Then the device and peer-access errors of psm_create_multi.
 *   - Slices: slice d of the range is built and filtered exactly as on a [0, max_disp) context, in every filter path; its
 *     raw and filtered costs are bit-identical to that context's slice d.
 *   - Selection: the candidates are d in [max(1, min_disp), max_disp) in the arg-min's order (strict <, lowest d on ties,
 *     NaN and +inf never win).  Maps hold the absolute disparity; 0 still means "no winner".
 *   - PSM_OPT_COSTS: entry k is q(m + k - 1), the quiet NaN 0x7FC00000 for an index outside [min_disp, max_disp).
 *     PSM_OPT_RUNNER_UP: the first candidate with |d - m| >= 2, 0 with a NaN cost when there is none.  Both are allowed.
 *   - The left-right check and the post-filter work on the absolute maps unchanged; the post-filter's value range is
 *     max_disp.
 *   - psm_read_cost_slice / psm_write_cost_slice / psm_read_ab_slice take a global d in the range (PSM_EINVAL outside
 *     it); on an unblocked context psm_device_ptr selectors 0 / 1 hold slice d at offset d - min_disp.
 * Every other call behaves as on the context of the same kind over [0, max_disp).  See DESIGN.md section 22. */
int psm_create_range(psm_ctx** out, int width, int height, int min_disp, int max_disp,
                     const int* devices, int n_devices, int block_slices, int map_bits);

/* Waits for the context's work on the stream it is bound to (psm_set_stream), on its own stream and on its copy stream,
 * then frees everything: a caller's stream bound with psm_set_stream must still exist when this is called. */
int psm_destroy(psm_ctx* ctx);

int psm_set_option(psm_ctx* ctx, int key, int value);

/* Guided-filter window (the reference's GIF_R_WIN: box Size(window, window), anchor window/2, BORDER_REFLECT_101)
 * and regulariser (GIF_EPS) for every later filtering call of this context. Default (8, 0.0001f).
 * Valid: 1 <= window <= 32, eps finite and > 0; anything else returns PSM_EINVAL and leaves the context unchanged.
 * Applies to psm_cost_filter, psm_read_guide_plane (planes 3-11), psm_read_ab_slice and psm_cost_filter_fgf (box
 * K = 2*(window/s)+1 with this eps, as FastGuidedFilter(img, GIF_R_WIN, GIF_EPS, s) does; PSM_EINVAL when the FGF kernel's
 * shared memory cannot hold that box, e.g. window 16 at s = 1).  Changing either value invalidates the cached guide planes.
 * At the defaults every call runs exactly the tuned 8 x 8 kernels; any other setting runs a generic-window streaming filter
 * (PSM_CVF_EXACT only: psm_cost_filter returns PSM_EINVAL in PSM_CVF_MIXED / PSM_CVF_NAIVE mode) whose results are
 * bit-exact under the same condition as the default path, with 2^23 replaced by 2^(29 - ceil(log2 window^2)).
 * Sharded contexts filter slice by slice as before: every rank must set the same parameters. */
int psm_set_guided_filter(psm_ctx* ctx, int window, float eps);

/* Matching cost (the reference's ALPHA_32F and truncation thresholds TAU_1_32F / TAU_2_32F, include/CVC.h:18-23) for every
 * later psm_cost_const of this context: src/CVC.cpp:18-39 with the truncation lines 24-25 and 36-37 restored, all in float:
 *   clr = (|dB| + |dG|) + |dR|,  grd = |dGradX|   (border pixels: the BC_32F differences in double, rounded once)
 *   if (clr > tau_color) clr = tau_color;  if (grd > tau_grad) grd = tau_grad;   (a NaN difference stays NaN)
 *   cost = alpha * clr + (1 - alpha) * grd       (every operation rounded separately, no FMA)
 * Default (0.9f, +inf, +inf): the reference as shipped, with the truncation commented out.  Valid: 0 <= alpha <= 1, each
 * tau >= 0 or +inf (no truncation); anything else, NaN included, returns PSM_EINVAL and leaves the context unchanged.
 * The guide planes do not depend on it.  At the default every call runs exactly the tuned cost-volume kernels; any other
 * setting runs a parameterised build of the shipped one (options 106 and 108 do not apply to it).  Sharded contexts build
 * their own slices: every rank must set the same values. */
int psm_set_matching_cost(psm_ctx* ctx, float alpha, float tau_color, float tau_grad);

/* Post-filter weight types: JointWMF::filter's weightType, numbered as in include/JointWMF.h:503-508 ("cos" = 3 and
 * "jac" = 4 are not functions of the colour difference and are not supported). */
enum { PSM_WMF_EXP = 0, PSM_WMF_IV1 = 1, PSM_WMF_IV2 = 2, PSM_WMF_OFF = 5 };

/* Post-filter (JointWMF::filter(disp, img8UC3, radius, sigma, 256, 256, iterations, weight_type), the reference's
 * PP::processDM with MED_SZ = 2 * radius + 1) for every later psm_post_process / psm_post_process_device of this context.
 * With s = sigma / 256 * 64 and the 6-bit colour difference (d0, d1, d2), in float with the reference's operation order:
 *   exp: expf(-(float)(d0^2+d1^2+d2^2) * (1 / ((2*s)*s)))    iv1: 1 / ((float)(|d0|+|d1|+|d2|) + s)
 *   iv2: 1 / ((float)(d0^2+d1^2+d2^2) + s*s)                  off: 1
 * held as W = lrintf(w / w(0) * 2^22); out(p) = min { v : 2 * sum_{q, I_q <= v} W >= sum_q W } over the (2r+1)^2 window
 * clipped at the image border, exact integer sums.  Each iteration filters the previous one's output with the original
 * feature image.  Default (9, 25.5f, 1, PSM_WMF_EXP): the reference as shipped.  Valid: 1 <= radius <= 32, sigma finite
 * in [2^-16, 2^16], 1 <= iterations <= 16, one of the four weight types; anything else, NaN included, returns PSM_EINVAL
 * and leaves the context unchanged.  At radius 9, sigma 25.5 and exp every pass runs exactly the tuned kernel pair; any
 * other setting runs a generic-radius kernel (two launches per pass and view in both cases).  The weight table is cached
 * on the context and rebuilt after a change of sigma or weight type.  See DESIGN.md section 13. */
int psm_set_post_filter(psm_ctx* ctx, int radius, float sigma, int iterations, int weight_type);

/* Left-right check modes of psm_set_lr_check */
enum { PSM_LR_OFF = 0, PSM_LR_FILL_WMF = 1, PSM_LR_FILL = 2 };

/* Left-right consistency check and occlusion fill (the reference's lrCheck and fillInv, src/PP.cpp:17-143, which
 * PP::processDM has commented out at :405-406) for every later psm_post_process / _u16 / _device of this context:
 *   PSM_LR_OFF (default): the post-filter alone, exactly as before (2 * 2 * iterations launches per call);
 *   PSM_LR_FILL_WMF: processDM with lines 405-406 restored: check, fill, then the post-filter of psm_set_post_filter on
 *                    the filled maps with the original feature image (1 + 4 * iterations launches);
 *   PSM_LR_FILL: check and fill only; the filled maps are the result (one launch).
 * Per row, on integer map values, W = width and mod the non-negative (Euclidean) remainder:
 *   lValid[x] = l[x] == r[(x - l[x]) mod W] && l[x] >= 2      rValid[x] = r[x] == l[(x + r[x]) mod W] && r[x] >= 2
 * both on the unmodified maps (disparities 0 and 1 are never valid; the gathers wrap around the row).  The reference
 * writes (x - d + W) % W, a C remainder, which equals this wherever d <= x + W and reads out of bounds beyond (a map
 * value above the width).  Then each view with its own mask: a valid pixel keeps its value, an invalid pixel x takes
 * min(map[L], map[R]) of the nearest valid pixels L <= x <= R, or the one of them that exists; a row with no valid pixel
 * is unchanged.  u16 maps use the same expressions.  The stage reads the maps of the last selection stage (or the
 * exchange block's complete maps) and never writes them: the filled maps go to psm_device_ptr selectors 4 / 5, the masks
 * to selectors 6 / 7.  Stage 5 of psm_stage_ms covers it.  Any other mode returns PSM_EINVAL and leaves the context
 * unchanged.  Sharded contexts: every rank must set the same mode.  See DESIGN.md section 15. */
int psm_set_lr_check(psm_ctx* ctx, int mode);

/* The left-right check's mask of one view (0 / 1, W x H, row step in bytes >= W) to HOST memory; synchronises.
 * PSM_ESTATE unless the last post-process call since the last selection stage ran the check. */
int psm_read_valid_mask(psm_ctx* ctx, int view, uint8_t* dst, size_t dst_step);

/* Speckle filter modes of psm_set_speckle_filter */
enum { PSM_SPECKLE_OFF = 0, PSM_SPECKLE_FIRST = 1, PSM_SPECKLE_ONLY = 2 };

/* Speckle removal (OpenCV's cv::filterSpeckles(map, 0, max_size, max_diff), as StereoBM / StereoSGBM users configure it
 * with speckleWindowSize and speckleRange) for every later psm_post_process / _u16 / _device of this context:
 *   PSM_SPECKLE_OFF (default): the stage exactly as psm_set_lr_check and psm_set_post_filter configure it, launch for
 *                     launch;
 *   PSM_SPECKLE_FIRST: speckle removal on the selection maps (or on the result of the uniqueness test, disparity check
 *                     and median before it, where those are on), then the configured check and / or post-filter on its
 *                     result (4 more launches);
 *   PSM_SPECKLE_ONLY: the chain up to and including speckle removal; its maps are the result and neither the check nor
 *                     the post-filter runs, so psm_read_valid_mask returns PSM_ESTATE (4 launches).
 * Definition, on each view's map on its own (u8, or u16 on a 16-bit context; cv::filterSpeckles on the map as CV_16S):
 * pixels of value 0 belong to no blob; two 4-neighbours p, q, both non-zero, are in the same blob when
 * |m(p) - m(q)| <= max_diff (in whole disparities, compared as int); blobs are the connected components of that graph;
 * every pixel of a blob of at most max_size pixels becomes 0, every other pixel keeps its value.  The result does not
 * depend on any visiting order.  Removed pixels are 0, which the check never accepts: with PSM_LR_FILL_WMF / PSM_LR_FILL
 * they are filled like occlusions and psm_read_valid_mask shows them as invalid.  With PSM_LR_OFF and
 * PSM_SPECKLE_FIRST the post-filter sees them as disparity 0 (a removed blob pulls its neighbours' medians down).  Range
 * contexts filter their absolute maps; left-only contexts filter the left map (PSM_SPECKLE_FIRST with a check mode keeps
 * the check's PSM_ESTATE).  The stage reads the maps of the last selection stage and never writes them, the costs or the
 * runner-up; the result goes to psm_device_ptr selectors 4 / 5 and psm_copy_maps_device(which = 1).  Stage 5 of
 * psm_stage_ms covers it.  Valid: one of the three modes and, unless the mode is PSM_SPECKLE_OFF, max_size >= 1 and
 * max_diff >= 0; anything else returns PSM_EINVAL and leaves the context unchanged.  Multi-device contexts forward it to
 * every shard.  See DESIGN.md section 23. */
int psm_set_speckle_filter(psm_ctx* ctx, int mode, int max_size, int max_diff);

/* Disparity check modes of psm_set_disparity_check */
enum { PSM_DCHECK_OFF = 0, PSM_DCHECK_FIRST = 1, PSM_DCHECK_ONLY = 2 };

/* One-view disparity check (OpenCV's cv::validateDisparity, StereoSGBM's disp12MaxDiff, which the reference's SGBM
 * matcher sets to 1) for every later psm_post_process / _u16 / _device of this context:
 *   PSM_DCHECK_OFF (default): the stage exactly as psm_set_speckle_filter, psm_set_lr_check and psm_set_post_filter
 *                     configure it, launch for launch;
 *   PSM_DCHECK_FIRST: the check on the selection maps (or on the uniqueness test's result, where it is on), then the
 *                     configured median, speckle removal, left-right check / fill and post-filter on its result, in
 *                     that order (one more launch);
 *   PSM_DCHECK_ONLY:  the chain up to and including the check; its maps are the result, nothing else runs and
 *                     psm_read_valid_mask returns PSM_ESTATE (one launch).
 * Definition, per row of one view's selection map m (u8 or u16), c = plane 1 of PSM_OPT_COSTS (the winner's cost q(m))
 * of the same selection, W = width, D = max_disp:
 *   1. only columns x in [D, W) with m[x] != 0 take part; every other pixel keeps its value;
 *   2. every participating x claims column x - m[x] with cost c[x]; per column the lowest cost wins, compared in the
 *      arg-min's order (-0 equal to +0), and on equal costs the lowest x; d2[column] is the winner's m;
 *   3. a participating x becomes 0 when |d2[x - m[x]] - m[x]| > max_diff (as int);
 *   4. the right view is the mirror image: fliplr(check(fliplr(r), fliplr(c_right))).
 * This equals cv::validateDisparity(m * 16 as CV_16S, c's order as CV_32S, 1, D - 1, max_diff) with 0 for 0; it does not
 * depend on min_disp.  With PSM_DCHECK_FIRST and PSM_LR_FILL / PSM_LR_FILL_WMF, a left-only context fills with the mask
 * valid[x] = v[x] >= 2 of its checked (and speckle-filtered) map v instead of the two-view check, and psm_read_valid_mask
 * of the left view returns that mask; two-view contexts run the left-right check on the checked maps, so the pixels
 * the check zeroed are filled like occlusions.  The stage reads the costs the last selection wrote: without them
 * (PSM_OPT_COSTS off for that selection) psm_post_process* returns PSM_ESTATE.  It writes nothing but the post-processed
 * maps and the masks.  Stage 5 of psm_stage_ms covers it.  Valid: one of the three modes and max_diff in [0, 4095];
 * anything else returns PSM_EINVAL and leaves the context unchanged, as does a mode other than PSM_DCHECK_OFF on a
 * context that owns part of the range (psm_create_sharded).  Multi-device contexts forward it to every shard; the stage
 * runs on the first.  Rows wider than 6144 columns use 8 * W * H bytes of scratch per computed view, allocated on first
 * use.
 * See DESIGN.md section 26. */
int psm_set_disparity_check(psm_ctx* ctx, int mode, int max_diff);

/* The post-process chain.  psm_post_process* runs the steps that are on in StereoSGBM's order,
 *   uniqueness test -> disparity check -> median -> speckle removal -> left-right check / fill -> post-filter,
 * each on the previous step's result.  A step's _ONLY mode (and PSM_LR_FILL) ends the chain after it: its maps are the
 * result.  With every step but the post-filter off, the stage is the post-filter alone.  Each of the first four adds one
 * launch (speckle removal four) and writes nothing but the post-processed maps and the masks.  On a left-only context,
 * PSM_UNIQUE_FIRST or PSM_DCHECK_FIRST with PSM_LR_FILL / PSM_LR_FILL_WMF fills the left map where the chain's map v is
 * below 2 (valid[x] = v[x] >= 2), and psm_read_valid_mask of the left view returns that mask. */

/* Uniqueness test modes of psm_set_uniqueness_check */
enum { PSM_UNIQUE_OFF = 0, PSM_UNIQUE_FIRST = 1, PSM_UNIQUE_ONLY = 2 };

/* Uniqueness test (OpenCV StereoSGBM's uniquenessRatio, which the reference's SGBM matcher sets to 10) for every later
 * psm_post_process / _u16 / _device of this context:
 *   PSM_UNIQUE_OFF (default): the stage exactly as the other steps configure it, launch for launch;
 *   PSM_UNIQUE_FIRST: the test on the selection maps, then the rest of the chain on its result (one more launch);
 *   PSM_UNIQUE_ONLY:  the test alone; its maps are the result and psm_read_valid_mask returns PSM_ESTATE (one launch).
 * Definition, per pixel of one view's selection map m (u8 or u16), with q(m) = plane 1 of PSM_OPT_COSTS and q(r) =
 * plane 1 of PSM_OPT_RUNNER_UP of the same selection: a pixel with m != 0 becomes 0 when
 *   (double)q(r) * (100 - ratio) < (double)q(m) * 100;
 * every other pixel keeps its value.  Both products are exact, so the comparison is the exact one on finite costs and
 * IEEE's on the rest: where there is no runner-up (r = 0, q(r) NaN) the pixel is kept.  This is computeDisparitySGBM's
 * `Sp[d]*(100 - uniquenessRatio) < minS*100 && abs(bestDisp - d) > 1` over the selection's candidates
 * [max(1, min_disp), max_disp) on float costs: the runner-up is the lowest of them with |d - m| >= 2, and multiplying
 * by a constant >= 0 keeps their order, so testing r alone tests them all.  Ratio 0 rejects nothing (q(r) >= q(m)).
 * StereoBM's variant (`<=` on integer sums with an integer division) is not this test.  Rejected pixels are 0, so they
 * claim no column in the disparity check that follows.  The stage reads the costs and the runner-up the last selection
 * wrote: without both (PSM_OPT_COSTS or PSM_OPT_RUNNER_UP off for that selection) psm_post_process* returns PSM_ESTATE.
 * Stage 5 of psm_stage_ms covers it.  Valid: one of the three modes and ratio in [0, 100]; anything else returns
 * PSM_EINVAL and leaves the context unchanged, as does a mode other than PSM_UNIQUE_OFF on a context that owns part of
 * the range (psm_create_sharded).  Multi-device contexts forward it to every shard; the stage runs on the first.
 * See DESIGN.md section 30. */
int psm_set_uniqueness_check(psm_ctx* ctx, int mode, int ratio);

/* Median modes of psm_set_median_blur */
enum { PSM_MEDIAN_OFF = 0, PSM_MEDIAN_FIRST = 1, PSM_MEDIAN_ONLY = 2 };

/* ksize x ksize median (OpenCV's cv::medianBlur, which StereoSGBM::compute runs with ksize 3 between its winner-take-all
 * and filterSpeckles) for every later psm_post_process / _u16 / _device of this context:
 *   PSM_MEDIAN_OFF (default): the stage exactly as the other steps configure it, launch for launch;
 *   PSM_MEDIAN_FIRST: the median after the uniqueness test and the disparity check, then speckle removal, the left-right
 *                     check / fill and the post-filter on its result (one more launch);
 *   PSM_MEDIAN_ONLY:  the chain up to and including the median; its maps are the result and psm_read_valid_mask
 *                     returns PSM_ESTATE (one launch).
 * Definition, per view: out(x, y) = the median of the ksize * ksize map values around (x, y), rows and columns clamped
 * to the map (BORDER_REPLICATE): exactly cv::medianBlur(map, ksize) on the u8 map, or on the u16 map as CV_16U.  Zeros
 * (invalid) take part as values, the lowest, as SGBM's invalid (minD - 1) * 16 does, so the result commutes with SGBM's
 * fixed-point scaling.  Stage 5 of psm_stage_ms covers it.  Valid: one of the three modes and ksize 3 or 5; anything
 * else returns PSM_EINVAL and leaves the context unchanged.  Multi-device contexts forward it to every shard; the stage
 * runs on the first.  See DESIGN.md section 30. */
int psm_set_median_blur(psm_ctx* ctx, int mode, int ksize);

/* Use an existing CUDA stream (cudaStream_t passed as void*) for all work; NULL restores the
 * context's own stream.  Lets a caller time with its own events on that stream.  Waits for the work already enqueued
 * on the stream the context was using.  The stream must outlive the context, or be replaced before psm_destroy. */
int psm_set_stream(psm_ctx* ctx, void* cuda_stream);

/* Ordering against a caller's stream (cudaStream_t passed as void*, NULL = the legacy default stream, on the context's
 * first device) with CUDA events only: neither call waits on the host, and both work on every kind of context.
 *   psm_wait_stream:   the context's later work waits for all work enqueued on the stream so far (e.g. the kernel
 *                      that wrote the frame psm_set_images_device_planes is about to read);
 *   psm_signal_stream: later work on the stream waits for all work the context has enqueued so far (e.g. a consumer of
 *                      the maps of psm_copy_maps_device, or the overwrite or free of the input frames).
 * "The context" is its compute and copy streams, on every shard of a multi-device context, including the
 * device-to-device copies that broadcast a frame.  The binding of psm_set_stream is unchanged.  PSM_EINVAL for a null
 * context. */
int psm_wait_stream(psm_ctx* ctx, void* cuda_stream);
int psm_signal_stream(psm_ctx* ctx, void* cuda_stream);

/* Inputs: interleaved 3-channel float images (cv::Mat CV_32FC3, BGR, values in [0,1]) in HOST
 * memory, row steps in BYTES.  Copies H2D and builds planar channels + x-gradients
 * (CVC::preprocess, src/CVC.cpp:41-46) on the device.
 * The buffers may be reused as soon as the call returns, page-locked or not: the copy runs on the context's copy
 * stream into a device staging set, once the last ingest from that set has read it (and after a pending
 * psm_set_images_async upload), and the call waits for it; the ingest kernels follow on the context's stream.  It does
 * not wait for the rest of the context's stream. */
int psm_set_images(psm_ctx* ctx, const float* left, size_t left_step,
                   const float* right, size_t right_step);

/* Same, 8-bit interleaved BGR input; the convertTo(CV_32F, 1/255.0f) of
 * src/StereoMatch.cpp:193-197 is done on the device (4x less H2D traffic).  Buffers reusable on return. */
int psm_set_images_u8(psm_ctx* ctx, const uint8_t* left, size_t left_step,
                      const uint8_t* right, size_t right_step);

/* Same as psm_set_images but the interleaved float images already live in DEVICE memory.  Asynchronous: the images are
 * read by the ingest kernels on the context's stream, so the caller orders the work that produces them, and any later
 * overwrite of them, against that stream (psm_set_stream, or events).  The pointers and steps must be multiples of 4
 * bytes (PSM_EINVAL before any CUDA call otherwise). */
int psm_set_images_device(psm_ctx* ctx, const float* d_left, size_t left_step,
                          const float* d_right, size_t right_step);

/* Sample types of psm_set_images_device_planes */
enum { PSM_PIX_U8 = 1, PSM_PIX_F32 = 2 };

/* Device frames in any 8-bit or float pixel layout (NVDEC / nvJPEG output, a tensor another model produced), read in
 * place: no staging copy, no host wait.  left[c] / right[c] point at channel c of pixel (0, 0) in B, G, R order; sample
 * (x, y) of channel c is at left[c] + y * row_step + x * col_step (bytes), in device memory of the context's (first)
 * device.  elem = 1 (PSM_PIX_U8) or 4 (PSM_PIX_F32) bytes; plane = the byte offset between channel planes:
 *   HWC BGR   p + 0, p + 1, p + 2 (times elem)   col_step 3 * elem
 *   HWC RGB   p + 2, p + 1, p + 0 (times elem)   col_step 3 * elem
 *   CHW RGB   p + 2 * plane, p + plane, p        col_step elem       (torchvision's decode_jpeg)
 *   BGRA      p + 0, p + 1, p + 2 (times elem)   col_step 4 * elem
 * The planes, gradients and guide flags equal those psm_set_images / _u8 build from the same sample values (u8 samples
 * scaled by 1/255.0f as convertTo does), so every later result is the same bit for bit; float frames take the same
 * flagged or unflagged filter route.  One ingest_kernel launch and one halo pass per view; stage 0 times it.
 *   - PSM_EINVAL before any CUDA call: a null array or channel pointer, an unknown pix_type, col_step < elem,
 *     row_step < (W - 1) * col_step + elem, and for float samples a pointer or step that is not a multiple of 4.
 *   - Asynchronous like psm_set_images_device: the kernels read the frames on the context's stream.  Order their
 *     producer before the call with psm_wait_stream, and their next overwrite or free after it with psm_signal_stream.
 *   - Multi-device contexts: the frames are read on the first device only; every other shard receives the first shard's
 *     ingested planes device to device, ordered by events (DESIGN.md section 19). */
int psm_set_images_device_planes(psm_ctx* ctx, int pix_type, const void* const left[3], const void* const right[3],
                                 size_t row_step, size_t col_step);

/* Rectify raw camera frames in ingest (the reference's video-mode remap and crop, src/StereoMatch.cpp:149-153, 464-478).
 * The maps are those initUndistortRectifyMap(..., CV_16SC2) returns for each view, cropped to the context's W x H: xy
 * holds W x H int16 pairs (sx, sy) (map[0], CV_16SC2), a holds W x H uint16 values (map[1], CV_16UC1), in HOST memory
 * with row steps in bytes.  They are copied once into device memory (6 bytes per pixel per view); synchronous.  From then
 * on every frame is 8-bit BGR of src_width x src_height, and output pixel (x, y) of each channel is
 *   a' = a[y][x] & 1023, fx = a' & 31, fy = a' >> 5,  taps (sx, sy), (sx + 1, sy), (sx, sy + 1), (sx + 1, sy + 1) with
 *   weights (32 - fx)(32 - fy) * 32, fx (32 - fy) * 32, (32 - fx) fy * 32, fx fy * 32;  a tap outside the frame reads 0;
 *   out = (sum of weight * sample + 16384) >> 15
 * -- cv::remap(frame, xy, a, INTER_LINEAR) with its default BORDER_CONSTANT 0, bit for bit -- and that u8 frame is
 * ingested as psm_set_images_u8 ingests a W x H frame (the gradient mirrors at the crop's borders).
 *   - psm_set_images_u8, _u8_async and psm_set_images_device_planes with PSM_PIX_U8 take src_width x src_height frames
 *     (steps checked against src_width); float frames (psm_set_images, _device, _async, PSM_PIX_F32 planes) return
 *     PSM_EINVAL.  One ingest_kernel launch and one halo pass per view, as without it.  The staging sets grow to hold
 *     the source frame here, so no frame allocates.
 *   - src_width = src_height = 0 with null maps and zero steps turns it off and frees the maps; the context then behaves
 *     as one that never rectified.
 *   - PSM_EINVAL before any CUDA work, context unchanged: a null map, a step below W * 4 (xy) or W * 2 (a) bytes, a source
 *     side outside 1..32767, or any other mix of zero and non-zero arguments.  PSM_ESTATE while a psm_set_images_async
 *     upload is pending.
 *   - Multi-device contexts keep the maps on the first shard; every kind of frame reaches the other shards as the first
 *     shard's ingested planes.  See DESIGN.md section 25. */
int psm_set_rectify(psm_ctx* ctx, int src_width, int src_height,
                    const int16_t* xy_left, size_t xy_left_step, const uint16_t* a_left, size_t a_left_step,
                    const int16_t* xy_right, size_t xy_right_step, const uint16_t* a_right, size_t a_right_step);

/* YUV frames (NVDEC surfaces, UVC cameras), converted to BGR in ingest.  A frame of Wf x Hf (the context's W x H, or the
 * source size while psm_set_rectify is on) has luma Y(x, y) and chroma U, V at (x >> 1, y >> vs), vs = 1 for 4:2:0 and 0
 * for 4:2:2.  Its BGR pixel is OpenCV's cvtColor(COLOR_YUV2BGR_*) (BT.601 limited range, fixed point, cv2 4.13.0), each
 * value clamped to 0..255:
 *   y' = max(0, Y - 16) * 1220542,  u = U - 128,  v = V - 128,  h = 1 << 19
 *   R = (y' + h + 1673527 v) >> 20,  G = (y' + h - 852492 v - 409993 u) >> 20,  B = (y' + h + 2116026 u) >> 20
 * and that u8 frame is ingested exactly as psm_set_images_u8 ingests it; with psm_set_rectify on, the frame is
 * remap(cvtColor(yuv), xy, a, INTER_LINEAR), each tap the converted pixel at its source position.  Wf must be even, and
 * Hf too for 4:2:0, as cv2 requires.  BT.709, full-range and 10-bit (P010 / P016) frames are not accepted: cv2 defines no
 * such conversion to pin them to.  One ingest_kernel launch and one halo pass per view, as for u8 frames.
 *
 * psm_set_images_device_yuv: device frames read in place, ordered like psm_set_images_device_planes (psm_wait_stream /
 * psm_signal_stream).  left[k] / right[k] point at Y, U, V of pixel (0, 0): Y(x, y) at p[0] + y * y_row_step + x *
 * y_col_step, U and V at p[1] / p[2] + (y >> vs) * c_row_step + (x >> 1) * c_col_step (bytes).  Separate luma and chroma
 * pitches (NVDEC) and the two halves of one side-by-side frame fit:
 *   NV12   Y p, 1;  U uv + 0, V uv + 1, c_col_step 2        I420   Y, U, V planes, c_col_step 1
 *   YUYV   Y p + 0, y_col_step 2;  U p + 1, V p + 3, c_col_step 4 (UYVY: U p, Y p + 1, V p + 2; YVYU: V p + 1, U p + 3)
 * psm_set_images_yuv / _yuv_async (finished by psm_set_images_commit): HOST frames in cv2's contiguous layouts, rows
 * `step` bytes apart: 4:2:0 formats are Hf * 3 / 2 rows (the luma rows, then the chroma; I420 and YV12 need step == Wf),
 * 4:2:2 formats Hf rows of 2 * Wf bytes.  They are copied into the u8 staging sets (1.5 or 2 bytes per pixel), so no
 * frame allocates, and converted in ingest; buffers reusable as for psm_set_images_u8 / _u8_async.
 *   - PSM_EINVAL before any CUDA work, context unchanged: an unknown format or sampling, a null pointer, an odd Wf or (4:2:0)
 *     Hf, a step below what a row spans (y_row_step < (Wf - 1) * y_col_step + 1, c_row_step < (Wf / 2 - 1) * c_col_step
 *     + 1, a zero column step, a host step below Wf or 2 * Wf).  psm_set_images_yuv_async returns PSM_ESTATE while
 *     another asynchronous upload is pending, and PSM_EINVAL on a multi-device context, as psm_set_images_u8_async does.
 *   - Multi-device contexts read the frame on the first device; the other shards receive its ingested planes.
 * See DESIGN.md section 27. */
enum { PSM_YUV_420 = 1, PSM_YUV_422 = 2 };
enum { PSM_YUV_NV12 = 1, PSM_YUV_NV21 = 2, PSM_YUV_I420 = 3, PSM_YUV_YV12 = 4, PSM_YUV_YUYV = 5, PSM_YUV_UYVY = 6,
       PSM_YUV_YVYU = 7 };
int psm_set_images_device_yuv(psm_ctx* ctx, int sampling, const void* const left[3], const void* const right[3],
                              size_t y_row_step, size_t y_col_step, size_t c_row_step, size_t c_col_step);
int psm_set_images_yuv(psm_ctx* ctx, int format, const uint8_t* left, size_t left_step, const uint8_t* right,
                       size_t right_step);
int psm_set_images_yuv_async(psm_ctx* ctx, int format, const uint8_t* left, size_t left_step, const uint8_t* right,
                             size_t right_step);

/* Bayer raw frames (machine-vision and CSI cameras), demosaiced to BGR in ingest.  A frame of Wf x Hf (the context's
 * W x H, or the source size while psm_set_rectify is on) has one u8 sample raw(x, y) per pixel; the pattern names the
 * colours of the 2 x 2 cell at (0, 0) in reading order (PSM_BAYER_RGGB is cv2's COLOR_BayerRGGB2BGR = COLOR_BayerBG2BGR,
 * BGGR = BayerRG, GRBG = BayerGB, GBRG = BayerGR: cv2's two-letter names are shifted by one cell).  Its BGR pixel is
 * OpenCV's cvtColor(COLOR_Bayer<PATTERN>2BGR) (PSM_DEMOSAIC_BILINEAR) or _EA (PSM_DEMOSAIC_EA), cv2 4.13.0:
 *   - interior pixel (1 <= x <= Wf - 2, 1 <= y <= Hf - 2) of colour c: channel c is raw(x, y).  At an R or B site
 *     G = (n4 + 2) >> 2 and the opposite colour = (d4 + 2) >> 2, n4 / d4 the sums of the four edge / diagonal neighbours.
 *     At a G site the colour of the horizontal neighbours is (raw(x - 1, y) + raw(x + 1, y) + 1) >> 1, the other colour
 *     (raw(x, y - 1) + raw(x, y + 1) + 1) >> 1.
 *   - edge-aware: G at an R or B site is the horizontal pair's (a + b + 1) >> 1 when |raw(x - 1, y) - raw(x + 1, y)| <=
 *     |raw(x, y - 1) - raw(x, y + 1)| (ties go horizontal), the vertical pair's otherwise; R and B as bilinear.
 *   - border: BGR(x, y) = interior(clamp(x, 1, Wf - 2), clamp(y, 1, Hf - 2)); every pixel is 0 when Wf < 3 or Hf < 3.
 * That u8 frame is ingested exactly as psm_set_images_u8 ingests it; with psm_set_rectify on, the frame is
 * remap(cvtColor(bayer), xy, a, INTER_LINEAR), each tap the demosaiced pixel at its source position.  One ingest_kernel
 * launch and one halo pass per view, as for u8 frames.
 *
 * Side-by-side frames: each view is demosaiced as a frame of its own, equal to cvtColor on the half as a separate array,
 * with borders at the half's own edges (demosaicing the whole side-by-side frame first differs at the two seam columns).
 * `pattern` names each view's own pixel (0, 0): a half that starts at an odd column has the horizontally shifted pattern.
 *
 * psm_set_images_device_bayer: device frames read in place, raw(x, y) at p + y * row_step + x * col_step (bytes), ordered
 * like psm_set_images_device_planes (psm_wait_stream / psm_signal_stream).
 * psm_set_images_bayer / _bayer_async (finished by psm_set_images_commit): HOST frames of Hf rows of Wf bytes, `step`
 * bytes apart, copied into the u8 staging sets (1 byte per pixel), so no frame allocates; buffers reusable as for
 * psm_set_images_u8 / _u8_async.
 *   - PSM_EINVAL before any CUDA work, context unchanged: an unknown pattern or method, a null pointer, a zero column
 *     step, row_step < (Wf - 1) * col_step + 1, a host step below Wf.  psm_set_images_bayer_async returns PSM_ESTATE while
 *     another asynchronous upload is pending, and PSM_EINVAL on a multi-device context, as psm_set_images_u8_async does.
 *   - Multi-device contexts read the frame on the first device; the other shards receive its ingested planes.
 * See DESIGN.md section 28. */
enum { PSM_BAYER_RGGB = 1, PSM_BAYER_BGGR = 2, PSM_BAYER_GRBG = 3, PSM_BAYER_GBRG = 4 };
enum { PSM_DEMOSAIC_BILINEAR = 1, PSM_DEMOSAIC_EA = 2 };
int psm_set_images_device_bayer(psm_ctx* ctx, int pattern, int method, const void* left, const void* right,
                                size_t row_step, size_t col_step);
int psm_set_images_bayer(psm_ctx* ctx, int pattern, int method, const uint8_t* left, size_t left_step,
                         const uint8_t* right, size_t right_step);
int psm_set_images_bayer_async(psm_ctx* ctx, int pattern, int method, const uint8_t* left, size_t left_step,
                               const uint8_t* right, size_t right_step);

/* Pipelined upload (extension; the reference's DispEst is synchronous per frame): start the H2D copy
 * of the NEXT frame on the context's copy stream into a second staging set while the current frame
 * is still being computed, then make it the current frame.  Host buffers must be page-locked for the
 * copy to overlap and must stay valid until psm_set_images_commit has returned; they may be reused after that.
 *   psm_set_images_async(k+1) ... stages of frame k ... psm_set_images_commit()  ->  frame k+1 is current
 * The copy waits until frame k-1's ingest has read the staging set it overwrites.  commit = the compute stream waits for
 * the upload, then the same ingest kernels as psm_set_images, then the host waits for the copy (in the two-deep pipeline
 * the frames already enqueued keep the device busy meanwhile). */
int psm_set_images_async(psm_ctx* ctx, const float* left, size_t left_step,
                         const float* right, size_t right_step);
int psm_set_images_u8_async(psm_ctx* ctx, const uint8_t* left, size_t left_step,
                            const uint8_t* right, size_t right_step);
int psm_set_images_commit(psm_ctx* ctx);

/* Stage 1: both raw cost volumes (CostConst_GPU). Asynchronous on the context stream. */
int psm_cost_const(psm_ctx* ctx);

/* Stage 2: guide precompute + guided filter of every slice of both volumes, in place
 * (CostFilter_GPU). Asynchronous on the context stream. */
int psm_cost_filter(psm_ctx* ctx);

/* Stage 2, Fast-Guided-Filter variant (DispEst::CostFilter_FGF, what the reference's CPU branch runs today): every
 * slice is sub-sampled by `sub_sample_rate` (1, 2, 4 or 8; the reference's `s` key cycles 2, 4, 8, default 4),
 * guided-filtered there with a (2*(8/s)+1)^2 box and the coefficient means are bilinearly up-sampled.  In place,
 * asynchronous.  Results equal the CPU restatement orc_cost_filter_fgf (test infrastructure, oracle/) bit for bit at any
 * input, including wide-range, outlier and non-finite costs, which is pinned against OpenCV's own (non-IPP) cv::blur /
 * cv::resize arithmetic (tests/golden/make_golden_fgf.py).  The K x K box is defined as the direct fp64 sum: from 0.0,
 * the K taps of a row left to right, then the K row sums top to bottom, times 1/K^2 in double, one rounding.  That equals
 * cv::blur wherever the fp64 sums are exact (values within 2^(29 - ceil(log2 K^2)) of each other in exponent); beyond
 * that the direct order is this library's definition, and cv::blur, which slides part of its sums, may differ. */
int psm_cost_filter_fgf(psm_ctx* ctx, int sub_sample_rate);

/* Stage 3: WTA over d in [1, max_disp) for both views; copies the u8 maps to HOST memory
 * (row steps in bytes) and synchronises (DispSelect_GPU).  Only valid on an unsharded context.
 * The destinations are checked before the selection runs: a null left map, or a step below a row, returns PSM_EINVAL
 * with nothing enqueued and the context unchanged; on a two-view context the same holds for the right map. */
int psm_disp_select(psm_ctx* ctx, uint8_t* left, size_t left_step,
                    uint8_t* right, size_t right_step);

/* Stage 3 with the D2H copies enqueued but NOT synchronised: the host maps are valid after psm_sync
 * (or any later synchronising call).  Page-locked host memory keeps the call asynchronous.  Destinations are checked
 * before the selection runs, as in psm_disp_select. */
int psm_disp_select_async(psm_ctx* ctx, uint8_t* left, size_t left_step,
                          uint8_t* right, size_t right_step);

/* Stage 3 without the D2H copy: maps stay on the device (see psm_device_ptr). Asynchronous. */
int psm_disp_select_device(psm_ctx* ctx);

/* Stage 3 on a u16 context (psm_create_u16): as psm_disp_select / psm_disp_select_async with uint16_t maps over
 * d in [1, max_disp); row steps in bytes (at least 2 * W), checked before the selection runs. */
int psm_disp_select_u16(psm_ctx* ctx, uint16_t* left, size_t left_step,
                        uint16_t* right, size_t right_step);
int psm_disp_select_u16_async(psm_ctx* ctx, uint16_t* left, size_t left_step,
                              uint16_t* right, size_t right_step);

/* Stage 4: post-processing of both maps -- the joint weighted-median filter of PP::processDM (window 19x19,
 * "exp" colour weights on the 6-bit-quantised left / right image, JointWMF defaults), on the device; the
 * reference runs this stage on the CPU even in GPU mode (src/DispEst.cpp:338-344).  Input: the maps of the last
 * selection stage (for a sharded context with the fused exchange: the complete maps of psm_disp_reduce_p2p);
 * output: filtered u8 maps copied to HOST memory (row steps in bytes), synchronises.  The destinations are checked before
 * the post-filter runs: a null left map, or a step below a row (the right map's too on a two-view context), returns
 * PSM_EINVAL with nothing enqueued and the context unchanged.
 * Parity: equals the reference's JointWMF whenever the feature image has <= 256 distinct 6-bit colours; beyond
 * that the reference clusters colours with an RNG-seeded cv::kmeans (an approximation by its own documentation,
 * JointWMF.h:70-72) while this stage evaluates the un-clustered weights -- see DESIGN.md. */
int psm_post_process(psm_ctx* ctx, uint8_t* left, size_t left_step, uint8_t* right, size_t right_step);
/* Same without the D2H copy (maps stay on the device: psm_device_ptr selectors 4, 5). Asynchronous. */
int psm_post_process_device(psm_ctx* ctx);
/* Stage 4 on a u16 context: as psm_post_process with uint16_t maps (row steps in bytes, checked before the post-filter). */
int psm_post_process_u16(psm_ctx* ctx, uint16_t* left, size_t left_step, uint16_t* right, size_t right_step);

/* Both maps into caller DEVICE buffers (row steps in bytes, at least W * map bytes), device to device on the context's
 * stream, asynchronous, in the context's map format (uint8_t, or uint16_t on a 16-bit context).  which = 0: the maps of
 * the last selection stage (psm_device_ptr selectors 2 / 3; a fused-exchange context's complete maps, as
 * psm_disp_fetch_p2p copies them); which = 1: the post-processed maps (selectors 4 / 5).  A multi-device context copies
 * the first shard's.  d_right must be NULL on a left-only context and is required otherwise.
 *   - PSM_EINVAL before any CUDA call: which not 0 / 1, a null pointer or a step below a row.
 *   - PSM_ESTATE: no selection (which = 0) or post-process (which = 1) since the context was created or PSM_OPT_VIEWS
 *     last changed, and under the exchanged-map rules of psm_disp_fetch_p2p. */
int psm_copy_maps_device(psm_ctx* ctx, int which, void* d_left, size_t left_step, void* d_right, size_t right_step);

/* The filtered costs at and beside each pixel's winning disparity (PSM_OPT_COSTS = 1), for sub-pixel refinement,
 * confidence masks or a cost threshold in the caller.  Per computed view, three float planes of H x W: plane k holds
 * q(x, y, m + k - 1), where m is the map of the last selection stage and q the filtered volume it scanned (the exact
 * filter in any mode, window or order, PSM_CVF_MIXED's q, or the Fast Guided Filter's q).  Every value is the volume's,
 * bit for bit (-0, +-inf and NaN payloads included).  An index outside [0, D) gives the quiet NaN 0x7FC00000, so a pixel
 * with no winner (map 0: every cost NaN or +inf) gets (NaN, q(0), q(1)).  The post-filter and the left-right check do not
 * change them: they belong to the selection maps.  Only a selection stage writes them, so on every kind of context they
 * stay the last selection's through the next frame's psm_set_images*, psm_cost_const and filter stage.
 *   - PSM_OPT_COSTS takes 0 or 1, anything else returns PSM_EINVAL and changes nothing.  Turning it on allocates the
 *     planes: 12 * H * W bytes per view, plus 16 * H * W on a blocked context, which tracks its winners' neighbours
 *     during the walk (a multi-device context: the result planes on the first shard only, the tracking planes on every
 *     blocked shard, 20 * H * W on a shard that owns no slice 0).  A failed allocation changes no setting, on any shard.
 *     A change resets the frame's stages as PSM_OPT_VIEWS does: the next stage must be psm_cost_const.  Turning it on
 *     returns PSM_EINVAL on a context that owns part of the range (psm_create_sharded, or psm_create_u16 /
 *     psm_create_blocked with d_count < max_disp); 0, the default, is accepted there.  A multi-device context passes it
 *     to every shard, since it spans [0, max_disp).
 *   - The work: after selection, one kernel per view writes the costs, from the volume on an unblocked context and from
 *     the tracking planes on a blocked one (whose block folds track them, in the same launches); on multi-device
 *     contexts every shard writes the entries it owns into the first shard's planes after the reduce.  Stage 3
 *     (psm_stage_ms) covers these kernels; psm_launch_count counts them.  With the option off nothing of this runs.
 *   - psm_disp_select_keys does not write the costs, and neither do the fused-exchange calls.
 * psm_copy_costs_device writes view v's planes to caller DEVICE memory on the context's stream, asynchronously: plane k
 * starts at dst + k * H * row_step (a contiguous (3, H, W) float32 tensor: row_step = 4 * W).  d_right must be NULL on a
 * left-only context and is required otherwise.  psm_read_costs writes one view's planes to HOST memory, same layout,
 * and synchronises.  A multi-device context copies the first shard's planes.
 *   - PSM_EINVAL before any CUDA call: a null pointer, a row_step below 4 * W, a bad view.
 *   - PSM_ESTATE: the last selection stage (psm_disp_select*) since the context was created or PSM_OPT_VIEWS /
 *     PSM_OPT_COSTS last changed did not run with PSM_OPT_COSTS = 1; a right-view read on a left-only context. */
int psm_copy_costs_device(psm_ctx* ctx, float* d_left, float* d_right, size_t row_step);
int psm_read_costs(psm_ctx* ctx, int view, float* dst, size_t row_step);

/* Each pixel's runner-up away from its winner (PSM_OPT_RUNNER_UP = 1), for the confidence tests a caller builds on it
 * (a uniqueness ratio as OpenCV's StereoBM / StereoSGBM uniquenessRatio, the peak ratio, the maximum margin).  The
 * reference has no confidence output; this is not part of its pipeline.  Take the filtered volume q the last selection
 * stage scanned (any filter path) and its map m.  The candidates are the arg-min's: d in [1, D) whose cost compares below
 * +inf (NaN and +inf never are, -0 ties with +0), lowest cost first and the lowest d first on ties.  The runner-up r is
 * the first candidate with |d - m| >= 2, and 0 when there is none (m = 0, D <= 3, or every cost away from m is +inf or
 * NaN).  Per computed view, two float planes of H x W: plane 0 holds r (an exact integer), plane 1 q(r), bit for bit
 * (the quiet NaN 0x7FC00000 where r = 0).  The exclusion width is 1 and fixed.  With PSM_OPT_COSTS the plain second
 * minimum is the first of q(m - 1) (m - 1 >= 1), q(m + 1) (m + 1 < D) and q(r) in that order.  The post-filter and the
 * left-right check do not change the planes; only a selection stage writes them, so on every kind of context they stay
 * the last selection's through the next frame's psm_set_images*, psm_cost_const and filter stage.
 *   - PSM_OPT_RUNNER_UP takes 0 or 1, anything else returns PSM_EINVAL and changes nothing.  Turning it on allocates
 *     8 * H * W bytes per view of result planes; a blocked context also keeps the running list's entries beside its
 *     running keys (28 * H * W bytes per view: four costs and three disparities), and a multi-device context keeps the
 *     result planes and one slot per shard on the first shard (12 * H * W bytes per shard and view) and the lists on
 *     every blocked shard.  A failed allocation changes no setting, on any shard.  A change resets the frame's stages as
 *     PSM_OPT_VIEWS does: the next stage must be psm_cost_const.  Turning it on returns PSM_EINVAL on a context that owns
 *     part of the range; 0, the default, is accepted there.  It may be on together with PSM_OPT_COSTS.
 *   - The work, all in stage 3 (psm_stage_ms) except the fold: an unblocked context selects the map and the runner-up in
 *     one kernel per view, in place of the plain selection (no extra launch); a blocked context's block folds keep the
 *     lists in the launches they make anyway, and one kernel per view picks the runner-up after selection; on a
 *     multi-device context every shard picks its candidate after the reduce (one kernel per view, a list scan of its
 *     slices when unblocked) into its slot on the first shard, which reduces the slots (one kernel per view).
 *     psm_launch_count counts them.  With the option off nothing of this runs.
 *   - psm_disp_select_keys does not write the runner-up, and neither do the fused-exchange calls.
 * psm_copy_runner_up_device writes view v's planes to caller DEVICE memory on the context's stream, asynchronously: plane
 * k starts at dst + k * H * row_step (a contiguous (2, H, W) float32 tensor: row_step = 4 * W).  psm_read_runner_up writes
 * one view's planes to HOST memory, same layout, and synchronises.  Arguments, left-only contexts and states as for
 * psm_copy_costs_device / psm_read_costs, with PSM_OPT_RUNNER_UP in place of PSM_OPT_COSTS. */
int psm_copy_runner_up_device(psm_ctx* ctx, float* d_left, float* d_right, size_t row_step);
int psm_read_runner_up(psm_ctx* ctx, int view, float* dst, size_t row_step);

/* The 3D point of every pixel of a map (OpenCV's cv::reprojectImageTo3D(map, xyz, Q, handleMissingValues) with a map of
 * integer disparities), for the rig's 4 x 4 reprojection matrix Q (row-major doubles, as cv::stereoRectify returns it);
 * the reference computes Q (src/StereoMatch.cpp:456-457, camProps.Q) and never reads it.  Per requested view, X, Y, Z
 * interleaved as float32 (CV_32FC3: 12 bytes per pixel), rows row_step bytes apart.  For pixel (x, y) with map value d,
 * in fp64 with each product and sum rounded on its own (no fused multiply-add) and the sum started from +0.0:
 *     h[i] = (((+0.0 + Q[i][0] x) + Q[i][1] y) + Q[i][2] d) + Q[i][3],  r = 1 / h[3] (correctly rounded),
 *     X = (float)((double)(float)h[0] * r), Y and Z likewise from h[1] and h[2];
 * with handle_missing = 1, Z = 10000 wherever d equals the minimum of that view's map (OpenCV takes the minimum for the
 * missing value, zero or not).  This is cv2's result bit for bit, except that a NaN (0 * inf, a NaN in Q) may carry
 * another payload.  Q may hold any doubles (0, +-inf, NaN): the result is what IEEE arithmetic gives.
 * which = 0: the maps of the last selection stage (a fused-exchange context's complete maps; a range context's absolute
 * disparities); which = 1: the post-processed maps -- as psm_copy_maps_device reads them.  A multi-device context
 * reprojects the first shard's.  The maps, masks, costs and runner-up are not touched.
 * psm_reproject_device: a view is reprojected when both its Q and its DEVICE point buffer are given; one launch covers
 * every requested view, plus one launch in front of it with handle_missing (the maps' minima, into context scratch), on
 * the context's stream, asynchronous; psm_launch_count counts them (a fused-exchange context's first reader of a frame
 * also enqueues the exchange wait, as psm_copy_maps_device does).  psm_read_points: one view into HOST memory through
 * a context-owned device buffer of 12 * W * H bytes (allocated on first use), then synchronises.
 *   - PSM_EINVAL before any CUDA work, with nothing changed: a Q without a point buffer or a buffer without a Q, no view
 *     requested, which not 0 / 1, handle_missing not 0 / 1, a bad view, row_step below 12 * W, a buffer or row_step that
 *     is not a multiple of 4 bytes.
 *   - PSM_ESTATE: no selection (which = 0) or post-process (which = 1) yet, as for psm_copy_maps_device; the right view
 *     on a left-only context.  See DESIGN.md section 24. */
int psm_reproject_device(psm_ctx* ctx, int which, const double* q_left, const double* q_right, int handle_missing,
                         float* d_left, float* d_right, size_t row_step);
int psm_read_points(psm_ctx* ctx, int which, int view, const double q[16], int handle_missing, float* dst, size_t row_step);

/* Sharded stage 3a: per-pixel packed minima over this context's slices, written to DEVICE
 * buffers of H*W uint64 each:  key = (order_preserving_u32(cost) << 32) | global_d.
 * min() over ranks' keys reproduces the reference's strict-< / lowest-d tie-break. Asynchronous. */
int psm_disp_select_keys(psm_ctx* ctx, uint64_t* d_keys_left, uint64_t* d_keys_right);

/* Sharded stage 3b: reduce `nranks` gathered key planes (DEVICE, [nranks][H*W] per view) to the
 * final u8 maps in HOST memory and synchronise.  A null left map (or a null right map on a two-view context) keeps the
 * maps on the device.  Otherwise a step below a row returns PSM_EINVAL before the reduction runs, with nothing enqueued
 * and the context unchanged. */
int psm_disp_reduce_keys(psm_ctx* ctx, const uint64_t* d_gathered_left,
                         const uint64_t* d_gathered_right, int nranks,
                         uint8_t* left, size_t left_step, uint8_t* right, size_t right_step);
/* Same on a u16 context: the low 16 bits of the winning key. */
int psm_disp_reduce_keys_u16(psm_ctx* ctx, const uint64_t* d_gathered_left,
                             const uint64_t* d_gathered_right, int nranks,
                             uint16_t* left, size_t left_step, uint16_t* right, size_t right_step);

/* ---- Sharded stage 3 fused with its exchange over NVLink peer memory ------------------------------
 * Instead of "local WTA kernel, then library collectives", the min-reduction over ranks is done by two
 * kernels that read/write PEER device memory directly (reduce-scatter + all-gather, hand-rolled):
 *   psm_disp_select_keys_p2p : WTA over this rank's slices; the packed minimum of every pixel is stored
 *                              straight into the exchange block of the rank that reduces that pixel;
 *   psm_disp_reduce_p2p      : this rank reduces its pixel chunk over all ranks' minima and stores the
 *                              winning disparity into EVERY rank's result map;
 *   psm_disp_fetch_p2p       : copy this rank's (complete) result maps to host memory and synchronise; a null left
 *                              map or a step below a row (the right map's too on a two-view context) returns
 *                              PSM_EINVAL before the DONE wait is enqueued, with the context unchanged.
 * The three kernels order themselves across ranks through ARRIVE / DONE flag words in the exchange blocks
 * (release stores over NVLink, acquire loads; PSM_OPT_P2P_SYNC = 1, default): select -> reduce -> fetch can be
 * enqueued back to back on every rank without any library collective or host barrier, provided every rank runs
 * the same sequence of frames and each rank's GPU can run its kernels independently of the others (one context
 * per GPU).  With PSM_OPT_P2P_SYNC = 0 a cross-rank barrier must separate select from reduce and reduce from
 * fetch.  All launches of one context must stay on ONE stream (psm_set_stream); collectives the caller issues
 * around them must be ordered against that stream.  Every rank owns one exchange block
 * (psm_p2p_create_buffer), shared with the other per-GPU processes through CUDA IPC (psm_ipc_export /
 * psm_ipc_import).  At most 8 ranks. */
int psm_p2p_create_buffer(psm_ctx* ctx, int nranks, void** d_buffer);
int psm_ipc_export(psm_ctx* ctx, void* d_ptr, unsigned char handle_out[64]);
int psm_ipc_import(psm_ctx* ctx, const unsigned char handle[64], void** d_ptr);
/* d_buffers[r] = exchange block of rank r as seen from this process (own pointer for r == rank). */
int psm_p2p_set_peers(psm_ctx* ctx, void* const* d_buffers, int nranks, int rank);
int psm_disp_select_keys_p2p(psm_ctx* ctx);
int psm_disp_reduce_p2p(psm_ctx* ctx);
int psm_disp_fetch_p2p(psm_ctx* ctx, uint8_t* left, size_t left_step, uint8_t* right, size_t right_step);
int psm_disp_fetch_p2p_u16(psm_ctx* ctx, uint16_t* left, size_t left_step, uint16_t* right, size_t right_step);

/* Debug / parity reads (synchronising). `d` is a GLOBAL disparity index owned by this context. */
int psm_read_cost_slice(psm_ctx* ctx, int view, int d, float* dst, size_t dst_step);
int psm_write_cost_slice(psm_ctx* ctx, int view, int d, const float* src, size_t src_step);
/* plane ids: 0-2 I (split channels), 3-5 mean_I, 6-11 var_I (rr,rg,rb,gg,gb,bb), 12 x-gradient */
int psm_read_guide_plane(psm_ctx* ctx, int view, int plane, float* dst, size_t dst_step);
/* guided-filter coefficients of one raw slice (a0,a1,a2,b; each H*W floats, dense rows), computed
 * from the CURRENT content of slice d (call between psm_cost_const and psm_cost_filter). */
int psm_read_ab_slice(psm_ctx* ctx, int view, int d, float* a3, float* b);

/* Device pointers for zero-copy callers / benchmarks. what: 0 left volume, 1 right volume,
 * 2 left u8 map, 3 right u8 map, 4 / 5 post-processed left / right u8 map (uint16_t maps on a psm_create_u16 context,
 * pitch_elems = W), 6 / 7 left / right mask of the left-right check (uint8_t 0 / 1 on both map formats, pitch_elems = W;
 * NULL until a post-process has run the check).  pitch_elems receives the row pitch in elements. */
int psm_device_ptr(psm_ctx* ctx, int what, void** ptr, size_t* pitch_elems);

/* Last measured stage durations in milliseconds (cudaEvent pairs on the context stream):
 * stage 0 ingest (H2D + planar/gradient), 1 CVC, 2 CVF (guide + filter), 3 WTA, 4 CVF filter kernel only, 5 post-process
 * (left-right check and fill included).
 * Synchronises on the stage's end event. */
int psm_stage_ms(psm_ctx* ctx, int stage, float* ms);

/* Number of kernels this context launched since creation (bench.py "gpu_launches"). */
int psm_launch_count(psm_ctx* ctx, uint64_t* n);

int psm_sync(psm_ctx* ctx);

/* Human-readable text of the last error on this context (or the last creation error if ctx==NULL). */
const char* psm_last_error(psm_ctx* ctx);

/* Library build info string: version, arch, compile flags. */
const char* psm_build_info(void);

#ifdef __cplusplus
}
#endif
#endif /* PRIME_STEREO_B200_H */
