// psm_capi.cu -- the C-ABI (include/prime_stereo_b200.h) over the sm_90a kernels.
// Host logic only: context/buffer ownership, stage ordering, launches, timers.  No CPU
// compute path exists here: every stage is a CUDA kernel launch or it fails.
#include "../../include/prime_stereo_b200.h"

#include <algorithm>
#include <climits>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <map>
#include <mutex>
#include <new>
#include <type_traits>

#include <cmath>

#include "psm_cvf_stream.cuh"
#include "psm_cvf_window.cuh"
#include "psm_cvf_ref.cuh"
#include "psm_pp.cuh"
#include "psm_pp_param.cuh"
#include "psm_fgf.cuh"
#include "psm_lr.cuh"
#include "psm_speckle.cuh"
#include "psm_dcheck.cuh"
#include "psm_unique.cuh"
#include "psm_median.cuh"
#include "psm_reproject.cuh"

#ifndef PSM_BUILD_FLAGS
#define PSM_BUILD_FLAGS "unknown"
#endif

using namespace psm;

namespace {

constexpr int kNumStages = 6;  // ingest, cvc, cvf, wta, cvf-filter-kernel, post-process

thread_local char g_create_error[512] = "";  // per host thread: psm_last_error(NULL) reports the calling thread's last failed creation

// The per-pixel outputs a selection stage writes beside the maps when their option is on, and the facts every host path
// of an output reads from here: its option, the noun of its messages and its result planes per view.
enum SelOut { kOutCosts, kOutRunnerUp, kNumOuts };
struct SelOutInfo {
    int key;
    const char* option;
    const char* noun;
    int planes;
};
constexpr SelOutInfo kSelOut[kNumOuts] = {
    {PSM_OPT_COSTS, "PSM_OPT_COSTS", "costs", kCostOut},
    {PSM_OPT_RUNNER_UP, "PSM_OPT_RUNNER_UP", "runner-up", kRunnerUpOut},
};

// The post-process steps in front of the post-filter, in chain order (StereoSGBM's); kPpStep holds what each one is.
// Every step's modes are 0 (off), 1 and kPpEnd, which ends the chain after the step.
enum PpStepId { kPpUnique, kPpDcheck, kPpMedian, kPpSpeckle, kPpLr, kNumPpSteps };
constexpr int kPpEnd = 2;
static_assert(PSM_UNIQUE_OFF == 0 && PSM_DCHECK_OFF == 0 && PSM_MEDIAN_OFF == 0 && PSM_SPECKLE_OFF == 0 && PSM_LR_OFF == 0,
              "mode 0 turns a post-process step off");
static_assert(PSM_UNIQUE_ONLY == kPpEnd && PSM_DCHECK_ONLY == kPpEnd && PSM_MEDIAN_ONLY == kPpEnd &&
              PSM_SPECKLE_ONLY == kPpEnd && PSM_LR_FILL == kPpEnd, "mode 2 ends the post-process chain");

}  // namespace

struct psm_ctx {
    int W = 0, H = 0, Wp = 0, D = 0, d_begin = 0, d_count = 0, device = 0;
    // The problem's range is [d_lo, D): 0 on every context but those of psm_create_range (and their shards).  The context
    // owns [d_begin, d_begin + d_count) of it.
    int d_lo = 0;
    // the context owns the whole problem range: selection, PSM_OPT_COSTS and PSM_OPT_RUNNER_UP need no other context
    bool owns_problem() const { return d_begin == d_lo && d_count == D - d_lo; }
    size_t plane = 0;  // H * Wp
    cudaStream_t own_stream = nullptr, stream = nullptr;
    float* guide[2] = {nullptr, nullptr};   // kGuidePlanes planes per view
    float* grd[2] = {nullptr, nullptr};
    float* vol[2] = {nullptr, nullptr};     // current volumes (raw after CVC, filtered after CVF)
    float* vol_alt[2] = {nullptr, nullptr}; // the other half of the ping-pong
    void* stage_in[2] = {nullptr, nullptr}; // device staging for the interleaved upload (the set the synchronous calls use)
    void* stage_alt[2] = {nullptr, nullptr};// second staging set: psm_set_images_async uploads frame k+1 while frame k is in flight
    size_t stage_bytes = 0;                 // bytes per view of each staging set: a float frame of W x H, or more (psm_set_rectify)
    // psm_set_rectify: frames are rect_sw x rect_sh and ingest remaps each view through its maps (W x H entries each) into
    // the context's W x H; 0 x 0 = off.  A multi-device context keeps the maps on its first shard.
    int rect_sw = 0, rect_sh = 0;
    short2* rect_xy[2] = {nullptr, nullptr};
    uint16_t* rect_a[2] = {nullptr, nullptr};
    int frame_w() const { return rect_sw ? rect_sw : W; }   // the size of the frames the psm_set_images* calls take
    int frame_h() const { return rect_sw ? rect_sh : H; }
    cudaStream_t copy_stream = nullptr;     // H2D stream of every host upload
    cudaEvent_t up_done = nullptr;          // async upload finished (recorded on copy_stream)
    cudaEvent_t host_copied = nullptr;      // H2D of a synchronous host upload finished (recorded on copy_stream)
    cudaEvent_t ingest_done[2] = {nullptr, nullptr};  // ingest kernels consumed staging set k (recorded on the compute stream)
    bool ingest_done_valid[2] = {false, false};
    int stage_cur = 0;                      // staging set holding the current frame: 0 = stage_in, 1 = stage_alt
    int up_pending = 0;                     // frame format (PSM_PIX_*, kFmtYuv + PSM_YUV_* or bayer_fmt) of the pending asynchronous upload, 0 none
    uint8_t* dis[2] = {nullptr, nullptr};    // disparity maps: u8, or u16 (map_bytes = 2, psm_create_u16) behind the same pointer
    int map_bytes = 1;                       // bytes per disparity-map element
    // Fast Guided Filter branch (lazy): low-res guide planes per view, low-res coefficient scratch, up-sampling plan
    float* fgf_lo[2] = {nullptr, nullptr};
    float* fgf_mean = nullptr;
    void* fgf_plan = nullptr;               // FgfTap x[W], y[H]: INTER_LINEAR source indices and weights
    int fgf_s = 0;                          // sub-sampling rate the buffers / plan were built for
    uint8_t* dis_pp[2] = {nullptr, nullptr}; // post-processed maps (map_bytes per element)
    uint8_t* pp_tmp[2] = {nullptr, nullptr}; // per computed view, lazy: the maps between two post-process steps
    uint32_t* pp_packed = nullptr;          // packed (disparity, 6-bit colour) image of one view, lazy
    uint32_t* pp_lut = nullptr;             // weight table of the current post-filter setting (kPpMaxD2 + 1 entries), lazy
    bool pp_lut_valid = false;              // pp_lut holds the table of (pp_sigma, pp_type)
    bool have_maps = false;                 // disparity maps valid (a select / reduce stage ran)
    int* guide_flags = nullptr;             // [2] device flags: guide outside the integer-widening domain (see psm_cvf_stream.cuh)
    unsigned char* p2p_own = nullptr;       // own exchange block (P2pLayout): keys, maps and flag words of both views
    unsigned char* p2p_peer[kMaxRanks] = {};// every rank's exchange block as mapped here
    void* p2p_imported[kMaxRanks] = {};     // IPC mappings to close at destroy
    int p2p_nimported = 0, p2p_nranks = 0, p2p_rank = 0;
    unsigned* p2p_counter = nullptr;        // device-local CTA counter of the publishing kernels
    unsigned p2p_seq = 0;                   // frame sequence number of the device-side exchange flags
    unsigned p2p_waited_seq = 0;            // last sequence number whose DONE flags a wait kernel was enqueued for
    int p2p_sync = 1;                       // 1: device-side ARRIVE/DONE flags; 0: the caller separates the kernels by its own barriers
    float* alloc[16] = {};                  // raw cudaMalloc pointers behind the halo-offset pointers above
    int nalloc = 0;
    int* slice_flags = nullptr;             // [2][res.count] device flags: slices the reference-order pass filters again
    bool slices_flagged = false;            // some slice flag is set (psm_write_cost_slice found a special cost)
    bool float_images = false;              // the current images came in as floats: the ingest flags may be set
    double* ref_rs = nullptr;               // reference-order scratch (psm_cvf_ref.cuh): [4][H][W] row sums, lazy
    float* ref_pl = nullptr;                // ... and [4][H][W] float planes
    int ref_blocks = 0;                     // grid of the cooperative reference-order kernels
    cudaEvent_t ev0[kNumStages] = {}, ev1[kNumStages] = {};
    bool ev_valid[kNumStages] = {};
    int cvf_mode = PSM_CVF_EXACT, gray_mode = 0, timing = 1, cvf_variant = 0, cvf_target_rows = 0, cvf_extra_smem = 0, cvf_threads = 0, cvf_remap = 0, cvf_no_pack = 0, cvc_variant = 0, guide_seg_rows = 0, cvc_chunk = 0;
    bool have_images = false, guide_valid = false, have_cvc = false, filtered = false;
    int gif_win = kBoxK;                    // guided-filter window (GIF_R_WIN) and regulariser (GIF_EPS), psm_set_guided_filter
    float gif_eps = kGifEps;
    bool gif_default() const { return gif_win == kBoxK && gif_eps == kGifEps; }
    CvcCost cost = {0.9f, INFINITY, INFINITY};   // matching cost (ALPHA_32F, TAU_1_32F, TAU_2_32F), psm_set_matching_cost
    bool cost_default() const { return cost.alpha == 0.9f && cost.tau_color == INFINITY && cost.tau_grad == INFINITY; }
    int pp_radius = kPpRadius;              // post-filter (JointWMF::filter's r, sigma, iter, weightType), psm_set_post_filter
    float pp_sigma = 25.5f;
    int pp_iter = 1, pp_type = PSM_WMF_EXP;
    bool pp_tuned() const { return pp_radius == kPpRadius && pp_sigma == 25.5f && pp_type == PSM_WMF_EXP; }   // any pp_iter
    // the post-process steps' settings by PpStepId: the mode and the arguments of the step's psm_set_* call (uniqueness
    // ratio 10, disparity check max_diff 1, median ksize 3, speckle max_size and max_diff 0)
    struct PpSetting { int mode, a, b; } pp_steps[kNumPpSteps] = {{0, 10, 0}, {0, 1, 0}, {0, 3, 0}, {0, 0, 0}, {0, 0, 0}};
    uint8_t* lr_valid[2] = {nullptr, nullptr};  // the left-right check's masks (W x H, 0/1), lazy
    bool lr_masks_ok = false;               // lr_valid holds the masks of the current maps (psm_read_valid_mask)
    int* sp_lab = nullptr;                  // speckle removal's labels and counts: 2 x W x H each (view v at v * W * H), lazy
    int* sp_cnt = nullptr;
    unsigned long long* dc_claims[2] = {nullptr, nullptr};  // W > kDcStageCols: the claim words, W x H per computed view, lazy
    // psm_create_blocked: the volumes hold blk_slices slices; the filter stages walk [d_begin, d_begin + d_count) in
    // blocks of that many and fold each into the running keys.  0 = unblocked (the volumes hold every owned slice).
    int blk_slices = 0;
    // The global slices [begin, begin + count) the volumes and the per-slice scratch hold, which every launcher works on:
    // the owned range on an unblocked context; on a blocked one nothing before psm_cost_const, then its first block,
    // each block in turn during a filter stage's walk and the last block after it.
    struct Slices { int begin, count; } res = {0, 0};
    unsigned long long* run_keys[2] = {nullptr, nullptr};  // blocked: running (cost, d) keys per view, [H][W]
    int vol_slices() const { return blk_slices ? blk_slices : d_count; }   // slices the volumes and per-slice scratch hold
    // psm_create_multi: the context drives nshards shard contexts (shard k on its own device, owning the slices
    // shard_range(D, nshards, k)) through the fused exchange, ordered by these events; every other context has none
    int nshards = 0;
    psm_ctx* shard[kMaxRanks] = {};
    cudaEvent_t ev_scattered[kMaxRanks] = {};  // shard k's scatter of the current frame (on its stream)
    cudaEvent_t ev_reduced[kMaxRanks] = {};    // shard k's reduce of the last frame (on its stream)
    bool reduced_valid = false;
    cudaEvent_t ev_copied[kMaxRanks] = {};     // shard k (k >= 1) has read the frame it receives from the first shard
    cudaEvent_t ev_written[kMaxRanks] = {};    // shard k's writes of the enabled outputs of the current frame (on its stream)
    cudaEvent_t ev_images = nullptr;           // psm_set_images_device: the caller's images as the first shard's stream sees them
    // PSM_OPT_VIEWS: 2 (both views) or 1 (the left view alone: the right view's guide, volume, selection and post-filter
    // are skipped).  stages_reset: PSM_OPT_VIEWS, PSM_OPT_COSTS or PSM_OPT_RUNNER_UP changed since the last psm_cost_const,
    // so the volumes, maps, masks, costs and runner-up are stale.
    int views = 2;
    bool stages_reset = false;
    // One per output (kSelOut): on = 1 while the selection stages also write it into planes[view] (its result planes; a
    // multi-device context's shards write the first shard's, the others have none), allocated when the option is turned
    // on.  have: the last selection stage since the last reset wrote them.
    struct OutState {
        int on = 0;
        bool have = false;
        float* planes[2] = {nullptr, nullptr};
    } outs[kNumOuts];
    bool outs_on() const { return std::any_of(outs, outs + kNumOuts, [](const OutState& o) { return o.on; }); }
    // PSM_OPT_COSTS: a blocked walk tracks the costs in track[view] (track_planes(); kCostFirst only where a neighbour
    // shard below reads it)
    float* track[2] = {nullptr, nullptr};
    int track_planes() const { return d_begin > d_lo ? kCostFirst + 1 : kCostLast + 1; }
    // PSM_OPT_RUNNER_UP: a blocked walk keeps the running list in ru_list[view] (kListPlanes), and a multi-device
    // context's first shard reduces its shards' picks from ru_slots[view]
    float* ru_list[2] = {nullptr, nullptr};
    unsigned char* ru_slots[2] = {nullptr, nullptr};
    unsigned p2p_seq_right = 0;                // frames whose exchange included the right view (p2p_seq counts every frame)
    bool p2p_right_current = false;            // the last frame's exchange included the right view
    bool have_pp = false;                      // dis_pp holds the maps of a post-process since the last PSM_OPT_VIEWS change
    unsigned* rp_min = nullptr;                // psm_reproject_device with handle_missing: each requested map's minimum, lazy
    float* rp_buf = nullptr;                   // psm_read_points: one view's points (12 * W * H bytes), lazy
    cudaEvent_t ev_user = nullptr;             // psm_wait_stream: the caller's stream, recorded
    cudaEvent_t ev_signal[2] = {nullptr, nullptr};  // psm_signal_stream: the compute and the copy stream, recorded
    uint64_t launches = 0;
    char err[512] = "";
};

namespace {

int fail(psm_ctx* c, int code, const char* fmt, ...)
{
    char* dst = c ? c->err : g_create_error;
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(dst, 512, fmt, ap);
    va_end(ap);
    return code;
}

#define PSM_CUDA(c, call)                                                                          \
    do {                                                                                           \
        cudaError_t e__ = (call);                                                                  \
        if (e__ != cudaSuccess)                                                                    \
            return fail((c), PSM_ECUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__),   \
                        __FILE__, __LINE__);                                                       \
    } while (0)

#define PSM_LAUNCH_CHECK(c)                                                                        \
    do {                                                                                           \
        (c)->launches++;                                                                           \
        PSM_CUDA((c), cudaGetLastError());                                                         \
    } while (0)

// Make `bytes` of dynamic shared memory launchable for `kern` on `device` (the current device).  The limit is one value per
// kernel per device for the whole process, and setting it then launching is not atomic: a context that lowered it
// between another thread's set and launch would make that launch fail.  So the limit only ever goes up: a size at or
// below the one already set is a no-op, and the record moves only once the runtime has accepted the new size.
cudaError_t raise_smem_limit(const void* kern, size_t bytes, int device)
{
    static std::mutex mu;
    static std::map<std::pair<int, const void*>, size_t> limit;
    std::lock_guard<std::mutex> lock(mu);
    size_t& have = limit[{device, kern}];
    if (bytes <= have) return cudaSuccess;
    const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) have = bytes;
    return e;
}

template <typename K>
cudaError_t raise_smem_limit(K* kern, size_t bytes, int device)
{
    return raise_smem_limit(reinterpret_cast<const void*>(kern), bytes, device);
}

// cudaMalloc into p while it is null; p stays null unless the allocation succeeds
template <typename T>
cudaError_t alloc_if_null(T*& p, size_t bytes)
{
    if (p) return cudaSuccess;
    void* q = nullptr;
    const cudaError_t e = cudaMalloc(&q, bytes);
    if (e == cudaSuccess) p = static_cast<T*>(q);
    return e;
}

int bind(psm_ctx* c)
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    PSM_CUDA(c, cudaSetDevice(c->device));
    return PSM_OK;
}

// a call that would read or return right-view data: PSM_ESTATE on a left-only context, and after a PSM_OPT_VIEWS,
// PSM_OPT_COSTS or PSM_OPT_RUNNER_UP change
// until psm_cost_const has built the current frame's volumes again
int check_right_view(psm_ctx* c, const char* call)
{
    if (c->views == 1)
        return fail(c, PSM_ESTATE, "%s of the right view on a left-only context (PSM_OPT_VIEWS = PSM_VIEWS_LEFT): the right "
                    "view is not computed; set PSM_VIEWS_BOTH", call);
    if (c->stages_reset)
        return fail(c, PSM_ESTATE, "%s of the right view after a PSM_OPT_VIEWS, PSM_OPT_COSTS or PSM_OPT_RUNNER_UP change: "
                    "call psm_cost_const first", call);
    return PSM_OK;
}

// a right-view output of a selection / map call: must be NULL on a left-only context, and is required otherwise
int check_right_arg(psm_ctx* c, const void* right, const char* call)
{
    if (c->views == 1 && right)
        return fail(c, PSM_EINVAL, "%s: the right map / key buffer must be NULL on a left-only context "
                    "(PSM_OPT_VIEWS = PSM_VIEWS_LEFT)", call);
    return PSM_OK;
}

// a stage that needs the stage state a PSM_OPT_VIEWS, PSM_OPT_COSTS or PSM_OPT_RUNNER_UP change reset
int check_stages_reset(psm_ctx* c, const char* call)
{
    if (c->stages_reset)
        return fail(c, PSM_ESTATE, "%s after a PSM_OPT_VIEWS, PSM_OPT_COSTS or PSM_OPT_RUNNER_UP change: the next stage must "
                    "be psm_cost_const", call);
    return PSM_OK;
}

int stage_begin(psm_ctx* c, int s)
{
    if (c->timing) PSM_CUDA(c, cudaEventRecord(c->ev0[s], c->stream));
    return PSM_OK;
}
int stage_end(psm_ctx* c, int s)
{
    if (c->timing) { PSM_CUDA(c, cudaEventRecord(c->ev1[s], c->stream)); c->ev_valid[s] = true; }
    return PSM_OK;
}

// mirror the column halos of `nrows` rows starting at `base` (pointer to row 0, column 0)
int pad_rows(psm_ctx* c, float* base, size_t nrows)
{
    const unsigned blocks = (unsigned)((nrows + 7) / 8);
    pad_cols_kernel<<<blocks, 256, 0, c->stream>>>(base, nrows, c->W, c->Wp);
    PSM_LAUNCH_CHECK(c);
    return PSM_OK;
}

void* stage_buf(psm_ctx* c, int set, int view) { return set ? c->stage_alt[view] : c->stage_in[view]; }

// a new frame's planes are (being) written: every stage after ingest starts again
void images_ingested(psm_ctx* c, bool float_images)
{
    c->have_images = true;
    c->float_images = float_images;   // u8 images lie in {0} U [1/255, 1]: they never raise an ingest flag
    c->guide_valid = false;
    c->have_cvc = false;
    c->filtered = false;
}

size_t pix_bytes(int pix) { return pix == PSM_PIX_U8 ? 1 : sizeof(float); }

// A host frame's format: PSM_PIX_U8 or PSM_PIX_F32 for interleaved BGR, kFmtYuv + PSM_YUV_* for a YUV frame in cv2's
// contiguous layout (psm_set_images_yuv), bayer_fmt(PSM_BAYER_*, PSM_DEMOSAIC_*) for a Bayer frame
// (psm_set_images_bayer).  Uploads, staging sets and the asynchronous commit go by it.
constexpr int kFmtYuv = 16, kFmtBayer = 32;
bool is_yuv(int fmt) { return fmt > kFmtYuv && fmt < kFmtBayer; }
int yuv_vs(int format) { return format <= PSM_YUV_YV12 ? 1 : 0; }   // the chroma row shift: 1 for 4:2:0, 0 for 4:2:2
int bayer_fmt(int pattern, int method) { return kFmtBayer | (method & 3) << 3 | (pattern & 7); }
bool is_bayer(int fmt) { return fmt > kFmtBayer; }

// bytes of one row, and rows, of a host frame of format fmt as the staging sets hold it
size_t host_row_bytes(psm_ctx* c, int fmt)
{
    if (is_yuv(fmt)) return (size_t)c->frame_w() * (yuv_vs(fmt - kFmtYuv) ? 1 : 2);
    if (is_bayer(fmt)) return (size_t)c->frame_w();
    return (size_t)c->frame_w() * 3 * pix_bytes(fmt);
}
int host_rows(psm_ctx* c, int fmt) { return is_yuv(fmt) && yuv_vs(fmt - kFmtYuv) ? c->frame_h() / 2 * 3 : c->frame_h(); }

// the YuvSrc of a YUV frame of format PSM_YUV_* in cv2's layout at p, rows `step` bytes apart, of the context's frame
// size: 4:2:0 frames are the luma rows followed by the chroma (NV12 / NV21: interleaved U, V rows of `step` bytes; I420 /
// YV12: two planes of Wf / 2 x Hf / 2, step == Wf), 4:2:2 frames rows of packed pairs (YUYV: Y0 U Y1 V)
YuvSrc yuv_host_src(psm_ctx* c, int format, const void* p, size_t step)
{
    const char* b = static_cast<const char*>(p);
    const char* uv = b + (size_t)c->frame_h() * step;
    const size_t cw = (size_t)c->frame_w() / 2, q = cw * (c->frame_h() / 2);
    switch (format) {
    case PSM_YUV_NV12: return YuvSrc{{b, uv, uv + 1}, step, 1, step, 2, 1};
    case PSM_YUV_NV21: return YuvSrc{{b, uv + 1, uv}, step, 1, step, 2, 1};
    case PSM_YUV_I420: return YuvSrc{{b, uv, uv + q}, step, 1, cw, 1, 1};
    case PSM_YUV_YV12: return YuvSrc{{b, uv + q, uv}, step, 1, cw, 1, 1};
    case PSM_YUV_YUYV: return YuvSrc{{b, b + 1, b + 3}, step, 2, step, 4, 0};
    case PSM_YUV_UYVY: return YuvSrc{{b + 1, b, b + 2}, step, 2, step, 4, 0};
    default: return YuvSrc{{b, b + 3, b + 1}, step, 2, step, 4, 0};   // PSM_YUV_YVYU
    }
}

// the BayerSrc of a checked Bayer frame of the context's frame size at p, samples col_step and rows row_step bytes apart,
// whose pixel (0, 0) has pattern PSM_BAYER_*'s first colour
BayerSrc bayer_src(psm_ctx* c, int pattern, int method, const void* p, size_t row_step, size_t col_step)
{
    const int rx = pattern == PSM_BAYER_BGGR || pattern == PSM_BAYER_GRBG;
    const int ry = pattern == PSM_BAYER_BGGR || pattern == PSM_BAYER_GBRG;
    return BayerSrc{static_cast<const char*>(p), row_step, col_step, c->frame_w(), c->frame_h(), rx, ry,
                    method == PSM_DEMOSAIC_EA};
}

// the frame's planes, gradients and ingest flags: one ingest_kernel launch and one pad_rows per view on the context's
// stream.  With psm_set_rectify on, the frame (u8, YUV or Bayer, checked by the caller) is read through each view's maps.
template <typename T, class Src>
int ingest(psm_ctx* c, const Src src[2])
{
    PSM_CUDA(c, cudaMemsetAsync(c->guide_flags, 0, 2 * sizeof(int), c->stream));
    for (int v = 0; v < 2; ++v) {
        float* g = c->guide[v];
        dim3 blk(128), grd((c->W + 3 + 127) / 128, c->H);
        auto launch = [&](auto k, const auto& s) {
            k<<<grd, blk, 0, c->stream>>>(s, c->W, c->H, c->Wp, g, g + c->plane, g + 2 * c->plane, c->grd[v], c->gray_mode,
                                          c->guide_flags + v);
        };
        if (c->rect_sw)
            launch(ingest_kernel<uint8_t, RectifySrc<Src>>,
                   RectifySrc<Src>{src[v], c->rect_xy[v], c->rect_a[v], c->rect_sw, c->rect_sh, c->W});
        else
            launch(ingest_kernel<T, Src>, src[v]);
        PSM_LAUNCH_CHECK(c);
        if (int rc = pad_rows(c, g, (size_t)3 * c->H)) return rc;  // mirrored halo of the 3 guide channels
    }
    images_ingested(c, !std::is_same<T, uint8_t>::value);
    return PSM_OK;
}

int ingest(psm_ctx* c, int pix, const PlanesSrc src[2])
{
    return pix == PSM_PIX_U8 ? ingest<uint8_t>(c, src) : ingest<float>(c, src);
}

// Copy a checked host frame of format fmt (src[v].ch[0] its first byte, src[v].row_step its row step) into staging set
// `set` on the copy stream and record `done` there.  The copy starts once the last ingest from that set has read it, so
// that it does not queue behind the compute stream's backlog.
int upload(psm_ctx* c, int set, int fmt, const PlanesSrc src[2], cudaEvent_t done)
{
    const size_t row_bytes = host_row_bytes(c, fmt);
    if (c->ingest_done_valid[set]) PSM_CUDA(c, cudaStreamWaitEvent(c->copy_stream, c->ingest_done[set], 0));
    for (int v = 0; v < 2; ++v)
        PSM_CUDA(c, cudaMemcpy2DAsync(stage_buf(c, set, v), row_bytes, src[v].ch[0], src[v].row_step, row_bytes,
                                      host_rows(c, fmt), cudaMemcpyHostToDevice, c->copy_stream));
    PSM_CUDA(c, cudaEventRecord(done, c->copy_stream));
    return PSM_OK;
}

// ingest staging set `set`, which holds a frame of format fmt, once the copy that filled it (`copied`) is done; the next
// copy into the set waits for this
int ingest_staged(psm_ctx* c, int set, int fmt, cudaEvent_t copied)
{
    PSM_CUDA(c, cudaStreamWaitEvent(c->stream, copied, 0));
    const size_t row_bytes = host_row_bytes(c, fmt);
    if (is_yuv(fmt)) {
        const YuvSrc src[2] = {yuv_host_src(c, fmt - kFmtYuv, stage_buf(c, set, 0), row_bytes),
                               yuv_host_src(c, fmt - kFmtYuv, stage_buf(c, set, 1), row_bytes)};
        if (int rc = ingest<uint8_t>(c, src)) return rc;
    } else if (is_bayer(fmt)) {
        const int pattern = fmt & 7, method = fmt >> 3 & 3;
        const BayerSrc src[2] = {bayer_src(c, pattern, method, stage_buf(c, set, 0), row_bytes, 1),
                                 bayer_src(c, pattern, method, stage_buf(c, set, 1), row_bytes, 1)};
        if (int rc = ingest<uint8_t>(c, src)) return rc;
    } else {
        const size_t elem = pix_bytes(fmt);
        const PlanesSrc src[2] = {interleaved_src(stage_buf(c, set, 0), elem, row_bytes),
                                  interleaved_src(stage_buf(c, set, 1), elem, row_bytes)};
        if (int rc = ingest(c, fmt, src)) return rc;
    }
    PSM_CUDA(c, cudaEventRecord(c->ingest_done[set], c->stream));
    c->ingest_done_valid[set] = true;
    return PSM_OK;
}

// a frame of pixel type pix while psm_set_rectify is on: the maps remap 8-bit frames alone
int check_rectify_pix(psm_ctx* c, int pix)
{
    if (c->rect_sw && pix != PSM_PIX_U8)
        return fail(c, PSM_EINVAL, "float frame on a context that rectifies (psm_set_rectify): rectification reads 8-bit "
                    "frames only, as OpenCV's remap of the camera frame does; pass the u8 frame, or turn it off");
    return PSM_OK;
}

// psm_set_images[_u8|_device][_async]: two interleaved BGR frames -> src, or PSM_EINVAL before any CUDA call.  The
// kernel reads a device frame in place with loads of whole samples, so its pointers and steps are multiples of a sample.
int check_interleaved(psm_ctx* c, int pix, bool device, const void* l, size_t lstep, const void* r, size_t rstep,
                      PlanesSrc src[2])
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    if (int rc = check_rectify_pix(c, pix)) return rc;
    const void* p[2] = {l, r};
    const size_t step[2] = {lstep, rstep};
    const size_t elem = pix_bytes(pix);
    for (int v = 0; v < 2; ++v) {
        if (!p[v] || step[v] < (size_t)c->frame_w() * 3 * elem)
            return fail(c, PSM_EINVAL, "bad image pointer/step for view %d", v);
        if (device && ((uintptr_t)p[v] % elem || step[v] % elem))
            return fail(c, PSM_EINVAL, "pointer or step %zu of view %d is not a multiple of the %zu bytes of a float sample",
                        step[v], v, elem);
        src[v] = interleaved_src(p[v], elem, step[v]);
    }
    return PSM_OK;
}

// psm_set_images_device_planes: the caller's two frames and their layout -> src, or PSM_EINVAL before any CUDA call
int check_planes(psm_ctx* c, int pix_type, const void* const left[3], const void* const right[3], size_t row_step,
                 size_t col_step, PlanesSrc src[2])
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    if (pix_type != PSM_PIX_U8 && pix_type != PSM_PIX_F32)
        return fail(c, PSM_EINVAL, "unknown pixel type %d (PSM_PIX_U8 = 1, PSM_PIX_F32 = 2)", pix_type);
    if (int rc = check_rectify_pix(c, pix_type)) return rc;
    const size_t elem = pix_bytes(pix_type);
    const void* const* ch[2] = {left, right};
    for (int v = 0; v < 2; ++v) {
        if (!ch[v]) return fail(c, PSM_EINVAL, "null channel pointer array for view %d", v);
        for (int k = 0; k < 3; ++k) {
            if (!ch[v][k]) return fail(c, PSM_EINVAL, "null pointer for channel %d of view %d", k, v);
            if ((uintptr_t)ch[v][k] % elem)
                return fail(c, PSM_EINVAL, "channel %d of view %d is not aligned to the %zu bytes of a float sample", k, v, elem);
            src[v].ch[k] = static_cast<const char*>(ch[v][k]);
        }
        src[v].row_step = row_step;
        src[v].col_step = col_step;
    }
    if (col_step < elem) return fail(c, PSM_EINVAL, "col_step %zu is below the %zu bytes of one sample", col_step, elem);
    const size_t span = (size_t)(c->frame_w() - 1);
    if ((span && col_step > (SIZE_MAX - elem) / span) || row_step < span * col_step + elem)
        return fail(c, PSM_EINVAL, "row_step %zu is below the (W - 1) * col_step + %zu bytes a row of W = %d spans", row_step,
                    elem, c->frame_w());
    if (row_step % elem || col_step % elem)
        return fail(c, PSM_EINVAL, "row_step %zu / col_step %zu are not multiples of the %zu bytes of a float sample",
                    row_step, col_step, elem);
    return PSM_OK;
}

// a YUV frame of the context's frame size with chroma rows y >> vs: cv2 converts even widths, and even heights for 4:2:0
int check_yuv_size(psm_ctx* c, int vs)
{
    if (c->frame_w() % 2 || (vs && c->frame_h() % 2))
        return fail(c, PSM_EINVAL, "YUV frame of %d x %d: the width must be even%s", c->frame_w(), c->frame_h(),
                    vs ? ", and the height too for 4:2:0" : "");
    return PSM_OK;
}

// psm_set_images_yuv[_async]: two host frames of format PSM_YUV_* -> src (ch[0] and row_step, as upload reads them), or
// PSM_EINVAL before any CUDA call
int check_yuv_host(psm_ctx* c, int format, const void* l, size_t lstep, const void* r, size_t rstep, PlanesSrc src[2])
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    if (format < PSM_YUV_NV12 || format > PSM_YUV_YVYU)
        return fail(c, PSM_EINVAL, "unknown YUV format %d (PSM_YUV_NV12 = 1 .. PSM_YUV_YVYU = 7)", format);
    if (int rc = check_yuv_size(c, yuv_vs(format))) return rc;
    const void* p[2] = {l, r};
    const size_t step[2] = {lstep, rstep};
    const size_t row = host_row_bytes(c, kFmtYuv + format);
    const bool planar = format == PSM_YUV_I420 || format == PSM_YUV_YV12;
    for (int v = 0; v < 2; ++v) {
        if (!p[v]) return fail(c, PSM_EINVAL, "null frame pointer for view %d", v);
        if (step[v] < row) return fail(c, PSM_EINVAL, "step %zu of view %d is below the %zu bytes of a row", step[v], v, row);
        if (planar && step[v] != row)
            return fail(c, PSM_EINVAL, "step %zu of view %d: I420 / YV12 frames are contiguous (step == width %zu)", step[v],
                        v, row);
        src[v] = PlanesSrc{{static_cast<const char*>(p[v]), nullptr, nullptr}, step[v], 0};
    }
    return PSM_OK;
}

// psm_set_images_device_yuv: the caller's two frames and their layout -> src, or PSM_EINVAL before any CUDA call
int check_yuv_device(psm_ctx* c, int sampling, const void* const left[3], const void* const right[3], size_t y_row_step,
                     size_t y_col_step, size_t c_row_step, size_t c_col_step, YuvSrc src[2])
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    if (sampling != PSM_YUV_420 && sampling != PSM_YUV_422)
        return fail(c, PSM_EINVAL, "unknown YUV sampling %d (PSM_YUV_420 = 1, PSM_YUV_422 = 2)", sampling);
    const int vs = sampling == PSM_YUV_420;
    if (int rc = check_yuv_size(c, vs)) return rc;
    const void* const* p[2] = {left, right};
    for (int v = 0; v < 2; ++v) {
        if (!p[v]) return fail(c, PSM_EINVAL, "null Y, U, V pointer array for view %d", v);
        for (int k = 0; k < 3; ++k)
            if (!p[v][k]) return fail(c, PSM_EINVAL, "null %c pointer of view %d", "YUV"[k], v);
        src[v] = YuvSrc{{static_cast<const char*>(p[v][0]), static_cast<const char*>(p[v][1]),
                         static_cast<const char*>(p[v][2])}, y_row_step, y_col_step, c_row_step, c_col_step, vs};
    }
    // a row of n samples col_step apart spans (n - 1) * col_step + 1 bytes
    auto short_row = [](size_t row_step, size_t col_step, size_t n) {
        return !col_step || (n > 1 && col_step > (SIZE_MAX - 1) / (n - 1)) || row_step < (n - 1) * col_step + 1;
    };
    if (short_row(y_row_step, y_col_step, c->frame_w()))
        return fail(c, PSM_EINVAL, "y_row_step %zu / y_col_step %zu: the column step must be nonzero and a row of %d luma "
                    "samples fit in the row step", y_row_step, y_col_step, c->frame_w());
    if (short_row(c_row_step, c_col_step, c->frame_w() / 2))
        return fail(c, PSM_EINVAL, "c_row_step %zu / c_col_step %zu: the column step must be nonzero and a row of %d chroma "
                    "samples fit in the row step", c_row_step, c_col_step, c->frame_w() / 2);
    return PSM_OK;
}

// a Bayer pattern and demosaicing method, or PSM_EINVAL
int check_bayer_kind(psm_ctx* c, int pattern, int method)
{
    if (pattern < PSM_BAYER_RGGB || pattern > PSM_BAYER_GBRG)
        return fail(c, PSM_EINVAL, "unknown Bayer pattern %d (PSM_BAYER_RGGB = 1 .. PSM_BAYER_GBRG = 4)", pattern);
    if (method != PSM_DEMOSAIC_BILINEAR && method != PSM_DEMOSAIC_EA)
        return fail(c, PSM_EINVAL, "unknown demosaicing method %d (PSM_DEMOSAIC_BILINEAR = 1, PSM_DEMOSAIC_EA = 2)", method);
    return PSM_OK;
}

// psm_set_images_bayer[_async]: two host frames -> src (ch[0] and row_step, as upload reads them), or PSM_EINVAL before
// any CUDA call
int check_bayer_host(psm_ctx* c, int pattern, int method, const void* l, size_t lstep, const void* r, size_t rstep,
                     PlanesSrc src[2])
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    if (int rc = check_bayer_kind(c, pattern, method)) return rc;
    const void* p[2] = {l, r};
    const size_t step[2] = {lstep, rstep};
    for (int v = 0; v < 2; ++v) {
        if (!p[v]) return fail(c, PSM_EINVAL, "null frame pointer for view %d", v);
        if (step[v] < (size_t)c->frame_w())
            return fail(c, PSM_EINVAL, "step %zu of view %d is below the %d bytes of a row", step[v], v, c->frame_w());
        src[v] = PlanesSrc{{static_cast<const char*>(p[v]), nullptr, nullptr}, step[v], 0};
    }
    return PSM_OK;
}

// psm_set_images_device_bayer: the caller's two frames and their layout -> src, or PSM_EINVAL before any CUDA call
int check_bayer_device(psm_ctx* c, int pattern, int method, const void* left, const void* right, size_t row_step,
                       size_t col_step, BayerSrc src[2])
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    if (int rc = check_bayer_kind(c, pattern, method)) return rc;
    if (!left || !right) return fail(c, PSM_EINVAL, "null frame pointer for view %d", left ? 1 : 0);
    // a row of Wf samples col_step apart spans (Wf - 1) * col_step + 1 bytes
    const size_t span = (size_t)(c->frame_w() - 1);
    if (!col_step || (span && col_step > (SIZE_MAX - 1) / span) || row_step < span * col_step + 1)
        return fail(c, PSM_EINVAL, "row_step %zu / col_step %zu: the column step must be nonzero and a row of %d samples "
                    "fit in the row step", row_step, col_step, c->frame_w());
    src[0] = bayer_src(c, pattern, method, left, row_step, col_step);
    src[1] = bayer_src(c, pattern, method, right, row_step, col_step);
    return PSM_OK;
}

// how a checked frame reaches the context: host buffers through a staging set, or device memory read in place
enum class Frame { host, device, planes };

// stage 0 of one context.  A host frame is copied into the current staging set and ingested from there; the call returns
// once the copy has read the caller's buffers (from page-locked memory it would otherwise still be reading them after the
// return).  A device frame is ingested in place.
int set_images_one(psm_ctx* c, Frame kind, int fmt, const PlanesSrc src[2])
{
    if (int rc = bind(c)) return rc;
    if (int rc = stage_begin(c, 0)) return rc;
    if (kind == Frame::host) {
        if (int rc = upload(c, c->stage_cur, fmt, src, c->host_copied)) return rc;
        if (int rc = ingest_staged(c, c->stage_cur, fmt, c->host_copied)) return rc;
        PSM_CUDA(c, cudaEventSynchronize(c->host_copied));
    } else if (int rc = ingest(c, fmt, src)) {
        return rc;
    }
    return stage_end(c, 0);
}

int launch_guide(psm_ctx* c);

// the raw volumes were replaced or filtered: no slice is flagged any more
int clear_slice_flags(psm_ctx* c)
{
    if (!c->slices_flagged) return PSM_OK;
    PSM_CUDA(c, cudaMemsetAsync(c->slice_flags, 0, 2 * (size_t)c->vol_slices() * sizeof(int), c->stream));
    c->slices_flagged = false;
    return PSM_OK;
}

// The cooperative reference-order kernels (psm_cvf_ref.cuh): scratch of one slice (48 bytes per pixel, allocated on the
// first launch) and a grid that fits on the device at once.
int launch_ref(psm_ctx* c, void* kernel, int mode, int one_view = 0, int one_d = 0)
{
    const size_t n = (size_t)c->W * c->H;
    PSM_CUDA(c, alloc_if_null(c->ref_rs, 4 * n * sizeof(double)));
    PSM_CUDA(c, alloc_if_null(c->ref_pl, 4 * n * sizeof(float)));
    if (c->ref_blocks == 0) {
        int nsm = 0, per_sm = 0;
        PSM_CUDA(c, cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, c->device));
        PSM_CUDA(c, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, cvf_ref_kernel, kRefThreads, 0));
        int per_sm_g = 0;
        PSM_CUDA(c, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_g, guide_ref_kernel, kRefThreads, 0));
        c->ref_blocks = nsm * std::min(2, std::min(per_sm, per_sm_g));
    }
    RefParams P;
    for (int v = 0; v < 2; ++v) { P.vol_in[v] = c->vol[v]; P.vol_out[v] = c->vol_alt[v]; P.guide[v] = c->guide[v]; }
    P.guide_flags = c->guide_flags;
    P.slice_flags = c->slice_flags;
    P.rs = c->ref_rs; P.pl = c->ref_pl;
    P.W = c->W; P.H = c->H; P.Wp = c->Wp; P.Dloc = c->res.count;
    P.K = c->gif_win; P.a = c->gif_win / 2;
    P.scale = 1.0 / ((double)P.K * P.K);
    P.eps = c->gif_eps;
    P.mode = mode; P.one_view = one_view; P.one_d = one_d;
    P.nviews = c->views;
    void* args[] = {&P};
    PSM_CUDA(c, cudaLaunchCooperativeKernel(kernel, dim3(c->ref_blocks), dim3(kRefThreads), args, 0, c->stream));
    PSM_LAUNCH_CHECK(c);
    return PSM_OK;
}

int ensure_guide(psm_ctx* c)
{
    if (c->guide_valid) return PSM_OK;
    if (int rc = launch_guide(c)) return rc;
    // a view whose ingest found values outside {0} U [2^-12, 1] gets its guide again in OpenCV's order (the kernel
    // leaves at once when no view is flagged; u8 images never are)
    if (c->float_images)
        if (int rc = launch_ref(c, (void*)guide_ref_kernel, kRefFlagged)) return rc;
    c->guide_valid = true;
    return PSM_OK;
}

int launch_guide(psm_ctx* c)
{
    if (!c->gif_default()) {   // any other window / eps: the generic precompute (psm_cvf_window.cuh)
        WinGuideParams P;
        P.guide[0] = c->guide[0]; P.guide[1] = c->guide[1];
        P.guide_flags = c->guide_flags;
        P.W = c->W; P.H = c->H; P.Wp = c->Wp; P.K = c->gif_win; P.a = c->gif_win / 2;
        P.seg_rows = kWinGuideSegRows;
        P.scale = 1.0 / ((double)P.K * P.K);
        P.eps = c->gif_eps;
        dim3 grd((c->W + 127) / 128, (c->H + P.seg_rows - 1) / P.seg_rows, c->views);
        guide_window_kernel<<<grd, 128, 0, c->stream>>>(P);
        PSM_LAUNCH_CHECK(c);
        return PSM_OK;
    }
    GuideParams P;
    P.guide[0] = c->guide[0]; P.guide[1] = c->guide[1];
    P.guide_flags = c->guide_flags;
    P.W = c->W; P.H = c->H; P.Wp = c->Wp;
    P.nstrips = (c->W + kGuideStripOut - 1) / kGuideStripOut;
    P.seg_rows = c->guide_seg_rows > 0 ? c->guide_seg_rows : kGuideSegRows;   // option 107 (tuning)
    P.nseg = (c->H + P.seg_rows - 1) / P.seg_rows;
    const int tasks = c->views * P.nstrips * P.nseg;  // one warp each
    if (c->views == 2)
        guide_kernel<<<(tasks + 3) / 4, 128, 0, c->stream>>>(P);
    else   // one warp per CTA: a spare warp of the last CTA would take a right-view task
        guide_kernel<<<tasks, 32, 0, c->stream>>>(P);
    PSM_LAUNCH_CHECK(c);
    return PSM_OK;
}

// FastGuidedFilter(img, r = GIF_R_WIN, eps = GIF_EPS, s) (DispEst.cpp:283-284) at rate s: box K = 2 * (r / s) + 1 at low
// resolution
FgfGeom fgf_geom(const psm_ctx* c, int s)
{
    FgfGeom g;
    g.W = c->W; g.H = c->H; g.Wp = c->Wp; g.s = s; g.w2 = c->W / s; g.h2 = c->H / s; g.K = 2 * (c->gif_win / s) + 1;
    g.ifx = 1.0 / ((double)g.w2 / g.W); g.ify = 1.0 / ((double)g.h2 / g.H);
    return g;
}

// The Fast Guided Filter at rate s: PSM_EINVAL for a rate it does not take; otherwise the low-resolution buffers and the
// INTER_LINEAR plan, (re)built when the rate changes
int ensure_fgf(psm_ctx* c, int s)
{
    if (s != 1 && s != 2 && s != 4 && s != 8) return fail(c, PSM_EINVAL, "sub-sampling rate must be 1, 2, 4 or 8 (got %d)", s);
    if (c->W / s < 1 || c->H / s < 1) return fail(c, PSM_EINVAL, "image smaller than the sub-sampling rate");
    const FgfGeom g = fgf_geom(c, s);
    int smem_max = 0;
    PSM_CUDA(c, cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, c->device));
    if (fgf_smem_bytes(g.K) > (size_t)smem_max)
        return fail(c, PSM_EINVAL, "Fast Guided Filter box %d (window %d, rate %d) needs %zu bytes of shared memory, more than "
                    "the %d a block may have", g.K, c->gif_win, s, fgf_smem_bytes(g.K), smem_max);
    if (c->fgf_s == s) return PSM_OK;
    const size_t n2 = (size_t)g.w2 * g.h2;
    cudaFree(c->fgf_lo[0]); cudaFree(c->fgf_lo[1]); cudaFree(c->fgf_mean); cudaFree(c->fgf_plan);
    c->fgf_lo[0] = c->fgf_lo[1] = c->fgf_mean = nullptr; c->fgf_plan = nullptr; c->fgf_s = 0;
    for (int v = 0; v < 2; ++v) PSM_CUDA(c, cudaMalloc(&c->fgf_lo[v], 12 * n2 * sizeof(float)));
    PSM_CUDA(c, cudaMalloc(&c->fgf_mean, (size_t)4 * c->vol_slices() * n2 * sizeof(float)));
    PSM_CUDA(c, cudaMalloc(&c->fgf_plan, (size_t)(c->W + c->H) * sizeof(FgfTap)));
    // cv::resize INTER_LINEAR coordinates (OpenCV's own implementation; same expressions as the CPU restatement fgf_build in oracle/)
    FgfTap* hp = new (std::nothrow) FgfTap[c->W + c->H];
    if (!hp) return fail(c, PSM_ENOMEM, "out of host memory");
    { const double sc = (double)g.w2 / g.W;
      for (int x = 0; x < c->W; ++x) {
          float f = (float)((x + 0.5) * sc - 0.5); int i = (int)floorf(f); f -= (float)i;
          if (i < 0) { f = 0.f; i = 0; }
          if (i >= g.w2 - 1) { f = 0.f; i = g.w2 - 1; }
          hp[x].i0 = i; hp[x].i1 = i + 1 < g.w2 ? i + 1 : g.w2 - 1; hp[x].f = f; hp[x].pad = 0.f; } }
    { const double sc = (double)g.h2 / g.H;
      for (int y = 0; y < c->H; ++y) {
          float f = (float)((y + 0.5) * sc - 0.5); int i = (int)floorf(f); f -= (float)i;
          FgfTap& t = hp[c->W + y];
          t.i0 = i < 0 ? 0 : (i > g.h2 - 1 ? g.h2 - 1 : i);
          t.i1 = i + 1 < 0 ? 0 : (i + 1 > g.h2 - 1 ? g.h2 - 1 : i + 1);
          t.f = f; t.pad = 0.f; } }
    // on the context's stream: a cudaMemcpy from pageable memory may return before its DMA lands, and it is not ordered
    // before the kernels of the context's non-blocking stream, which read the plan at once
    cudaError_t e = cudaMemcpyAsync(c->fgf_plan, hp, (size_t)(c->W + c->H) * sizeof(FgfTap), cudaMemcpyHostToDevice, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    delete[] hp;
    PSM_CUDA(c, e);
    c->fgf_s = s;
    return PSM_OK;
}

// The Fast Guided Filter at rate s, view by view: the view's low-resolution guide if `guide`, then the filter of its
// resident slices if `slices`
int fgf_views(psm_ctx* c, int s, bool guide, bool slices)
{
    const FgfGeom g = fgf_geom(c, s);
    FgfPlan pl;
    pl.x = static_cast<const FgfTap*>(c->fgf_plan);
    pl.y = pl.x + c->W;
    for (int v = 0; v < c->views; ++v) {
        if (guide) {
            dim3 blk(128), g2((g.w2 + 127) / 128, g.h2);
            fgf_guide_kernel<<<g2, blk, 0, c->stream>>>(c->guide[v], c->plane, g, c->gif_eps, c->fgf_lo[v]);
            PSM_LAUNCH_CHECK(c);
        }
        if (!slices) continue;
        dim3 blk(128);
        dim3 g3((g.w2 + kFgfTX - 1) / kFgfTX, (g.h2 + kFgfTY - 1) / kFgfTY, c->res.count);
        const size_t fsmem = fgf_smem_bytes(g.K);
        PSM_CUDA(c, raise_smem_limit(fgf_lowres_kernel, fsmem, c->device));
        fgf_lowres_kernel<<<g3, kFgfThreads, fsmem, c->stream>>>(c->vol[v], c->plane, g, c->fgf_lo[v], c->fgf_mean);
        PSM_LAUNCH_CHECK(c);
        dim3 g5((((c->W + 3) / 4) + 127) / 128, c->H, c->res.count);
        fgf_up_kernel<<<g5, blk, 0, c->stream>>>(c->vol[v], c->plane, c->guide[v], c->plane, g, pl, c->fgf_mean);
        PSM_LAUNCH_CHECK(c);
    }
    return PSM_OK;
}

// Row segmentation of the streaming kernel: segments are multiples of 8 rows, >= 16 rows, and the
// last one keeps >= 8 rows so that only the first/last segment ever sees a reflected row.
void plan_segments(int H, int target_rows, int* nseg, int* seg_rows)
{
    int n = H / target_rows;
    if (n < 1) n = 1;
    for (; n > 1; --n) {
        int rows = (H + n - 1) / n;
        rows = (rows + 7) & ~7;
        if (rows < 16) continue;
        const int last = H - (n - 1) * rows;
        if (last >= 8) { *nseg = n; *seg_rows = rows; return; }
    }
    *nseg = 1;
    *seg_rows = (H + 7) & ~7;
}

// The streaming kernel's work decomposition as a pure host function (no CUDA calls) so that the host logic can be
// tested without a GPU (psm_cvf_plan, tests/test_cvf_plan.py).
struct CvfPlan {
    int nthreads, nstrips, ndgroups, nseg, seg_rows;
    int pack_gl, pack_x0, pack_ndg, pack_first;
    unsigned grid;
};

// nviews: 2, or 1 for a left-only context (the grid holds the left view's CTAs alone)
CvfPlan plan_cvf(int W, int H, int d_count, int nsm, int threads_override, int target_rows, bool allow_pack, int nviews)
{
    CvfPlan q{};
    q.nstrips = (W + kStripOut - 1) / kStripOut;
    // packed remainder strips (psm_cvf_stream.cuh): the columns past the last full strip, 4 or 2 slices per warp
    const int nfull = W / kStripOut, rem = W - nfull * kStripOut;
    if (allow_pack && nfull >= 1 && rem > 0) {
        for (int gl = 8; gl <= 16; gl *= 2) {
            const int x0 = (W - 4 * (gl - 4) + 3) & ~3;
            if (x0 <= nfull * kStripOut) { q.pack_gl = gl; q.pack_x0 = x0; q.nstrips = nfull; break; }
        }
    }
    // slice-warps per CTA: 3 (4 CTAs per SM) or 4 (3 CTAs per SM) -- the same 12 warps per SM either way; take the one that
    // leaves no warp slot idle in the last slice group (16 slices per rank at 8 GPUs: 4 x 4 instead of 6 x 3 with two idle)
    const int auto_threads = (d_count % 3 != 0 && d_count % 4 == 0) ? 128 : kCvfThreads;
    q.nthreads = threads_override > 0 ? threads_override : auto_threads;
    const int wpc = q.nthreads / 32;
    q.ndgroups = (d_count + wpc - 1) / wpc;
    if (q.pack_gl) q.pack_ndg = (d_count + wpc * (32 / q.pack_gl) - 1) / (wpc * (32 / q.pack_gl));
    // Row segmentation, wave-aware: every segment pays ~11 warm-up rows, and the grid runs in waves of (SMs x resident
    // CTAs) -- with few slices per rank (16 at 8 GPUs) a badly chosen segment count leaves the last wave nearly empty.
    // Pick the count that minimises (waves + ragged end) x (rows per segment + warm-up).
    int best_ns = 1, best_rows = (H + 7) & ~7;
    {
        const long slots = (long)nsm * (65536 / (168 * q.nthreads));        // resident CTAs: 168 registers per thread
        long best_cost = -1;
        for (int want = 1; want <= 12; ++want) {
            int ns = 1, rows = H;
            plan_segments(H, (H + want - 1) / want, &ns, &rows);
            const long ctas = (long)nviews * ns * (q.nstrips * q.ndgroups + q.pack_ndg);
            const long waves = (ctas + slots - 1) / slots;
            // the last wave rarely runs full length: count it in proportion to its fill, but never below half a wave
            const long rem_ctas = ctas - (waves - 1) * slots;
            const double last = rem_ctas >= slots ? 1.0 : (0.5 + 0.5 * (double)rem_ctas / (double)slots);
            // + half a CTA duration: CTAs do not finish in lock-step, and the shorter they are the shorter the ragged end of the
            // kernel.  At 132 SMs (H100): C4 -> 5 segments, C3 -> 6, 16 slices of C4 (one of 8 ranks) -> 8, 32 slices of C5 -> 10,
            // each the fastest count in an A/B over forced counts or within 1.5 % of it.
            const long cost = (long)(((double)(waves - 1) + last + 0.5) * (rows + 11) * 16);
            if (best_cost < 0 || cost < best_cost) { best_cost = cost; best_ns = ns; best_rows = rows; }
        }
    }
    q.nseg = best_ns; q.seg_rows = best_rows;
    if (target_rows > 0) plan_segments(H, target_rows, &q.nseg, &q.seg_rows);
    q.pack_first = nviews * q.nseg * q.nstrips * q.ndgroups;
    q.grid = (unsigned)q.pack_first + (unsigned)nviews * q.nseg * q.pack_ndg;
    return q;
}

int launch_cvf_stream(psm_ctx* c)
{
    CvfParams P;
    for (int v = 0; v < 2; ++v) { P.vol_in[v] = c->vol[v]; P.vol_out[v] = c->vol_alt[v]; P.guide[v] = c->guide[v]; }
    P.W = c->W; P.H = c->H; P.Wp = c->Wp; P.Dloc = c->res.count;
    // the packed remainder needs no CTA-level staging (variant 9 stages the guide rows of one strip); variants 1 and 2
    // keep the plain decomposition of the round-1 kernel; option 105 = 1 disables it
    const bool plain_variant = c->cvf_variant == 9 || c->cvf_variant == 2 || (c->cvf_mode != PSM_CVF_MIXED && c->cvf_variant == 1);
    int nsm = 0;
    PSM_CUDA(c, cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, c->device));
    const CvfPlan plan = plan_cvf(c->W, c->H, c->res.count, nsm, c->cvf_threads, c->cvf_target_rows,
                                  !c->cvf_no_pack && !plain_variant && !c->cvf_remap, c->views);
    const int nthreads = plan.nthreads;
    P.nstrips = plan.nstrips; P.ndgroups = plan.ndgroups; P.nseg = plan.nseg; P.seg_rows = plan.seg_rows;
    P.pack_gl = plan.pack_gl; P.pack_x0 = plan.pack_x0; P.pack_ndg = plan.pack_ndg; P.pack_first = plan.pack_first;
    P.remap_sms = 0; P.remap_ctas = 0;
    if (c->cvf_remap) {
        P.remap_sms = nsm;
        P.remap_ctas = (int)((227 * 1024) / ((size_t)8 * 4 * nthreads * sizeof(float4) + 1024));  // resident CTAs by shared memory
        if (P.remap_ctas * nthreads * 170 > 65536) P.remap_ctas = 65536 / (nthreads * 170);      // ... and by registers
    }
    // kernel selection: mode (exact / mixed) x tuning variant (PSM option 100); every build keeps its history ring in
    // shared memory
    //   variant 0 (shipped): integer widening (+ L1 prefetch of the next guide rows in exact mode)
    //   variant 1: F2F conversions (the round-1 kernel, kept as the A/B baseline; exact only)
    //   variant 2: integer widening, plain decomposition
    //   variant 3: F2F conversions (exact only)
    //   variant 4: as 0 with <= 128 registers
    //   variants 5-8: experiments recorded in DESIGN.md (prefetch on/off, stage-2 F2F, 144/152-register builds)
    using kern_t = void (*)(CvfParams);
    kern_t kern = nullptr;
    bool staged = false;
    if (c->cvf_mode == PSM_CVF_MIXED) {
        switch (c->cvf_variant) {
        case 2: kern = cvf_stream_kernel<3, 1, kS2Mixed>; break;
        case 4: kern = cvf_stream_kernel<4, 1, kS2Mixed>; break;
        case 5: kern = cvf_stream_kernel<3, 1, kS2Mixed, 1>; break;
        case 6: kern = cvf_stream_kernel<4, 1, kS2Mixed, 1>; break;
        case 7: kern = cvf_stream_kernel<5, 1, kS2Mixed, 0>; break;   // 144 registers
        case 8: kern = cvf_stream_kernel<6, 1, kS2Mixed, 0>; break;   // 152 registers
        case 9: kern = cvf_stream_kernel<3, 1, kS2Mixed, 2>; staged = true; break;   // TMA-staged guide rows
        case 10: kern = cvf_stream_kernel<4, 1, kS2Mixed, 3>; break;  // light prefetch, <= 128 registers
        case 11: kern = cvf_stream_kernel<3, 1, kS2Mixed, 3>; break;  // light prefetch, 168 registers
        case 12: kern = cvf_stream_kernel<3, 1, kS2Mixed, 0, 1>; break;  // exact adds as fma
        case 14: kern = cvf_stream_kernel<3, 1, kS2Mixed, 4, 0>; break;  // coefficient rows one step ahead
        case 15: kern = cvf_stream_kernel<3, 1, kS2Mixed, 4, 1>; break;  // ... + exact adds as fma
        case 13: kern = cvf_stream_kernel<4, 1, kS2Mixed, 3, 1>; break;  // exact adds as fma + light prefetch, 128 registers
        default: kern = cvf_stream_kernel<3, 1, kS2Mixed>; break;
        }
    } else {
        switch (c->cvf_variant) {
        case 1: kern = cvf_stream_kernel<3, 0, kS2Exact>; break;
        case 2: kern = cvf_stream_kernel<3, 1, kS2Exact>; break;
        case 3: kern = cvf_stream_kernel<3, 0, kS2Exact>; break;
        case 4: kern = cvf_stream_kernel<4, 1, kS2Exact>; break;
        case 6: kern = cvf_stream_kernel<3, 2, kS2Exact, 0>; break;
        case 7: kern = cvf_stream_kernel<3, 2, kS2Exact, 1>; break;
        case 8: kern = cvf_stream_kernel<3, 1, kS2Exact, 0>; break;
        case 9: kern = cvf_stream_kernel<3, 1, kS2Exact, 2>; staged = true; break;   // TMA-staged guide rows
        case 10: kern = cvf_stream_kernel<4, 1, kS2Exact, 3>; break;  // light prefetch, <= 128 registers
        case 11: kern = cvf_stream_kernel<3, 1, kS2Exact, 3>; break;  // light prefetch, 168 registers
        case 12: kern = cvf_stream_kernel<3, 1, kS2Exact, 1, 1>; break;  // exact adds as fma
        case 14: kern = cvf_stream_kernel<3, 1, kS2Exact, 4, 0>; break;  // coefficient rows one step ahead
        default: kern = cvf_stream_kernel<3, 1, kS2Exact, 1>; break;
        }
    }
    const size_t smem = (staged ? (size_t)kStSmemBytes : 0) + (size_t)8 * 4 * nthreads * sizeof(float4) + (size_t)c->cvf_extra_smem;
    int smem_max = 0;
    PSM_CUDA(c, cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, c->device));
    if (smem > (size_t)smem_max)
        return fail(c, PSM_EINVAL, "streaming filter: %zu bytes of shared memory for %d threads exceed the %d a block may have",
                    smem, nthreads, smem_max);
    PSM_CUDA(c, raise_smem_limit(kern, smem, c->device));
    P.guide_flags = c->guide_flags;
    P.one = 1.0f; P.mone = -1.0f;
    const unsigned grid = plan.grid;
    kern<<<grid, nthreads, smem, c->stream>>>(P);
    PSM_LAUNCH_CHECK(c);
    return PSM_OK;
}

// The guided filter at a non-default window / eps (psm_cvf_window.cuh): strips of kWinThreads - 2K + 2 output columns, and
// as many row segments (of >= 4K rows, so that the ~2K warm-up rows stay a small share) as it takes to give every SM a few CTAs.
int launch_cvf_window(psm_ctx* c)
{
    WinParams P;
    for (int v = 0; v < 2; ++v) { P.vol_in[v] = c->vol[v]; P.vol_out[v] = c->vol_alt[v]; P.guide[v] = c->guide[v]; }
    P.W = c->W; P.H = c->H; P.Wp = c->Wp; P.Dloc = c->res.count;
    P.K = c->gif_win; P.a = c->gif_win / 2;
    P.scale = 1.0 / ((double)P.K * P.K);
    P.tw = kWinThreads - 2 * P.K + 2;
    P.nstrips = (c->W + P.tw - 1) / P.tw;
    P.ring_stride = (c->W < P.tw ? c->W : P.tw) + P.K - 1;
    int nsm = 0, smem_max = 0;
    PSM_CUDA(c, cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, c->device));
    PSM_CUDA(c, cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, c->device));
    const long base = (long)c->views * P.Dloc * P.nstrips;
    int nseg = 1;
    while (base * nseg < 4L * nsm && c->H / (nseg + 1) >= 4 * P.K) ++nseg;
    P.seg_rows = (c->H + nseg - 1) / nseg;
    P.nseg = (c->H + P.seg_rows - 1) / P.seg_rows;
    const size_t smem = win_smem_bytes(P.K, P.ring_stride);
    if (smem > (size_t)smem_max)
        return fail(c, PSM_EINVAL, "guided filter window %d: %zu bytes of shared memory exceed the %d a block may have", P.K, smem, smem_max);
    PSM_CUDA(c, raise_smem_limit(cvf_window_kernel, smem, c->device));
    cvf_window_kernel<<<(unsigned)(base * P.nseg), kWinThreads, smem, c->stream>>>(P);
    PSM_LAUNCH_CHECK(c);
    return PSM_OK;
}

// K1: both raw volumes of the resident slices
int launch_cvc(psm_ctx* c)
{
    CvcParams2 P2;
    for (int v = 0; v < 2; ++v) {
        CvcParams& P = P2.v[v];
        const float* gs = c->guide[v];
        const float* go = c->guide[1 - v];
        for (int k = 0; k < 3; ++k) { P.self[k] = gs + k * c->plane; P.other[k] = go + k * c->plane; }
        P.self[3] = c->grd[v];
        P.other[3] = c->grd[1 - v];
        P.vol = c->vol[v];
        P.W = c->W; P.H = c->H; P.Wp = c->Wp; P.d_begin = c->res.begin; P.d_count = c->res.count;
        P.fold_halo = c->W >= 32 ? 1 : 0;
    }
    // option 108 (tuning): slices per CTA (0 = all resident slices in one CTA, the shipped decomposition)
    P2.chunk = (c->cvc_chunk > 0 && c->cvc_chunk < c->res.count) ? c->cvc_chunk : 0;
    const int nchunks = P2.chunk ? (c->res.count + P2.chunk - 1) / P2.chunk : 1;
    dim3 blk(128), grd((((c->W + 3) / 4) + 127) / 128, c->H, c->views * nchunks);
    // option 106 (tuning): 0 shipped = interior fast path + scalar window loads; 2 = no fast path (the round-1 loop);
    // 1 / 3 = fast path + grouped 128-bit window loads for the border warps without / with a register cap (DESIGN.md section 10)
    const auto both = [&](auto nviews) {
        constexpr int NV = decltype(nviews)::value;
        switch (c->cvc_variant) {
        case 1: cvc_both_kernel<4, 1, NV><<<grd, blk, 0, c->stream>>>(P2); break;
        case 2: cvc_both_kernel<7, 2, NV><<<grd, blk, 0, c->stream>>>(P2); break;
        case 3: cvc_both_kernel<5, 1, NV><<<grd, blk, 0, c->stream>>>(P2); break;
        default: cvc_both_kernel<7, 0, NV><<<grd, blk, 0, c->stream>>>(P2); break;
        }
    };
    // Any matching cost other than the default runs the parameterised build of the shipped variant, all resident slices
    // per CTA: options 106 and 108 do not apply to it.  A left-only context runs the one-view builds.
    if (!c->cost_default()) {
        grd.z = c->views;
        if (c->views == 2) cvc_cost_kernel<<<grd, blk, 0, c->stream>>>(P2, c->cost);
        else cvc_cost_kernel<1><<<grd, blk, 0, c->stream>>>(P2, c->cost);
    } else if (c->views == 2) {
        both(std::integral_constant<int, 2>());
    } else {
        both(std::integral_constant<int, 1>());
    }
    PSM_LAUNCH_CHECK(c);
    if (!P2.v[0].fold_halo)  // narrow images: separate halo pass (general reflection)
        for (int v = 0; v < c->views; ++v)
            if (int rc = pad_rows(c, c->vol[v], (size_t)c->res.count * c->H)) return rc;
    return PSM_OK;
}

// of view v: the result planes of output o, the costs' tracking planes, the runner-up's running list and (on the first
// shard of a multi-device context of nslots shards) its slots
CostPlanes out_planes(const psm_ctx* c, int o, int v) { return {c->outs[o].planes[v], (size_t)c->W * c->H}; }
CostPlanes track_planes(const psm_ctx* c, int v) { return {c->track[v], (size_t)c->W * c->H}; }
CostPlanes list_planes(const psm_ctx* c, int v) { return {c->ru_list[v], (size_t)c->W * c->H}; }
RunnerUpSlots runner_up_slots(const psm_ctx* c, int v, int nslots) { return {c->ru_slots[v], (size_t)c->W * c->H, nslots}; }

// the filtered block in the volumes -> the running keys (stored by the first block, min-folded by the others), with
// PSM_OPT_COSTS the costs beside the running winners, and with PSM_OPT_RUNNER_UP the running lists
int launch_fold(psm_ctx* c, bool first)
{
    FoldParams P;
    for (int v = 0; v < 2; ++v) {
        P.vol[v] = c->vol[v]; P.keys[v] = c->run_keys[v]; P.track[v] = track_planes(c, v); P.list[v] = list_planes(c, v);
    }
    P.W = c->W; P.H = c->H; P.Wp = c->Wp; P.d_begin = c->res.begin; P.d_count = c->res.count; P.first = first ? 1 : 0;
    P.write_first = c->track_planes() > kCostFirst;
    dim3 blk(256), grd(((c->W + 3) / 4 + 255) / 256, c->H, c->views);
    const bool costs = c->outs[kOutCosts].on;
    if (c->outs[kOutRunnerUp].on)
        (costs ? wta_fold_kernel<true, true> : wta_fold_kernel<false, true>)<<<grd, blk, 0, c->stream>>>(P);
    else
        (costs ? wta_fold_kernel<true, false> : wta_fold_kernel<false, false>)<<<grd, blk, 0, c->stream>>>(P);
    PSM_LAUNCH_CHECK(c);
    return PSM_OK;
}

// The cost entries context c owns (cost_write_kernel) from `map` (the complete selection map of view v) into dst: from
// its resident volume on an unblocked context, from its tracking planes on a blocked one
int launch_cost_write(psm_ctx* c, int v, const void* map, CostPlanes dst)
{
    CostWriteParams P;
    P.map = map; P.vol = c->vol[v]; P.src = track_planes(c, v); P.dst = dst;
    P.W = c->W; P.H = c->H; P.Wp = c->Wp; P.D = c->D; P.d_lo = c->d_lo; P.d_begin = c->d_begin; P.d_count = c->d_count;
    dim3 blk(256), grd((c->W + 255) / 256, c->H);
    if (c->map_bytes == 2)
        (c->blk_slices ? cost_write_kernel<uint16_t, true> : cost_write_kernel<uint16_t, false>)<<<grd, blk, 0, c->stream>>>(P);
    else
        (c->blk_slices ? cost_write_kernel<uint8_t, true> : cost_write_kernel<uint8_t, false>)<<<grd, blk, 0, c->stream>>>(P);
    PSM_LAUNCH_CHECK(c);
    return PSM_OK;
}

// The runner-up of the slices context c owns (runner_up_write_kernel), from `map` (the complete selection map of view v):
// from a list scan of its resident volume on an unblocked context, from its running lists on a blocked one.  Into its
// own result planes, or, where slots.base is set, into slot `slot` of the first shard's.
int launch_runner_up_write(psm_ctx* c, int v, const void* map, RunnerUpSlots slots, int slot)
{
    RunnerUpWriteParams P;
    P.map = map; P.vol = c->vol[v]; P.keys = c->run_keys[v]; P.list = list_planes(c, v);
    P.dst = out_planes(c, kOutRunnerUp, v); P.slots = slots; P.slot = slot;
    P.W = c->W; P.H = c->H; P.Wp = c->Wp; P.d_begin = c->d_begin; P.d_count = c->d_count;
    dim3 blk(256), grd(((c->W + 3) / 4 + 255) / 256, c->H);
    if (c->map_bytes == 2)
        (c->blk_slices ? runner_up_write_kernel<uint16_t, true> : runner_up_write_kernel<uint16_t, false>)<<<grd, blk, 0, c->stream>>>(P);
    else
        (c->blk_slices ? runner_up_write_kernel<uint8_t, true> : runner_up_write_kernel<uint8_t, false>)<<<grd, blk, 0, c->stream>>>(P);
    PSM_LAUNCH_CHECK(c);
    return PSM_OK;
}

// Output o of view v once `map` (its complete selection map) is written: context c's writer of the entries it owns.  On a
// single-device context (n = 0) into its own result planes; on shard k of a multi-device context of n shards into the
// first shard s0's result planes (the costs) or into its slot there (the runner-up, which s0 then reduces).
int launch_out_write(psm_ctx* c, int o, int v, const void* map, psm_ctx* s0, int k, int n)
{
    if (o == kOutCosts) return launch_cost_write(c, v, map, out_planes(s0, kOutCosts, v));
    if (!n && !c->blk_slices) return PSM_OK;   // an unblocked context's selection kernel wrote it beside the map
    return launch_runner_up_write(c, v, map, n ? runner_up_slots(s0, v, n) : RunnerUpSlots{}, k);
}

// The slices the volumes hold while the context's stages work from global slice `b` on: up to vol_slices() of the owned
// range, so the owned range itself on an unblocked context and the block starting at b on a blocked one.
psm_ctx::Slices block_at(const psm_ctx* c, int b)
{
    return {b, std::min(c->vol_slices(), c->d_begin + c->d_count - b)};
}

// The destinations of a map call `call`: rows of W elements of the map format, the right map's on a two-view context only.
// Checked before the call's first launch: a bad one returns PSM_EINVAL with nothing enqueued and no state changed.
int check_map_dst(psm_ctx* c, const char* call, const void* left, size_t left_step, const void* right, size_t right_step)
{
    if (int rc = check_right_arg(c, right, call)) return rc;
    const size_t row = (size_t)c->W * c->map_bytes;
    if (!left || left_step < row || (c->views == 2 && (!right || right_step < row)))
        return c->map_bytes == 1 ? fail(c, PSM_EINVAL, "bad disparity map pointer/step")
                                 : fail(c, PSM_EINVAL, "bad disparity map pointer/step (u16 maps need a step of at least %zu bytes)", row);
    return PSM_OK;
}

// device maps src[view] -> the checked destinations, on the context's stream; then waits for the copies if `sync`
int copy_maps_out(psm_ctx* c, const uint8_t* const src[2], void* left, size_t left_step, void* right, size_t right_step,
                  cudaMemcpyKind kind, bool sync)
{
    const size_t row = (size_t)c->W * c->map_bytes;
    PSM_CUDA(c, cudaMemcpy2DAsync(left, left_step, src[0], row, row, c->H, kind, c->stream));
    if (c->views == 2) PSM_CUDA(c, cudaMemcpy2DAsync(right, right_step, src[1], row, row, c->H, kind, c->stream));
    if (sync) PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    return PSM_OK;
}

// The exchange block of one rank (psm_p2p_create_buffer), as byte offsets: keys [2 views][nranks][chunk] u64, maps
// [2 views][H*W] of the map format rounded up to 256 bytes, flag words [2 views][2 * kMaxRanks] u32 (ARRIVE, DONE per rank).
struct P2pLayout {
    size_t chunk, keys_view, maps_at, map_view, flags_at, bytes;
    unsigned long long* keys(unsigned char* base, int v) const { return reinterpret_cast<unsigned long long*>(base + v * keys_view); }
    unsigned char* maps(unsigned char* base, int v) const { return base + maps_at + v * map_view; }
    unsigned* flags(unsigned char* base, int v) const { return reinterpret_cast<unsigned*>(base + flags_at) + v * 2 * kMaxRanks; }
};

P2pLayout p2p_layout(const psm_ctx* c, int nranks)
{
    const size_t npix = (size_t)c->W * c->H, chunk = (npix + nranks - 1) / nranks, keys_view = nranks * chunk * sizeof(uint64_t);
    const size_t map_view = npix * c->map_bytes, flags_at = 2 * keys_view + ((2 * map_view + 255) & ~(size_t)255);
    return {chunk, keys_view, 2 * keys_view, map_view, flags_at, flags_at + 2 * 2 * kMaxRanks * sizeof(unsigned)};
}

// the current maps are the exchange block's: from the first exchanged frame on, also after a later local selection
bool exchanged(const psm_ctx* c) { return c->p2p_own && c->p2p_seq > 0; }

// a selection stage wrote new maps (`own`: the context's own, not an exchange block's): the left-right masks are stale
// and so are the costs and the runner-up, until the stage writes them too
void selection_ran(psm_ctx* c, bool own)
{
    c->lr_masks_ok = false;
    c->have_maps = c->have_maps || own;
    for (psm_ctx::OutState& o : c->outs) o.have = false;
}

// a map call for maps of type T, named u8_call / u16_call in its two formats, on a context of the other format:
// PSM_EINVAL naming the right call
template <typename T>
int check_map_format(psm_ctx* c, const char* u8_call, const char* u16_call)
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    if (c->map_bytes == (int)sizeof(T)) return PSM_OK;
    if (sizeof(T) == 1) return fail(c, PSM_EINVAL, "%s on a context with 16-bit maps (psm_create_u16): use %s", u8_call, u16_call);
    return fail(c, PSM_EINVAL, "%s on a context with 8-bit maps (psm_create / psm_create_sharded): use %s", u16_call, u8_call);
}

// ---- multi-device contexts (psm_create_multi) ----
// The context aliases the first shard's stream and complete maps (the maps in its exchange block), so the map calls that
// copy out or sync run unchanged on it; every other call is forwarded to the shards, or rejected.

bool is_multi(const psm_ctx* c) { return c && c->nshards; }

// a call on shard k failed: its error becomes the multi-device context's
int relay(psm_ctx* c, int k, int rc)
{
    if (rc) {
        char text[512];
        snprintf(text, sizeof(text), "%s", c->shard[k]->err);
        fail(c, rc, "shard %d (device %d): %s", k, c->shard[k]->device, text);
    }
    return rc;
}

// the same call on every shard in turn, up to the first failure.  The setters judge the value alone, the same way on
// every shard, so a value that one shard rejects is rejected by the first one, before any shard has changed.
template <class F>
int forward(psm_ctx* c, F f)
{
    for (int k = 0; k < c->nshards; ++k)
        if (int rc = f(c->shard[k])) return relay(c, k, rc);
    return PSM_OK;
}

int reject_multi(psm_ctx* c, const char* call, const char* why)
{
    return fail(c, PSM_EINVAL, "%s on a multi-device context (psm_create_multi): %s", call, why);
}

// psm_set_images[_u8|_device] on a multi-device context, after the first shard's stage 0.  Every other shard receives
// the frame device to device into its own staging set and runs its own ingest kernels; its stage 0 covers the copy.
// The staging sets' readers and writers:
//   - shard k's copy starts once the source holds the frame (the first shard's staging set after its upload, or the
//     caller's device images at the first shard's ingest) and once shard k's last ingest has read shard k's staging set;
//   - the source's next writer follows every copy: the first shard's copy stream (its next upload) for a host frame, the
//     first shard's stream (which the caller orders its overwrites against) for device images;
//   - shard k's ingest kernels follow its copy, and its next copy follows them (ingest_done).
int multi_send_frame(psm_ctx* c, Frame kind, int pix, const PlanesSrc src[2])
{
    psm_ctx* s0 = c->shard[0];
    const size_t row = (size_t)c->W * 3 * pix_bytes(pix);
    const void* from[2] = {src[0].ch[0], src[1].ch[0]};
    size_t step[2] = {src[0].row_step, src[1].row_step};
    cudaEvent_t ready = s0->host_copied;
    cudaStream_t next_writer = s0->copy_stream;
    if (kind == Frame::device) {
        PSM_CUDA(c, cudaEventRecord(c->ev_images, s0->stream));
        ready = c->ev_images;
        next_writer = s0->stream;
    } else {
        for (int v = 0; v < 2; ++v) { from[v] = stage_buf(s0, s0->stage_cur, v); step[v] = row; }
    }
    for (int k = 1; k < c->nshards; ++k) {
        psm_ctx* s = c->shard[k];
        int rc = bind(s);
        if (rc) return relay(c, k, rc);
        if (s->ingest_done_valid[0]) PSM_CUDA(c, cudaStreamWaitEvent(s->copy_stream, s->ingest_done[0], 0));
        PSM_CUDA(c, cudaStreamWaitEvent(s->copy_stream, ready, 0));
        if (s->timing) PSM_CUDA(c, cudaEventRecord(s->ev0[0], s->copy_stream));
        for (int v = 0; v < 2; ++v)   // a peer copy between distinct devices
            PSM_CUDA(c, cudaMemcpy2DAsync(s->stage_in[v], row, from[v], step[v], row, c->H, cudaMemcpyDefault, s->copy_stream));
        PSM_CUDA(c, cudaEventRecord(c->ev_copied[k], s->copy_stream));
        PSM_CUDA(c, cudaStreamWaitEvent(next_writer, c->ev_copied[k], 0));
        if ((rc = ingest_staged(s, 0, pix, c->ev_copied[k])) || (rc = stage_end(s, 0))) return relay(c, k, rc);
    }
    return PSM_OK;
}

// psm_set_images_device_planes on a multi-device context, after the first shard's stage 0.  Every other shard copies what
// the first shard's ingest wrote (the three channel planes with their mirrored halos, the gradient planes and the ingest
// flags, byte for byte) device to device on its own stream, so the caller's buffers are read on the first device only and
// every shard holds the planes its own ingest would have written.  The broadcast's readers and writers:
//   - shard k's copy follows the first shard's ingest (ev_images) and, on its own stream, shard k's earlier work, which
//     reads the planes the copy overwrites;
//   - the first shard's later work (its next ingest, and the guide precompute, which adds to the flags) follows every
//     copy (ev_copied), and so does whatever orders itself after the first shard's stream (psm_signal_stream).
int multi_send_planes(psm_ctx* c, int pix)
{
    psm_ctx* s0 = c->shard[0];
    PSM_CUDA(c, cudaEventRecord(c->ev_images, s0->stream));
    for (int k = 1; k < c->nshards; ++k) {
        psm_ctx* s = c->shard[k];
        int rc = bind(s);
        if (rc) return relay(c, k, rc);
        PSM_CUDA(c, cudaStreamWaitEvent(s->stream, c->ev_images, 0));
        if ((rc = stage_begin(s, 0))) return relay(c, k, rc);
        for (int v = 0; v < 2; ++v) {   // from the first row's left halo: 3 channel planes, then the gradient plane
            PSM_CUDA(c, cudaMemcpyAsync(s->guide[v] - kPadLeft, s0->guide[v] - kPadLeft, 3 * s0->plane * sizeof(float),
                                        cudaMemcpyDefault, s->stream));
            PSM_CUDA(c, cudaMemcpyAsync(s->grd[v] - kPadLeft, s0->grd[v] - kPadLeft, s0->plane * sizeof(float),
                                        cudaMemcpyDefault, s->stream));
        }
        PSM_CUDA(c, cudaMemcpyAsync(s->guide_flags, s0->guide_flags, 2 * sizeof(int), cudaMemcpyDefault, s->stream));
        PSM_CUDA(c, cudaEventRecord(c->ev_copied[k], s->stream));
        PSM_CUDA(c, cudaStreamWaitEvent(s0->stream, c->ev_copied[k], 0));
        images_ingested(s, pix == PSM_PIX_F32);
        if ((rc = stage_end(s, 0))) return relay(c, k, rc);
    }
    return PSM_OK;
}

// the body of every synchronous psm_set_images* call once its frame is checked.  A multi-device context runs stage 0 on
// its first shard and sends the other shards the frame, or the planes the first shard ingested.  With psm_set_rectify on,
// only the first shard holds the maps, so every kind of frame reaches the others as its planes; so does a YUV or Bayer
// frame.
int set_images(psm_ctx* c, Frame kind, int fmt, const PlanesSrc src[2])
{
    if (!is_multi(c)) return set_images_one(c, kind, fmt, src);
    if (int rc = set_images_one(c->shard[0], kind, fmt, src)) return relay(c, 0, rc);
    return kind == Frame::planes || c->rect_sw || is_yuv(fmt) || is_bayer(fmt) ? multi_send_planes(c, fmt)
                                                                                : multi_send_frame(c, kind, fmt, src);
}

// psm_set_images_device_yuv / _device_bayer once its frames are checked: stage 0 on the context (a multi-device context's
// first shard, whose ingested planes the other shards receive)
template <class Src>
int set_images_device_converted(psm_ctx* c, const Src src[2])
{
    psm_ctx* s = is_multi(c) ? c->shard[0] : c;
    int rc = bind(s);
    if (!rc) rc = stage_begin(s, 0);
    if (!rc) rc = ingest<uint8_t>(s, src);
    if (!rc) rc = stage_end(s, 0);
    if (!is_multi(c)) return rc;
    return rc ? relay(c, 0, rc) : multi_send_planes(c, PSM_PIX_U8);
}

// psm_set_images[_u8|_yuv|_bayer]_async: the frame of format fmt that check(src) checks is uploaded into the staging set that is
// not in use, on the copy stream
template <class Check>
int set_images_async(psm_ctx* c, int fmt, const char* call, Check check)
{
    if (is_multi(c)) return reject_multi(c, call, "the asynchronous upload pipeline is not available on it; use psm_set_images / _u8");
    if (int rc = bind(c)) return rc;
    if (c->up_pending) return fail(c, PSM_ESTATE, "an asynchronous upload is already pending: call psm_set_images_commit first");
    PlanesSrc src[2];
    if (int rc = check(src)) return rc;
    if (!c->stage_alt[0]) {  // allocated on first use: synchronous callers never pay for the second set
        for (int v = 0; v < 2; ++v) PSM_CUDA(c, cudaMalloc(&c->stage_alt[v], c->stage_bytes));
    }
    if (int rc = upload(c, c->stage_cur ^ 1, fmt, src, c->up_done)) return rc;
    c->up_pending = fmt;
    return PSM_OK;
}

// the contexts whose streams carry a context's work: the shards of a multi-device context, or the context itself
int ctx_parts(psm_ctx* c, psm_ctx** parts)
{
    if (!is_multi(c)) { parts[0] = c; return 1; }
    for (int k = 0; k < c->nshards; ++k) parts[k] = c->shard[k];
    return c->nshards;
}

// psm_cost_filter: the MIXED and NAIVE modes exist for the default guided filter alone
int check_cvf_mode(psm_ctx* c)
{
    if (!c->gif_default() && c->cvf_mode != PSM_CVF_EXACT)
        return fail(c, PSM_EINVAL, "CVF mode %s exists only for the default guided filter (window 8, eps 1e-4); "
                    "this context has window %d, eps %g: use PSM_CVF_EXACT", c->cvf_mode == PSM_CVF_MIXED ? "MIXED" : "NAIVE",
                    c->gif_win, (double)c->gif_eps);
    return PSM_OK;
}

// psm_cost_filter on the resident slices.  NAIVE and images below one strip: every slice in OpenCV's order.  Otherwise
// the tuned kernel, then, in OpenCV's order, the slices psm_write_cost_slice flagged and every slice of a view whose image
// is outside the integer domain or whose solve terms are not finite (psm_cvf_ref.cuh).  The second launch is needed only
// where a flag can be set: flagged slices, float images, a non-default window or eps.  u8 frames at the defaults run the
// tuned kernel alone.
int cvf_block(psm_ctx* c)
{
    if (c->gif_default() && (c->cvf_mode == PSM_CVF_NAIVE || c->W < 16 || c->H < 16)) {
        if (int rc = launch_ref(c, (void*)cvf_ref_kernel, kRefAll)) return rc;
    } else {
        if (int rc = c->gif_default() ? launch_cvf_stream(c) : launch_cvf_window(c)) return rc;
        if (c->slices_flagged || c->float_images || !c->gif_default())
            if (int rc = launch_ref(c, (void*)cvf_ref_kernel, kRefFlagged)) return rc;
    }
    if (int rc = clear_slice_flags(c)) return rc;
    // the right view's pair is not swapped on a left-only context: its volume buffers keep their roles
    for (int v = 0; v < c->views; ++v) { float* t = c->vol[v]; c->vol[v] = c->vol_alt[v]; c->vol_alt[v] = t; }
    return PSM_OK;
}

// The filter stage of entry point `call`.  `prepare` checks the entry point's own arguments and sets up its buffers; then
// stage 2 runs `guide` once and `filter`, which leaves the resident slices filtered in c->vol, on the range.  An unblocked
// context filters every slice it owns in one pass, timed as stage 4.  A blocked context walks its range block by block:
// the block's raw costs (psm_cost_const built the first block's), `filter`, and the fold into the running keys.  It
// records no stage 4, whose kernels would interleave with every block's CVC and fold.
template <class Prepare, class Guide, class Filter>
int filter_stage(psm_ctx* c, const char* call, Prepare prepare, Guide guide, Filter filter)
{
    if (is_multi(c)) return forward(c, [&](psm_ctx* s) { return filter_stage(s, call, prepare, guide, filter); });
    if (int rc = bind(c)) return rc;
    if (int rc = check_stages_reset(c, call)) return rc;
    if (!c->have_cvc) return fail(c, PSM_ESTATE, "%s before psm_cost_const", call);
    if (int rc = prepare(c)) return rc;
    if (int rc = stage_begin(c, 2)) return rc;
    if (int rc = guide(c)) return rc;
    if (!c->blk_slices) {
        if (int rc = stage_begin(c, 4)) return rc;
        if (int rc = filter(c)) return rc;
        if (int rc = stage_end(c, 4)) return rc;
    } else {
        for (int b = c->d_begin; b < c->d_begin + c->d_count; b += c->blk_slices) {
            const bool first = b == c->d_begin;
            c->res = block_at(c, b);
            if (!first)
                if (int rc = launch_cvc(c)) return rc;
            if (int rc = filter(c)) return rc;
            if (int rc = launch_fold(c, first)) return rc;
        }
    }
    c->have_cvc = false;  // the volumes now hold filtered costs; filtering again needs a new CVC
    c->filtered = true;
    return stage_end(c, 2);
}

}  // namespace

// ----------------------------------------------------------------------------------------------

extern "C" {

int psm_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

const char* psm_build_info(void)
{
    return "prime_stereo_b200 0.1 (sm_90a; " PSM_BUILD_FLAGS ")";
}

const char* psm_last_error(psm_ctx* ctx) { return ctx ? ctx->err : g_create_error; }

int psm_cvf_plan(int width, int height, int d_count, int sm_count, int no_pack, int* out, int n)
{
    if (width < 1 || height < 1 || d_count < 1 || sm_count < 1 || !out || n < 10) return PSM_EINVAL;
    const CvfPlan q = plan_cvf(width, height, d_count, sm_count, 0, 0, !no_pack, 2);
    const int v[10] = {q.nthreads, q.nstrips, q.ndgroups, q.nseg, q.seg_rows, q.pack_gl, q.pack_x0, q.pack_ndg, q.pack_first, (int)q.grid};
    for (int i = 0; i < 10; ++i) out[i] = v[i];
    return PSM_OK;
}

}  // extern "C"

// geometry already validated by the caller; map_bytes 1 (u8 maps) or 2 (u16 maps)
static int create_ctx(psm_ctx** out, int width, int height, int max_disp, int d_begin, int d_count, int device, int map_bytes,
                      int block_slices = 0, int d_lo = 0)
{
    int ndev = psm_device_count();
    if (device < 0 || device >= ndev) return fail(nullptr, PSM_ECUDA, "CUDA device %d not available (%d devices)", device, ndev);
    psm_ctx* c = new (std::nothrow) psm_ctx();
    if (!c) return fail(nullptr, PSM_ENOMEM, "out of host memory");
    c->W = width; c->H = height; c->Wp = pitch_for_width(width); c->D = max_disp;
    c->d_begin = d_begin; c->d_count = d_count; c->device = device; c->d_lo = d_lo;
    c->plane = (size_t)c->H * c->Wp;
    c->map_bytes = map_bytes;
    c->blk_slices = block_slices;
    if (!block_slices) c->res = {d_begin, d_count};
    auto bail = [&](int code) {
        snprintf(g_create_error, sizeof(g_create_error), "%s", c->err);
        psm_destroy(c);
        return code;
    };
#define PSM_CREATE_CUDA(call)                                                                    \
    do {                                                                                         \
        cudaError_t e__ = (call);                                                                \
        if (e__ != cudaSuccess) {                                                                \
            fail(c, PSM_ECUDA, "%s failed: %s", #call, cudaGetErrorString(e__));                 \
            return bail(e__ == cudaErrorMemoryAllocation ? PSM_ENOMEM : PSM_ECUDA);              \
        }                                                                                        \
    } while (0)
    PSM_CREATE_CUDA(cudaSetDevice(device));
    PSM_CREATE_CUDA(cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking));
    c->stream = c->own_stream;
    // every float buffer is allocated with kPadLeft floats in front so that the (row 0, column 0)
    // pointer may be indexed at negative columns (left halo of row 0); rows are Wp floats apart
    auto halo_alloc = [&](float** out, size_t rows) -> cudaError_t {
        float* raw = nullptr;
        const size_t n = rows * (size_t)c->Wp + kPadLeft + 32;
        cudaError_t e = cudaMalloc(&raw, n * sizeof(float));
        if (e != cudaSuccess) return e;
        c->alloc[c->nalloc++] = raw;
        e = cudaMemsetAsync(raw, 0, n * sizeof(float), c->stream);  // DispEst.cpp:31-37 zero-init
        *out = raw + kPadLeft;
        return e;
    };
    const size_t vol_rows = (size_t)c->vol_slices() * c->H;
    c->stage_bytes = (size_t)c->W * c->H * 3 * sizeof(float);
    for (int v = 0; v < 2; ++v) {
        PSM_CREATE_CUDA(halo_alloc(&c->guide[v], (size_t)kGuidePlanes * c->H));
        PSM_CREATE_CUDA(halo_alloc(&c->grd[v], (size_t)c->H));
        PSM_CREATE_CUDA(halo_alloc(&c->vol[v], vol_rows));
        PSM_CREATE_CUDA(halo_alloc(&c->vol_alt[v], vol_rows));
        PSM_CREATE_CUDA(cudaMalloc(&c->stage_in[v], c->stage_bytes));
        PSM_CREATE_CUDA(cudaMalloc(&c->dis[v], (size_t)c->W * c->H * map_bytes));
        PSM_CREATE_CUDA(cudaMemsetAsync(c->dis[v], 0, (size_t)c->W * c->H * map_bytes, c->stream));
        if (block_slices) PSM_CREATE_CUDA(cudaMalloc(&c->run_keys[v], (size_t)c->W * c->H * sizeof(unsigned long long)));
    }
    PSM_CREATE_CUDA(cudaMalloc(&c->guide_flags, 2 * sizeof(int)));
    PSM_CREATE_CUDA(cudaMalloc(&c->slice_flags, 2 * (size_t)c->vol_slices() * sizeof(int)));
    PSM_CREATE_CUDA(cudaMemsetAsync(c->slice_flags, 0, 2 * (size_t)c->vol_slices() * sizeof(int), c->stream));
    PSM_CREATE_CUDA(cudaMemsetAsync(c->guide_flags, 0, 2 * sizeof(int), c->stream));
    PSM_CREATE_CUDA(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
    PSM_CREATE_CUDA(cudaEventCreateWithFlags(&c->up_done, cudaEventDisableTiming));
    PSM_CREATE_CUDA(cudaEventCreateWithFlags(&c->host_copied, cudaEventDisableTiming));
    for (int k = 0; k < 2; ++k) PSM_CREATE_CUDA(cudaEventCreateWithFlags(&c->ingest_done[k], cudaEventDisableTiming));
    PSM_CREATE_CUDA(cudaEventCreateWithFlags(&c->ev_user, cudaEventDisableTiming));
    for (int k = 0; k < 2; ++k) PSM_CREATE_CUDA(cudaEventCreateWithFlags(&c->ev_signal[k], cudaEventDisableTiming));
    for (int s = 0; s < kNumStages; ++s) {
        PSM_CREATE_CUDA(cudaEventCreate(&c->ev0[s]));
        PSM_CREATE_CUDA(cudaEventCreate(&c->ev1[s]));
    }
    PSM_CREATE_CUDA(cudaStreamSynchronize(c->stream));
#undef PSM_CREATE_CUDA
    *out = c;
    return PSM_OK;
}

extern "C" {

int psm_create_sharded(psm_ctx** out, int width, int height, int max_disp, int d_begin, int d_count, int device)
{
    if (!out) return fail(nullptr, PSM_EINVAL, "out is null");
    *out = nullptr;
    if (width < 1 || height < 1 || max_disp < 2 || max_disp > MapFormat<uint8_t>::kMaxDisp)
        return fail(nullptr, PSM_EINVAL, "bad geometry W=%d H=%d D=%d (need W,H>=1, 2<=D<=%d)", width, height, max_disp,
                    MapFormat<uint8_t>::kMaxDisp);
    if (d_begin < 0 || d_count < 1 || d_begin + d_count > max_disp)
        return fail(nullptr, PSM_EINVAL, "bad shard [%d,%d) of %d", d_begin, d_begin + d_count, max_disp);
    return create_ctx(out, width, height, max_disp, d_begin, d_count, device, 1);
}

int psm_create_u16(psm_ctx** out, int width, int height, int max_disp, int d_begin, int d_count, int device)
{
    if (!out) return fail(nullptr, PSM_EINVAL, "out is null");
    *out = nullptr;
    if (width < 1 || height < 1 || max_disp < 2 || max_disp > MapFormat<uint16_t>::kMaxDisp)
        return fail(nullptr, PSM_EINVAL, "bad geometry W=%d H=%d D=%d (need W,H>=1, 2<=D<=%d)", width, height, max_disp,
                    MapFormat<uint16_t>::kMaxDisp);
    if (d_begin < 0 || d_count < 1 || d_begin + d_count > max_disp)
        return fail(nullptr, PSM_EINVAL, "bad shard [%d,%d) of %d", d_begin, d_begin + d_count, max_disp);
    return create_ctx(out, width, height, max_disp, d_begin, d_count, device, 2);
}

int psm_create_blocked(psm_ctx** out, int width, int height, int max_disp, int d_begin, int d_count, int block_slices,
                       int map_bits, int device)
{
    if (!out) return fail(nullptr, PSM_EINVAL, "out is null");
    *out = nullptr;
    if (map_bits != 8 && map_bits != 16) return fail(nullptr, PSM_EINVAL, "map_bits must be 8 or 16 (got %d)", map_bits);
    const int dmax = map_bits == 8 ? MapFormat<uint8_t>::kMaxDisp : MapFormat<uint16_t>::kMaxDisp;
    if (width < 1 || height < 1 || max_disp < 2 || max_disp > dmax)
        return fail(nullptr, PSM_EINVAL, "bad geometry W=%d H=%d D=%d (need W,H>=1, 2<=D<=%d with %d-bit maps)", width, height,
                    max_disp, dmax, map_bits);
    if (d_begin < 0 || d_count < 1 || d_begin + d_count > max_disp)
        return fail(nullptr, PSM_EINVAL, "bad shard [%d,%d) of %d", d_begin, d_begin + d_count, max_disp);
    if (block_slices < 1 || block_slices > d_count)
        return fail(nullptr, PSM_EINVAL, "block_slices %d outside 1..%d (the context's d_count)", block_slices, d_count);
    return create_ctx(out, width, height, max_disp, d_begin, d_count, device, map_bits / 8, block_slices);
}

int psm_create(psm_ctx** out, int width, int height, int max_disp, int device)
{
    return psm_create_sharded(out, width, height, max_disp, 0, max_disp, device);
}

}  // extern "C"

// The multi-device context over the problem range [d_lo, max_disp), its arguments checked up to the devices' existence:
// shard k owns the k-th part of sharding.py's shard_range split of the range.
static int create_multi(psm_ctx** out, int width, int height, int d_lo, int max_disp, const int* devices, int n_devices,
                        int block_slices, int map_bits)
{
    const int ndev = psm_device_count();
    for (int k = 0; k < n_devices; ++k)
        if (devices[k] >= ndev)
            return fail(nullptr, PSM_EINVAL, "devices[%d] = %d: CUDA device not available (%d devices)", k, devices[k], ndev);
    // Shards on distinct devices store into each other's memory: every such pair needs peer access both ways.  Peer
    // access is process-wide and another context may rely on it, so it is enabled here and never disabled.
    for (int i = 0; i < n_devices; ++i)
        for (int j = 0; j < n_devices; ++j) {
            const int a = devices[i], b = devices[j];
            if (a == b) continue;
            int ok = 0;
            cudaError_t e = cudaDeviceCanAccessPeer(&ok, a, b);
            if (e != cudaSuccess) return fail(nullptr, PSM_ECUDA, "cudaDeviceCanAccessPeer(%d, %d) failed: %s", a, b, cudaGetErrorString(e));
            if (!ok) return fail(nullptr, PSM_EINVAL, "device %d cannot access the memory of device %d (no peer access)", a, b);
            if ((e = cudaSetDevice(a)) == cudaSuccess) e = cudaDeviceEnablePeerAccess(b, 0);
            if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); e = cudaSuccess; }
            if (e != cudaSuccess) return fail(nullptr, PSM_ECUDA, "enabling peer access %d -> %d failed: %s", a, b, cudaGetErrorString(e));
        }
    psm_ctx* c = new (std::nothrow) psm_ctx();
    if (!c) return fail(nullptr, PSM_ENOMEM, "out of host memory");
    c->W = width; c->H = height; c->Wp = pitch_for_width(width); c->D = max_disp;
    c->d_begin = d_lo; c->d_count = max_disp - d_lo; c->d_lo = d_lo; c->device = devices[0];
    c->map_bytes = map_bits / 8;
    auto bail = [&](int code) {
        snprintf(g_create_error, sizeof(g_create_error), "%s", c->err);
        psm_destroy(c);
        return code;
    };
    // the split of sharding.py's shard_range: contiguous slices, the last shard takes the remainder
    const int base = c->d_count / n_devices;
    for (int k = 0; k < n_devices; ++k) {
        const int d_begin = d_lo + k * base, d_count = k < n_devices - 1 ? base : max_disp - d_begin;
        if (int rc = create_ctx(&c->shard[k], width, height, max_disp, d_begin, d_count, devices[k], c->map_bytes,
                                block_slices ? std::min(block_slices, d_count) : 0, d_lo)) {
            snprintf(c->err, sizeof(c->err), "shard %d (device %d): %.400s", k, devices[k], g_create_error);
            return bail(rc);
        }
        c->nshards = k + 1;
        c->shard[k]->p2p_sync = 0;   // the shards' exchange kernels never spin on a flag: events order them
    }
    // every shard's exchange block, its peers' blocks as raw pointers (one process, no IPC), and the ordering events
    void* blocks[kMaxRanks] = {};
    for (int k = 0; k < n_devices; ++k) {
        if (int rc = psm_p2p_create_buffer(c->shard[k], n_devices, &blocks[k])) {
            const bool oom = cudaGetLastError() == cudaErrorMemoryAllocation;
            relay(c, k, rc);
            return bail(oom ? PSM_ENOMEM : rc);
        }
    }
    for (int k = 0; k < n_devices; ++k) {
        if (int rc = psm_p2p_set_peers(c->shard[k], blocks, n_devices, k)) { relay(c, k, rc); return bail(rc); }
        cudaError_t e = cudaSetDevice(devices[k]);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_scattered[k], cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_reduced[k], cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_copied[k], cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->ev_written[k], cudaEventDisableTiming);
        if (e == cudaSuccess && k == 0) e = cudaEventCreateWithFlags(&c->ev_images, cudaEventDisableTiming);
        if (e != cudaSuccess) { fail(c, PSM_ECUDA, "event creation on device %d failed: %s", devices[k], cudaGetErrorString(e)); return bail(PSM_ECUDA); }
    }
    // the first shard's stream and complete maps stand for the context's (see is_multi)
    psm_ctx* s0 = c->shard[0];
    c->stream = s0->stream;
    for (int v = 0; v < 2; ++v) c->dis[v] = p2p_layout(c, n_devices).maps(static_cast<unsigned char*>(blocks[0]), v);
    *out = c;
    return PSM_OK;
}

extern "C" {

int psm_create_multi(psm_ctx** out, int width, int height, int max_disp, const int* devices, int n_devices, int block_slices,
                     int map_bits)
{
    if (!out) return fail(nullptr, PSM_EINVAL, "out is null");
    *out = nullptr;
    if (map_bits != 8 && map_bits != 16) return fail(nullptr, PSM_EINVAL, "map_bits must be 8 or 16 (got %d)", map_bits);
    const int dmax = map_bits == 8 ? MapFormat<uint8_t>::kMaxDisp : MapFormat<uint16_t>::kMaxDisp;
    if (width < 1 || height < 1 || max_disp < 2 || max_disp > dmax)
        return fail(nullptr, PSM_EINVAL, "bad geometry W=%d H=%d D=%d (need W,H>=1, 2<=D<=%d with %d-bit maps)", width, height,
                    max_disp, dmax, map_bits);
    if (n_devices < 1 || n_devices > kMaxRanks || n_devices > max_disp)
        return fail(nullptr, PSM_EINVAL, "n_devices %d outside 1..%d (at most %d shards, each owning at least one of the %d slices)",
                    n_devices, std::min(kMaxRanks, max_disp), kMaxRanks, max_disp);
    if (!devices) return fail(nullptr, PSM_EINVAL, "devices is null");
    if (block_slices < 0) return fail(nullptr, PSM_EINVAL, "block_slices %d is negative (0 = unblocked shards)", block_slices);
    for (int k = 0; k < n_devices; ++k)
        if (devices[k] < 0) return fail(nullptr, PSM_EINVAL, "devices[%d] = %d is negative", k, devices[k]);
    return create_multi(out, width, height, 0, max_disp, devices, n_devices, block_slices, map_bits);
}

int psm_create_range(psm_ctx** out, int width, int height, int min_disp, int max_disp, const int* devices, int n_devices,
                     int block_slices, int map_bits)
{
    if (!out) return fail(nullptr, PSM_EINVAL, "out is null");
    *out = nullptr;
    if (width < 1 || height < 1) return fail(nullptr, PSM_EINVAL, "bad geometry W=%d H=%d (need W,H>=1)", width, height);
    if (min_disp < 0) return fail(nullptr, PSM_EINVAL, "min_disp %d is negative", min_disp);
    if (max_disp < 2) return fail(nullptr, PSM_EINVAL, "max_disp %d is below 2", max_disp);
    if (min_disp >= max_disp)
        return fail(nullptr, PSM_EINVAL, "min_disp %d is not below max_disp %d: the range [min_disp, max_disp) is empty",
                    min_disp, max_disp);
    if (map_bits != 8 && map_bits != 16) return fail(nullptr, PSM_EINVAL, "map_bits must be 8 or 16 (got %d)", map_bits);
    const int dmax = map_bits == 8 ? MapFormat<uint8_t>::kMaxDisp : MapFormat<uint16_t>::kMaxDisp;
    if (max_disp > dmax)
        return fail(nullptr, PSM_EINVAL, "max_disp %d above %d: %d-bit maps hold disparities up to %d", max_disp, dmax,
                    map_bits, dmax - 1);
    const int n = max_disp - min_disp;
    if (n_devices < 1 || n_devices > kMaxRanks || n_devices > n)
        return fail(nullptr, PSM_EINVAL, "n_devices %d outside 1..%d (at most %d shards, each owning at least one of the %d "
                    "slices)", n_devices, std::min(kMaxRanks, n), kMaxRanks, n);
    if (block_slices < 0) return fail(nullptr, PSM_EINVAL, "block_slices %d is negative (0 = unblocked)", block_slices);
    if (!devices) return fail(nullptr, PSM_EINVAL, "devices is null");
    for (int k = 0; k < n_devices; ++k)
        if (devices[k] < 0) return fail(nullptr, PSM_EINVAL, "devices[%d] = %d is negative", k, devices[k]);
    if (n_devices == 1)
        return create_ctx(out, width, height, max_disp, min_disp, n, devices[0], map_bits / 8, std::min(block_slices, n),
                          min_disp);
    return create_multi(out, width, height, min_disp, max_disp, devices, n_devices, block_slices, map_bits);
}

int psm_destroy(psm_ctx* c)
{
    if (!c) return PSM_OK;
    if (c->nshards) {
        // every shard's work first: a shard's kernels store into the other shards' exchange blocks, and its copies read
        // the first shard's staging set
        for (int k = 0; k < c->nshards; ++k) {
            cudaSetDevice(c->shard[k]->device);
            cudaStreamSynchronize(c->shard[k]->stream);
            cudaStreamSynchronize(c->shard[k]->copy_stream);
        }
        for (int k = 0; k < c->nshards; ++k) {
            cudaSetDevice(c->shard[k]->device);
            if (c->ev_scattered[k]) cudaEventDestroy(c->ev_scattered[k]);
            if (c->ev_reduced[k]) cudaEventDestroy(c->ev_reduced[k]);
            if (c->ev_copied[k]) cudaEventDestroy(c->ev_copied[k]);
            if (c->ev_written[k]) cudaEventDestroy(c->ev_written[k]);
            if (k == 0 && c->ev_images) cudaEventDestroy(c->ev_images);
            psm_destroy(c->shard[k]);
        }
        cudaGetLastError();
        delete c;
        return PSM_OK;
    }
    cudaSetDevice(c->device);
    // every stream that may still run work on the buffers below: the caller's (psm_set_stream), the context's own one
    // (work enqueued before a psm_set_stream) and the copy stream
    if (c->stream) cudaStreamSynchronize(c->stream);
    if (c->own_stream) cudaStreamSynchronize(c->own_stream);
    if (c->copy_stream) cudaStreamSynchronize(c->copy_stream);
    for (int i = 0; i < c->p2p_nimported; ++i) cudaIpcCloseMemHandle(c->p2p_imported[i]);
    cudaFree(c->p2p_own);
    cudaFree(c->p2p_counter);
    for (int i = 0; i < c->nalloc; ++i) cudaFree(c->alloc[i]);
    for (int v = 0; v < 2; ++v) { cudaFree(c->stage_in[v]); cudaFree(c->stage_alt[v]); cudaFree(c->dis[v]); }
    if (c->up_done) cudaEventDestroy(c->up_done);
    if (c->host_copied) cudaEventDestroy(c->host_copied);
    for (int k = 0; k < 2; ++k) if (c->ingest_done[k]) cudaEventDestroy(c->ingest_done[k]);
    if (c->ev_user) cudaEventDestroy(c->ev_user);
    for (int k = 0; k < 2; ++k) if (c->ev_signal[k]) cudaEventDestroy(c->ev_signal[k]);
    if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
    cudaFree(c->slice_flags);
    cudaFree(c->ref_rs);
    cudaFree(c->ref_pl);
    cudaFree(c->guide_flags);
    cudaFree(c->pp_packed); cudaFree(c->pp_lut);
    cudaFree(c->fgf_lo[0]); cudaFree(c->fgf_lo[1]); cudaFree(c->fgf_mean); cudaFree(c->fgf_plan);
    cudaFree(c->sp_lab); cudaFree(c->sp_cnt);
    cudaFree(c->rp_min); cudaFree(c->rp_buf);
    for (int v = 0; v < 2; ++v) { cudaFree(c->rect_xy[v]); cudaFree(c->rect_a[v]); }
    for (int v = 0; v < 2; ++v) { cudaFree(c->dis_pp[v]); cudaFree(c->lr_valid[v]); cudaFree(c->run_keys[v]);
                                   cudaFree(c->pp_tmp[v]); cudaFree(c->dc_claims[v]);
                                   cudaFree(c->track[v]); cudaFree(c->ru_list[v]); cudaFree(c->ru_slots[v]);
                                   for (psm_ctx::OutState& o : c->outs) cudaFree(o.planes[v]); }
    for (int s = 0; s < kNumStages; ++s) {
        if (c->ev0[s]) cudaEventDestroy(c->ev0[s]);
        if (c->ev1[s]) cudaEventDestroy(c->ev1[s]);
    }
    if (c->own_stream) cudaStreamDestroy(c->own_stream);
    cudaGetLastError();
    delete c;
    return PSM_OK;
}

}  // extern "C"

// PSM_OPT_VIEWS, PSM_OPT_COSTS or PSM_OPT_RUNNER_UP changed: the frame's stages start again from psm_cost_const on the
// current images; nothing computed for the other setting (volumes, maps, masks, costs, runner-up, the guide of the right
// view) can be read or selected from
static void reset_stages(psm_ctx* c)
{
    c->stages_reset = true;
    c->guide_valid = false;
    c->have_cvc = false;
    c->filtered = false;
    c->have_maps = false;
    c->have_pp = false;
    c->lr_masks_ok = false;
    for (psm_ctx::OutState& o : c->outs) o.have = false;
}

// the output whose option is `key`, or -1
static int out_of_key(int key)
{
    for (int o = 0; o < kNumOuts; ++o)
        if (kSelOut[o].key == key) return o;
    return -1;
}

// output o = 1 on one context, a multi-device context's shards included: the planes it reads or writes.  The result
// planes where `result` (a single-device context, the first shard), then the output's own scratch: the costs' tracking
// planes on a blocked context; the runner-up's running lists on a blocked context and the slots of `nslots` shards (the
// first shard of a multi-device context).  Only allocates: a failure leaves the setting as it was.
static int alloc_out(psm_ctx* c, int o, bool result, int nslots)
{
    if (int rc = bind(c)) return rc;
    const size_t npix = (size_t)c->W * c->H, plane = npix * sizeof(float);
    for (int v = 0; v < 2; ++v) {
        if (result) PSM_CUDA(c, alloc_if_null(c->outs[o].planes[v], kSelOut[o].planes * plane));
        if (o == kOutCosts) {
            if (c->blk_slices) PSM_CUDA(c, alloc_if_null(c->track[v], c->track_planes() * plane));
        } else {
            if (nslots) PSM_CUDA(c, alloc_if_null(c->ru_slots[v], RunnerUpSlots::bytes(npix, nslots)));
            if (c->blk_slices) PSM_CUDA(c, alloc_if_null(c->ru_list[v], kListPlanes * plane));
        }
    }
    return PSM_OK;
}

// output o = value, its planes allocated: a blocked context's walk keeps the output's running state, so a change
// restarts the frame
static void apply_out(psm_ctx* c, int o, int value)
{
    if (value != c->outs[o].on) {
        reset_stages(c);
        c->outs[o].on = value;
    }
}

static int check_out_value(psm_ctx* c, int o, int value)
{
    if (value != 0 && value != 1) return fail(c, PSM_EINVAL, "%s must be 0 or 1 (got %d)", kSelOut[o].option, value);
    return PSM_OK;
}

extern "C" {

int psm_set_option(psm_ctx* c, int key, int value)
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    const int o = out_of_key(key);
    if (c->nshards) {
        if (key == PSM_OPT_P2P_SYNC)
            return reject_multi(c, "PSM_OPT_P2P_SYNC", "its shards' exchange is ordered by events, never by flags");
        if (o >= 0) {   // the shards own part of the range, the context as a whole spans it
            if (int rc = check_out_value(c, o, value)) return rc;
            // every shard's planes first (the first shard's hold the results and every shard's slot), then the setting
            // on all of them: a failed allocation changes no shard's setting
            for (int k = 0; value && k < c->nshards; ++k)
                if (int rc = alloc_out(c->shard[k], o, k == 0, k == 0 ? c->nshards : 0)) return relay(c, k, rc);
            for (int k = 0; k < c->nshards; ++k) apply_out(c->shard[k], o, value);
            c->outs[o].on = value;
            return PSM_OK;
        }
        if (int rc = forward(c, [&](psm_ctx* s) { return psm_set_option(s, key, value); })) return rc;
        if (key == PSM_OPT_VIEWS) c->views = value;   // the map calls check the right-view arguments on the context itself
        return PSM_OK;
    }
    if (o >= 0) {
        if (int rc = check_out_value(c, o, value)) return rc;
        if (value && !c->owns_problem())
            return fail(c, PSM_EINVAL, "%s on a context that owns slices [%d,%d) of %d: the %s may depend on slices "
                        "another context owns; use a context over the whole range (psm_create, psm_create_u16 / "
                        "psm_create_blocked over [0, max_disp), psm_create_multi or psm_create_range)", kSelOut[o].option,
                        c->d_begin, c->d_begin + c->d_count, c->D, kSelOut[o].noun);
        if (int rc = value ? alloc_out(c, o, true, 0) : PSM_OK) return rc;
        apply_out(c, o, value);
        return PSM_OK;
    }
    switch (key) {
    case PSM_OPT_VIEWS:
        if (value != PSM_VIEWS_LEFT && value != PSM_VIEWS_BOTH)
            return fail(c, PSM_EINVAL, "PSM_OPT_VIEWS must be PSM_VIEWS_LEFT (1) or PSM_VIEWS_BOTH (2) (got %d)", value);
        if (value != c->views) {
            c->views = value;
            reset_stages(c);
        }
        return PSM_OK;
    case PSM_OPT_CVF_MODE:
        if (value != PSM_CVF_EXACT && value != PSM_CVF_MIXED && value != PSM_CVF_NAIVE)
            return fail(c, PSM_EINVAL, "unknown CVF mode %d", value);
        c->cvf_mode = value;
        return PSM_OK;
    case PSM_OPT_GRAY_MODE:
        if (value != 0 && value != 1) return fail(c, PSM_EINVAL, "gray mode must be 0 or 1");
        c->gray_mode = value;
        return PSM_OK;
    case PSM_OPT_TIMING:
        c->timing = value ? 1 : 0;
        return PSM_OK;
    case PSM_OPT_P2P_SYNC:
        c->p2p_sync = value ? 1 : 0;
        return PSM_OK;
    case 100:  // streaming-kernel variant selector for tuning experiments
        c->cvf_variant = value;
        return PSM_OK;
    case 108:  // tuning: slices per CTA of the CVC kernel (0 = all)
        if (value < 0) return fail(c, PSM_EINVAL, "bad CVC chunk");
        c->cvc_chunk = value;
        return PSM_OK;
    case 107:  // tuning: rows per warp of the guide precompute (0 = default)
        if (value < 0 || value > 4096) return fail(c, PSM_EINVAL, "bad guide segment rows");
        c->guide_seg_rows = value;
        c->guide_valid = false;
        return PSM_OK;
    case 106:  // tuning: CVC kernel build (see psm_cost_const)
        c->cvc_variant = value;
        return PSM_OK;
    case 105:  // tuning: 1 = no packed remainder strips (one warp per slice for the last W % 112 columns, as in round 1)
        c->cvf_no_pack = value ? 1 : 0;
        return PSM_OK;
    case 104:  // undocumented: block->work remap so that co-resident CTAs are work neighbours (0/1)
        c->cvf_remap = value;
        return PSM_OK;
    case 103:  // undocumented: threads per CTA of the streaming kernel (64 / 96 / 128)
        if (value != 0 && (value % 32 != 0 || value < 32 || value > kCvfMaxThreads)) return fail(c, PSM_EINVAL, "bad thread count");
        c->cvf_threads = value;
        return PSM_OK;
    case 102:  // undocumented: extra dynamic shared memory per CTA (bytes) to throttle occupancy in experiments
        c->cvf_extra_smem = value;
        return PSM_OK;
    case 101:  // undocumented: rows per segment of the streaming kernel (0 = automatic)
        c->cvf_target_rows = value;
        return PSM_OK;
    default:
        return fail(c, PSM_EINVAL, "unknown option %d", key);
    }
}

int psm_set_guided_filter(psm_ctx* c, int window, float eps)
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    if (c->nshards) return forward(c, [&](psm_ctx* s) { return psm_set_guided_filter(s, window, eps); });
    if (window < 1 || window > kWinMax) return fail(c, PSM_EINVAL, "guided-filter window %d outside 1..%d", window, kWinMax);
    if (!(eps > 0.0f) || !std::isfinite(eps)) return fail(c, PSM_EINVAL, "guided-filter eps %g is not a finite value > 0", (double)eps);
    if (window != c->gif_win || eps != c->gif_eps) c->guide_valid = false;   // mean_I, var_I and the solve depend on both
    c->gif_win = window;
    c->gif_eps = eps;
    return PSM_OK;
}

int psm_set_matching_cost(psm_ctx* c, float alpha, float tau_color, float tau_grad)
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    if (c->nshards) return forward(c, [&](psm_ctx* s) { return psm_set_matching_cost(s, alpha, tau_color, tau_grad); });
    if (!(alpha >= 0.0f && alpha <= 1.0f)) return fail(c, PSM_EINVAL, "matching-cost alpha %g is not in [0, 1]", (double)alpha);
    if (!(tau_color >= 0.0f)) return fail(c, PSM_EINVAL, "colour threshold %g is not >= 0 or +inf", (double)tau_color);
    if (!(tau_grad >= 0.0f)) return fail(c, PSM_EINVAL, "gradient threshold %g is not >= 0 or +inf", (double)tau_grad);
    c->cost = CvcCost{alpha, tau_color, tau_grad};
    return PSM_OK;
}

int psm_set_post_filter(psm_ctx* c, int radius, float sigma, int iterations, int weight_type)
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    if (c->nshards) return forward(c, [&](psm_ctx* s) { return psm_set_post_filter(s, radius, sigma, iterations, weight_type); });
    if (radius < 1 || radius > kPpParamMaxRadius) return fail(c, PSM_EINVAL, "post-filter radius %d outside 1..%d", radius, kPpParamMaxRadius);
    if (!(sigma >= 0x1p-16f && sigma <= 0x1p16f)) return fail(c, PSM_EINVAL, "post-filter sigma %g outside [2^-16, 2^16]", (double)sigma);
    if (iterations < 1 || iterations > 16) return fail(c, PSM_EINVAL, "post-filter iterations %d outside 1..16", iterations);
    if (weight_type != PSM_WMF_EXP && weight_type != PSM_WMF_IV1 && weight_type != PSM_WMF_IV2 && weight_type != PSM_WMF_OFF)
        return fail(c, PSM_EINVAL, "post-filter weight type %d is not exp (0), iv1 (1), iv2 (2) or off (5)", weight_type);
    if (sigma != c->pp_sigma || weight_type != c->pp_type) c->pp_lut_valid = false;   // the table depends on both
    c->pp_radius = radius;
    c->pp_sigma = sigma;
    c->pp_iter = iterations;
    c->pp_type = weight_type;
    return PSM_OK;
}

int psm_set_rectify(psm_ctx* c, int src_width, int src_height, const int16_t* xy_left, size_t xy_left_step,
                    const uint16_t* a_left, size_t a_left_step, const int16_t* xy_right, size_t xy_right_step,
                    const uint16_t* a_right, size_t a_right_step)
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    const void* map[4] = {xy_left, a_left, xy_right, a_right};
    const size_t step[4] = {xy_left_step, a_left_step, xy_right_step, a_right_step};
    const bool off = !src_width && !src_height && std::none_of(map, map + 4, [](const void* p) { return p; }) &&
                     std::none_of(step, step + 4, [](size_t s) { return s; });
    if (!off) {
        if (src_width < 1 || src_width > 32767 || src_height < 1 || src_height > 32767)
            return fail(c, PSM_EINVAL, "rectify source size %d x %d: each side must lie in 1..32767 (the int16 coordinate "
                        "range), or both be 0 with null maps and zero steps to turn rectification off", src_width, src_height);
        for (int k = 0; k < 4; ++k) {
            const char* what = k % 2 ? "a (CV_16UC1)" : "xy (CV_16SC2)";
            const char* view = k < 2 ? "left" : "right";
            const size_t row = (size_t)c->W * (k % 2 ? 2 : 4);
            if (!map[k]) return fail(c, PSM_EINVAL, "null %s map of the %s view", what, view);
            if (step[k] < row)
                return fail(c, PSM_EINVAL, "row step %zu of the %s map of the %s view is below the %zu bytes of a row of W = %d "
                            "entries", step[k], what, view, row, c->W);
        }
    }
    if (c->up_pending)
        return fail(c, PSM_ESTATE, "psm_set_rectify with an asynchronous upload pending: call psm_set_images_commit first");
    if (c->nshards) {
        if (int rc = psm_set_rectify(c->shard[0], src_width, src_height, xy_left, xy_left_step, a_left, a_left_step, xy_right,
                                     xy_right_step, a_right, a_right_step))
            return relay(c, 0, rc);
        c->rect_sw = src_width;
        c->rect_sh = src_height;
        return PSM_OK;
    }
    if (int rc = bind(c)) return rc;
    // the last ingest may still read the maps and the staging sets, and the last upload may still fill a staging set
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    PSM_CUDA(c, cudaStreamSynchronize(c->copy_stream));
    if (off) {
        for (int v = 0; v < 2; ++v) {
            PSM_CUDA(c, cudaFree(c->rect_xy[v]));
            PSM_CUDA(c, cudaFree(c->rect_a[v]));
            c->rect_xy[v] = nullptr;
            c->rect_a[v] = nullptr;
        }
        c->rect_sw = c->rect_sh = 0;
        return PSM_OK;
    }
    const size_t n = (size_t)c->W * c->H;
    for (int v = 0; v < 2; ++v) {
        PSM_CUDA(c, alloc_if_null(c->rect_xy[v], n * sizeof(short2)));
        PSM_CUDA(c, alloc_if_null(c->rect_a[v], n * sizeof(uint16_t)));
    }
    // the staging sets hold a u8 source frame as well as a float frame of W x H, so no frame allocates
    const size_t need = std::max(c->stage_bytes, (size_t)src_width * src_height * 3);
    if (need > c->stage_bytes) {
        for (void** set : {c->stage_in, c->stage_alt})
            for (int v = 0; v < 2; ++v) {
                if (!set[v]) continue;
                void* p = nullptr;
                PSM_CUDA(c, cudaMalloc(&p, need));
                cudaFree(set[v]);
                set[v] = p;
            }
        c->stage_bytes = need;
    }
    for (int v = 0; v < 2; ++v) {
        PSM_CUDA(c, cudaMemcpy2DAsync(c->rect_xy[v], (size_t)c->W * sizeof(short2), map[2 * v], step[2 * v],
                                      (size_t)c->W * sizeof(short2), c->H, cudaMemcpyHostToDevice, c->stream));
        PSM_CUDA(c, cudaMemcpy2DAsync(c->rect_a[v], (size_t)c->W * sizeof(uint16_t), map[2 * v + 1], step[2 * v + 1],
                                      (size_t)c->W * sizeof(uint16_t), c->H, cudaMemcpyHostToDevice, c->stream));
    }
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    c->rect_sw = src_width;
    c->rect_sh = src_height;
    return PSM_OK;
}

int psm_set_stream(psm_ctx* c, void* cuda_stream)
{
    if (is_multi(c)) return reject_multi(c, "psm_set_stream", "a stream belongs to one device, the context spans several");
    if (int rc = bind(c)) return rc;
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    c->stream = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : c->own_stream;
    return PSM_OK;
}

int psm_set_images(psm_ctx* c, const float* left, size_t left_step, const float* right, size_t right_step)
{
    PlanesSrc src[2];
    if (int rc = check_interleaved(c, PSM_PIX_F32, false, left, left_step, right, right_step, src)) return rc;
    return set_images(c, Frame::host, PSM_PIX_F32, src);
}

int psm_set_images_u8(psm_ctx* c, const uint8_t* left, size_t left_step, const uint8_t* right, size_t right_step)
{
    PlanesSrc src[2];
    if (int rc = check_interleaved(c, PSM_PIX_U8, false, left, left_step, right, right_step, src)) return rc;
    return set_images(c, Frame::host, PSM_PIX_U8, src);
}

int psm_set_images_device(psm_ctx* c, const float* d_left, size_t left_step, const float* d_right, size_t right_step)
{
    PlanesSrc src[2];
    if (int rc = check_interleaved(c, PSM_PIX_F32, true, d_left, left_step, d_right, right_step, src)) return rc;
    return set_images(c, Frame::device, PSM_PIX_F32, src);
}

int psm_set_images_device_planes(psm_ctx* c, int pix_type, const void* const left[3], const void* const right[3],
                                 size_t row_step, size_t col_step)
{
    PlanesSrc src[2];
    if (int rc = check_planes(c, pix_type, left, right, row_step, col_step, src)) return rc;
    return set_images(c, Frame::planes, pix_type, src);
}

// Events only: the caller's stream is recorded once (on the context's first device) and every stream of the context
// waits for that record.
int psm_wait_stream(psm_ctx* c, void* cuda_stream)
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    psm_ctx* parts[kMaxRanks];
    const int n = ctx_parts(c, parts);
    if (int rc = bind(parts[0])) return rc;
    PSM_CUDA(c, cudaEventRecord(parts[0]->ev_user, static_cast<cudaStream_t>(cuda_stream)));
    for (int k = 0; k < n; ++k) {
        if (int rc = bind(parts[k])) return rc;
        PSM_CUDA(c, cudaStreamWaitEvent(parts[k]->stream, parts[0]->ev_user, 0));
        PSM_CUDA(c, cudaStreamWaitEvent(parts[k]->copy_stream, parts[0]->ev_user, 0));
    }
    return PSM_OK;
}

// Events only: every stream of the context is recorded and the caller's stream waits for each record.
int psm_signal_stream(psm_ctx* c, void* cuda_stream)
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    psm_ctx* parts[kMaxRanks];
    const int n = ctx_parts(c, parts);
    const cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    for (int k = 0; k < n; ++k) {
        psm_ctx* p = parts[k];
        if (int rc = bind(p)) return rc;
        PSM_CUDA(c, cudaEventRecord(p->ev_signal[0], p->stream));
        PSM_CUDA(c, cudaEventRecord(p->ev_signal[1], p->copy_stream));
    }
    if (int rc = bind(parts[0])) return rc;   // the caller's stream lives on the first device
    for (int k = 0; k < n; ++k)
        for (int e = 0; e < 2; ++e) PSM_CUDA(c, cudaStreamWaitEvent(s, parts[k]->ev_signal[e], 0));
    return PSM_OK;
}

int psm_set_images_async(psm_ctx* c, const float* left, size_t left_step, const float* right, size_t right_step)
{
    return set_images_async(c, PSM_PIX_F32, "psm_set_images_async", [&](PlanesSrc* src) {
        return check_interleaved(c, PSM_PIX_F32, false, left, left_step, right, right_step, src);
    });
}

int psm_set_images_u8_async(psm_ctx* c, const uint8_t* left, size_t left_step, const uint8_t* right, size_t right_step)
{
    return set_images_async(c, PSM_PIX_U8, "psm_set_images_u8_async", [&](PlanesSrc* src) {
        return check_interleaved(c, PSM_PIX_U8, false, left, left_step, right, right_step, src);
    });
}

int psm_set_images_yuv(psm_ctx* c, int format, const uint8_t* left, size_t left_step, const uint8_t* right,
                       size_t right_step)
{
    PlanesSrc src[2];
    if (int rc = check_yuv_host(c, format, left, left_step, right, right_step, src)) return rc;
    return set_images(c, Frame::host, kFmtYuv + format, src);
}

int psm_set_images_yuv_async(psm_ctx* c, int format, const uint8_t* left, size_t left_step, const uint8_t* right,
                             size_t right_step)
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    return set_images_async(c, kFmtYuv + format, "psm_set_images_yuv_async", [&](PlanesSrc* src) {
        return check_yuv_host(c, format, left, left_step, right, right_step, src);
    });
}

int psm_set_images_device_yuv(psm_ctx* c, int sampling, const void* const left[3], const void* const right[3],
                              size_t y_row_step, size_t y_col_step, size_t c_row_step, size_t c_col_step)
{
    YuvSrc src[2];
    if (int rc = check_yuv_device(c, sampling, left, right, y_row_step, y_col_step, c_row_step, c_col_step, src)) return rc;
    return set_images_device_converted(c, src);
}

int psm_set_images_bayer(psm_ctx* c, int pattern, int method, const uint8_t* left, size_t left_step, const uint8_t* right,
                         size_t right_step)
{
    PlanesSrc src[2];
    if (int rc = check_bayer_host(c, pattern, method, left, left_step, right, right_step, src)) return rc;
    return set_images(c, Frame::host, bayer_fmt(pattern, method), src);
}

int psm_set_images_bayer_async(psm_ctx* c, int pattern, int method, const uint8_t* left, size_t left_step,
                               const uint8_t* right, size_t right_step)
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    return set_images_async(c, bayer_fmt(pattern, method), "psm_set_images_bayer_async", [&](PlanesSrc* src) {
        return check_bayer_host(c, pattern, method, left, left_step, right, right_step, src);
    });
}

int psm_set_images_device_bayer(psm_ctx* c, int pattern, int method, const void* left, const void* right, size_t row_step,
                                size_t col_step)
{
    BayerSrc src[2];
    if (int rc = check_bayer_device(c, pattern, method, left, right, row_step, col_step, src)) return rc;
    return set_images_device_converted(c, src);
}

int psm_set_images_commit(psm_ctx* c)
{
    if (is_multi(c)) return reject_multi(c, "psm_set_images_commit", "the asynchronous upload pipeline is not available on it; use psm_set_images / _u8");
    if (int rc = bind(c)) return rc;
    if (!c->up_pending) return fail(c, PSM_ESTATE, "psm_set_images_commit without a pending psm_set_images_async");
    const int set = c->stage_cur ^ 1, fmt = c->up_pending;
    if (int rc = stage_begin(c, 0)) return rc;
    c->stage_cur = set;
    c->up_pending = 0;
    if (int rc = ingest_staged(c, set, fmt, c->up_done)) return rc;
    if (int rc = stage_end(c, 0)) return rc;
    // the caller may reuse its host buffers once this returns: wait for the copy that reads them (it may still be
    // waiting for the frame before last to leave this staging set); the ingest kernels are already queued behind it
    PSM_CUDA(c, cudaEventSynchronize(c->up_done));
    return PSM_OK;
}

int psm_cost_const(psm_ctx* c)
{
    if (is_multi(c)) return forward(c, [](psm_ctx* s) { return psm_cost_const(s); });
    if (int rc = bind(c)) return rc;
    if (!c->have_images) return fail(c, PSM_ESTATE, "psm_cost_const before psm_set_images");
    if (int rc = stage_begin(c, 1)) return rc;
    c->res = block_at(c, c->d_begin);   // a blocked context's first block; the filter stages build the others
    if (int rc = launch_cvc(c)) return rc;
    if (int rc = clear_slice_flags(c)) return rc;
    c->have_cvc = true;
    c->filtered = false;
    c->stages_reset = false;
    return stage_end(c, 1);
}

int psm_cost_filter(psm_ctx* c)
{
    return filter_stage(c, "psm_cost_filter", check_cvf_mode, ensure_guide, cvf_block);
}

// DispEst::CostFilter_FGF (reference src/DispEst.cpp:281-296): Fast Guided Filter with sub-sampling rate s.  An unblocked
// context computes each view's low-resolution guide just before that view's slices; a blocked one computes both guides
// before its walk.
int psm_cost_filter_fgf(psm_ctx* c, int s)
{
    return filter_stage(c, "psm_cost_filter_fgf", [s](psm_ctx* c) { return ensure_fgf(c, s); },
                        [s](psm_ctx* c) { return fgf_views(c, s, c->blk_slices != 0, false); },
                        [s](psm_ctx* c) { return fgf_views(c, s, c->blk_slices == 0, true); });
}

}  // extern "C"

// the WTA of both views into the context's maps of type T
template <typename T>
static int select_maps(psm_ctx* c)
{
    if (c->blk_slices) {   // a blocked context's selection is in its running keys: reduce them as one rank's
        const size_t npix = (size_t)c->W * c->H;
        for (int v = 0; v < c->views; ++v) {
            keys_reduce_kernel<T><<<(unsigned)((npix + 255) / 256), 256, 0, c->stream>>>(c->run_keys[v], 1, npix,
                                                                                         reinterpret_cast<T*>(c->dis[v]));
            PSM_LAUNCH_CHECK(c);
        }
        return PSM_OK;
    }
    for (int v = 0; v < c->views; ++v) {
        dim3 blk(256), grd(((c->W + 3) / 4 + 255) / 256, c->H);
        // with the runner-up, the map and the runner-up in one read of the volume
        (c->outs[kOutRunnerUp].on ? wta_kernel<T, true> : wta_kernel<T, false>)<<<grd, blk, 0, c->stream>>>(
            c->vol[v], c->W, c->H, c->Wp, c->d_begin, c->d_count, reinterpret_cast<T*>(c->dis[v]), nullptr,
            out_planes(c, kOutRunnerUp, v));
        PSM_LAUNCH_CHECK(c);
    }
    return PSM_OK;
}

// psm_disp_select[_u16][_async]: select on the device, copy both maps to the host, then wait for them unless async
template <typename T>
static int disp_select(psm_ctx* c, T* left, size_t left_step, T* right, size_t right_step, bool sync)
{
    if (int rc = sync ? check_map_format<T>(c, "psm_disp_select", "psm_disp_select_u16")
                      : check_map_format<T>(c, "psm_disp_select_async", "psm_disp_select_u16_async")) return rc;
    if (int rc = check_map_dst(c, "psm_disp_select", left, left_step, right, right_step)) return rc;
    if (int rc = psm_disp_select_device(c)) return rc;
    return copy_maps_out(c, c->dis, left, left_step, right, right_step, cudaMemcpyDeviceToHost, sync);
}

template <typename T>
static int disp_reduce_keys(psm_ctx* c, const uint64_t* d_gathered_left, const uint64_t* d_gathered_right, int nranks,
                            T* left, size_t left_step, T* right, size_t right_step)
{
    if (is_multi(c)) return reject_multi(c, sizeof(T) == 1 ? "psm_disp_reduce_keys" : "psm_disp_reduce_keys_u16", "the context already spans the whole disparity range; use psm_disp_select*");
    if (int rc = check_map_format<T>(c, "psm_disp_reduce_keys", "psm_disp_reduce_keys_u16")) return rc;
    if (int rc = bind(c)) return rc;
    if (int rc = check_stages_reset(c, "psm_disp_reduce_keys")) return rc;
    if (int rc = check_right_arg(c, d_gathered_right, "psm_disp_reduce_keys")) return rc;
    if (int rc = check_right_arg(c, right, "psm_disp_reduce_keys")) return rc;
    const bool to_host = left && (right || c->views == 1);   // a null map pointer: the maps stay on the device
    if (int rc = to_host ? check_map_dst(c, "psm_disp_reduce_keys", left, left_step, right, right_step) : PSM_OK) return rc;
    if (!d_gathered_left || (c->views == 2 && !d_gathered_right) || nranks < 1) return fail(c, PSM_EINVAL, "bad gathered keys");
    const uint64_t* g[2] = {d_gathered_left, d_gathered_right};
    const size_t npix = (size_t)c->W * c->H;
    for (int v = 0; v < c->views; ++v) {
        keys_reduce_kernel<T><<<(unsigned)((npix + 255) / 256), 256, 0, c->stream>>>(
            reinterpret_cast<const unsigned long long*>(g[v]), nranks, npix, reinterpret_cast<T*>(c->dis[v]));
        PSM_LAUNCH_CHECK(c);
    }
    selection_ran(c, true);
    if (to_host) return copy_maps_out(c, c->dis, left, left_step, right, right_step, cudaMemcpyDeviceToHost, true);
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    return PSM_OK;
}

extern "C" {

static int multi_select(psm_ctx* c);   // below

int psm_disp_select_device(psm_ctx* c)
{
    if (is_multi(c)) return multi_select(c);
    if (int rc = bind(c)) return rc;
    if (!c->owns_problem())
        return fail(c, PSM_ESTATE, "psm_disp_select on a sharded context: use psm_disp_select_keys + psm_disp_reduce_keys");
    if (!c->filtered) return fail(c, PSM_ESTATE, "psm_disp_select before psm_cost_filter");
    if (int rc = stage_begin(c, 3)) return rc;
    if (int rc = c->map_bytes == 2 ? select_maps<uint16_t>(c) : select_maps<uint8_t>(c)) return rc;
    selection_ran(c, true);
    for (int o = 0; o < kNumOuts; ++o) {
        if (!c->outs[o].on) continue;
        for (int v = 0; v < c->views; ++v)
            if (int rc = launch_out_write(c, o, v, c->dis[v], c, 0, 0)) return rc;
        c->outs[o].have = true;
    }
    return stage_end(c, 3);
}

int psm_disp_select(psm_ctx* c, uint8_t* left, size_t left_step, uint8_t* right, size_t right_step)
{
    return disp_select(c, left, left_step, right, right_step, true);
}

int psm_disp_select_async(psm_ctx* c, uint8_t* left, size_t left_step, uint8_t* right, size_t right_step)
{
    return disp_select(c, left, left_step, right, right_step, false);
}

int psm_disp_select_u16(psm_ctx* c, uint16_t* left, size_t left_step, uint16_t* right, size_t right_step)
{
    return disp_select(c, left, left_step, right, right_step, true);
}

int psm_disp_select_u16_async(psm_ctx* c, uint16_t* left, size_t left_step, uint16_t* right, size_t right_step)
{
    return disp_select(c, left, left_step, right, right_step, false);
}

int psm_disp_select_keys(psm_ctx* c, uint64_t* d_keys_left, uint64_t* d_keys_right)
{
    if (is_multi(c)) return reject_multi(c, "psm_disp_select_keys", "the context already spans the whole disparity range; use psm_disp_select*");
    if (int rc = bind(c)) return rc;
    if (int rc = check_right_arg(c, d_keys_right, "psm_disp_select_keys")) return rc;
    if (!d_keys_left || (c->views == 2 && !d_keys_right)) return fail(c, PSM_EINVAL, "null key buffer");
    if (!c->filtered) return fail(c, PSM_ESTATE, "psm_disp_select_keys before psm_cost_filter");
    if (int rc = stage_begin(c, 3)) return rc;
    for (psm_ctx::OutState& o : c->outs) o.have = false;   // keys carry no output beside the winner
    uint64_t* keys[2] = {d_keys_left, d_keys_right};
    if (c->blk_slices) {   // the running keys are this context's minima already
        for (int v = 0; v < c->views; ++v)
            PSM_CUDA(c, cudaMemcpyAsync(keys[v], c->run_keys[v], (size_t)c->W * c->H * sizeof(uint64_t),
                                        cudaMemcpyDeviceToDevice, c->stream));
        return stage_end(c, 3);
    }
    for (int v = 0; v < c->views; ++v) {   // keys only, on either map format
        dim3 blk(256), grd(((c->W + 3) / 4 + 255) / 256, c->H);
        wta_kernel<uint8_t, false><<<grd, blk, 0, c->stream>>>(c->vol[v], c->W, c->H, c->Wp, c->d_begin, c->d_count, nullptr,
                                                               reinterpret_cast<unsigned long long*>(keys[v]), CostPlanes{});
        PSM_LAUNCH_CHECK(c);
    }
    return stage_end(c, 3);
}

int psm_disp_reduce_keys(psm_ctx* c, const uint64_t* d_gathered_left, const uint64_t* d_gathered_right, int nranks,
                         uint8_t* left, size_t left_step, uint8_t* right, size_t right_step)
{
    return disp_reduce_keys(c, d_gathered_left, d_gathered_right, nranks, left, left_step, right, right_step);
}

int psm_disp_reduce_keys_u16(psm_ctx* c, const uint64_t* d_gathered_left, const uint64_t* d_gathered_right, int nranks,
                             uint16_t* left, size_t left_step, uint16_t* right, size_t right_step)
{
    return disp_reduce_keys(c, d_gathered_left, d_gathered_right, nranks, left, left_step, right, right_step);
}

int psm_p2p_create_buffer(psm_ctx* c, int nranks, void** d_buffer)
{
    if (is_multi(c)) return reject_multi(c, "psm_p2p_create_buffer", "the context already spans the whole disparity range; use psm_disp_select*");
    if (int rc = bind(c)) return rc;
    if (nranks < 1 || nranks > kMaxRanks || !d_buffer) return fail(c, PSM_EINVAL, "bad nranks %d (1..%d)", nranks, kMaxRanks);
    if (c->p2p_own) { cudaFree(c->p2p_own); c->p2p_own = nullptr; }
    for (int i = 0; i < c->p2p_nimported; ++i) cudaIpcCloseMemHandle(c->p2p_imported[i]);   // peers of a previous exchange set-up
    c->p2p_nimported = 0;
    for (int r = 0; r < kMaxRanks; ++r) c->p2p_peer[r] = nullptr;
    const P2pLayout L = p2p_layout(c, nranks);
    PSM_CUDA(c, cudaMalloc(&c->p2p_own, L.bytes));
    PSM_CUDA(c, cudaMemsetAsync(c->p2p_own, 0xff, L.flags_at, c->stream));   // keys and maps
    PSM_CUDA(c, cudaMemsetAsync(c->p2p_own + L.flags_at, 0, L.bytes - L.flags_at, c->stream));
    if (!c->p2p_counter) PSM_CUDA(c, cudaMalloc(&c->p2p_counter, sizeof(unsigned)));
    PSM_CUDA(c, cudaMemsetAsync(c->p2p_counter, 0, sizeof(unsigned), c->stream));
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    c->p2p_nranks = nranks;
    c->p2p_seq = 0;
    c->p2p_seq_right = 0;
    c->p2p_right_current = false;
    c->p2p_waited_seq = 0;
    *d_buffer = c->p2p_own;
    return PSM_OK;
}

int psm_ipc_export(psm_ctx* c, void* d_ptr, unsigned char handle_out[64])
{
    if (is_multi(c)) return reject_multi(c, "psm_ipc_export", "the context already spans the whole disparity range; use psm_disp_select*");
    if (int rc = bind(c)) return rc;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    cudaIpcMemHandle_t h;
    PSM_CUDA(c, cudaIpcGetMemHandle(&h, d_ptr));
    memcpy(handle_out, &h, 64);
    return PSM_OK;
}

int psm_ipc_import(psm_ctx* c, const unsigned char handle[64], void** d_ptr)
{
    if (is_multi(c)) return reject_multi(c, "psm_ipc_import", "the context already spans the whole disparity range; use psm_disp_select*");
    if (int rc = bind(c)) return rc;
    if (c->p2p_nimported >= kMaxRanks) return fail(c, PSM_EINVAL, "too many imported buffers");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    PSM_CUDA(c, cudaIpcOpenMemHandle(d_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    c->p2p_imported[c->p2p_nimported++] = *d_ptr;
    return PSM_OK;
}

int psm_p2p_set_peers(psm_ctx* c, void* const* d_buffers, int nranks, int rank)
{
    if (is_multi(c)) return reject_multi(c, "psm_p2p_set_peers", "the context already spans the whole disparity range; use psm_disp_select*");
    if (!c || !d_buffers) return fail(c, PSM_EINVAL, "null argument");
    if (nranks != c->p2p_nranks || rank < 0 || rank >= nranks) return fail(c, PSM_EINVAL, "bad peers (nranks %d, rank %d)", nranks, rank);
    for (int r = 0; r < nranks; ++r) {
        if (!d_buffers[r]) return fail(c, PSM_EINVAL, "null buffer for rank %d", r);
        c->p2p_peer[r] = static_cast<unsigned char*>(d_buffers[r]);
    }
    c->p2p_rank = rank;
    return PSM_OK;
}

static void p2p_fill(const psm_ctx* c, int view, P2pPeers& peers)
{
    const P2pLayout L = p2p_layout(c, c->p2p_nranks);
    peers.nranks = c->p2p_nranks; peers.rank = c->p2p_rank; peers.chunk = (unsigned)L.chunk;
    peers.counter = c->p2p_counter;
    // each view's flags carry the number of the last frame that exchanged that view
    peers.seq = c->p2p_sync ? (view ? c->p2p_seq_right : c->p2p_seq) : 0u;
    for (int r = 0; r < kMaxRanks; ++r) {
        unsigned char* base = r < c->p2p_nranks ? c->p2p_peer[r] : nullptr;
        peers.keys[r] = base ? L.keys(base, view) : nullptr;
        peers.maps[r] = base ? L.maps(base, view) : nullptr;
        peers.flags[r] = base ? L.flags(base, view) : nullptr;
    }
}

// the scatter of the fused exchange over this context's slices: wta_scatter_kernel over the filtered volumes, or, for a
// blocked shard of a multi-device context, keys_scatter_kernel over its running keys
static int p2p_scatter(psm_ctx* c)
{
    c->p2p_seq++;   // one sequence number per frame, identical on every rank (all ranks run the same frames and views)
    if (c->views == 2) c->p2p_seq_right++;
    c->p2p_right_current = c->views == 2;
    for (int v = 0; v < c->views; ++v) {
        P2pPeers peers;
        p2p_fill(c, v, peers);
        dim3 blk(256), grd(((c->W + 3) / 4 + 255) / 256, (c->H + kScatterRows - 1) / kScatterRows);
        if (c->blk_slices)
            keys_scatter_kernel<<<grd, blk, 0, c->stream>>>(c->run_keys[v], c->W, c->H, peers);
        else
            wta_scatter_kernel<<<grd, blk, 0, c->stream>>>(c->vol[v], c->W, c->H, c->Wp, c->d_begin, c->d_count, peers);
        PSM_LAUNCH_CHECK(c);
    }
    selection_ran(c, false);
    return PSM_OK;
}

int psm_disp_select_keys_p2p(psm_ctx* c)
{
    if (is_multi(c)) return reject_multi(c, "psm_disp_select_keys_p2p", "the context already spans the whole disparity range; use psm_disp_select*");
    if (int rc = bind(c)) return rc;
    if (c->blk_slices)
        return fail(c, PSM_EINVAL, "psm_disp_select_keys_p2p on a blocked context: the fused exchange scans whole volumes, a "
                    "blocked context holds one block; use psm_disp_select_keys + psm_disp_reduce_keys");
    if (!c->p2p_own || !c->p2p_peer[0]) return fail(c, PSM_ESTATE, "psm_p2p_create_buffer / psm_p2p_set_peers first");
    if (!c->filtered) return fail(c, PSM_ESTATE, "psm_disp_select_keys_p2p before psm_cost_filter");
    if (int rc = stage_begin(c, 3)) return rc;
    if (int rc = p2p_scatter(c)) return rc;
    return stage_end(c, 3);
}

int psm_disp_reduce_p2p(psm_ctx* c)
{
    if (is_multi(c)) return reject_multi(c, "psm_disp_reduce_p2p", "the context already spans the whole disparity range; use psm_disp_select*");
    if (int rc = bind(c)) return rc;
    if (!c->p2p_own || !c->p2p_peer[0]) return fail(c, PSM_ESTATE, "no exchange block");
    if (int rc = check_stages_reset(c, "psm_disp_reduce_p2p")) return rc;
    const unsigned npix = (unsigned)((size_t)c->W * c->H);
    const auto reduce = c->map_bytes == 2 ? chunk_reduce_kernel<uint16_t> : chunk_reduce_kernel<uint8_t>;
    for (int v = 0; v < c->views; ++v) {
        P2pPeers peers;
        p2p_fill(c, v, peers);
        reduce<<<(peers.chunk + 255) / 256, 256, 0, c->stream>>>(peers, npix);
        PSM_LAUNCH_CHECK(c);
    }
    selection_ran(c, false);
    return PSM_OK;
}

// the exchange block's right map is from an earlier frame than its left map (the last exchanged frame was left-only)
static int check_p2p_right_map(psm_ctx* c, const char* call)
{
    if (c->views == 2 && c->p2p_seq > 0 && !c->p2p_right_current)
        return fail(c, PSM_ESTATE, "%s: the exchanged right map is from a frame before the last left-only one; run a "
                    "selection stage with PSM_VIEWS_BOTH first", call);
    return PSM_OK;
}

// the exchanged maps are complete once every rank's DONE flag carries this frame's number: enqueue the wait in front
// of a consumer of the maps (once per frame)
static int p2p_wait_done(psm_ctx* c)
{
    if (!exchanged(c) || !c->p2p_sync || c->p2p_waited_seq == c->p2p_seq) return PSM_OK;
    const P2pLayout L = p2p_layout(c, c->p2p_nranks);
    unsigned char* own = c->p2p_peer[c->p2p_rank];
    if (c->views == 2 && c->p2p_seq_right == c->p2p_seq) {
        p2p_wait_done_kernel<<<1, 32, 0, c->stream>>>(L.flags(own, 0), c->p2p_nranks, c->p2p_seq);
        PSM_LAUNCH_CHECK(c);
    } else {   // the views' flags carry different frame numbers: one wait per view, nranks threads (the first view's words)
        for (int v = 0; v < c->views; ++v) {
            p2p_wait_done_kernel<<<1, c->p2p_nranks, 0, c->stream>>>(L.flags(own, v), c->p2p_nranks,
                                                                     v ? c->p2p_seq_right : c->p2p_seq);
            PSM_LAUNCH_CHECK(c);
        }
    }
    c->p2p_waited_seq = c->p2p_seq;
    return PSM_OK;
}

// Selection on a multi-device context: the fused exchange's two kernels on every shard, which never wait on a flag
// (PSM_OPT_P2P_SYNC = 0), ordered by events across the shards' streams instead.  The hazards, for frame f:
//   1. every shard's scatter overwrites key slots that every shard's reduce of frame f - 1 read: it waits for them;
//   2. every shard's reduce reads the slots of every shard's scatter of frame f: it waits for them;
//   3. whatever reads the first shard's complete maps after the select (D2H, post-filter, left-right check, psm_sync in
//      front of a psm_device_ptr user) runs on the first shard's stream, which waits for every shard's reduce;
//   4. every reduce writes the first shard's maps, which what the first shard enqueued before this select (a previous
//      post-filter, an asynchronous D2H) may still read: the wait of 2 on the first shard's scatter, queued behind
//      that work, covers it.
// With outputs on (kSelOut), every shard then writes, per enabled output, what it owns into the first shard: the cost
// entries into its cost planes, its runner-up pick into its own slot, which the first shard then reduces into its
// runner-up planes:
//   5. shard k's writes read its copy of the complete maps, which every shard's reduce writes: they wait for them;
//   6. the first shard's stream waits for every shard's writes.  It carries the slot reduce and every reader of the
//      result planes (psm_copy_*_device, psm_read_*), queued behind them;
//   7. the writes overwrite cost planes and slots that a copy-out or the slot reduce of frame f - 1 on the first shard's
//      stream may still read: each shard's writes follow its reduce, which waits for the first shard's scatter (2),
//      queued behind that work;
//   8. a shard's writes read its map, which the next frame's reduces overwrite: they wait for that shard's next scatter
//      (2), queued behind the writes; and the volumes, tracking planes or running lists they read are rewritten only by
//      later stages on its own stream.
// Every cost entry and every slot has one writer, and the slot reduce takes the first slot of the lowest key, so the
// result does not depend on the order in which the writes land.  The first shard's result planes are written by these
// writes and the slot reduce alone, never by a filter stage (its tracking planes and running lists are separate), so they
// hold frame f's outputs until the next select, as on a single-device context.
// No kernel waits for another queued behind it, so shards on one device are as safe as shards on several.
static int multi_select(psm_ctx* c)
{
    const int n = c->nshards;
    for (int k = 0; k < n; ++k)
        if (!c->shard[k]->filtered) return fail(c, PSM_ESTATE, "psm_disp_select before psm_cost_filter (shard %d)", k);
    for (int k = 0; k < n; ++k) {
        psm_ctx* s = c->shard[k];
        if (int rc = bind(s)) return relay(c, k, rc);
        if (c->reduced_valid)
            for (int j = 0; j < n; ++j)
                if (j != k) PSM_CUDA(c, cudaStreamWaitEvent(s->stream, c->ev_reduced[j], 0));   // 1
        if (k == 0)
            if (int rc = stage_begin(s, 3)) return relay(c, k, rc);
        if (int rc = p2p_scatter(s)) return relay(c, k, rc);
        PSM_CUDA(c, cudaEventRecord(c->ev_scattered[k], s->stream));
    }
    for (int k = 0; k < n; ++k) {
        psm_ctx* s = c->shard[k];
        if (int rc = bind(s)) return relay(c, k, rc);
        for (int j = 0; j < n; ++j)
            if (j != k) PSM_CUDA(c, cudaStreamWaitEvent(s->stream, c->ev_scattered[j], 0));   // 2, and 4
        if (int rc = psm_disp_reduce_p2p(s)) return relay(c, k, rc);
        PSM_CUDA(c, cudaEventRecord(c->ev_reduced[k], s->stream));
    }
    c->reduced_valid = true;
    psm_ctx* s0 = c->shard[0];
    for (int k = 0; c->outs_on() && k < n; ++k) {
        psm_ctx* s = c->shard[k];
        if (int rc = bind(s)) return relay(c, k, rc);
        for (int j = 0; j < n; ++j)
            if (j != k) PSM_CUDA(c, cudaStreamWaitEvent(s->stream, c->ev_reduced[j], 0));   // 5
        const P2pLayout L = p2p_layout(s, s->p2p_nranks);
        for (int o = 0; o < kNumOuts; ++o)
            for (int v = 0; c->outs[o].on && v < s->views; ++v)   // peer stores between distinct devices
                if (int rc = launch_out_write(s, o, v, L.maps(s->p2p_own, v), s0, k, n)) return relay(c, k, rc);
        PSM_CUDA(c, cudaEventRecord(c->ev_written[k], s->stream));
    }
    if (int rc = bind(s0)) return relay(c, 0, rc);
    for (int j = 1; j < n; ++j) PSM_CUDA(c, cudaStreamWaitEvent(s0->stream, c->ev_reduced[j], 0));   // 3
    for (int j = 1; c->outs_on() && j < n; ++j) PSM_CUDA(c, cudaStreamWaitEvent(s0->stream, c->ev_written[j], 0));   // 6
    if (c->outs[kOutRunnerUp].on) {
        const size_t npix = (size_t)s0->W * s0->H;
        for (int v = 0; v < s0->views; ++v) {
            runner_up_reduce_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, s0->stream>>>(runner_up_slots(s0, v, n),
                                                                                           out_planes(s0, kOutRunnerUp, v));
            PSM_LAUNCH_CHECK(s0);
        }
    }
    for (int o = 0; o < kNumOuts; ++o) s0->outs[o].have = c->outs[o].on;   // its reduce cleared them (selection_ran)
    return relay(c, 0, stage_end(s0, 3));
}

}  // extern "C"

template <typename T>
static int disp_fetch_p2p(psm_ctx* c, T* left, size_t left_step, T* right, size_t right_step)
{
    if (is_multi(c)) return reject_multi(c, sizeof(T) == 1 ? "psm_disp_fetch_p2p" : "psm_disp_fetch_p2p_u16", "the context already spans the whole disparity range; use psm_disp_select*");
    if (int rc = check_map_format<T>(c, "psm_disp_fetch_p2p", "psm_disp_fetch_p2p_u16")) return rc;
    if (int rc = bind(c)) return rc;
    if (!c->p2p_own) return fail(c, PSM_ESTATE, "no exchange block");
    if (int rc = check_stages_reset(c, "psm_disp_fetch_p2p")) return rc;
    if (int rc = check_map_dst(c, "psm_disp_fetch_p2p", left, left_step, right, right_step)) return rc;
    if (int rc = check_p2p_right_map(c, "psm_disp_fetch_p2p")) return rc;
    if (int rc = p2p_wait_done(c)) return rc;
    const P2pLayout L = p2p_layout(c, c->p2p_nranks);
    const uint8_t* maps[2] = {L.maps(c->p2p_own, 0), L.maps(c->p2p_own, 1)};
    return copy_maps_out(c, maps, left, left_step, right, right_step, cudaMemcpyDeviceToHost, true);
}

extern "C" {

int psm_disp_fetch_p2p(psm_ctx* c, uint8_t* left, size_t left_step, uint8_t* right, size_t right_step)
{
    return disp_fetch_p2p(c, left, left_step, right, right_step);
}

int psm_disp_fetch_p2p_u16(psm_ctx* c, uint16_t* left, size_t left_step, uint16_t* right, size_t right_step)
{
    return disp_fetch_p2p(c, left, left_step, right, right_step);
}

// ---- post-processing (PP::processDM) ----------------------------------------------------------------
// the maps of the last selection stage for psm_post_process* and psm_copy_maps_device, under the exchanged-map rules of
// psm_disp_fetch_p2p; the caller enqueues p2p_wait_done before it reads them
static int selection_maps(psm_ctx* c, const char* call, const uint8_t* maps[2])
{
    if (!exchanged(c)) {
        if (!c->have_maps) return fail(c, PSM_ESTATE, "%s before a disparity-selection stage", call);
        maps[0] = c->dis[0]; maps[1] = c->dis[1];
        return PSM_OK;
    }
    const P2pLayout L = p2p_layout(c, c->p2p_nranks);
    maps[0] = L.maps(c->p2p_own, 0); maps[1] = L.maps(c->p2p_own, 1);
    return check_p2p_right_map(c, call);
}

static int pp_weight_table_size(int type)
{
    return type == PSM_WMF_IV1 ? 3 * 63 + 1 : (type == PSM_WMF_OFF ? 1 : kPpMaxD2 + 1);
}

// The post-filter's 2^-22 fixed-point weight table: JointWMF.h:620-648's float formulas on the 6-bit colour difference
// (index: squared distance for exp / iv2, L1 distance for iv1, one entry for off), normalised by w(0) so that the centre
// tap is always 2^22.  Built with -ffp-contract=off.  Both post-filter kernels read it: pp_wmf_kernel its first
// kPpLutN entries, the generic kernels all of them.  -> entries
static int pp_weight_table(float sigma, int type, uint32_t* t)
{
    const float s = sigma / 256.0f * 64;
    auto w = [&](int k) -> float {
        switch (type) {
        case PSM_WMF_EXP: return expf(-(float)k * (1.0f / (2 * s * s)));
        case PSM_WMF_IV1: return 1.0f / ((float)k + s);
        case PSM_WMF_IV2: return 1.0f / ((float)k + s * s);
        default: return 1.0f;
        }
    };
    const float w0 = w(0);
    const int n = pp_weight_table_size(type);
    for (int k = 0; k < n; ++k) t[k] = (uint32_t)lrintf((w(k) / w0) * 4194304.0f);
    return n;
}

}  // extern "C"

// speckle removal (psm_speckle.cuh) of the maps in[view] into out[view], both views in each of its four launches
template <typename T>
static int speckle_filter(psm_ctx* c, const uint8_t* const in[2], uint8_t* const out[2])
{
    const int max_size = c->pp_steps[kPpSpeckle].a, max_diff = c->pp_steps[kPpSpeckle].b;
    const SpeckleArgs<T> a = {{reinterpret_cast<const T*>(in[0]), reinterpret_cast<const T*>(in[1])}, c->sp_lab, c->sp_cnt,
                              c->W, c->H, max_diff};
    const unsigned ntx = (unsigned)(c->W + kSpTile - 1) / kSpTile, nty = (unsigned)(c->H + kSpTile - 1) / kSpTile;
    const dim3 blk(kSpTile, kSpRows);
    speckle_local_kernel<T><<<dim3(ntx, nty, c->views), blk, 0, c->stream>>>(a);
    PSM_LAUNCH_CHECK(c);
    const int nv = (int)(ntx - 1) * c->H, nh = (int)(nty - 1) * c->W;   // edges across vertical / horizontal seams
    const unsigned sgrid = std::max(1u, (unsigned)((nv + nh + kSpSeamThreads - 1) / kSpSeamThreads));
    speckle_seam_kernel<T><<<dim3(sgrid, 1, c->views), kSpSeamThreads, 0, c->stream>>>(a, nv, nh);
    PSM_LAUNCH_CHECK(c);
    const dim3 grd(ntx, (unsigned)(c->H + kSpRows - 1) / kSpRows, c->views);
    speckle_count_kernel<T><<<grd, blk, 0, c->stream>>>(a);
    PSM_LAUNCH_CHECK(c);
    speckle_paint_kernel<T><<<grd, blk, 0, c->stream>>>(a, max_size, reinterpret_cast<T*>(out[0]),
                                                         reinterpret_cast<T*>(out[1]));
    PSM_LAUNCH_CHECK(c);
    return PSM_OK;
}

// the one-view disparity check (psm_dcheck.cuh) of the maps in[view] into out[view], every computed view in one launch
template <typename T>
static int disparity_check(psm_ctx* c, const uint8_t* const in[2], uint8_t* const out[2])
{
    const float* q[2];
    for (int v = 0; v < 2; ++v) q[v] = c->outs[kOutCosts].planes[v] ? c->outs[kOutCosts].planes[v] + (size_t)c->W * c->H : nullptr;
    const DcheckArgs<T> a = {{reinterpret_cast<const T*>(in[0]), reinterpret_cast<const T*>(in[1])}, {q[0], q[1]},
                             {reinterpret_cast<T*>(out[0]), reinterpret_cast<T*>(out[1])}, {c->dc_claims[0], c->dc_claims[1]}, c->W, c->H, c->D,
                             c->pp_steps[kPpDcheck].a};
    const size_t smem = c->W <= kDcStageCols ? (size_t)c->W * sizeof(unsigned long long) : 0;
    dcheck_kernel<T><<<dim3((unsigned)c->H, (unsigned)c->views), kDcThreads, smem, c->stream>>>(a);
    PSM_LAUNCH_CHECK(c);
    return PSM_OK;
}

// the uniqueness test (psm_unique.cuh) of the maps in[view] into out[view], every computed view in one launch
template <typename T>
static int unique_check(psm_ctx* c, const uint8_t* const in[2], uint8_t* const out[2])
{
    const size_t npix = (size_t)c->W * c->H;
    const float* qm[2];
    const float* qr[2];
    for (int v = 0; v < 2; ++v) {
        qm[v] = c->outs[kOutCosts].planes[v] ? c->outs[kOutCosts].planes[v] + npix : nullptr;
        qr[v] = c->outs[kOutRunnerUp].planes[v] ? c->outs[kOutRunnerUp].planes[v] + npix : nullptr;
    }
    const UniqueArgs<T> a = {{reinterpret_cast<const T*>(in[0]), reinterpret_cast<const T*>(in[1])}, {qm[0], qm[1]},
                             {qr[0], qr[1]}, {reinterpret_cast<T*>(out[0]), reinterpret_cast<T*>(out[1])}, npix,
                             c->pp_steps[kPpUnique].a};
    unique_kernel<T><<<dim3((unsigned)((npix + kUnThreads - 1) / kUnThreads), (unsigned)c->views), kUnThreads, 0, c->stream>>>(a);
    PSM_LAUNCH_CHECK(c);
    return PSM_OK;
}

// the ksize x ksize median (psm_median.cuh) of the maps in[view] into out[view], every computed view in one launch
template <typename T>
static int median_blur(psm_ctx* c, const uint8_t* const in[2], uint8_t* const out[2])
{
    const MedianArgs<T> a = {{reinterpret_cast<const T*>(in[0]), reinterpret_cast<const T*>(in[1])},
                             {reinterpret_cast<T*>(out[0]), reinterpret_cast<T*>(out[1])}, c->W, c->H};
    const dim3 grd((unsigned)(c->W + kMdTileX - 1) / kMdTileX, (unsigned)(c->H + kMdTileY - 1) / kMdTileY, c->views);
    (c->pp_steps[kPpMedian].a == 3 ? median_kernel<T, 1> : median_kernel<T, 2>)<<<grd, dim3(kMdTileX, kMdTileY), 0, c->stream>>>(a);
    PSM_LAUNCH_CHECK(c);
    return PSM_OK;
}

// lrCheck + fillInv (PP.cpp:405-406) of in[view] into out[view] and lr_valid; on a left-only context the left view
// alone, its mask from the map itself (post_process_maps runs the step there only after a step that reads selection
// outputs)
template <typename T>
static int lr_check_fill(psm_ctx* c, const uint8_t* const in[2], uint8_t* const out[2])
{
    const bool own = c->views == 1;
    const size_t smem = c->W <= kLrStageCols ? (size_t)c->W * (2 * sizeof(T) + 2) : 0;
    (own ? lr_check_fill_kernel<T, true> : lr_check_fill_kernel<T, false>)<<<(unsigned)c->H, kLrThreads, smem, c->stream>>>(
        reinterpret_cast<const T*>(in[0]), own ? nullptr : reinterpret_cast<const T*>(in[1]), c->W,
        reinterpret_cast<T*>(out[0]), own ? nullptr : reinterpret_cast<T*>(out[1]), c->lr_valid[0], own ? nullptr : c->lr_valid[1]);
    PSM_LAUNCH_CHECK(c);
    c->lr_masks_ok = true;
    return PSM_OK;
}

// What each post-process step is, by PpStepId: the noun and the setter its messages name, the selection outputs
// (kSelOut) it reads as a bit mask, and its launcher on maps of type T.  A step that reads selection outputs needs a context over the
// whole range, and after it a left-only context's left-right step fills from the chain's own map.
template <typename T>
struct PpStepInfo {
    const char* noun;
    const char* setter;
    unsigned reads;
    int (*launch)(psm_ctx* c, const uint8_t* const in[2], uint8_t* const out[2]);
};
template <typename T>
constexpr PpStepInfo<T> kPpStep[kNumPpSteps] = {
    {"uniqueness check", "psm_set_uniqueness_check", 1u << kOutCosts | 1u << kOutRunnerUp, unique_check<T>},
    {"disparity check", "psm_set_disparity_check", 1u << kOutCosts, disparity_check<T>},
    {"median blur", "psm_set_median_blur", 0, median_blur<T>},
    {"speckle filter", "psm_set_speckle_filter", 0, speckle_filter<T>},
    {"left-right check", "psm_set_lr_check", 0, lr_check_fill<T>},
};

// the options of the selection outputs in `reads` (a kSelOut bit mask), joined by " and "
static const char* reads_text(unsigned reads, char (&buf)[64])
{
    buf[0] = 0;
    for (int o = 0; o < kNumOuts; ++o)
        if (reads >> o & 1) {
            const size_t n = strlen(buf);
            snprintf(buf + n, sizeof(buf) - n, "%s%s", n ? " and " : "", kSelOut[o].option);
        }
    return buf;
}

// psm_set_<step>: mode 0, 1 or kPpEnd and the step's own arguments; a mode other than off, for a step that reads
// selection outputs, only on a context over the whole range.  A multi-device context spans the range and its first
// shard holds the complete maps and outputs: it judges the value once, then every shard takes it.
static int set_pp_step(psm_ctx* c, int step, int mode, int a = 0, int b = 0)
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    const PpStepInfo<uint8_t>& f = kPpStep<uint8_t>[step];   // everything but the launcher is the same for every map type
    if (mode < 0 || mode > kPpEnd) return fail(c, PSM_EINVAL, "%s mode %d is not off (0), 1 or 2", f.noun, mode);
    if (step == kPpUnique && (a < 0 || a > 100)) return fail(c, PSM_EINVAL, "uniqueness ratio %d outside 0..100", a);
    if (step == kPpDcheck && (a < 0 || a > 4095)) return fail(c, PSM_EINVAL, "disparity check max_diff %d outside 0..4095", a);
    if (step == kPpMedian && a != 3 && a != 5) return fail(c, PSM_EINVAL, "median blur ksize %d is not 3 or 5", a);
    if (step == kPpSpeckle && mode && (a < 1 || b < 0))
        return fail(c, PSM_EINVAL, "speckle filter max_size %d / max_diff %d: need max_size >= 1 and max_diff >= 0", a, b);
    if (mode && f.reads && !c->owns_problem()) {
        char outs[64];
        return fail(c, PSM_EINVAL, "%s on a context that owns slices [%d,%d) of %d: the %s reads %s, which such a "
                    "context cannot write; use a context over the whole range", f.setter, c->d_begin,
                    c->d_begin + c->d_count, c->D, f.noun, reads_text(f.reads, outs));
    }
    c->pp_steps[step] = {mode, a, b};
    for (int k = 0; k < c->nshards; ++k) c->shard[k]->pp_steps[step] = c->pp_steps[step];
    return PSM_OK;
}

extern "C" {

int psm_set_uniqueness_check(psm_ctx* c, int mode, int ratio) { return set_pp_step(c, kPpUnique, mode, ratio); }
int psm_set_disparity_check(psm_ctx* c, int mode, int max_diff) { return set_pp_step(c, kPpDcheck, mode, max_diff); }
int psm_set_median_blur(psm_ctx* c, int mode, int ksize) { return set_pp_step(c, kPpMedian, mode, ksize); }
int psm_set_speckle_filter(psm_ctx* c, int mode, int max_size, int max_diff)
{
    return set_pp_step(c, kPpSpeckle, mode, max_size, max_diff);
}
int psm_set_lr_check(psm_ctx* c, int mode) { return set_pp_step(c, kPpLr, mode); }

}  // extern "C"

// psm_post_process's steps in front of the post-filter (wmf): the steps that are on, in chain order, up to the first
// whose mode is kPpEnd; the post-filter runs when no step ends the chain
struct PpChain {
    int step[kNumPpSteps];   // PpStepId
    int n = 0;
    bool wmf = true;
    explicit PpChain(const psm_ctx* c)
    {
        for (int s = 0; s < kNumPpSteps && wmf; ++s) {
            if (c->pp_steps[s].mode) step[n++] = s;
            wmf = c->pp_steps[s].mode != kPpEnd;
        }
    }
};

// the post-process stage on maps of type T
template <typename T>
static int post_process_maps(psm_ctx* c)
{
    // the generic kernel: one histogram level over the 256 values of u8 maps, two levels on u16 maps
    const auto generic = [] {
        if constexpr (sizeof(T) == 1) return pp_wmf_param_kernel; else return pp_wmf_param_two_level_kernel;
    }();
    c->lr_masks_ok = false;
    if (!c->have_images) return fail(c, PSM_ESTATE, "psm_post_process before psm_set_images");
    if (int rc = check_stages_reset(c, "psm_post_process")) return rc;
    const uint8_t* maps[2];
    if (int rc = selection_maps(c, "psm_post_process", maps)) return rc;
    const size_t npix = (size_t)c->W * c->H;
    const PpChain p(c);
    bool read_outs = false;   // a step so far reads selection outputs
    for (int i = 0; i < p.n; ++i) {
        const int s = p.step[i], mode = c->pp_steps[s].mode;
        const PpStepInfo<T>& f = kPpStep<T>[s];
        for (int o = 0; o < kNumOuts; ++o)
            if ((f.reads >> o & 1) && !c->outs[o].have) {
                char outs[64];
                return fail(c, PSM_ESTATE, "psm_post_process: the %s (%s mode %d) reads %s, and the last selection stage "
                            "did not write them all: set each to 1 before it", f.noun, f.setter, mode, reads_text(f.reads, outs));
            }
        read_outs = read_outs || f.reads;
        if (s == kPpLr && c->views == 1 && !read_outs)
            return fail(c, PSM_ESTATE, "psm_post_process: the left-right check (psm_set_lr_check mode %d) needs both maps, "
                        "and this context computes the left view alone (PSM_OPT_VIEWS = PSM_VIEWS_LEFT): set PSM_LR_OFF or "
                        "PSM_VIEWS_BOTH", mode);
        if (s == kPpSpeckle && npix > (size_t)INT_MAX)
            return fail(c, PSM_EINVAL, "psm_post_process: speckle removal labels pixels with int32 indices (W * H <= 2^31 - 1)");
    }
    // Each buffer is allocated while its own pointer is null and the table is marked valid only once it is on the
    // device, so a call that failed part-way leaves nothing a launch could trip over: the next call completes the set-up
    // or fails in turn.
    if (p.wmf) {
        PSM_CUDA(c, alloc_if_null(c->pp_lut, (kPpMaxD2 + 1) * sizeof(uint32_t)));
        PSM_CUDA(c, alloc_if_null(c->pp_packed, npix * sizeof(uint32_t)));
    }
    for (int v = 0; v < 2; ++v) PSM_CUDA(c, alloc_if_null(c->dis_pp[v], npix * c->map_bytes));
    if (p.n >= 2)
        for (int v = 0; v < c->views; ++v) PSM_CUDA(c, alloc_if_null(c->pp_tmp[v], npix * c->map_bytes));
    for (int i = 0; i < p.n; ++i) {   // each step's own scratch
        if (p.step[i] == kPpLr)
            for (int v = 0; v < 2; ++v) PSM_CUDA(c, alloc_if_null(c->lr_valid[v], npix));
        if (p.step[i] == kPpDcheck && c->W > kDcStageCols)
            for (int v = 0; v < c->views; ++v) PSM_CUDA(c, alloc_if_null(c->dc_claims[v], npix * sizeof(unsigned long long)));
        if (p.step[i] == kPpSpeckle) {
            PSM_CUDA(c, alloc_if_null(c->sp_lab, 2 * npix * sizeof(int)));
            PSM_CUDA(c, alloc_if_null(c->sp_cnt, 2 * npix * sizeof(int)));
        }
    }
    if (p.wmf && !c->pp_lut_valid) {
        const size_t smem = kPpParamWarps * 256 * sizeof(unsigned long long) + (size_t)(kPpMaxD2 + 1) * sizeof(uint32_t);
        PSM_CUDA(c, raise_smem_limit(generic, smem, c->device));
        uint32_t* host = new (std::nothrow) uint32_t[kPpMaxD2 + 1];
        if (!host) return fail(c, PSM_ENOMEM, "out of host memory");
        const int n = pp_weight_table(c->pp_sigma, c->pp_type, host);
        // stream-ordered: a previous frame's filter may still be reading the old table
        cudaError_t e = cudaMemcpyAsync(c->pp_lut, host, n * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
        delete[] host;
        PSM_CUDA(c, e);
        c->pp_lut_valid = true;
    }
    const bool tuned = c->pp_tuned();
    if (int rc = p2p_wait_done(c)) return rc;
    if (int rc = stage_begin(c, 5)) return rc;
    // the last step writes dis_pp, the ones before alternate back through pp_tmp: no step writes the maps it reads
    for (int i = 0; i < p.n; ++i) {
        uint8_t* const* out = (p.n - 1 - i) % 2 ? c->pp_tmp : c->dis_pp;
        if (int rc = kPpStep<T>[p.step[i]].launch(c, maps, out)) return rc;
        maps[0] = out[0]; maps[1] = out[1];
    }
    if (!p.wmf) return stage_end(c, 5);
    int nsm = 0;
    PSM_CUDA(c, cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, c->device));
    const int lut_n = pp_weight_table_size(c->pp_type);
    const int idx_mode = c->pp_type == PSM_WMF_IV1 ? kIdxL1 : (c->pp_type == PSM_WMF_OFF ? kIdxOne : kIdxSq);
    const size_t psmem = kPpParamWarps * 256 * sizeof(unsigned long long) + (size_t)lut_n * sizeof(uint32_t);
    const long pgrid = std::min<long>((long)nsm * 8, ((long)npix + kPpParamWarps - 1) / kPpParamWarps);
    int steps = 0;
    while ((1 << steps) < c->D) ++steps;   // u16 maps: ceil(log2 max_disp) bisection steps over [0, max_disp - 1]
    for (int v = 0; v < c->views; ++v) {
        const float* g = c->guide[v];
        T* dst = reinterpret_cast<T*>(c->dis_pp[v]);
        dim3 blk(256), grd((c->W + 255) / 256, c->H);
        // JointWMF.h:126-131: the feature image stays the original, each pass filters the previous pass's output (after
        // the earlier steps, the first pass filters their result; it packs its input before it writes dis_pp)
        for (int it = 0; it < c->pp_iter; ++it) {
            const T* src = reinterpret_cast<const T*>(it == 0 ? maps[v] : c->dis_pp[v]);
            pp_pack_kernel<T><<<grd, blk, 0, c->stream>>>(g, g + c->plane, g + 2 * c->plane, c->Wp, src, c->W, c->H, c->pp_packed);
            PSM_LAUNCH_CHECK(c);
            if (tuned)
                pp_wmf_kernel<T><<<nsm * 8, kPpWarps * 32, 0, c->stream>>>(c->pp_packed, c->pp_lut, c->W, c->H, dst, c->D, steps);
            else
                generic<<<(unsigned)pgrid, kPpParamWarps * 32, psmem, c->stream>>>(c->pp_packed, c->pp_lut, lut_n, idx_mode,
                                                                                    c->pp_radius, c->W, c->H, dst);
            PSM_LAUNCH_CHECK(c);
        }
    }
    return stage_end(c, 5);
}

// psm_post_process[_u16]: the post-filter on the device, then both maps to the host
template <typename T>
static int post_process(psm_ctx* c, T* left, size_t left_step, T* right, size_t right_step)
{
    if (int rc = check_map_format<T>(c, "psm_post_process", "psm_post_process_u16")) return rc;
    if (int rc = check_map_dst(c, "psm_post_process", left, left_step, right, right_step)) return rc;
    if (int rc = psm_post_process_device(c)) return rc;
    return copy_maps_out(c, c->dis_pp, left, left_step, right, right_step, cudaMemcpyDeviceToHost, true);
}

extern "C" {

int psm_post_process_device(psm_ctx* c)
{
    if (is_multi(c)) {   // on the first shard, which holds the complete maps; its outputs stand for the context's
        psm_ctx* s0 = c->shard[0];
        if (int rc = psm_post_process_device(s0)) return relay(c, 0, rc);
        for (int v = 0; v < 2; ++v) { c->dis_pp[v] = s0->dis_pp[v]; c->lr_valid[v] = s0->lr_valid[v]; }
        return PSM_OK;
    }
    if (int rc = bind(c)) return rc;
    const int rc = c->map_bytes == 2 ? post_process_maps<uint16_t>(c) : post_process_maps<uint8_t>(c);
    if (!rc) c->have_pp = true;
    return rc;
}

int psm_post_process(psm_ctx* c, uint8_t* left, size_t left_step, uint8_t* right, size_t right_step)
{
    return post_process(c, left, left_step, right, right_step);
}

int psm_post_process_u16(psm_ctx* c, uint16_t* left, size_t left_step, uint16_t* right, size_t right_step)
{
    return post_process(c, left, left_step, right, right_step);
}

// `which` of a map call `call`: PSM_EINVAL unless 0 (the selection maps) or 1 (the post-processed maps)
static int check_which(psm_ctx* c, const char* call, int which)
{
    if (which != 0 && which != 1)
        return fail(c, PSM_EINVAL, "%s: which %d is neither 0 (selection maps) nor 1 (post-processed maps)", call, which);
    return PSM_OK;
}

// the maps `which` names for a reader `call` on a single-device context (bound): the selection maps, with the wait for
// the exchanged maps enqueued in front of the reader, or the post-processed maps
static int result_maps(psm_ctx* c, const char* call, int which, const uint8_t* maps[2])
{
    if (int rc = check_stages_reset(c, call)) return rc;
    maps[0] = c->dis_pp[0]; maps[1] = c->dis_pp[1];
    if (which == 0) {
        if (int rc = selection_maps(c, call, maps)) return rc;
        return p2p_wait_done(c);
    }
    if (!c->have_pp) return fail(c, PSM_ESTATE, "%s of the post-processed maps before a post-process", call);
    return PSM_OK;
}

int psm_copy_maps_device(psm_ctx* c, int which, void* d_left, size_t left_step, void* d_right, size_t right_step)
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    if (int rc = check_which(c, "psm_copy_maps_device", which)) return rc;
    if (int rc = check_map_dst(c, "psm_copy_maps_device", d_left, left_step, d_right, right_step)) return rc;
    // a multi-device context's maps are the first shard's (its exchange block, and its post-filter's outputs)
    if (is_multi(c)) return relay(c, 0, psm_copy_maps_device(c->shard[0], which, d_left, left_step, d_right, right_step));
    if (int rc = bind(c)) return rc;
    const uint8_t* maps[2];
    if (int rc = result_maps(c, "psm_copy_maps_device", which, maps)) return rc;
    return copy_maps_out(c, maps, d_left, left_step, d_right, right_step, cudaMemcpyDefault, false);
}

}  // extern "C"

// the points of each requested view v (q[v] given) of maps[v] into out[v]: with handle_missing the maps' minima first,
// then one launch over every requested view
template <typename T>
static int reproject_maps(psm_ctx* c, const uint8_t* const maps[2], const double* const q[2], int handle_missing,
                          float* const out[2], size_t row_step)
{
    ReprojArgs<T> a = {};
    unsigned nz = 0;   // the launch's slots: the requested views in order
    for (int v = 0; v < 2; ++v) {
        if (!q[v]) continue;
        a.map[nz] = reinterpret_cast<const T*>(maps[v]);
        a.out[nz] = out[v];
        std::memcpy(a.q[nz], q[v], sizeof a.q[nz]);
        ++nz;
    }
    a.row_step = row_step;
    a.W = c->W;
    a.H = c->H;
    if (handle_missing) {
        PSM_CUDA(c, alloc_if_null(c->rp_min, 2 * sizeof(unsigned)));
        PSM_CUDA(c, cudaMemsetAsync(c->rp_min, 0xff, 2 * sizeof(unsigned), c->stream));
        const size_t npix = (size_t)c->W * c->H;
        const unsigned grid = (unsigned)std::min<size_t>(kRpMinBlocks, (npix + kRpThreads - 1) / kRpThreads);
        reproject_min_kernel<T><<<dim3(grid, 1, nz), kRpThreads, 0, c->stream>>>(a, c->rp_min);
        PSM_LAUNCH_CHECK(c);
        a.minv = c->rp_min;
    }
    const unsigned segs = (unsigned)((c->W + kRpPix - 1) / kRpPix);
    reproject_kernel<T><<<dim3(segs * (unsigned)c->H, 1, nz), kRpThreads, 0, c->stream>>>(a, segs);
    PSM_LAUNCH_CHECK(c);
    return PSM_OK;
}

// the arguments of psm_reproject_device / psm_read_points `call`, before any CUDA work: a view is requested when its Q
// and its point buffer are both given
static int check_reproject_args(psm_ctx* c, const char* call, int which, const double* const q[2], int handle_missing,
                                float* const out[2], size_t row_step)
{
    if (int rc = check_which(c, call, which)) return rc;
    if (handle_missing != 0 && handle_missing != 1)
        return fail(c, PSM_EINVAL, "%s: handle_missing %d is neither 0 nor 1", call, handle_missing);
    for (int v = 0; v < 2; ++v)
        if (!q[v] != !out[v])
            return fail(c, PSM_EINVAL, "%s: the %s view has %s; give both or neither", call, v ? "right" : "left",
                        q[v] ? "a Q without a point buffer" : "a point buffer without a Q");
    if (!q[0] && !q[1]) return fail(c, PSM_EINVAL, "%s: no view requested (no Q and point buffer given)", call);
    const size_t row = (size_t)c->W * 3 * sizeof(float);
    const auto misaligned = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3) != 0; };
    if (row_step < row || row_step % 4 || misaligned(out[0]) || misaligned(out[1]))
        return fail(c, PSM_EINVAL, "%s: bad point buffer/row_step (row_step must be a multiple of 4 and at least 12 * W = "
                    "%zu bytes, buffers 4-byte aligned)", call, row);
    return PSM_OK;
}

// the maps `which` names and the requested views' state, on a bound single-device context
static int reproject_maps_of(psm_ctx* c, const char* call, int which, const double* const q[2], const uint8_t* maps[2])
{
    if (q[1])
        if (int rc = check_right_view(c, call)) return rc;
    return result_maps(c, call, which, maps);
}

static int reproject_run(psm_ctx* c, const uint8_t* const maps[2], const double* const q[2], int handle_missing,
                         float* const out[2], size_t row_step)
{
    return c->map_bytes == 2 ? reproject_maps<uint16_t>(c, maps, q, handle_missing, out, row_step)
                             : reproject_maps<uint8_t>(c, maps, q, handle_missing, out, row_step);
}

extern "C" {

int psm_reproject_device(psm_ctx* c, int which, const double* q_left, const double* q_right, int handle_missing,
                         float* d_left, float* d_right, size_t row_step)
{
    static const char* call = "psm_reproject_device";
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    const double* const q[2] = {q_left, q_right};
    float* const out[2] = {d_left, d_right};
    if (int rc = check_reproject_args(c, call, which, q, handle_missing, out, row_step)) return rc;
    if (is_multi(c))
        return relay(c, 0, psm_reproject_device(c->shard[0], which, q_left, q_right, handle_missing, d_left, d_right, row_step));
    if (int rc = bind(c)) return rc;
    const uint8_t* maps[2];
    if (int rc = reproject_maps_of(c, call, which, q, maps)) return rc;
    return reproject_run(c, maps, q, handle_missing, out, row_step);
}

int psm_read_points(psm_ctx* c, int which, int view, const double q_view[16], int handle_missing, float* dst, size_t row_step)
{
    static const char* call = "psm_read_points";
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    if (view != PSM_LEFT && view != PSM_RIGHT) return fail(c, PSM_EINVAL, "%s: bad view %d", call, view);
    const double* q[2] = {nullptr, nullptr};
    float* out[2] = {nullptr, nullptr};
    q[view] = q_view;
    out[view] = dst;
    if (int rc = check_reproject_args(c, call, which, q, handle_missing, out, row_step)) return rc;
    if (is_multi(c)) return relay(c, 0, psm_read_points(c->shard[0], which, view, q_view, handle_missing, dst, row_step));
    if (int rc = bind(c)) return rc;
    const uint8_t* maps[2];
    if (int rc = reproject_maps_of(c, call, which, q, maps)) return rc;
    const size_t row = (size_t)c->W * 3 * sizeof(float);
    PSM_CUDA(c, alloc_if_null(c->rp_buf, row * c->H));
    out[view] = c->rp_buf;
    if (int rc = reproject_run(c, maps, q, handle_missing, out, row)) return rc;
    PSM_CUDA(c, cudaMemcpy2DAsync(dst, row_step, c->rp_buf, row, row, c->H, cudaMemcpyDeviceToHost, c->stream));
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    return PSM_OK;
}

// output o of the last selection stage, for its copy-out call `call`
static int check_out_ready(psm_ctx* c, int o, const char* call)
{
    if (int rc = check_stages_reset(c, call)) return rc;
    if (!c->outs[o].have)
        return fail(c, PSM_ESTATE, "%s: no %s; the last selection stage since the context was created or the last "
                    "PSM_OPT_VIEWS / PSM_OPT_COSTS / PSM_OPT_RUNNER_UP change did not write the %s (psm_disp_select* with "
                    "%s = 1)", call, kSelOut[o].noun, kSelOut[o].noun, kSelOut[o].option);
    return PSM_OK;
}

// the destination of a copy-out call of output o: `given` (its pointers are set) and rows of at least W floats
static int check_out_dst(psm_ctx* c, int o, const char* call, bool given, size_t row_step)
{
    const size_t row = (size_t)c->W * sizeof(float);
    if (!given || row_step < row)
        return fail(c, PSM_EINVAL, "%s: bad %s plane pointer/step (row_step must be at least %zu bytes)", call,
                    kSelOut[o].noun, row);
    return PSM_OK;
}

// nplanes planes of H x W floats at src -> dst (plane k at dst + k * H * row_step) on the context's stream: one copy of
// nplanes * H rows
static int copy_planes_out(psm_ctx* c, const float* src, int nplanes, float* dst, size_t row_step, cudaMemcpyKind kind)
{
    const size_t row = (size_t)c->W * sizeof(float);
    PSM_CUDA(c, cudaMemcpy2DAsync(dst, row_step, src, row, row, (size_t)nplanes * c->H, kind, c->stream));
    return PSM_OK;
}

// psm_copy_*_device: both views' result planes of output o -> device memory, asynchronously
static int copy_out_device(psm_ctx* c, int o, const char* call, float* d_left, float* d_right, size_t row_step)
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    if (int rc = check_right_arg(c, d_right, call)) return rc;
    if (int rc = check_out_dst(c, o, call, d_left && (c->views == 1 || d_right), row_step)) return rc;
    // a multi-device context's outputs are the first shard's
    if (is_multi(c)) return relay(c, 0, copy_out_device(c->shard[0], o, call, d_left, d_right, row_step));
    if (int rc = bind(c)) return rc;
    if (int rc = check_out_ready(c, o, call)) return rc;
    float* dst[2] = {d_left, d_right};
    for (int v = 0; v < c->views; ++v)
        if (int rc = copy_planes_out(c, c->outs[o].planes[v], kSelOut[o].planes, dst[v], row_step, cudaMemcpyDefault))
            return rc;
    return PSM_OK;
}

// psm_read_*: one view's result planes of output o -> host memory, then waits for the copy
static int read_out(psm_ctx* c, int o, const char* call, int view, float* dst, size_t row_step)
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    if (view != PSM_LEFT && view != PSM_RIGHT) return fail(c, PSM_EINVAL, "bad view %d", view);
    if (int rc = check_out_dst(c, o, call, dst, row_step)) return rc;
    if (is_multi(c)) return relay(c, 0, read_out(c->shard[0], o, call, view, dst, row_step));
    if (int rc = bind(c)) return rc;
    if (view == PSM_RIGHT)
        if (int rc = check_right_view(c, call)) return rc;
    if (int rc = check_out_ready(c, o, call)) return rc;
    if (int rc = copy_planes_out(c, c->outs[o].planes[view], kSelOut[o].planes, dst, row_step, cudaMemcpyDeviceToHost))
        return rc;
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    return PSM_OK;
}

int psm_copy_costs_device(psm_ctx* c, float* d_left, float* d_right, size_t row_step)
{
    return copy_out_device(c, kOutCosts, "psm_copy_costs_device", d_left, d_right, row_step);
}

int psm_read_costs(psm_ctx* c, int view, float* dst, size_t row_step)
{
    return read_out(c, kOutCosts, "psm_read_costs", view, dst, row_step);
}

int psm_copy_runner_up_device(psm_ctx* c, float* d_left, float* d_right, size_t row_step)
{
    return copy_out_device(c, kOutRunnerUp, "psm_copy_runner_up_device", d_left, d_right, row_step);
}

int psm_read_runner_up(psm_ctx* c, int view, float* dst, size_t row_step)
{
    return read_out(c, kOutRunnerUp, "psm_read_runner_up", view, dst, row_step);
}

static int check_slice(psm_ctx* c, int view, int d)
{
    if (view != PSM_LEFT && view != PSM_RIGHT) return fail(c, PSM_EINVAL, "bad view %d", view);
    if (d < c->d_begin || d >= c->d_begin + c->d_count)
        return fail(c, PSM_EINVAL, "slice %d not owned by this context [%d,%d)", d, c->d_begin, c->d_begin + c->d_count);
    if (d < c->res.begin || d >= c->res.begin + c->res.count)
        return fail(c, PSM_EINVAL, "slice %d is not resident: this blocked context holds slices [%d,%d) only (the first block "
                    "after psm_cost_const, the last after a filter stage)", d, c->res.begin, c->res.begin + c->res.count);
    return PSM_OK;
}

}  // extern "C"

// a per-slice call on a multi-device context: routed to the shard that owns global slice d
template <class F>
static int route_slice(psm_ctx* c, int d, F f)
{
    for (int k = 0; k < c->nshards; ++k)
        if (d >= c->shard[k]->d_begin && d < c->shard[k]->d_begin + c->shard[k]->d_count) return relay(c, k, f(c->shard[k]));
    return fail(c, PSM_EINVAL, "slice %d outside [%d,%d)", d, c->d_lo, c->D);
}

extern "C" {

// the offset of a checked slice in the volumes
static size_t slice_offset(const psm_ctx* c, int d) { return (size_t)(d - c->res.begin) * c->plane; }

int psm_read_cost_slice(psm_ctx* c, int view, int d, float* dst, size_t dst_step)
{
    if (is_multi(c)) return route_slice(c, d, [&](psm_ctx* s) { return psm_read_cost_slice(s, view, d, dst, dst_step); });
    if (int rc = bind(c)) return rc;
    if (int rc = check_slice(c, view, d)) return rc;
    if (view == PSM_RIGHT)
        if (int rc = check_right_view(c, "psm_read_cost_slice")) return rc;
    if (!dst || dst_step < (size_t)c->W * sizeof(float)) return fail(c, PSM_EINVAL, "bad dst/step");
    PSM_CUDA(c, cudaMemcpy2DAsync(dst, dst_step, c->vol[view] + slice_offset(c, d),
                                  c->Wp * sizeof(float), c->W * sizeof(float), c->H, cudaMemcpyDeviceToHost, c->stream));
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    return PSM_OK;
}

int psm_write_cost_slice(psm_ctx* c, int view, int d, const float* src, size_t src_step)
{
    if (is_multi(c)) return route_slice(c, d, [&](psm_ctx* s) { return psm_write_cost_slice(s, view, d, src, src_step); });
    if (int rc = bind(c)) return rc;
    if (c->blk_slices)
        return fail(c, PSM_EINVAL, "psm_write_cost_slice on a blocked context: the filter stages rebuild every block after the "
                    "first from the images, so a written slice would not be filtered");
    if (int rc = check_slice(c, view, d)) return rc;
    if (!src || src_step < (size_t)c->W * sizeof(float)) return fail(c, PSM_EINVAL, "bad src/step");
    PSM_CUDA(c, cudaMemcpy2DAsync(c->vol[view] + slice_offset(c, d), c->Wp * sizeof(float), src, src_step,
                                  c->W * sizeof(float), c->H, cudaMemcpyHostToDevice, c->stream));
    if (int rc = pad_rows(c, c->vol[view] + slice_offset(c, d), (size_t)c->H)) return rc;
    // A negative, -0, inf, NaN or >= 2^63 cost (bit patterns >= that of 2^63; the sign bit sorts last) makes the fp64 box
    // sums order-dependent: flag the slice for the reference-order pass.  psm_cost_const never produces one from images
    // without kGuideOutside, so this is the only other way such a cost enters a volume.
    bool special = false;
    for (int y = 0; y < c->H && !special; ++y) {
        const uint32_t* row = reinterpret_cast<const uint32_t*>(reinterpret_cast<const char*>(src) + (size_t)y * src_step);
        for (int x = 0; x < c->W; ++x) special |= row[x] >= 0x5f000000u;
    }
    if (special) {
        static const int one = 1;
        PSM_CUDA(c, cudaMemcpyAsync(c->slice_flags + (size_t)view * c->res.count + (d - c->res.begin), &one, sizeof(int),
                                    cudaMemcpyHostToDevice, c->stream));
        c->slices_flagged = true;
    }
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    c->have_cvc = true;  // caller-provided raw costs may be filtered
    return PSM_OK;
}

int psm_read_guide_plane(psm_ctx* c, int view, int plane_id, float* dst, size_t dst_step)
{
    if (is_multi(c)) return relay(c, 0, psm_read_guide_plane(c->shard[0], view, plane_id, dst, dst_step));
    if (int rc = bind(c)) return rc;
    if (view != PSM_LEFT && view != PSM_RIGHT) return fail(c, PSM_EINVAL, "bad view %d", view);
    if (!c->have_images) return fail(c, PSM_ESTATE, "no images set");
    if (!dst || dst_step < (size_t)c->W * sizeof(float)) return fail(c, PSM_EINVAL, "bad dst/step");
    const float* src = nullptr;
    if (plane_id >= 0 && plane_id <= 2) src = c->guide[view] + (size_t)plane_id * c->plane;
    else if (plane_id >= 3 && plane_id <= 5) src = c->guide[view] + (size_t)(kGuideMean + plane_id - 3) * c->plane;
    else if (plane_id >= 6 && plane_id <= 11) src = c->guide[view] + (size_t)(kGuideVar + plane_id - 6) * c->plane;
    else if (plane_id == 12) src = c->grd[view];
    else return fail(c, PSM_EINVAL, "bad plane id %d", plane_id);
    if (plane_id >= 3 && plane_id <= 11) {
        if (view == PSM_RIGHT && c->views == 1) return check_right_view(c, "psm_read_guide_plane (planes 3-11)");
        if (int rc = ensure_guide(c)) return rc;
    }
    PSM_CUDA(c, cudaMemcpy2DAsync(dst, dst_step, src, c->Wp * sizeof(float), c->W * sizeof(float), c->H,
                                  cudaMemcpyDeviceToHost, c->stream));
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    return PSM_OK;
}

int psm_read_ab_slice(psm_ctx* c, int view, int d, float* a3, float* b)
{
    if (is_multi(c)) return route_slice(c, d, [&](psm_ctx* s) { return psm_read_ab_slice(s, view, d, a3, b); });
    if (int rc = bind(c)) return rc;
    if (int rc = check_slice(c, view, d)) return rc;
    if (view == PSM_RIGHT)
        if (int rc = check_right_view(c, "psm_read_ab_slice")) return rc;
    if (!a3 || !b) return fail(c, PSM_EINVAL, "null output");
    if (!c->have_images) return fail(c, PSM_ESTATE, "no images set");
    if (int rc = ensure_guide(c)) return rc;
    // a, b in OpenCV's order (psm_cvf_ref.cuh), left in the scratch planes [4][H][W]
    if (int rc = launch_ref(c, (void*)cvf_ref_kernel, kRefAbOnly, view, d - c->res.begin)) return rc;
    const size_t n = (size_t)c->W * c->H;
    PSM_CUDA(c, cudaMemcpyAsync(a3, c->ref_pl, 3 * n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    PSM_CUDA(c, cudaMemcpyAsync(b, c->ref_pl + 3 * n, n * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    return PSM_OK;
}

int psm_device_ptr(psm_ctx* c, int what, void** ptr, size_t* pitch_elems)
{
    if (!c || !ptr) return fail(c, PSM_EINVAL, "null argument");
    if (c->nshards && (what == 0 || what == 1))
        return reject_multi(c, "psm_device_ptr selectors 0 / 1", "the volumes are split across the shards");
    switch (what) {
    case 0: case 1: *ptr = c->vol[what]; if (pitch_elems) *pitch_elems = c->Wp; return PSM_OK;
    case 2: case 3: *ptr = c->dis[what - 2]; if (pitch_elems) *pitch_elems = c->W; return PSM_OK;
    case 4: case 5: *ptr = c->dis_pp[what - 4]; if (pitch_elems) *pitch_elems = c->W; return PSM_OK;
    case 6: case 7: *ptr = c->lr_valid[what - 6]; if (pitch_elems) *pitch_elems = c->W; return PSM_OK;
    default: return fail(c, PSM_EINVAL, "bad selector %d", what);
    }
}

int psm_read_valid_mask(psm_ctx* c, int view, uint8_t* dst, size_t dst_step)
{
    if (is_multi(c)) return relay(c, 0, psm_read_valid_mask(c->shard[0], view, dst, dst_step));
    if (int rc = bind(c)) return rc;
    if (view != PSM_LEFT && view != PSM_RIGHT) return fail(c, PSM_EINVAL, "bad view %d", view);
    if (!dst || dst_step < (size_t)c->W) return fail(c, PSM_EINVAL, "bad dst/step");
    // the left-right check never runs on a left-only context; the fill after the disparity check masks the left view
    if (c->views == 1 && (view == PSM_RIGHT || !c->lr_masks_ok))
        return fail(c, PSM_ESTATE, "psm_read_valid_mask on a left-only context (PSM_OPT_VIEWS = PSM_VIEWS_LEFT): the "
                    "left-right check needs both maps; set PSM_VIEWS_BOTH, or fill the left view after "
                    "psm_set_disparity_check(PSM_DCHECK_FIRST) or psm_set_uniqueness_check(PSM_UNIQUE_FIRST)");
    if (!c->lr_masks_ok)
        return fail(c, PSM_ESTATE, "no valid mask: the last post-process since the last selection stage did not run the left-right check");
    PSM_CUDA(c, cudaMemcpy2DAsync(dst, dst_step, c->lr_valid[view], c->W, c->W, c->H, cudaMemcpyDeviceToHost, c->stream));
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    return PSM_OK;
}

int psm_stage_ms(psm_ctx* c, int stage, float* ms)
{
    if (is_multi(c)) {
        // stages 3 (timed across the shards) and 5 (the post-process) run on the first shard; the others are the
        // longest of the shards' own times
        if (stage == 3 || stage == 5) return relay(c, 0, psm_stage_ms(c->shard[0], stage, ms));
        float worst = 0.0f, t = 0.0f;
        for (int k = 0; k < c->nshards; ++k) {
            if (int rc = psm_stage_ms(c->shard[k], stage, &t)) return relay(c, k, rc);
            worst = std::max(worst, t);
        }
        *ms = worst;
        return PSM_OK;
    }
    if (int rc = bind(c)) return rc;
    if (stage < 0 || stage >= kNumStages || !ms) return fail(c, PSM_EINVAL, "bad stage %d", stage);
    if (!c->ev_valid[stage]) return fail(c, PSM_ESTATE, "stage %d has not been timed", stage);
    PSM_CUDA(c, cudaEventSynchronize(c->ev1[stage]));
    PSM_CUDA(c, cudaEventElapsedTime(ms, c->ev0[stage], c->ev1[stage]));
    return PSM_OK;
}

int psm_launch_count(psm_ctx* c, uint64_t* n)
{
    if (!c || !n) return fail(c, PSM_EINVAL, "null argument");
    *n = c->launches;
    for (int k = 0; k < c->nshards; ++k) *n += c->shard[k]->launches;
    return PSM_OK;
}

int psm_sync(psm_ctx* c)
{
    if (is_multi(c)) return forward(c, [](psm_ctx* s) { return psm_sync(s); });
    if (int rc = bind(c)) return rc;
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    return PSM_OK;
}

}  // extern "C"
