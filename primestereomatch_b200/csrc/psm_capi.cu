// psm_capi.cu -- the C-ABI (include/prime_stereo_b200.h) over the sm_90a kernels.
// Host logic only: context/buffer ownership, stage ordering, launches, timers.  No CPU
// compute path exists here: every stage is a CUDA kernel launch or it fails.
#include "../../include/prime_stereo_b200.h"

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <new>

#include <cmath>

#include "psm_cvf_stream.cuh"
#include "psm_cvf_window.cuh"
#include "psm_pp.cuh"
#include "psm_pp_param.cuh"
#include "psm_fgf.cuh"

#ifndef PSM_BUILD_FLAGS
#define PSM_BUILD_FLAGS "unknown"
#endif

using namespace psm;

namespace {

constexpr int kNumStages = 6;  // ingest, cvc, cvf, wta, cvf-filter-kernel, post-process

thread_local char g_create_error[512] = "";  // per host thread: psm_last_error(NULL) reports the calling thread's last failed creation

}  // namespace

struct psm_ctx {
    int W = 0, H = 0, Wp = 0, D = 0, d_begin = 0, d_count = 0, device = 0;
    size_t plane = 0;  // H * Wp
    cudaStream_t own_stream = nullptr, stream = nullptr;
    float* guide[2] = {nullptr, nullptr};   // kGuidePlanes planes per view
    float* grd[2] = {nullptr, nullptr};
    float* vol[2] = {nullptr, nullptr};     // current volumes (raw after CVC, filtered after CVF)
    float* vol_alt[2] = {nullptr, nullptr}; // the other half of the ping-pong
    void* stage_in[2] = {nullptr, nullptr}; // device staging for the interleaved upload (the set the synchronous calls use)
    void* stage_alt[2] = {nullptr, nullptr};// second staging set: psm_set_images_async uploads frame k+1 while frame k is in flight
    cudaStream_t copy_stream = nullptr;     // H2D stream of the asynchronous upload
    cudaEvent_t up_done = nullptr;          // async upload finished (recorded on copy_stream)
    cudaEvent_t ingest_done[2] = {nullptr, nullptr};  // ingest kernels consumed staging set k (recorded on the compute stream)
    bool ingest_done_valid[2] = {false, false};
    int stage_cur = 0;                      // staging set holding the current frame: 0 = stage_in, 1 = stage_alt
    int up_pending = 0;                     // 0 none, 1 f32 upload pending, 2 u8 upload pending
    uint8_t* dis[2] = {nullptr, nullptr};    // disparity maps: u8, or u16 (map_bytes = 2, psm_create_u16) behind the same pointer
    int map_bytes = 1;                       // bytes per disparity-map element
    // Fast Guided Filter branch (lazy): low-res guide planes per view, low-res coefficient scratch, up-sampling plan
    float* fgf_lo[2] = {nullptr, nullptr};
    float* fgf_mean = nullptr;
    void* fgf_plan = nullptr;               // FgfTap x[W], y[H]: INTER_LINEAR source indices and weights
    int fgf_s = 0;                          // sub-sampling rate the buffers / plan were built for
    uint8_t* dis_pp[2] = {nullptr, nullptr}; // post-processed maps (map_bytes per element)
    uint32_t* pp_packed = nullptr;          // packed (disparity, 6-bit colour) image of one view, lazy
    uint32_t* pp_lut = nullptr;             // weight table of the current post-filter setting (kPpMaxD2 + 1 entries), lazy
    bool pp_lut_valid = false;              // pp_lut holds the table of (pp_sigma, pp_type)
    bool have_maps = false;                 // disparity maps valid (a select / reduce stage ran)
    int* guide_flags = nullptr;             // [2] device flags: guide outside the integer-widening domain (see psm_cvf_stream.cuh)
    unsigned char* p2p_own = nullptr;       // own exchange block: keys [2 views][nranks][chunk] u64, maps [2 views][H*W] u8, flag words
    unsigned char* p2p_peer[kMaxRanks] = {};// every rank's exchange block as mapped here
    void* p2p_imported[kMaxRanks] = {};     // IPC mappings to close at destroy
    int p2p_nimported = 0, p2p_nranks = 0, p2p_rank = 0;
    unsigned* p2p_counter = nullptr;        // device-local CTA counter of the publishing kernels
    unsigned p2p_seq = 0;                   // frame sequence number of the device-side exchange flags
    unsigned p2p_waited_seq = 0;            // last sequence number whose DONE flags a wait kernel was enqueued for
    int p2p_sync = 1;                       // 1: device-side ARRIVE/DONE flags; 0: the caller separates the kernels by its own barriers
    float* alloc[16] = {};                  // raw cudaMalloc pointers behind the halo-offset pointers above
    int nalloc = 0;
    float* ab = nullptr;                    // naive-mode scratch [4][d_count][H][Wp], lazy
    size_t ab_slices = 0;
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

template <typename T>
int ingest(psm_ctx* c, const T* l, size_t lstep, const T* r, size_t rstep, bool from_device)
{
    const T* src[2] = {l, r};
    const size_t step[2] = {lstep, rstep};
    const size_t row_bytes = (size_t)c->W * 3 * sizeof(T);
    PSM_CUDA(c, cudaMemsetAsync(c->guide_flags, 0, 2 * sizeof(int), c->stream));
    for (int v = 0; v < 2; ++v) {
        if (!src[v] || step[v] < row_bytes) return fail(c, PSM_EINVAL, "bad image pointer/step for view %d", v);
        const T* dsrc = src[v];
        size_t dstep = step[v];
        if (!from_device) {
            PSM_CUDA(c, cudaMemcpy2DAsync(stage_buf(c, c->stage_cur, v), row_bytes, src[v], step[v], row_bytes, c->H,
                                          cudaMemcpyHostToDevice, c->stream));
            dsrc = static_cast<const T*>(stage_buf(c, c->stage_cur, v));
            dstep = row_bytes;
        }
        float* g = c->guide[v];
        dim3 blk(128), grd((c->W + 3 + 127) / 128, c->H);
        ingest_kernel<T><<<grd, blk, 0, c->stream>>>(dsrc, dstep, c->W, c->H, c->Wp, g, g + c->plane,
                                                      g + 2 * c->plane, c->grd[v], c->gray_mode, c->guide_flags + v);
        PSM_LAUNCH_CHECK(c);
        if (int rc = pad_rows(c, g, (size_t)3 * c->H)) return rc;  // mirrored halo of the 3 guide channels
    }
    c->have_images = true;
    c->guide_valid = false;
    c->have_cvc = false;
    c->filtered = false;
    return PSM_OK;
}

// asynchronous upload of the NEXT frame into the staging set that is not in use (copy stream)
template <typename T>
int upload_async(psm_ctx* c, const T* l, size_t lstep, const T* r, size_t rstep)
{
    const T* src[2] = {l, r};
    const size_t step[2] = {lstep, rstep};
    const size_t row_bytes = (size_t)c->W * 3 * sizeof(T);
    if (c->up_pending) return fail(c, PSM_ESTATE, "an asynchronous upload is already pending: call psm_set_images_commit first");
    const int set = c->stage_cur ^ 1;
    if (!c->stage_alt[0]) {  // allocated on first use: synchronous callers never pay for the second set
        for (int v = 0; v < 2; ++v) PSM_CUDA(c, cudaMalloc(&c->stage_alt[v], (size_t)c->W * c->H * 3 * sizeof(float)));
    }
    if (c->ingest_done_valid[set]) PSM_CUDA(c, cudaStreamWaitEvent(c->copy_stream, c->ingest_done[set], 0));
    for (int v = 0; v < 2; ++v) {
        if (!src[v] || step[v] < row_bytes) return fail(c, PSM_EINVAL, "bad image pointer/step for view %d", v);
        PSM_CUDA(c, cudaMemcpy2DAsync(stage_buf(c, set, v), row_bytes, src[v], step[v], row_bytes, c->H,
                                      cudaMemcpyHostToDevice, c->copy_stream));
    }
    PSM_CUDA(c, cudaEventRecord(c->up_done, c->copy_stream));
    c->up_pending = sizeof(T) == 1 ? 2 : 1;
    return PSM_OK;
}

int ensure_guide(psm_ctx* c)
{
    if (c->guide_valid) return PSM_OK;
    if (!c->gif_default()) {   // any other window / eps: the generic precompute (psm_cvf_window.cuh)
        WinGuideParams P;
        P.guide[0] = c->guide[0]; P.guide[1] = c->guide[1];
        P.W = c->W; P.H = c->H; P.Wp = c->Wp; P.K = c->gif_win; P.a = c->gif_win / 2;
        P.seg_rows = kWinGuideSegRows;
        P.scale = 1.0 / ((double)P.K * P.K);
        P.eps = c->gif_eps;
        dim3 grd((c->W + 127) / 128, (c->H + P.seg_rows - 1) / P.seg_rows, 2);
        guide_window_kernel<<<grd, 128, 0, c->stream>>>(P);
        PSM_LAUNCH_CHECK(c);
        c->guide_valid = true;
        return PSM_OK;
    }
    GuideParams P;
    P.guide[0] = c->guide[0]; P.guide[1] = c->guide[1];
    P.guide_flags = c->guide_flags;
    P.W = c->W; P.H = c->H; P.Wp = c->Wp;
    P.nstrips = (c->W + kGuideStripOut - 1) / kGuideStripOut;
    P.seg_rows = c->guide_seg_rows > 0 ? c->guide_seg_rows : kGuideSegRows;   // option 107 (tuning)
    P.nseg = (c->H + P.seg_rows - 1) / P.seg_rows;
    const int tasks = 2 * P.nstrips * P.nseg;  // one warp each
    guide_kernel<<<(tasks + 3) / 4, 128, 0, c->stream>>>(P);
    PSM_LAUNCH_CHECK(c);
    c->guide_valid = true;
    return PSM_OK;
}

int ensure_ab(psm_ctx* c, size_t slices)
{
    if (c->ab && c->ab_slices >= slices) return PSM_OK;
    if (c->ab) { cudaFree(c->ab); c->ab = nullptr; c->ab_slices = 0; }
    PSM_CUDA(c, cudaMalloc(&c->ab, 4 * slices * c->plane * sizeof(float)));
    c->ab_slices = slices;
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

CvfPlan plan_cvf(int W, int H, int d_count, int nsm, int threads_override, int target_rows, bool allow_pack)
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
            const long ctas = 2L * ns * (q.nstrips * q.ndgroups + q.pack_ndg);
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
    q.pack_first = 2 * q.nseg * q.nstrips * q.ndgroups;
    q.grid = (unsigned)q.pack_first + 2u * q.nseg * q.pack_ndg;
    return q;
}

int launch_cvf_stream(psm_ctx* c)
{
    CvfParams P;
    for (int v = 0; v < 2; ++v) { P.vol_in[v] = c->vol[v]; P.vol_out[v] = c->vol_alt[v]; P.guide[v] = c->guide[v]; }
    P.W = c->W; P.H = c->H; P.Wp = c->Wp; P.Dloc = c->d_count;
    // the packed remainder needs no CTA-level staging (variant 9 stages the guide rows of one strip); variants 1 and 2
    // keep the plain decomposition of the round-1 kernel; option 105 = 1 disables it
    const bool plain_variant = c->cvf_variant == 9 || c->cvf_variant == 2 || (c->cvf_mode != PSM_CVF_MIXED && c->cvf_variant == 1);
    int nsm = 0;
    PSM_CUDA(c, cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, c->device));
    const CvfPlan plan = plan_cvf(c->W, c->H, c->d_count, nsm, c->cvf_threads, c->cvf_target_rows,
                                  !c->cvf_no_pack && !plain_variant && !c->cvf_remap);
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
    PSM_CUDA(c, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
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
    P.W = c->W; P.H = c->H; P.Wp = c->Wp; P.Dloc = c->d_count;
    P.K = c->gif_win; P.a = c->gif_win / 2;
    P.scale = 1.0 / ((double)P.K * P.K);
    P.tw = kWinThreads - 2 * P.K + 2;
    P.nstrips = (c->W + P.tw - 1) / P.tw;
    P.ring_stride = (c->W < P.tw ? c->W : P.tw) + P.K - 1;
    int nsm = 0, smem_max = 0;
    PSM_CUDA(c, cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, c->device));
    PSM_CUDA(c, cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, c->device));
    const long base = 2L * P.Dloc * P.nstrips;
    int nseg = 1;
    while (base * nseg < 4L * nsm && c->H / (nseg + 1) >= 4 * P.K) ++nseg;
    P.seg_rows = (c->H + nseg - 1) / nseg;
    P.nseg = (c->H + P.seg_rows - 1) / P.seg_rows;
    const size_t smem = win_smem_bytes(P.K, P.ring_stride);
    if (smem > (size_t)smem_max)
        return fail(c, PSM_EINVAL, "guided filter window %d: %zu bytes of shared memory exceed the %d a block may have", P.K, smem, smem_max);
    PSM_CUDA(c, cudaFuncSetAttribute(cvf_window_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cvf_window_kernel<<<(unsigned)(base * P.nseg), kWinThreads, smem, c->stream>>>(P);
    PSM_LAUNCH_CHECK(c);
    return PSM_OK;
}

// device map -> host rows of W elements of the context's map format
int copy_map_out(psm_ctx* c, const uint8_t* dsrc, void* dst, size_t step)
{
    const size_t row = (size_t)c->W * c->map_bytes;
    if (!dst || step < row)
        return c->map_bytes == 1 ? fail(c, PSM_EINVAL, "bad disparity map pointer/step")
                                 : fail(c, PSM_EINVAL, "bad disparity map pointer/step (u16 maps need a step of at least %zu bytes)", row);
    PSM_CUDA(c, cudaMemcpy2DAsync(dst, step, dsrc, row, row, c->H, cudaMemcpyDeviceToHost, c->stream));
    return PSM_OK;
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
    const CvfPlan q = plan_cvf(width, height, d_count, sm_count, 0, 0, !no_pack);
    const int v[10] = {q.nthreads, q.nstrips, q.ndgroups, q.nseg, q.seg_rows, q.pack_gl, q.pack_x0, q.pack_ndg, q.pack_first, (int)q.grid};
    for (int i = 0; i < 10; ++i) out[i] = v[i];
    return PSM_OK;
}

}  // extern "C"

// geometry already validated by the caller; map_bytes 1 (u8 maps) or 2 (u16 maps)
static int create_ctx(psm_ctx** out, int width, int height, int max_disp, int d_begin, int d_count, int device, int map_bytes)
{
    int ndev = psm_device_count();
    if (device < 0 || device >= ndev) return fail(nullptr, PSM_ECUDA, "CUDA device %d not available (%d devices)", device, ndev);
    psm_ctx* c = new (std::nothrow) psm_ctx();
    if (!c) return fail(nullptr, PSM_ENOMEM, "out of host memory");
    c->W = width; c->H = height; c->Wp = pitch_for_width(width); c->D = max_disp;
    c->d_begin = d_begin; c->d_count = d_count; c->device = device;
    c->plane = (size_t)c->H * c->Wp;
    c->map_bytes = map_bytes;
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
    const size_t vol_rows = (size_t)d_count * c->H;
    for (int v = 0; v < 2; ++v) {
        PSM_CREATE_CUDA(halo_alloc(&c->guide[v], (size_t)kGuidePlanes * c->H));
        PSM_CREATE_CUDA(halo_alloc(&c->grd[v], (size_t)c->H));
        PSM_CREATE_CUDA(halo_alloc(&c->vol[v], vol_rows));
        PSM_CREATE_CUDA(halo_alloc(&c->vol_alt[v], vol_rows));
        PSM_CREATE_CUDA(cudaMalloc(&c->stage_in[v], (size_t)c->W * c->H * 3 * sizeof(float)));
        PSM_CREATE_CUDA(cudaMalloc(&c->dis[v], (size_t)c->W * c->H * map_bytes));
        PSM_CREATE_CUDA(cudaMemsetAsync(c->dis[v], 0, (size_t)c->W * c->H * map_bytes, c->stream));
    }
    PSM_CREATE_CUDA(cudaMalloc(&c->guide_flags, 2 * sizeof(int)));
    PSM_CREATE_CUDA(cudaMemsetAsync(c->guide_flags, 0, 2 * sizeof(int), c->stream));
    PSM_CREATE_CUDA(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
    PSM_CREATE_CUDA(cudaEventCreateWithFlags(&c->up_done, cudaEventDisableTiming));
    for (int k = 0; k < 2; ++k) PSM_CREATE_CUDA(cudaEventCreateWithFlags(&c->ingest_done[k], cudaEventDisableTiming));
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

int psm_create(psm_ctx** out, int width, int height, int max_disp, int device)
{
    return psm_create_sharded(out, width, height, max_disp, 0, max_disp, device);
}

int psm_destroy(psm_ctx* c)
{
    if (!c) return PSM_OK;
    cudaSetDevice(c->device);
    if (c->own_stream) cudaStreamSynchronize(c->own_stream);
    for (int i = 0; i < c->p2p_nimported; ++i) cudaIpcCloseMemHandle(c->p2p_imported[i]);
    cudaFree(c->p2p_own);
    cudaFree(c->p2p_counter);
    for (int i = 0; i < c->nalloc; ++i) cudaFree(c->alloc[i]);
    if (c->copy_stream) cudaStreamSynchronize(c->copy_stream);
    for (int v = 0; v < 2; ++v) { cudaFree(c->stage_in[v]); cudaFree(c->stage_alt[v]); cudaFree(c->dis[v]); }
    if (c->up_done) cudaEventDestroy(c->up_done);
    for (int k = 0; k < 2; ++k) if (c->ingest_done[k]) cudaEventDestroy(c->ingest_done[k]);
    if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
    cudaFree(c->ab);
    cudaFree(c->guide_flags);
    cudaFree(c->pp_packed); cudaFree(c->pp_lut);
    cudaFree(c->fgf_lo[0]); cudaFree(c->fgf_lo[1]); cudaFree(c->fgf_mean); cudaFree(c->fgf_plan);
    for (int v = 0; v < 2; ++v) cudaFree(c->dis_pp[v]);
    for (int s = 0; s < kNumStages; ++s) {
        if (c->ev0[s]) cudaEventDestroy(c->ev0[s]);
        if (c->ev1[s]) cudaEventDestroy(c->ev1[s]);
    }
    if (c->own_stream) cudaStreamDestroy(c->own_stream);
    cudaGetLastError();
    delete c;
    return PSM_OK;
}

int psm_set_option(psm_ctx* c, int key, int value)
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
    switch (key) {
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
    if (!(alpha >= 0.0f && alpha <= 1.0f)) return fail(c, PSM_EINVAL, "matching-cost alpha %g is not in [0, 1]", (double)alpha);
    if (!(tau_color >= 0.0f)) return fail(c, PSM_EINVAL, "colour threshold %g is not >= 0 or +inf", (double)tau_color);
    if (!(tau_grad >= 0.0f)) return fail(c, PSM_EINVAL, "gradient threshold %g is not >= 0 or +inf", (double)tau_grad);
    c->cost = CvcCost{alpha, tau_color, tau_grad};
    return PSM_OK;
}

int psm_set_post_filter(psm_ctx* c, int radius, float sigma, int iterations, int weight_type)
{
    if (!c) return fail(nullptr, PSM_EINVAL, "null context");
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

int psm_set_stream(psm_ctx* c, void* cuda_stream)
{
    if (int rc = bind(c)) return rc;
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    c->stream = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : c->own_stream;
    return PSM_OK;
}

int psm_set_images(psm_ctx* c, const float* left, size_t left_step, const float* right, size_t right_step)
{
    if (int rc = bind(c)) return rc;
    if (int rc = stage_begin(c, 0)) return rc;
    if (int rc = ingest<float>(c, left, left_step, right, right_step, false)) return rc;
    return stage_end(c, 0);
}

int psm_set_images_u8(psm_ctx* c, const uint8_t* left, size_t left_step, const uint8_t* right, size_t right_step)
{
    if (int rc = bind(c)) return rc;
    if (int rc = stage_begin(c, 0)) return rc;
    if (int rc = ingest<uint8_t>(c, left, left_step, right, right_step, false)) return rc;
    return stage_end(c, 0);
}

int psm_set_images_device(psm_ctx* c, const float* d_left, size_t left_step, const float* d_right, size_t right_step)
{
    if (int rc = bind(c)) return rc;
    if (int rc = stage_begin(c, 0)) return rc;
    if (int rc = ingest<float>(c, d_left, left_step, d_right, right_step, true)) return rc;
    return stage_end(c, 0);
}

int psm_set_images_async(psm_ctx* c, const float* left, size_t left_step, const float* right, size_t right_step)
{
    if (int rc = bind(c)) return rc;
    return upload_async<float>(c, left, left_step, right, right_step);
}

int psm_set_images_u8_async(psm_ctx* c, const uint8_t* left, size_t left_step, const uint8_t* right, size_t right_step)
{
    if (int rc = bind(c)) return rc;
    return upload_async<uint8_t>(c, left, left_step, right, right_step);
}

int psm_set_images_commit(psm_ctx* c)
{
    if (int rc = bind(c)) return rc;
    if (!c->up_pending) return fail(c, PSM_ESTATE, "psm_set_images_commit without a pending psm_set_images_async");
    const int set = c->stage_cur ^ 1;
    const bool u8 = c->up_pending == 2;
    if (int rc = stage_begin(c, 0)) return rc;
    PSM_CUDA(c, cudaStreamWaitEvent(c->stream, c->up_done, 0));
    c->stage_cur = set;
    c->up_pending = 0;
    int rc;
    if (u8) rc = ingest<uint8_t>(c, static_cast<const uint8_t*>(stage_buf(c, set, 0)), (size_t)c->W * 3,
                                 static_cast<const uint8_t*>(stage_buf(c, set, 1)), (size_t)c->W * 3, true);
    else rc = ingest<float>(c, static_cast<const float*>(stage_buf(c, set, 0)), (size_t)c->W * 3 * sizeof(float),
                            static_cast<const float*>(stage_buf(c, set, 1)), (size_t)c->W * 3 * sizeof(float), true);
    if (rc) return rc;
    PSM_CUDA(c, cudaEventRecord(c->ingest_done[set], c->stream));
    c->ingest_done_valid[set] = true;
    return stage_end(c, 0);
}

int psm_cost_const(psm_ctx* c)
{
    if (int rc = bind(c)) return rc;
    if (!c->have_images) return fail(c, PSM_ESTATE, "psm_cost_const before psm_set_images");
    if (int rc = stage_begin(c, 1)) return rc;
    CvcParams2 P2;
    for (int v = 0; v < 2; ++v) {
        CvcParams& P = P2.v[v];
        const float* gs = c->guide[v];
        const float* go = c->guide[1 - v];
        for (int k = 0; k < 3; ++k) { P.self[k] = gs + k * c->plane; P.other[k] = go + k * c->plane; }
        P.self[3] = c->grd[v];
        P.other[3] = c->grd[1 - v];
        P.vol = c->vol[v];
        P.W = c->W; P.H = c->H; P.Wp = c->Wp; P.d_begin = c->d_begin; P.d_count = c->d_count;
        P.fold_halo = c->W >= 32 ? 1 : 0;
    }
    {
        // option 108 (tuning): slices per CTA (0 = all owned slices in one CTA, the shipped decomposition)
        P2.chunk = (c->cvc_chunk > 0 && c->cvc_chunk < c->d_count) ? c->cvc_chunk : 0;
        const int nchunks = P2.chunk ? (c->d_count + P2.chunk - 1) / P2.chunk : 1;
        dim3 blk(128), grd((((c->W + 3) / 4) + 127) / 128, c->H, 2 * nchunks);
        // option 106 (tuning): 0 shipped = interior fast path + scalar window loads; 2 = no fast path (the round-1 loop);
        // 1 / 3 = fast path + grouped 128-bit window loads for the border warps without / with a register cap (DESIGN.md section 10)
        // Any matching cost other than the default runs the parameterised build of the shipped variant, all owned slices
        // per CTA: options 106 and 108 do not apply to it.
        if (!c->cost_default()) {
            grd.z = 2;
            cvc_cost_kernel<<<grd, blk, 0, c->stream>>>(P2, c->cost);
        } else {
            switch (c->cvc_variant) {
            case 1: cvc_both_kernel<4, 1><<<grd, blk, 0, c->stream>>>(P2); break;
            case 2: cvc_both_kernel<7, 2><<<grd, blk, 0, c->stream>>>(P2); break;
            case 3: cvc_both_kernel<5, 1><<<grd, blk, 0, c->stream>>>(P2); break;
            default: cvc_both_kernel<7, 0><<<grd, blk, 0, c->stream>>>(P2); break;
            }
        }
        PSM_LAUNCH_CHECK(c);
        if (!P2.v[0].fold_halo)  // narrow images: separate halo pass (general reflection)
            for (int v = 0; v < 2; ++v)
                if (int rc = pad_rows(c, c->vol[v], (size_t)c->d_count * c->H)) return rc;
    }
    c->have_cvc = true;
    c->filtered = false;
    return stage_end(c, 1);
}

int psm_cost_filter(psm_ctx* c)
{
    if (int rc = bind(c)) return rc;
    if (!c->have_cvc) return fail(c, PSM_ESTATE, "psm_cost_filter before psm_cost_const");
    if (!c->gif_default() && c->cvf_mode != PSM_CVF_EXACT)
        return fail(c, PSM_EINVAL, "CVF mode %s exists only for the default guided filter (window 8, eps 1e-4); "
                    "this context has window %d, eps %g: use PSM_CVF_EXACT", c->cvf_mode == PSM_CVF_MIXED ? "MIXED" : "NAIVE",
                    c->gif_win, (double)c->gif_eps);
    if (int rc = stage_begin(c, 2)) return rc;
    if (int rc = ensure_guide(c)) return rc;
    if (!c->gif_default()) {
        if (int rc = stage_begin(c, 4)) return rc;
        if (int rc = launch_cvf_window(c)) return rc;
        if (int rc = stage_end(c, 4)) return rc;
        for (int v = 0; v < 2; ++v) { float* t = c->vol[v]; c->vol[v] = c->vol_alt[v]; c->vol_alt[v] = t; }
        c->have_cvc = false;
        c->filtered = true;
        return stage_end(c, 2);
    }
    const bool tiny = c->W < 16 || c->H < 16;
    if (c->cvf_mode == PSM_CVF_NAIVE || tiny) {
        if (int rc = ensure_ab(c, (size_t)c->d_count)) return rc;
        if (int rc = stage_begin(c, 4)) return rc;
        for (int v = 0; v < 2; ++v) {
            dim3 blk(128), grd((c->W + 127) / 128, c->H, c->d_count);
            cvf_naive_ab_kernel<<<grd, blk, 0, c->stream>>>(c->vol[v], c->guide[v], c->plane, c->W, c->H, c->Wp,
                                                          c->d_count, c->ab);
            PSM_LAUNCH_CHECK(c);
            cvf_naive_q_kernel<<<grd, blk, 0, c->stream>>>(c->ab, c->guide[v], c->plane, c->W, c->H, c->Wp,
                                                         c->d_count, c->vol_alt[v]);
            PSM_LAUNCH_CHECK(c);
        }
        if (int rc = stage_end(c, 4)) return rc;
    } else {
        if (int rc = stage_begin(c, 4)) return rc;
        int rc = launch_cvf_stream(c);
        if (rc) return rc;
        if (int rc2 = stage_end(c, 4)) return rc2;
    }
    for (int v = 0; v < 2; ++v) { float* t = c->vol[v]; c->vol[v] = c->vol_alt[v]; c->vol_alt[v] = t; }
    c->have_cvc = false;  // the volumes now hold filtered costs; filtering again needs a new CVC
    c->filtered = true;
    return stage_end(c, 2);
}

// DispEst::CostFilter_FGF (reference src/DispEst.cpp:281-296): Fast Guided Filter with sub-sampling rate s
int psm_cost_filter_fgf(psm_ctx* c, int s)
{
    if (int rc = bind(c)) return rc;
    if (!c->have_cvc) return fail(c, PSM_ESTATE, "psm_cost_filter_fgf before psm_cost_const");
    if (s != 1 && s != 2 && s != 4 && s != 8) return fail(c, PSM_EINVAL, "sub-sampling rate must be 1, 2, 4 or 8 (got %d)", s);
    if (c->W / s < 1 || c->H / s < 1) return fail(c, PSM_EINVAL, "image smaller than the sub-sampling rate");
    FgfGeom g;
    // FastGuidedFilter(img, r = GIF_R_WIN, eps = GIF_EPS, s) (DispEst.cpp:283-284): box K = 2 * (r / s) + 1 at low resolution
    g.W = c->W; g.H = c->H; g.Wp = c->Wp; g.s = s; g.w2 = c->W / s; g.h2 = c->H / s; g.K = 2 * (c->gif_win / s) + 1;
    {
        int smem_max = 0;
        PSM_CUDA(c, cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, c->device));
        if (fgf_smem_bytes(g.K) > (size_t)smem_max)
            return fail(c, PSM_EINVAL, "Fast Guided Filter box %d (window %d, rate %d) needs %zu bytes of shared memory, more than "
                        "the %d a block may have", g.K, c->gif_win, s, fgf_smem_bytes(g.K), smem_max);
    }
    g.ifx = 1.0 / ((double)g.w2 / g.W); g.ify = 1.0 / ((double)g.h2 / g.H);
    const size_t n2 = (size_t)g.w2 * g.h2;
    if (c->fgf_s != s) {   // (re)build buffers and the INTER_LINEAR plan for this rate
        cudaFree(c->fgf_lo[0]); cudaFree(c->fgf_lo[1]); cudaFree(c->fgf_mean); cudaFree(c->fgf_plan);
        c->fgf_lo[0] = c->fgf_lo[1] = c->fgf_mean = nullptr; c->fgf_plan = nullptr; c->fgf_s = 0;
        for (int v = 0; v < 2; ++v) PSM_CUDA(c, cudaMalloc(&c->fgf_lo[v], 12 * n2 * sizeof(float)));
        PSM_CUDA(c, cudaMalloc(&c->fgf_mean, (size_t)4 * c->d_count * n2 * sizeof(float)));
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
        cudaError_t e = cudaMemcpy(c->fgf_plan, hp, (size_t)(c->W + c->H) * sizeof(FgfTap), cudaMemcpyHostToDevice);
        delete[] hp;
        PSM_CUDA(c, e);
        c->fgf_s = s;
    }
    FgfPlan pl;
    pl.x = static_cast<const FgfTap*>(c->fgf_plan);
    pl.y = pl.x + c->W;
    if (int rc = stage_begin(c, 2)) return rc;
    if (int rc = stage_begin(c, 4)) return rc;
    for (int v = 0; v < 2; ++v) {
        dim3 blk(128), g2((g.w2 + 127) / 128, g.h2);
        fgf_guide_kernel<<<g2, blk, 0, c->stream>>>(c->guide[v], c->plane, g, c->gif_eps, c->fgf_lo[v]);
        PSM_LAUNCH_CHECK(c);
        dim3 g3((g.w2 + kFgfTX - 1) / kFgfTX, (g.h2 + kFgfTY - 1) / kFgfTY, c->d_count);
        const size_t fsmem = fgf_smem_bytes(g.K);
        PSM_CUDA(c, cudaFuncSetAttribute(fgf_lowres_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem));
        fgf_lowres_kernel<<<g3, kFgfThreads, fsmem, c->stream>>>(c->vol[v], c->plane, g, c->fgf_lo[v], c->fgf_mean);
        PSM_LAUNCH_CHECK(c);
        dim3 g5((((c->W + 3) / 4) + 127) / 128, c->H, c->d_count);
        fgf_up_kernel<<<g5, blk, 0, c->stream>>>(c->vol[v], c->plane, c->guide[v], c->plane, g, pl, c->fgf_mean);
        PSM_LAUNCH_CHECK(c);
    }
    if (int rc = stage_end(c, 4)) return rc;
    c->have_cvc = false;
    c->filtered = true;
    return stage_end(c, 2);
}

}  // extern "C"

// the WTA of both views into the context's maps of type T
template <typename T>
static int select_maps(psm_ctx* c)
{
    for (int v = 0; v < 2; ++v) {
        dim3 blk(256), grd(((c->W + 3) / 4 + 255) / 256, c->H);
        wta_kernel<T><<<grd, blk, 0, c->stream>>>(c->vol[v], c->W, c->H, c->Wp, c->d_begin, c->d_count,
                                                  reinterpret_cast<T*>(c->dis[v]), nullptr);
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
    if (int rc = psm_disp_select_device(c)) return rc;
    if (int rc = copy_map_out(c, c->dis[0], left, left_step)) return rc;
    if (int rc = copy_map_out(c, c->dis[1], right, right_step)) return rc;
    if (sync) PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    return PSM_OK;
}

template <typename T>
static int disp_reduce_keys(psm_ctx* c, const uint64_t* d_gathered_left, const uint64_t* d_gathered_right, int nranks,
                            T* left, size_t left_step, T* right, size_t right_step)
{
    if (int rc = check_map_format<T>(c, "psm_disp_reduce_keys", "psm_disp_reduce_keys_u16")) return rc;
    if (int rc = bind(c)) return rc;
    if (!d_gathered_left || !d_gathered_right || nranks < 1) return fail(c, PSM_EINVAL, "bad gathered keys");
    const uint64_t* g[2] = {d_gathered_left, d_gathered_right};
    const size_t npix = (size_t)c->W * c->H;
    for (int v = 0; v < 2; ++v) {
        keys_reduce_kernel<T><<<(unsigned)((npix + 255) / 256), 256, 0, c->stream>>>(
            reinterpret_cast<const unsigned long long*>(g[v]), nranks, npix, reinterpret_cast<T*>(c->dis[v]));
        PSM_LAUNCH_CHECK(c);
    }
    c->have_maps = true;
    if (left && right) {
        if (int rc = copy_map_out(c, c->dis[0], left, left_step)) return rc;
        if (int rc = copy_map_out(c, c->dis[1], right, right_step)) return rc;
    }
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    return PSM_OK;
}

extern "C" {

int psm_disp_select_device(psm_ctx* c)
{
    if (int rc = bind(c)) return rc;
    if (c->d_begin != 0 || c->d_count != c->D)
        return fail(c, PSM_ESTATE, "psm_disp_select on a sharded context: use psm_disp_select_keys + psm_disp_reduce_keys");
    if (!c->filtered) return fail(c, PSM_ESTATE, "psm_disp_select before psm_cost_filter");
    if (int rc = stage_begin(c, 3)) return rc;
    if (int rc = c->map_bytes == 2 ? select_maps<uint16_t>(c) : select_maps<uint8_t>(c)) return rc;
    c->have_maps = true;
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
    if (int rc = bind(c)) return rc;
    if (!d_keys_left || !d_keys_right) return fail(c, PSM_EINVAL, "null key buffer");
    if (!c->filtered) return fail(c, PSM_ESTATE, "psm_disp_select_keys before psm_cost_filter");
    if (int rc = stage_begin(c, 3)) return rc;
    uint64_t* keys[2] = {d_keys_left, d_keys_right};
    for (int v = 0; v < 2; ++v) {   // keys only, on either map format
        dim3 blk(256), grd(((c->W + 3) / 4 + 255) / 256, c->H);
        wta_kernel<uint8_t><<<grd, blk, 0, c->stream>>>(c->vol[v], c->W, c->H, c->Wp, c->d_begin, c->d_count, nullptr,
                                                        reinterpret_cast<unsigned long long*>(keys[v]));
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

// Exchange block of one rank: [2 views][nranks][chunk] uint64 keys, [2 views][H*W] result maps (u8, or u16 on a u16 context),
// [2 views][2 * kMaxRanks] u32 flag words (ARRIVE per rank, DONE per rank), each part 256-byte aligned.
static size_t p2p_chunk(const psm_ctx* c, int nranks) { return ((size_t)c->W * c->H + nranks - 1) / nranks; }
static size_t p2p_keys_bytes(const psm_ctx* c, int nranks) { return (size_t)2 * nranks * p2p_chunk(c, nranks) * sizeof(unsigned long long); }
static size_t p2p_maps_bytes(const psm_ctx* c) { return (((size_t)2 * c->W * c->H * c->map_bytes) + 255) & ~(size_t)255; }
static size_t p2p_flags_bytes() { return (size_t)2 * 2 * kMaxRanks * sizeof(unsigned); }

int psm_p2p_create_buffer(psm_ctx* c, int nranks, void** d_buffer)
{
    if (int rc = bind(c)) return rc;
    if (nranks < 1 || nranks > kMaxRanks || !d_buffer) return fail(c, PSM_EINVAL, "bad nranks %d (1..%d)", nranks, kMaxRanks);
    if (c->p2p_own) { cudaFree(c->p2p_own); c->p2p_own = nullptr; }
    for (int i = 0; i < c->p2p_nimported; ++i) cudaIpcCloseMemHandle(c->p2p_imported[i]);   // peers of a previous exchange set-up
    c->p2p_nimported = 0;
    for (int r = 0; r < kMaxRanks; ++r) c->p2p_peer[r] = nullptr;
    const size_t kb = p2p_keys_bytes(c, nranks), mb = p2p_maps_bytes(c), fb = p2p_flags_bytes();
    PSM_CUDA(c, cudaMalloc(&c->p2p_own, kb + mb + fb));
    PSM_CUDA(c, cudaMemsetAsync(c->p2p_own, 0xff, kb + mb, c->stream));
    PSM_CUDA(c, cudaMemsetAsync(c->p2p_own + kb + mb, 0, fb, c->stream));
    if (!c->p2p_counter) PSM_CUDA(c, cudaMalloc(&c->p2p_counter, sizeof(unsigned)));
    PSM_CUDA(c, cudaMemsetAsync(c->p2p_counter, 0, sizeof(unsigned), c->stream));
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    c->p2p_nranks = nranks;
    c->p2p_seq = 0;
    c->p2p_waited_seq = 0;
    *d_buffer = c->p2p_own;
    return PSM_OK;
}

int psm_ipc_export(psm_ctx* c, void* d_ptr, unsigned char handle_out[64])
{
    if (int rc = bind(c)) return rc;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    cudaIpcMemHandle_t h;
    PSM_CUDA(c, cudaIpcGetMemHandle(&h, d_ptr));
    memcpy(handle_out, &h, 64);
    return PSM_OK;
}

int psm_ipc_import(psm_ctx* c, const unsigned char handle[64], void** d_ptr)
{
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
    const size_t chunk = p2p_chunk(c, c->p2p_nranks);
    const size_t npix = (size_t)c->W * c->H;
    const size_t kb = p2p_keys_bytes(c, c->p2p_nranks), mb = p2p_maps_bytes(c);
    peers.nranks = c->p2p_nranks; peers.rank = c->p2p_rank; peers.chunk = (unsigned)chunk;
    peers.counter = c->p2p_counter;
    peers.seq = c->p2p_sync ? c->p2p_seq : 0u;
    for (int r = 0; r < kMaxRanks; ++r) {
        unsigned char* base = r < c->p2p_nranks ? c->p2p_peer[r] : nullptr;
        peers.keys[r] = base ? reinterpret_cast<unsigned long long*>(base) + (size_t)view * c->p2p_nranks * chunk : nullptr;
        peers.maps[r] = base ? base + kb + (size_t)view * npix * c->map_bytes : nullptr;
        peers.flags[r] = base ? reinterpret_cast<unsigned*>(base + kb + mb) + (size_t)view * 2 * kMaxRanks : nullptr;
    }
}

int psm_disp_select_keys_p2p(psm_ctx* c)
{
    if (int rc = bind(c)) return rc;
    if (!c->p2p_own || !c->p2p_peer[0]) return fail(c, PSM_ESTATE, "psm_p2p_create_buffer / psm_p2p_set_peers first");
    if (!c->filtered) return fail(c, PSM_ESTATE, "psm_disp_select_keys_p2p before psm_cost_filter");
    if (int rc = stage_begin(c, 3)) return rc;
    c->p2p_seq++;   // one sequence number per frame, identical on every rank (all ranks run the same frames)
    for (int v = 0; v < 2; ++v) {
        P2pPeers peers;
        p2p_fill(c, v, peers);
        dim3 blk(256), grd(((c->W + 3) / 4 + 255) / 256, (c->H + kScatterRows - 1) / kScatterRows);
        wta_scatter_kernel<<<grd, blk, 0, c->stream>>>(c->vol[v], c->W, c->H, c->Wp, c->d_begin, c->d_count, peers);
        PSM_LAUNCH_CHECK(c);
    }
    return stage_end(c, 3);
}

int psm_disp_reduce_p2p(psm_ctx* c)
{
    if (int rc = bind(c)) return rc;
    if (!c->p2p_own || !c->p2p_peer[0]) return fail(c, PSM_ESTATE, "no exchange block");
    const unsigned npix = (unsigned)((size_t)c->W * c->H);
    const auto reduce = c->map_bytes == 2 ? chunk_reduce_kernel<uint16_t> : chunk_reduce_kernel<uint8_t>;
    for (int v = 0; v < 2; ++v) {
        P2pPeers peers;
        p2p_fill(c, v, peers);
        reduce<<<(peers.chunk + 255) / 256, 256, 0, c->stream>>>(peers, npix);
        PSM_LAUNCH_CHECK(c);
    }
    return PSM_OK;
}

// the local result maps are complete once every rank's DONE flag carries this frame's number: enqueue the wait in front
// of a consumer of the maps (once per frame)
static int p2p_wait_done(psm_ctx* c)
{
    if (!c->p2p_sync || c->p2p_waited_seq == c->p2p_seq) return PSM_OK;
    P2pPeers peers;
    p2p_fill(c, 0, peers);
    p2p_wait_done_kernel<<<1, 32, 0, c->stream>>>(peers.flags[c->p2p_rank], c->p2p_nranks, c->p2p_seq);
    PSM_LAUNCH_CHECK(c);
    c->p2p_waited_seq = c->p2p_seq;
    return PSM_OK;
}

}  // extern "C"

template <typename T>
static int disp_fetch_p2p(psm_ctx* c, T* left, size_t left_step, T* right, size_t right_step)
{
    if (int rc = check_map_format<T>(c, "psm_disp_fetch_p2p", "psm_disp_fetch_p2p_u16")) return rc;
    if (int rc = bind(c)) return rc;
    if (!c->p2p_own) return fail(c, PSM_ESTATE, "no exchange block");
    if (int rc = p2p_wait_done(c)) return rc;
    const unsigned char* maps = c->p2p_own + p2p_keys_bytes(c, c->p2p_nranks);
    if (int rc = copy_map_out(c, maps, left, left_step)) return rc;
    if (int rc = copy_map_out(c, maps + (size_t)c->W * c->H * sizeof(T), right, right_step)) return rc;
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    return PSM_OK;
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
static const uint8_t* current_map(const psm_ctx* c, int v)
{
    if (c->p2p_own && c->p2p_seq > 0)   // sharded: the complete maps live in the exchange block
        return c->p2p_own + p2p_keys_bytes(c, c->p2p_nranks) + (size_t)v * c->W * c->H * c->map_bytes;
    return c->dis[v];
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

// the post-filter stage on maps of type T
template <typename T>
static int post_process_maps(psm_ctx* c)
{
    // the generic kernel: one histogram level over the 256 values of u8 maps, two levels on u16 maps
    const auto generic = [] {
        if constexpr (sizeof(T) == 1) return pp_wmf_param_kernel; else return pp_wmf_param_two_level_kernel;
    }();
    if (!c->have_images) return fail(c, PSM_ESTATE, "psm_post_process before psm_set_images");
    if (!c->have_maps && !(c->p2p_own && c->p2p_seq > 0)) return fail(c, PSM_ESTATE, "psm_post_process before a disparity-selection stage");
    const size_t npix = (size_t)c->W * c->H;
    // Each buffer is allocated while its own pointer is null and the table is marked valid only once it is on the
    // device, so a call that failed part-way leaves nothing a launch could trip over: the next call completes the set-up
    // or fails in turn.
    PSM_CUDA(c, alloc_if_null(c->pp_lut, (kPpMaxD2 + 1) * sizeof(uint32_t)));
    PSM_CUDA(c, alloc_if_null(c->pp_packed, npix * sizeof(uint32_t)));
    for (int v = 0; v < 2; ++v) PSM_CUDA(c, alloc_if_null(c->dis_pp[v], npix * c->map_bytes));
    if (!c->pp_lut_valid) {
        const size_t smem = kPpParamWarps * 256 * sizeof(unsigned long long) + (size_t)(kPpMaxD2 + 1) * sizeof(uint32_t);
        PSM_CUDA(c, cudaFuncSetAttribute(generic, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
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
    if (c->p2p_own && c->p2p_seq > 0)
        if (int rc = p2p_wait_done(c)) return rc;
    if (int rc = stage_begin(c, 5)) return rc;
    int nsm = 0;
    PSM_CUDA(c, cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, c->device));
    const int lut_n = pp_weight_table_size(c->pp_type);
    const int idx_mode = c->pp_type == PSM_WMF_IV1 ? kIdxL1 : (c->pp_type == PSM_WMF_OFF ? kIdxOne : kIdxSq);
    const size_t psmem = kPpParamWarps * 256 * sizeof(unsigned long long) + (size_t)lut_n * sizeof(uint32_t);
    const long pgrid = std::min<long>((long)nsm * 8, ((long)npix + kPpParamWarps - 1) / kPpParamWarps);
    int steps = 0;
    while ((1 << steps) < c->D) ++steps;   // u16 maps: ceil(log2 max_disp) bisection steps over [0, max_disp - 1]
    for (int v = 0; v < 2; ++v) {
        const float* g = c->guide[v];
        T* dst = reinterpret_cast<T*>(c->dis_pp[v]);
        dim3 blk(256), grd((c->W + 255) / 256, c->H);
        // JointWMF.h:126-131: the feature image stays the original, each pass filters the previous pass's output
        for (int it = 0; it < c->pp_iter; ++it) {
            const T* src = reinterpret_cast<const T*>(it == 0 ? current_map(c, v) : c->dis_pp[v]);
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
    if (int rc = psm_post_process_device(c)) return rc;
    if (int rc = copy_map_out(c, c->dis_pp[0], left, left_step)) return rc;
    if (int rc = copy_map_out(c, c->dis_pp[1], right, right_step)) return rc;
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    return PSM_OK;
}

extern "C" {

int psm_post_process_device(psm_ctx* c)
{
    if (int rc = bind(c)) return rc;
    return c->map_bytes == 2 ? post_process_maps<uint16_t>(c) : post_process_maps<uint8_t>(c);
}

int psm_post_process(psm_ctx* c, uint8_t* left, size_t left_step, uint8_t* right, size_t right_step)
{
    return post_process(c, left, left_step, right, right_step);
}

int psm_post_process_u16(psm_ctx* c, uint16_t* left, size_t left_step, uint16_t* right, size_t right_step)
{
    return post_process(c, left, left_step, right, right_step);
}

static int check_slice(psm_ctx* c, int view, int d)
{
    if (view != PSM_LEFT && view != PSM_RIGHT) return fail(c, PSM_EINVAL, "bad view %d", view);
    if (d < c->d_begin || d >= c->d_begin + c->d_count)
        return fail(c, PSM_EINVAL, "slice %d not owned by this context [%d,%d)", d, c->d_begin, c->d_begin + c->d_count);
    return PSM_OK;
}

int psm_read_cost_slice(psm_ctx* c, int view, int d, float* dst, size_t dst_step)
{
    if (int rc = bind(c)) return rc;
    if (int rc = check_slice(c, view, d)) return rc;
    if (!dst || dst_step < (size_t)c->W * sizeof(float)) return fail(c, PSM_EINVAL, "bad dst/step");
    PSM_CUDA(c, cudaMemcpy2DAsync(dst, dst_step, c->vol[view] + (size_t)(d - c->d_begin) * c->plane,
                                  c->Wp * sizeof(float), c->W * sizeof(float), c->H, cudaMemcpyDeviceToHost, c->stream));
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    return PSM_OK;
}

int psm_write_cost_slice(psm_ctx* c, int view, int d, const float* src, size_t src_step)
{
    if (int rc = bind(c)) return rc;
    if (int rc = check_slice(c, view, d)) return rc;
    if (!src || src_step < (size_t)c->W * sizeof(float)) return fail(c, PSM_EINVAL, "bad src/step");
    PSM_CUDA(c, cudaMemcpy2DAsync(c->vol[view] + (size_t)(d - c->d_begin) * c->plane, c->Wp * sizeof(float), src,
                                  src_step, c->W * sizeof(float), c->H, cudaMemcpyHostToDevice, c->stream));
    if (int rc = pad_rows(c, c->vol[view] + (size_t)(d - c->d_begin) * c->plane, (size_t)c->H)) return rc;
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    c->have_cvc = true;  // caller-provided raw costs may be filtered
    return PSM_OK;
}

int psm_read_guide_plane(psm_ctx* c, int view, int plane_id, float* dst, size_t dst_step)
{
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
    if (plane_id >= 3 && plane_id <= 11)
        if (int rc = ensure_guide(c)) return rc;
    PSM_CUDA(c, cudaMemcpy2DAsync(dst, dst_step, src, c->Wp * sizeof(float), c->W * sizeof(float), c->H,
                                  cudaMemcpyDeviceToHost, c->stream));
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    return PSM_OK;
}

int psm_read_ab_slice(psm_ctx* c, int view, int d, float* a3, float* b)
{
    if (int rc = bind(c)) return rc;
    if (int rc = check_slice(c, view, d)) return rc;
    if (!a3 || !b) return fail(c, PSM_EINVAL, "null output");
    if (!c->have_images) return fail(c, PSM_ESTATE, "no images set");
    if (int rc = ensure_guide(c)) return rc;
    if (int rc = ensure_ab(c, 1)) return rc;
    dim3 blk(128), grd((c->W + 127) / 128, c->H, 1);
    if (!c->gif_default())
        ab_window_kernel<<<grd, blk, 0, c->stream>>>(c->vol[view] + (size_t)(d - c->d_begin) * c->plane, c->guide[view], c->plane,
                                                     c->W, c->H, c->Wp, c->gif_win, c->gif_win / 2,
                                                     1.0 / ((double)c->gif_win * c->gif_win), c->ab);
    else
        cvf_naive_ab_kernel<<<grd, blk, 0, c->stream>>>(c->vol[view] + (size_t)(d - c->d_begin) * c->plane, c->guide[view],
                                                      c->plane, c->W, c->H, c->Wp, 1, c->ab);
    PSM_LAUNCH_CHECK(c);
    const size_t wb = c->W * sizeof(float);
    // scratch is laid out [4][ab_slices][plane]; only slice 0 of each plane group was written with nslices=1
    for (int k = 0; k < 4; ++k) {
        float* dst = k < 3 ? a3 + (size_t)k * c->W * c->H : b;
        PSM_CUDA(c, cudaMemcpy2DAsync(dst, wb, c->ab + (size_t)k * c->plane, c->Wp * sizeof(float), wb, c->H,
                                      cudaMemcpyDeviceToHost, c->stream));
    }
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    return PSM_OK;
}

int psm_device_ptr(psm_ctx* c, int what, void** ptr, size_t* pitch_elems)
{
    if (!c || !ptr) return fail(c, PSM_EINVAL, "null argument");
    switch (what) {
    case 0: case 1: *ptr = c->vol[what]; if (pitch_elems) *pitch_elems = c->Wp; return PSM_OK;
    case 2: case 3: *ptr = c->dis[what - 2]; if (pitch_elems) *pitch_elems = c->W; return PSM_OK;
    case 4: case 5: *ptr = c->dis_pp[what - 4]; if (pitch_elems) *pitch_elems = c->W; return PSM_OK;
    default: return fail(c, PSM_EINVAL, "bad selector %d", what);
    }
}

int psm_stage_ms(psm_ctx* c, int stage, float* ms)
{
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
    return PSM_OK;
}

int psm_sync(psm_ctx* c)
{
    if (int rc = bind(c)) return rc;
    PSM_CUDA(c, cudaStreamSynchronize(c->stream));
    return PSM_OK;
}

}  // extern "C"
