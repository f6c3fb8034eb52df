// psm_dcheck.cuh -- one-view disparity check of the post-process stage (psm_set_disparity_check; OpenCV's
// cv::validateDisparity, StereoSGBM's disp12MaxDiff).
//
// What is computed, per row of one view's map m (u8 or u16), with q = the winners' costs (plane 1 of PSM_OPT_COSTS),
// W = width, D = max_disp, in the view's own coordinate u (u = x on the left view; the right view is the mirror image,
// u = W - 1 - x):
//   pass 1: every u in [D, W) with m != 0 claims column u - m with key (order key of q, u); per column the lowest key
//           wins (the lowest cost, -0 equal to +0, then the lowest u), and d2[column] is the winner's m;
//   pass 2: a pixel u in [D, W) with m != 0 becomes 0 when |d2[u - m] - m| > max_diff; every other pixel keeps m.
// The key minimum does not depend on the order in which the claims arrive, so the result is exact.
//
// GPU mapping: one CTA per row and view (grid H x views).  Claims are packed (float_order_key(q) << 32 | u) and taken
// with a 64-bit atomicMin, in shared memory for rows of up to kDcStageCols columns and in the context's scratch rows
// beyond that.  Columns are addressed physically (x), so a right-view claim goes to x + m.
#pragma once
#include "psm_common.cuh"

namespace psm {

constexpr int kDcThreads = 256;
constexpr int kDcStageCols = 6144;   // 8 bytes per column: 48 KiB, the most that needs no opt-in

template <typename T>
struct DcheckArgs {
    const T* in[2];                  // the maps to check (read only)
    const float* cost[2];            // q at each pixel's m (row pitch W)
    T* out[2];                       // the checked maps
    unsigned long long* scratch[2];  // W > kDcStageCols: H x W claim words per view, else unused
    int W, H, D, max_diff;
};

template <typename T>
__global__ void __launch_bounds__(kDcThreads) dcheck_kernel(const DcheckArgs<T> a)
{
    extern __shared__ __align__(16) unsigned char dc_smem[];
    const int view = blockIdx.y, W = a.W;
    const bool staged = W <= kDcStageCols;
    const size_t row = (size_t)blockIdx.x * W;
    const T* m = (view ? a.in[1] : a.in[0]) + row;   // (selects, not a dynamic index into the parameter struct)
    const float* q = (view ? a.cost[1] : a.cost[0]) + row;
    unsigned long long* claim = staged ? reinterpret_cast<unsigned long long*>(dc_smem)
                                       : (view ? a.scratch[1] : a.scratch[0]) + row;
    for (int x = threadIdx.x; x < W; x += kDcThreads) claim[x] = ~0ull;
    __syncthreads();
    for (int x = threadIdx.x; x < W; x += kDcThreads) {
        const int d = __ldg(m + x), u = view ? W - 1 - x : x;
        if (u < a.D || d == 0) continue;
        atomicMin(claim + (view ? x + d : x - d), ((unsigned long long)float_order_key(__ldg(q + x)) << 32) | (unsigned)u);
    }
    __syncthreads();
    T* out = (view ? a.out[1] : a.out[0]) + row;
    for (int x = threadIdx.x; x < W; x += kDcThreads) {
        const int d = __ldg(m + x), u = view ? W - 1 - x : x;
        T v = (T)d;
        if (u >= a.D && d != 0) {
            const int x2 = view ? x + d : x - d;
            // the winner's column u2 (never empty: this pixel's own claim is in it); scratch claims bypass L1
            const int u2 = (int)(unsigned)(staged ? claim[x2] : __ldcg(claim + x2));
            const int d2 = __ldg(m + (view ? W - 1 - u2 : u2));
            if (abs(d2 - d) > a.max_diff) v = 0;
        }
        out[x] = v;
    }
}

}  // namespace psm
