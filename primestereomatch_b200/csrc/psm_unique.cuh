// psm_unique.cuh -- uniqueness test of the post-process stage (psm_set_uniqueness_check; OpenCV StereoSGBM's
// uniquenessRatio).
//
// What is computed, per pixel of one view's selection map m (u8 or u16), with q(m) = plane 1 of PSM_OPT_COSTS and
// q(r) = plane 1 of PSM_OPT_RUNNER_UP (the cost of the lowest candidate with |d - m| >= 2, NaN where there is none):
//   m != 0 and (double)q(r) * (100 - ratio) < (double)q(m) * 100  ->  0;  every other pixel keeps m.
// Both products are exact in fp64 (a 24-bit significand times an integer <= 100), so the comparison is the exact real
// one on finite costs and IEEE's on the rest: a NaN q(r) (no runner-up) or q(m) never rejects.  This is computeDisparity-
// SGBM's `Sp[d]*(100 - uniquenessRatio) < minS*100 && abs(bestDisp - d) > 1` over every candidate d: multiplying by a
// constant >= 0 keeps the order of the costs, so the lowest candidate away from the winner decides for all of them.
//
// GPU mapping: elementwise, one thread per pixel, grid (pixels / kUnThreads, views).
#pragma once
#include "psm_common.cuh"

namespace psm {

constexpr int kUnThreads = 256;

template <typename T>
struct UniqueArgs {
    const T* in[2];          // the maps to test (read only)
    const float* qm[2];      // q(m): plane 1 of the costs
    const float* qr[2];      // q(r): plane 1 of the runner-up
    T* out[2];               // the tested maps
    size_t npix;
    int ratio;               // [0, 100]
};

template <typename T>
__global__ void __launch_bounds__(kUnThreads) unique_kernel(const UniqueArgs<T> a)
{
    const size_t i = (size_t)blockIdx.x * kUnThreads + threadIdx.x;
    if (i >= a.npix) return;
    const int view = blockIdx.y;
    const T m = __ldg((view ? a.in[1] : a.in[0]) + i);
    T v = m;
    if (m != 0) {
        const double qr = __ldg((view ? a.qr[1] : a.qr[0]) + i), qm = __ldg((view ? a.qm[1] : a.qm[0]) + i);
        if (__dmul_rn(qr, (double)(100 - a.ratio)) < __dmul_rn(qm, 100.0)) v = 0;
    }
    (view ? a.out[1] : a.out[0])[i] = v;
}

}  // namespace psm
