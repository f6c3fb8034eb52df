// psm_pp.cuh -- post-processing: joint weighted-median filter of the disparity maps on the device.
//
// Reference: PP::processDM (/root/reference/src/PP.cpp:402-425), whose live code is
//   img.convertTo(img8UC3, CV_8UC3, 255);  disp = JointWMF::filter(disp, img8UC3, MED_SZ/2 = 9)
// (vendored include/JointWMF.h:81-155, filterCore :173-390) and which the reference runs on the CPU even in
// its GPU mode (src/DispEst.cpp:338-344).
//
// What is computed (exactly what the CPU restatement orc_wmf (test infrastructure, oracle/) restates, and what the reference's
// JointWMF computes whenever the feature image has <= 256 distinct 6-bit colours): for every pixel p
//   out(p) = min { v : sum_{q in window, I_q <= v} w(p,q)  >=  sum_{q in window, I_q > v} w(p,q) }
// window = (2r+1)^2 clipped at the image border, w = exp(-|c_p - c_q|^2 / (2 s^2)) on the 6-bit colours
// c = (B,G,R) >> 2, s = 25.5/256*64, held as 2^-22 fixed point: the context's one weight table, built on the host by
// pp_weight_table (psm_capi.cu) from the reference's float expression; this kernel reads its first kPpLutN entries.  The
// reference also clusters the colours to 256 indices with cv::kmeans (RNG-seeded, un-vendored): parity for natural
// images is unpinned by the reference itself; this kernel needs no clustering -- it evaluates the weights directly.
//
// GPU mapping (nothing like the reference's serial column scan with necklace tables): one WARP per pixel,
//   the 361 window taps dealt round-robin to the 32 lanes (12 rounds), each tap one 4-byte load of a packed
//   u32 image, d << kDispShift | R6 << 2 * kColourBits | G6 << kColourBits | B6 (MapFormat, psm_common.cuh):
//   d << 24 | R6 << 16 | G6 << 8 | B6 for u8 maps, d << 18 | R6 << 12 | G6 << 6 | B6 for u16 maps;
//   the taps ((disparity, fixed-point weight) pairs) stay in registers, 12 per lane; the weighted median is found by
//   bisection on the value, eight steps over [0, 255] on u8 maps and ceil(log2 D) steps over [0, D - 1] on u16 maps,
//   each a masked add per tap and one warp REDUX -- no shared memory, no atomics, integer sums (exact,
//   order-independent, identical to a histogram scan).
#pragma once
#include "psm_common.cuh"

namespace psm {

constexpr int kPpRadius = 9;                 // MED_SZ / 2, reference include/PP.h:12
constexpr int kPpMaxD2 = 3 * 63 * 63;        // largest squared distance between two 6-bit colours
constexpr int kPpWarps = 8;                  // warps (pixels in flight) per CTA
constexpr int kPpLutN = 1344;                // the 2^-22 fixed-point weight is zero beyond d2 = 1295 (exp(-d2/81.3) < 2^-23): only this
                                             // prefix of the table is ever non-zero; it lives in shared memory (random gathers: bank
                                             // conflicts cost a few cycles, L1 line wavefronts cost up to 32 per load)

// guide planes (float, BGR planar) + disparity map -> packed u32 image
template <typename T>
__global__ void pp_pack_kernel(const float* __restrict__ I0, const float* __restrict__ I1, const float* __restrict__ I2, int Wp,
                               const T* __restrict__ disp, int W, int H, uint32_t* __restrict__ packed)
{
    using F = MapFormat<T>;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= W || y >= H) return;
    const size_t o = (size_t)y * Wp + x;
    // convertTo(CV_8UC3, 255): saturate_cast<uchar>(cvRound(v * 255.0f)), round half to even (PP.cpp:416-417).  cvRound
    // on x86 returns INT_MIN for a NaN or a product >= 2^31, which saturates to 0 (__float2int_rn would give 255 there)
    auto q6 = [](float v) {
        const float f = fmul(v, 255.0f);
        int q = f < 2147483648.0f ? __float2int_rn(f) : 0;
        q = q < 0 ? 0 : (q > 255 ? 255 : q);
        return (uint32_t)(q >> 2);           // JointWMF.h:546,559-561: 8 bit -> 6 bit
    };
    const uint32_t b = q6(I0[o]), g = q6(I1[o]), r = q6(I2[o]);
    packed[(size_t)y * W + x] =
        ((uint32_t)disp[(size_t)y * W + x] << F::kDispShift) | (r << 2 * F::kColourBits) | (g << F::kColourBits) | b;
}

// max_disp and steps = ceil(log2 max_disp) bound the bisection on u16 maps; u8 maps always take eight steps over [0, 255]
template <typename T>
__global__ void __launch_bounds__(kPpWarps * 32) pp_wmf_kernel(const uint32_t* __restrict__ packed, const uint32_t* __restrict__ lut,
                                                              int W, int H, T* __restrict__ out, int max_disp, int steps)
{
    using F = MapFormat<T>;
    __shared__ uint32_t slut[kPpLutN];
    for (int i = threadIdx.x; i < kPpLutN; i += blockDim.x) slut[i] = __ldg(lut + i);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int kSide = 2 * kPpRadius + 1, kTaps = kSide * kSide, kRounds = (kTaps + 31) / 32;
    const long npix = (long)W * H;
    for (long pix = (long)blockIdx.x * kPpWarps + warp; pix < npix; pix += (long)gridDim.x * kPpWarps) {
        const int y = (int)(pix / W), x = (int)(pix - (long)y * W);
        const uint32_t cp = __ldg(packed + pix);
        const int pb = cp & 63, pg = (cp >> F::kColourBits) & 63, pr = (cp >> 2 * F::kColourBits) & 63;
        // the 361 window taps are dealt round-robin to the 32 lanes and stay in registers: (disparity, weight) x 12
        uint32_t dq[kRounds], wq[kRounds];
        uint32_t total = 0;
#pragma unroll
        for (int r = 0; r < kRounds; ++r) {
            const int i = r * 32 + lane;
            const int dy = i / kSide, dx = i - dy * kSide;
            const int yy = y - kPpRadius + dy, xx = x - kPpRadius + dx;
            const bool ok = i < kTaps && yy >= 0 && yy < H && xx >= 0 && xx < W;
            dq[r] = F::kSentinel;     // greater than every candidate value: never counted
            wq[r] = 0u;
            if (ok) {
                const uint32_t cq = __ldg(packed + (size_t)yy * W + xx);
                const int d0 = pb - (int)(cq & 63), d1 = pg - (int)((cq >> F::kColourBits) & 63),
                          d2 = pr - (int)((cq >> 2 * F::kColourBits) & 63);
                const int dd = d0 * d0 + d1 * d1 + d2 * d2;
                wq[r] = dd < kPpLutN ? slut[dd] : 0u;
                dq[r] = cq >> F::kDispShift;
            }
            total += wq[r];
        }
        total = __reduce_add_sync(0xffffffffu, total);
        // out = min { v : 2 * sum_{dq <= v} w >= total }: bisection steps, each one masked add per tap and one REDUX
        // (integer sums: exact and order-independent, identical to a histogram scan).  u8 maps: eight fully unrolled
        // steps over [0, 255]; u16 maps: `steps` rolled steps over [0, max_disp - 1]
        constexpr bool kU8 = sizeof(T) == 1;
        int lo = 0, hi = kU8 ? 255 : max_disp - 1;
        const int nsteps = kU8 ? 8 : steps;
#pragma unroll(kU8 ? 8 : 1)
        for (int it = 0; it < nsteps; ++it) {
            const int mid = (lo + hi) >> 1;
            uint32_t s = 0;
#pragma unroll
            for (int r = 0; r < kRounds; ++r) s += dq[r] <= (uint32_t)mid ? wq[r] : 0u;
            s = __reduce_add_sync(0xffffffffu, s);
            if (2u * s >= total) hi = mid; else lo = mid + 1;
        }
        if (lane == 0) out[pix] = (T)lo;
    }
}

}  // namespace psm
