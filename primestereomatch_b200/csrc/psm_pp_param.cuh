// psm_pp_param.cuh -- post-processing at any filter setting (psm_set_post_filter): the joint weighted median of
// psm_pp.cuh for any radius 1..32 and any of the exp / iv1 / iv2 / off weight tables.
//
// What is computed: for every pixel p
//   out(p) = min { v : 2 * sum_{q in window, I_q <= v} W(p,q)  >=  sum_{q in window} W(p,q) }
// window = (2r+1)^2 clipped at the image border, W = the 2^-22 fixed-point weight of the colour difference between the
// 6-bit colours of p and q, looked up in a host-built table (DESIGN.md section 13) indexed by
//   kIdxSq: the squared distance d0^2 + d1^2 + d2^2 (exp, iv2; 11908 entries)
//   kIdxL1: the L1 distance |d0| + |d1| + |d2|      (iv1; 190 entries)
//   kIdxOne: entry 0 for every tap                   (off; 1 entry)
// The window total stays below 2^35 (4225 taps of at most 2^22): bins and sums are u64.
//
// GPU mapping: one WARP per pixel, the pixels of a CTA consecutive in raster order (their windows overlap: the taps
// are L1 hits).  The window taps are walked in raster order, 32 per round (lane = tap), each one 4-byte load of the
// packed image of pp_pack_kernel.  Every warp owns a 256-bin u64 histogram in shared memory; a round adds its taps by
// disparity with warp aggregation: neighbouring taps nearly always share a disparity, so the round loops over its
// DISTINCT disparities (usually one to three), each one ballot + REDUX, and lane 0 adds the group's sum to its bin.
// Only lane 0 writes the histogram, so there are no atomics and the sums are exact and order-independent.  The
// median is then one warp scan of the 256 bins (8 per lane).  The weight table lives in shared memory next to the
// histograms (dynamic, up to 46.5 KiB + 2 KiB per warp).
#pragma once
#include "psm_common.cuh"

namespace psm {

constexpr int kPpParamMaxRadius = 32;
constexpr int kPpParamWarps = 8;             // warps (pixels in flight) per CTA
enum { kIdxSq = 0, kIdxL1 = 1, kIdxOne = 2 };

__global__ void __launch_bounds__(kPpParamWarps * 32) pp_wmf_param_kernel(const uint32_t* __restrict__ packed,
                                                                          const uint32_t* __restrict__ lut, int lut_n, int idx_mode,
                                                                          int radius, int W, int H, uint8_t* __restrict__ out)
{
    extern __shared__ __align__(16) unsigned char pp_smem[];
    unsigned long long* hist_all = reinterpret_cast<unsigned long long*>(pp_smem);     // [kPpParamWarps][256]
    uint32_t* slut = reinterpret_cast<uint32_t*>(hist_all + kPpParamWarps * 256);
    for (int i = threadIdx.x; i < lut_n; i += blockDim.x) slut[i] = __ldg(lut + i);
    for (int i = threadIdx.x; i < kPpParamWarps * 256; i += blockDim.x) hist_all[i] = 0ull;
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    unsigned long long* hist = hist_all + warp * 256;
    const int side = 2 * radius + 1, taps = side * side;
    // i / side for i < 2^16 by one multiply-high: floor(i * m / 2^32) with m = floor(2^32 / side) + 1 is exact for
    // i < 2^32 / side
    const uint32_t magic = (uint32_t)(0xffffffffu / (uint32_t)side) + 1u;
    const long npix = (long)W * H;
    for (long pix = (long)blockIdx.x * kPpParamWarps + warp; pix < npix; pix += (long)gridDim.x * kPpParamWarps) {
        const int y = (int)(pix / W), x = (int)(pix - (long)y * W);
        const uint32_t cp = __ldg(packed + pix);
        const int pb = cp & 63, pg = (cp >> 8) & 63, pr = (cp >> 16) & 63;
        for (int i = lane; i - lane < taps; i += 32) {
            const int dy = (int)__umulhi((uint32_t)i, magic), dx = i - dy * side;
            const int yy = y - radius + dy, xx = x - radius + dx;
            const bool ok = i < taps && yy >= 0 && yy < H && xx >= 0 && xx < W;
            uint32_t d = 256u, w = 0u;      // outside the clipped window: a bin no group ever adds to
            if (ok) {
                const uint32_t cq = __ldg(packed + (size_t)yy * W + xx);
                const int d0 = pb - (int)(cq & 63), d1 = pg - (int)((cq >> 8) & 63), d2 = pr - (int)((cq >> 16) & 63);
                const int k = idx_mode == kIdxSq ? d0 * d0 + d1 * d1 + d2 * d2
                            : idx_mode == kIdxL1 ? abs(d0) + abs(d1) + abs(d2) : 0;
                w = slut[k];
                d = cq >> 24;
            }
            // warp aggregation over the round's distinct disparities: one ballot + REDUX each (<= 2^27 per sum)
            unsigned todo = __ballot_sync(0xffffffffu, ok);
            while (todo) {
                const uint32_t dl = __shfl_sync(0xffffffffu, d, __ffs(todo) - 1);
                const bool mine = ok && d == dl;
                todo &= ~__ballot_sync(0xffffffffu, mine);
                const uint32_t s = __reduce_add_sync(0xffffffffu, mine ? w : 0u);
                if (lane == 0) hist[dl] += s;
            }
        }
        __syncwarp();
        // scan: lane owns bins 8*lane .. 8*lane+7; out = first v whose inclusive prefix c satisfies 2c >= total
        unsigned long long b[8], own = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) { b[k] = hist[lane * 8 + k]; own += b[k]; }
        unsigned long long incl = own;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        const unsigned long long total = __shfl_sync(0xffffffffu, incl, 31);
        unsigned long long cum = incl - own;
        int hit = 8;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            cum += b[k];
            if (hit == 8 && 2ull * cum >= total) hit = k;
        }
        const unsigned found = __ballot_sync(0xffffffffu, hit < 8);   // lane 31 always finds: its last prefix is the total
        const int src = __ffs(found) - 1;
        const int h = __shfl_sync(0xffffffffu, hit, src);
        if (lane == 0) out[pix] = (uint8_t)(src * 8 + h);
#pragma unroll
        for (int k = 0; k < 8; ++k) hist[lane * 8 + k] = 0ull;
        __syncwarp();
    }
}

}  // namespace psm
