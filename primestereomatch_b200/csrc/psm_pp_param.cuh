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
// Only lane 0 writes the histogram, so there are no atomics and the sums are exact and order-independent.  On u8 maps
// the median is then one warp scan of the 256 bins (8 per lane).  u16 maps have up to 4096 values, and a 4096-bin
// histogram per warp does not fit in shared memory: pp_wmf_param_two_level_kernel selects in two levels over the same
// 256 bins instead.  The weight table lives in shared memory next to the histograms (dynamic, up to 46.5 KiB + 2 KiB
// per warp).
#pragma once
#include "psm_common.cuh"

namespace psm {

constexpr int kPpParamMaxRadius = 32;
constexpr int kPpParamWarps = 8;             // warps (pixels in flight) per CTA
enum { kIdxSq = 0, kIdxL1 = 1, kIdxOne = 2 };

// The clipped window of one pixel in the packed image of pp_pack_kernel<T>.  tap(i) gives window tap i (raster order)
// as (disparity, weight) and whether it lies inside the clipped window; outside it d = the sentinel and w = 0.
template <typename T>
struct PpWindow {
    const uint32_t* __restrict__ packed;
    const uint32_t* slut;
    int idx_mode, radius, side, taps, W, H;
    uint32_t magic;   // i / side for i < 2^16 by one multiply-high: floor(i * m / 2^32) with m = floor(2^32 / side) + 1
                      // is exact for i < 2^32 / side
    int x, y, pb, pg, pr;

    __device__ __forceinline__ PpWindow(const uint32_t* __restrict__ packed_, const uint32_t* slut_, int idx_mode_, int radius_,
                                        int side_, int taps_, uint32_t magic_, int W_, int H_, long pix)
        : packed(packed_), slut(slut_), idx_mode(idx_mode_), radius(radius_), side(side_), taps(taps_), W(W_), H(H_), magic(magic_)
    {
        constexpr int kC = MapFormat<T>::kColourBits;
        y = (int)(pix / W); x = (int)(pix - (long)y * W);
        const uint32_t cp = __ldg(packed + pix);
        pb = cp & 63; pg = (cp >> kC) & 63; pr = (cp >> 2 * kC) & 63;
    }

    __device__ __forceinline__ bool tap(int i, uint32_t& d, uint32_t& w) const
    {
        using F = MapFormat<T>;
        const int dy = (int)__umulhi((uint32_t)i, magic), dx = i - dy * side;
        const int yy = y - radius + dy, xx = x - radius + dx;
        const bool ok = i < taps && yy >= 0 && yy < H && xx >= 0 && xx < W;
        d = F::kSentinel; w = 0u;
        if (ok) {
            const uint32_t cq = __ldg(packed + (size_t)yy * W + xx);
            const int d0 = pb - (int)(cq & 63), d1 = pg - (int)((cq >> F::kColourBits) & 63),
                      d2 = pr - (int)((cq >> 2 * F::kColourBits) & 63);
            const int k = idx_mode == kIdxSq ? d0 * d0 + d1 * d1 + d2 * d2
                        : idx_mode == kIdxL1 ? abs(d0) + abs(d1) + abs(d2) : 0;
            w = slut[k];
            d = cq >> F::kDispShift;
        }
        return ok;
    }
};

// warp aggregation of one round: hist[bin] += w over the lanes with `ok`, one ballot + REDUX per distinct bin
// (<= 2^27 per sum); only lane 0 writes the histogram
__device__ __forceinline__ void pp_bin_add(unsigned long long* hist, bool ok, uint32_t bin, uint32_t w, int lane)
{
    unsigned todo = __ballot_sync(0xffffffffu, ok);
    while (todo) {
        const uint32_t bl = __shfl_sync(0xffffffffu, bin, __ffs(todo) - 1);
        const bool mine = ok && bin == bl;
        todo &= ~__ballot_sync(0xffffffffu, mine);
        const uint32_t s = __reduce_add_sync(0xffffffffu, mine ? w : 0u);
        if (lane == 0) hist[bl] += s;
    }
}

// u8 maps: one histogram of the 256 values and one scan
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
    const uint32_t magic = (uint32_t)(0xffffffffu / (uint32_t)side) + 1u;
    const long npix = (long)W * H;
    for (long pix = (long)blockIdx.x * kPpParamWarps + warp; pix < npix; pix += (long)gridDim.x * kPpParamWarps) {
        const PpWindow<uint8_t> win(packed, slut, idx_mode, radius, side, taps, magic, W, H, pix);
        for (int i = lane; i - lane < taps; i += 32) {
            uint32_t d, w;
            const bool ok = win.tap(i, d, w);
            // pp_bin_add(hist, ok, d, w, lane) written out: through the helper, nvcc emits this kernel with the
            // operands of one compare swapped
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

// u16 maps: an exact two-level select.  Pass 1 fills the warp's 256-bin histogram with d >> 4; one warp scan finds the
// coarse bucket B holding the median and the weight below it.  Pass 2 walks the window again and adds the taps of
// bucket B by d & 15 into 16 bins; a second scan finds the fine bin.  Integer sums throughout:
// out = min { v : 2 * sum_{I_q <= v} W >= sum W }, bit-exact and order-independent.
__global__ void __launch_bounds__(kPpParamWarps * 32) pp_wmf_param_two_level_kernel(const uint32_t* __restrict__ packed,
                                                                                    const uint32_t* __restrict__ lut, int lut_n,
                                                                                    int idx_mode, int radius, int W, int H,
                                                                                    uint16_t* __restrict__ out)
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
    const uint32_t magic = (uint32_t)(0xffffffffu / (uint32_t)side) + 1u;
    const long npix = (long)W * H;
    for (long pix = (long)blockIdx.x * kPpParamWarps + warp; pix < npix; pix += (long)gridDim.x * kPpParamWarps) {
        const PpWindow<uint16_t> win(packed, slut, idx_mode, radius, side, taps, magic, W, H, pix);
        // pass 1: coarse histogram of d >> 4
        for (int i = lane; i - lane < taps; i += 32) {
            uint32_t d, w;
            const bool ok = win.tap(i, d, w);
            pp_bin_add(hist, ok, d >> 4, w, lane);
        }
        __syncwarp();
        unsigned long long b8[8], own = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) { b8[k] = hist[lane * 8 + k]; own += b8[k]; }
        unsigned long long incl = own;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        const unsigned long long total = __shfl_sync(0xffffffffu, incl, 31);
        unsigned long long cum = incl - own, below = 0;
        int hit = 8;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            if (hit == 8 && 2ull * (cum + b8[k]) >= total) { hit = k; below = cum; }
            cum += b8[k];
        }
        const unsigned found = __ballot_sync(0xffffffffu, hit < 8);
        const int src = __ffs(found) - 1;
        const uint32_t bucket = (uint32_t)(src * 8 + __shfl_sync(0xffffffffu, hit, src));
        below = __shfl_sync(0xffffffffu, below, src);   // weight of every tap below the bucket
#pragma unroll
        for (int k = 0; k < 8; ++k) hist[lane * 8 + k] = 0ull;
        __syncwarp();
        // pass 2: the bucket's taps by d & 15
        for (int i = lane; i - lane < taps; i += 32) {
            uint32_t d, w;
            const bool ok = win.tap(i, d, w) && (d >> 4) == bucket;
            pp_bin_add(hist, ok, d & 15u, w, lane);
        }
        __syncwarp();
        const unsigned long long fb = lane < 16 ? hist[lane] : 0ull;
        unsigned long long fin = fb;
#pragma unroll
        for (int o = 1; o < 16; o <<= 1) {
            const unsigned long long t = __shfl_up_sync(0xffffffffu, fin, o);
            if (lane >= o) fin += t;
        }
        // the bucket holds the median, so some fine bin of it satisfies the condition (lane 15 at the latest)
        const unsigned ffound = __ballot_sync(0xffffffffu, lane < 16 && 2ull * (below + fin) >= total);
        if (lane == 0) out[pix] = (uint16_t)(bucket * 16 + (uint32_t)(__ffs(ffound) - 1));
        if (lane < 16) hist[lane] = 0ull;
        __syncwarp();
    }
}

}  // namespace psm
