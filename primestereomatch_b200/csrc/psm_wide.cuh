// psm_wide.cuh -- 16-bit disparity maps (psm_create_u16): the selection, sharded reduction and post-filter kernels for
// contexts whose maps are uint16_t, so that max_disp may reach 4096.  Each kernel is a twin of a u8 kernel of
// psm_kernels.cuh / psm_pp.cuh / psm_pp_param.cuh with the same definition; only the map width changes.  The u8 kernels
// are not touched (their SASS stays what it was).
//
// Reference pins (DESIGN.md section 14): DispSel::CVSelect computes the arg-min as an int and stores it in a uchar, so
// for max_disp > 256 the reference's own map is the low byte of the u16 map here.  JointWMF::filter on a CV_32F map of
// integer values with nI = max_disp gives every value its own quantisation index and maps it back exactly: that is the
// reference definition of the post-filter on wide maps, and it is the same order-based weighted median as on u8 maps.
#pragma once
#include "psm_kernels.cuh"
#include "psm_pp.cuh"
#include "psm_pp_param.cuh"

namespace psm {

constexpr int kWideMaxDisp = 4096;   // 12-bit disparity + 18 colour bits fill the packed u32 of the post-filter

// wta_kernel with a u16 map: per pixel arg-min over global d in [1, D), strict <, ties -> lowest d, minCost starts at
// +inf, 0 when nothing compares below +inf.  One thread = 4 pixels; the same 4*V bytes of volume per view as the u8 twin.
__global__ void __launch_bounds__(256) wta16_kernel(const float* __restrict__ vol, int W, int H, int Wp, int d_begin, int d_count,
                                                    uint16_t* __restrict__ dis /* [H][W] */)
{
    const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const int y = blockIdx.y;
    if (x4 >= W) return;
    const size_t plane = (size_t)H * Wp;
    const float* p = vol + (size_t)y * Wp + x4;
    float mc[4] = {INFINITY, INFINITY, INFINITY, INFINITY};
    int md[4] = {0, 0, 0, 0};
    int dl = (d_begin == 0) ? 1 : 0;  // global d = 0 is never a candidate (DispSel.cpp:96)
#pragma unroll 8
    for (; dl < d_count; ++dl) {
        const float4 c = __ldg(reinterpret_cast<const float4*>(p + (size_t)dl * plane));
        const int d = d_begin + dl;
        if (c.x < mc[0]) { mc[0] = c.x; md[0] = d; }
        if (c.y < mc[1]) { mc[1] = c.y; md[1] = d; }
        if (c.z < mc[2]) { mc[2] = c.z; md[2] = d; }
        if (c.w < mc[3]) { mc[3] = c.w; md[3] = d; }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
        if (x4 + j < W) dis[(size_t)y * W + x4 + j] = (uint16_t)md[j];
}

// keys_reduce_kernel with a u16 map: min over ranks of the packed keys, low 16 bits of the winner
__global__ void keys_reduce16_kernel(const unsigned long long* __restrict__ gathered, int nranks, size_t npix,
                                     uint16_t* __restrict__ dis)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix) return;
    unsigned long long k = gathered[i];
    for (int r = 1; r < nranks; ++r) {
        const unsigned long long v = gathered[(size_t)r * npix + i];
        k = v < k ? v : k;
    }
    dis[i] = (uint16_t)(k & 0xffffu);
}

// chunk_reduce_kernel with u16 result maps (peers.maps[r] points at 2-byte maps): the same ARRIVE wait, min over the
// ranks' slots, store into every rank's map, DONE flag
__global__ void __launch_bounds__(256) chunk_reduce16_kernel(P2pPeers peers, unsigned npix)
{
    if (peers.seq) {
        if (threadIdx.x < (unsigned)peers.nranks) {
            const unsigned* f = peers.flags[peers.rank] + threadIdx.x;
            while ((int)(ld_acquire_sys(f) - peers.seq) < 0) __nanosleep(64);
        }
        __syncthreads();
    }
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned pix = (unsigned)peers.rank * peers.chunk + i;
    if (i < peers.chunk && pix < npix) {
        const unsigned long long* mine = peers.keys[peers.rank];
        unsigned long long k = __ldcg(mine + i);
        for (int r = 1; r < peers.nranks; ++r) {
            const unsigned long long v = __ldcg(mine + (size_t)r * peers.chunk + i);
            k = v < k ? v : k;
        }
        const uint16_t d = (uint16_t)(k & 0xffffu);
        for (int r = 0; r < peers.nranks; ++r) reinterpret_cast<uint16_t*>(peers.maps[r])[pix] = d;
    }
    if (peers.seq) p2p_publish(peers, kMaxRanks);   // DONE
}

// pp_pack_kernel for u16 maps: d << 18 | R6 << 12 | G6 << 6 | B6 (d < 4096)
__global__ void pp_pack16_kernel(const float* __restrict__ I0, const float* __restrict__ I1, const float* __restrict__ I2, int Wp,
                                 const uint16_t* __restrict__ disp, int W, int H, uint32_t* __restrict__ packed)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= W || y >= H) return;
    const size_t o = (size_t)y * Wp + x;
    auto q6 = [](float v) {   // convertTo(CV_8UC3, 255), then 8 bit -> 6 bit, as pp_pack_kernel
        int q = __float2int_rn(fmul(v, 255.0f));
        q = q < 0 ? 0 : (q > 255 ? 255 : q);
        return (uint32_t)(q >> 2);
    };
    const uint32_t b = q6(I0[o]), g = q6(I1[o]), r = q6(I2[o]);
    packed[(size_t)y * W + x] = ((uint32_t)disp[(size_t)y * W + x] << 18) | (r << 12) | (g << 6) | b;
}

// pp_wmf_kernel on u16 maps (radius 9, sigma 25.5, exp): the 361 taps stay in registers; `steps` = ceil(log2 max_disp)
// bisection steps over [0, max_disp - 1] instead of eight over [0, 255]
__global__ void __launch_bounds__(kPpWarps * 32) pp_wmf16_kernel(const uint32_t* __restrict__ packed, const uint32_t* __restrict__ lut,
                                                                int W, int H, int max_disp, int steps, uint16_t* __restrict__ out)
{
    __shared__ uint32_t slut[kPpLutN];
    for (int i = threadIdx.x; i < kPpLutN; i += blockDim.x) slut[i] = __ldg(lut + i);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int kSide = 2 * kPpRadius + 1, kTaps = kSide * kSide, kRounds = (kTaps + 31) / 32;
    const long npix = (long)W * H;
    for (long pix = (long)blockIdx.x * kPpWarps + warp; pix < npix; pix += (long)gridDim.x * kPpWarps) {
        const int y = (int)(pix / W), x = (int)(pix - (long)y * W);
        const uint32_t cp = __ldg(packed + pix);
        const int pb = cp & 63, pg = (cp >> 6) & 63, pr = (cp >> 12) & 63;
        uint32_t dq[kRounds], wq[kRounds];
        uint32_t total = 0;
#pragma unroll
        for (int r = 0; r < kRounds; ++r) {
            const int i = r * 32 + lane;
            const int dy = i / kSide, dx = i - dy * kSide;
            const int yy = y - kPpRadius + dy, xx = x - kPpRadius + dx;
            const bool ok = i < kTaps && yy >= 0 && yy < H && xx >= 0 && xx < W;
            dq[r] = 0xffffffffu;   // above every candidate value: never counted
            wq[r] = 0u;
            if (ok) {
                const uint32_t cq = __ldg(packed + (size_t)yy * W + xx);
                const int d0 = pb - (int)(cq & 63), d1 = pg - (int)((cq >> 6) & 63), d2 = pr - (int)((cq >> 12) & 63);
                const int dd = d0 * d0 + d1 * d1 + d2 * d2;
                wq[r] = dd < kPpLutN ? slut[dd] : 0u;
                dq[r] = cq >> 18;
            }
            total += wq[r];
        }
        total = __reduce_add_sync(0xffffffffu, total);
        int lo = 0, hi = max_disp - 1;
#pragma unroll 1
        for (int it = 0; it < steps; ++it) {
            const int mid = (lo + hi) >> 1;
            uint32_t s = 0;
#pragma unroll
            for (int r = 0; r < kRounds; ++r) s += dq[r] <= (uint32_t)mid ? wq[r] : 0u;
            s = __reduce_add_sync(0xffffffffu, s);
            if (2u * s >= total) hi = mid; else lo = mid + 1;
        }
        if (lane == 0) out[pix] = (uint16_t)lo;
    }
}

// pp_wmf_param_kernel on u16 maps: an exact two-level select.  Pass 1 fills the warp's 256-bin histogram with d >> 4 by
// the same warp aggregation; one warp scan finds the coarse bucket B holding the median and the weight below it.  Pass 2
// walks the window again and adds the taps of bucket B by d & 15 into 16 bins; a second scan finds the fine bin.  Integer
// sums throughout: out = min { v : 2 * sum_{I_q <= v} W >= sum W }, bit-exact and order-independent.
__global__ void __launch_bounds__(kPpParamWarps * 32) pp_wmf16_param_kernel(const uint32_t* __restrict__ packed,
                                                                            const uint32_t* __restrict__ lut, int lut_n, int idx_mode,
                                                                            int radius, int W, int H, uint16_t* __restrict__ out)
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
        const int y = (int)(pix / W), x = (int)(pix - (long)y * W);
        const uint32_t cp = __ldg(packed + pix);
        const int pb = cp & 63, pg = (cp >> 6) & 63, pr = (cp >> 12) & 63;
        // one tap of the window: (disparity, weight), ok = inside the clipped window
        auto tap = [&](int i, uint32_t& d, uint32_t& w) -> bool {
            const int dy = (int)__umulhi((uint32_t)i, magic), dx = i - dy * side;
            const int yy = y - radius + dy, xx = x - radius + dx;
            const bool ok = i < taps && yy >= 0 && yy < H && xx >= 0 && xx < W;
            d = 0xffffffffu; w = 0u;
            if (ok) {
                const uint32_t cq = __ldg(packed + (size_t)yy * W + xx);
                const int d0 = pb - (int)(cq & 63), d1 = pg - (int)((cq >> 6) & 63), d2 = pr - (int)((cq >> 12) & 63);
                const int k = idx_mode == kIdxSq ? d0 * d0 + d1 * d1 + d2 * d2
                            : idx_mode == kIdxL1 ? abs(d0) + abs(d1) + abs(d2) : 0;
                w = slut[k];
                d = cq >> 18;
            }
            return ok;
        };
        // pass 1: coarse histogram of d >> 4
        for (int i = lane; i - lane < taps; i += 32) {
            uint32_t d, w;
            const bool ok = tap(i, d, w);
            const uint32_t b = d >> 4;
            unsigned todo = __ballot_sync(0xffffffffu, ok);
            while (todo) {
                const uint32_t bl = __shfl_sync(0xffffffffu, b, __ffs(todo) - 1);
                const bool mine = ok && b == bl;
                todo &= ~__ballot_sync(0xffffffffu, mine);
                const uint32_t s = __reduce_add_sync(0xffffffffu, mine ? w : 0u);
                if (lane == 0) hist[bl] += s;
            }
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
            const bool ok = tap(i, d, w) && (d >> 4) == bucket;
            const uint32_t f = d & 15u;
            unsigned todo = __ballot_sync(0xffffffffu, ok);
            while (todo) {
                const uint32_t fl = __shfl_sync(0xffffffffu, f, __ffs(todo) - 1);
                const bool mine = ok && f == fl;
                todo &= ~__ballot_sync(0xffffffffu, mine);
                const uint32_t s = __reduce_add_sync(0xffffffffu, mine ? w : 0u);
                if (lane == 0) hist[fl] += s;
            }
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
