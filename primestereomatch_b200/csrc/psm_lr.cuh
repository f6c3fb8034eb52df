// psm_lr.cuh -- left-right consistency check and occlusion fill of the disparity maps (psm_set_lr_check).
//
// Reference: lrCheck and fillInv (the reference's src/PP.cpp:17-143), which PP::processDM has commented out in front of
// its weighted median (PP.cpp:405-406).  What is computed, per row, on integer map values (W = width, mod = the
// non-negative remainder; the reference's (x - d + W) % W equals it wherever d <= x + W and is undefined beyond):
//   lValid[x] = l[x] == r[(x - l[x]) mod W] && l[x] >= 2        rValid[x] = r[x] == l[(x + r[x]) mod W] && r[x] >= 2
// both on the unmodified maps; then each view with its own mask: a valid pixel keeps its value, an invalid pixel x takes
// min(map[L], map[R]) of the nearest valid pixels L <= x <= R, or the one of them that exists; a row with no valid pixel
// is unchanged.  Valid pixels are never written, so the result does not depend on the visiting order.
//
// GPU mapping: one CTA per row, both views.  Rows of up to kLrStageCols columns are staged in shared memory with their
// masks, so the check's gathers never leave the CTA; wider rows gather from global memory and keep their masks in the
// output masks (written, __syncthreads, read back by the same CTA).  The fill walks the row in chunks of
// kLrThreads * kLrItems columns, each thread owning kLrItems consecutive columns: a right-to-left chunk pass takes the
// block-wide min-scan of "index of the next valid pixel" and writes map[R] (or the pixel's own value when no R exists);
// a left-to-right pass takes the max-scan of "index of the last valid pixel" and combines map[L] with it.  Each pass
// carries its scan state from chunk to chunk, and every column is read and written by the same thread in both passes.
#pragma once
#include "psm_common.cuh"

namespace psm {

constexpr int kLrThreads = 256;
constexpr int kLrItems = 4;
constexpr int kLrChunk = kLrThreads * kLrItems;
constexpr int kLrStageCols = 7680;   // 2 maps + 2 masks, at most 6 bytes per column: 45 KiB, under the 48 KiB that needs
                                     // no opt-in

// Exclusive block scan of two values per thread (left and right view) in thread order (kForward, max) or reverse thread
// order (!kForward, min), seeded with carry; carry becomes the combination with every thread's value.
template <bool kForward>
__device__ __forceinline__ int2 lr_block_scan(int2 v, int2& carry, int2* warp_part)
{
    auto op = [](int a, int b) { return kForward ? max(a, b) : min(a, b); };
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int kWarps = kLrThreads / 32;
    int2 incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int ax = kForward ? __shfl_up_sync(0xffffffffu, incl.x, o) : __shfl_down_sync(0xffffffffu, incl.x, o);
        const int ay = kForward ? __shfl_up_sync(0xffffffffu, incl.y, o) : __shfl_down_sync(0xffffffffu, incl.y, o);
        if (kForward ? lane >= o : lane + o < 32) { incl.x = op(incl.x, ax); incl.y = op(incl.y, ay); }
    }
    if (lane == (kForward ? 31 : 0)) warp_part[warp] = incl;
    // this thread's exclusive value: the inclusive value of its predecessor lane in scan order
    int2 ex;
    ex.x = kForward ? __shfl_up_sync(0xffffffffu, incl.x, 1) : __shfl_down_sync(0xffffffffu, incl.x, 1);
    ex.y = kForward ? __shfl_up_sync(0xffffffffu, incl.y, 1) : __shfl_down_sync(0xffffffffu, incl.y, 1);
    if (lane == (kForward ? 0 : 31)) ex = carry;
    else { ex.x = op(ex.x, carry.x); ex.y = op(ex.y, carry.y); }
    __syncthreads();
    int2 total = carry;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) {
        const int2 p = warp_part[w];
        if (kForward ? w < warp : w > warp) { ex.x = op(ex.x, p.x); ex.y = op(ex.y, p.y); }
        total.x = op(total.x, p.x); total.y = op(total.y, p.y);
    }
    __syncthreads();   // warp_part is reused by the next scan
    carry = total;
    return ex;
}

// l, r: the maps to check (read only); out_l, out_r: the filled maps; valid_l, valid_r: the masks (0/1).  One CTA of
// kLrThreads threads per row, bounded for eight CTAs per SM (without the bound ptxas spills a register on u16 maps);
// dynamic shared memory W * (2 * sizeof(T) + 2) bytes when W <= kLrStageCols, else none.  kOwn: the left view alone,
// its mask its own map >= 2 instead of the check against the right view (the fill of a left-only context after
// psm_set_disparity_check); r, out_r and valid_r are never touched and may be null.  It is bounded for six CTAs per SM:
// at eight ptxas spills.
template <typename T, bool kOwn>
__global__ void __launch_bounds__(kLrThreads, kOwn ? 6 : 8) lr_check_fill_kernel(const T* __restrict__ l, const T* __restrict__ r, int W,
                                                                   T* __restrict__ out_l, T* __restrict__ out_r,
                                                                   uint8_t* valid_l, uint8_t* valid_r)
{
    extern __shared__ __align__(16) unsigned char lr_smem[];
    __shared__ int2 warp_part[kLrThreads / 32];
    const size_t row = (size_t)blockIdx.x * W;
    const bool staged = W <= kLrStageCols;
    const T* ml = l + row;
    constexpr bool kRight = !kOwn;   // the right view's half of every step
    const T* mr = kRight ? r + row : nullptr;
    uint8_t* vl = valid_l + row;
    uint8_t* vr = kRight ? valid_r + row : nullptr;
    if (staged) {
        T* sl = reinterpret_cast<T*>(lr_smem);
        T* sr = sl + W;
        for (int x = threadIdx.x; x < W; x += kLrThreads) {
            sl[x] = __ldg(ml + x);
            if constexpr (kRight) sr[x] = __ldg(mr + x);
        }
        ml = sl; mr = sr;
        vl = reinterpret_cast<uint8_t*>(sr + W);
        vr = vl + W;
        __syncthreads();
    }
    // the check, on the unmodified maps
    int2 own_last = make_int2(-1, -1);
    for (int x = threadIdx.x; x < W; x += kLrThreads) {
        const int dl = ml[x], dr = kRight ? mr[x] : 0;
        uint8_t okl, okr;
        if constexpr (kOwn) {
            okl = dl >= 2;
            okr = 0;
        } else {
            int xl = (x - dl) % W;
            if (xl < 0) xl += W;
            const int xr = (int)(((unsigned)x + (unsigned)dr) % (unsigned)W);
            okl = dl >= 2 && dl == (int)mr[xl];
            okr = dr >= 2 && dr == (int)ml[xr];
        }
        vl[x] = okl;
        if constexpr (kRight) vr[x] = okr;
        if (staged) {
            valid_l[row + x] = okl;
            if constexpr (kRight) valid_r[row + x] = okr;
        }
        if (okl) own_last.x = x;
        if (okr) own_last.y = x;
    }
    // the last valid column of each view (-1: none): a pixel x has a valid pixel at or right of it iff x <= last.  The
    // scan's barriers also publish the masks to the whole CTA.
    int2 last = make_int2(-1, -1);
    lr_block_scan<true>(own_last, last, warp_part);
    // right to left: R = the nearest valid column at or right of x (W: none); out = map[R], or map[x] without an R
    T* ol = out_l + row;
    T* orr = kRight ? out_r + row : nullptr;
    const int nchunks = (W + kLrChunk - 1) / kLrChunk;
    int2 carry = make_int2(W, W);
    for (int c = nchunks - 1; c >= 0; --c) {
        const int x0 = c * kLrChunk + threadIdx.x * kLrItems;
        int2 own = make_int2(W, W);
#pragma unroll
        for (int i = kLrItems - 1; i >= 0; --i) {
            const int x = x0 + i;
            if (x < W) {
                if (vl[x]) own.x = x;
                if (kRight && vr[x]) own.y = x;
            }
        }
        int2 nxt = lr_block_scan<false>(own, carry, warp_part);
#pragma unroll
        for (int i = kLrItems - 1; i >= 0; --i) {
            const int x = x0 + i;
            if (x < W) {
                if (vl[x]) nxt.x = x;
                if (kRight && vr[x]) nxt.y = x;
                ol[x] = ml[nxt.x < W ? nxt.x : x];
                if constexpr (kRight) orr[x] = mr[nxt.y < W ? nxt.y : x];
            }
        }
    }
    // left to right: L = the nearest valid column at or left of x (-1: none); out = min(map[L], map[R]) or map[L]
    carry = make_int2(-1, -1);
    for (int c = 0; c < nchunks; ++c) {
        const int x0 = c * kLrChunk + threadIdx.x * kLrItems;
        int2 own = make_int2(-1, -1);
#pragma unroll
        for (int i = 0; i < kLrItems; ++i) {
            const int x = x0 + i;
            if (x < W) {
                if (vl[x]) own.x = x;
                if (kRight && vr[x]) own.y = x;
            }
        }
        int2 prv = lr_block_scan<true>(own, carry, warp_part);
#pragma unroll
        for (int i = 0; i < kLrItems; ++i) {
            const int x = x0 + i;
            if (x < W) {
                const bool gl = vl[x], gr = kRight && vr[x];
                if (gl) prv.x = x;
                if (gr) prv.y = x;
                // ol[x] holds map[R] where x <= last, else map[x]: then map[L] alone
                if (!gl && prv.x >= 0) {
                    const T a = ml[prv.x], b = ol[x];
                    ol[x] = x <= last.x && b < a ? b : a;
                }
                if (kRight && !gr && prv.y >= 0) {
                    const T a = mr[prv.y], b = orr[x];
                    orr[x] = x <= last.y && b < a ? b : a;
                }
            }
        }
    }
}

}  // namespace psm
