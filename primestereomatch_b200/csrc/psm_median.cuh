// psm_median.cuh -- the 3x3 / 5x5 median of the post-process stage (psm_set_median_blur; OpenCV's medianBlur, the
// fixed medianBlur(disp, 3) that StereoSGBM::compute runs between its winner-take-all and filterSpeckles).
//
// What is computed, per view and pixel (x, y) of a map m (u8 or u16), k = ksize (3 or 5), R = k / 2:
//   out(x, y) = the median of the k * k values m(clamp(x + i, 0, W - 1), clamp(y + j, 0, H - 1)), -R <= i, j <= R,
// a plain median with BORDER_REPLICATE, exactly cv::medianBlur(m, k) on CV_8U and CV_16U.  Zeros (invalid) take part as
// values, the lowest ones, as SGBM's invalid (minD - 1) * 16 does; no value is compared with anything but another value.
//
// GPU mapping: one thread per pixel in kMdTileX x kMdTileY tiles, every computed view in one launch (grid z).  Each CTA
// stages its tile with the replicated halo in shared memory, then each thread runs a fixed selection network over its
// k * k values in registers: 19 compare-exchanges for 9 values, 113 for 25 (Batcher's odd-even merge sort of 16 / 32
// wires with the wires past 25 taken as +inf and every exchange that cannot reach the middle wire removed).  No
// atomics: the result does not depend on any order.  tests/test_oracle_median.py checks both networks on every 0-1
// input (the 0-1 principle), so they select the median of any input.
#pragma once
#include "psm_common.cuh"

namespace psm {

constexpr int kMdTileX = 32, kMdTileY = 8;

template <typename T>
struct MedianArgs {
    const T* in[2];   // the maps to filter (read only)
    T* out[2];        // the filtered maps
    int W, H;
};

// compare-exchange: p[a] takes the lower value, p[b] the higher (constant indices: p stays in registers)
template <int N>
__device__ __forceinline__ void cs(int (&p)[N], int a, int b)
{
    const int lo = min(p[a], p[b]);
    p[b] = max(p[a], p[b]);
    p[a] = lo;
}

// the median of 9 values -> p[4]
__device__ __forceinline__ int median9(int (&p)[9])
{
    cs(p, 1, 2); cs(p, 4, 5); cs(p, 7, 8); cs(p, 0, 1); cs(p, 3, 4); cs(p, 6, 7); cs(p, 1, 2); cs(p, 4, 5); cs(p, 7, 8);
    cs(p, 0, 3); cs(p, 5, 8); cs(p, 4, 7); cs(p, 3, 6); cs(p, 1, 4); cs(p, 2, 5); cs(p, 4, 7); cs(p, 4, 2); cs(p, 6, 4);
    cs(p, 4, 2);
    return p[4];
}

// the median of 25 values -> p[12]
__device__ __forceinline__ int median25(int (&p)[25])
{
    cs(p, 0, 1); cs(p, 2, 3); cs(p, 4, 5); cs(p, 6, 7); cs(p, 8, 9); cs(p, 10, 11); cs(p, 12, 13); cs(p, 14, 15); cs(p, 16, 17);
    cs(p, 18, 19); cs(p, 20, 21); cs(p, 22, 23); cs(p, 0, 2); cs(p, 1, 3); cs(p, 4, 6); cs(p, 5, 7); cs(p, 8, 10); cs(p, 9, 11);
    cs(p, 12, 14); cs(p, 13, 15); cs(p, 16, 18); cs(p, 17, 19); cs(p, 20, 22); cs(p, 21, 23); cs(p, 1, 2); cs(p, 5, 6); cs(p, 9, 10);
    cs(p, 13, 14); cs(p, 17, 18); cs(p, 21, 22); cs(p, 0, 4); cs(p, 1, 5); cs(p, 2, 6); cs(p, 3, 7); cs(p, 8, 12); cs(p, 9, 13);
    cs(p, 10, 14); cs(p, 11, 15); cs(p, 16, 20); cs(p, 17, 21); cs(p, 18, 22); cs(p, 19, 23); cs(p, 2, 4); cs(p, 3, 5); cs(p, 10, 12);
    cs(p, 11, 13); cs(p, 18, 20); cs(p, 19, 21); cs(p, 1, 2); cs(p, 3, 4); cs(p, 5, 6); cs(p, 9, 10); cs(p, 11, 12); cs(p, 13, 14);
    cs(p, 17, 18); cs(p, 19, 20); cs(p, 21, 22); cs(p, 0, 8); cs(p, 1, 9); cs(p, 2, 10); cs(p, 3, 11); cs(p, 4, 12); cs(p, 5, 13);
    cs(p, 6, 14); cs(p, 7, 15); cs(p, 16, 24); cs(p, 4, 8); cs(p, 5, 9); cs(p, 6, 10); cs(p, 7, 11); cs(p, 20, 24); cs(p, 2, 4);
    cs(p, 3, 5); cs(p, 6, 8); cs(p, 7, 9); cs(p, 10, 12); cs(p, 11, 13); cs(p, 18, 20); cs(p, 19, 21); cs(p, 22, 24); cs(p, 1, 2);
    cs(p, 3, 4); cs(p, 5, 6); cs(p, 7, 8); cs(p, 9, 10); cs(p, 11, 12); cs(p, 13, 14); cs(p, 17, 18); cs(p, 19, 20); cs(p, 21, 22);
    cs(p, 23, 24); cs(p, 0, 16); cs(p, 1, 17); cs(p, 2, 18); cs(p, 3, 19); cs(p, 4, 20); cs(p, 5, 21); cs(p, 6, 22); cs(p, 7, 23);
    cs(p, 8, 24); cs(p, 8, 16); cs(p, 9, 17); cs(p, 10, 18); cs(p, 11, 19); cs(p, 12, 20); cs(p, 13, 21); cs(p, 6, 10); cs(p, 7, 11);
    cs(p, 12, 16); cs(p, 13, 17); cs(p, 10, 12); cs(p, 11, 13); cs(p, 11, 12);
    return p[12];
}

template <typename T, int R>
__global__ void __launch_bounds__(kMdTileX * kMdTileY) median_kernel(const MedianArgs<T> a)
{
    constexpr int kTw = kMdTileX + 2 * R, kTh = kMdTileY + 2 * R, K = 2 * R + 1;
    __shared__ T tile[kTh][kTw];
    const int view = blockIdx.z, W = a.W, H = a.H;
    const int x0 = blockIdx.x * kMdTileX - R, y0 = blockIdx.y * kMdTileY - R;
    const T* in = view ? a.in[1] : a.in[0];
    for (int i = threadIdx.y * kMdTileX + threadIdx.x; i < kTw * kTh; i += kMdTileX * kMdTileY) {
        const int ty = i / kTw, tx = i - ty * kTw;
        const int y = min(max(y0 + ty, 0), H - 1), x = min(max(x0 + tx, 0), W - 1);
        tile[ty][tx] = __ldg(in + (size_t)y * W + x);
    }
    __syncthreads();
    const int x = x0 + R + threadIdx.x, y = y0 + R + threadIdx.y;
    if (x >= W || y >= H) return;
    int p[K * K];
#pragma unroll
    for (int j = 0; j < K; ++j)
#pragma unroll
        for (int i = 0; i < K; ++i) p[j * K + i] = tile[threadIdx.y + j][threadIdx.x + i];
    int v;
    if constexpr (R == 1) v = median9(p); else v = median25(p);
    (view ? a.out[1] : a.out[0])[(size_t)y * W + x] = (T)v;
}

}  // namespace psm
