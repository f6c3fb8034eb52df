// psm_common.cuh -- shared device helpers for the H100 (sm_90a) STEREO_GIF path.
//
// Numerics rule for this library: every float operation that the reference performs as a
// separate IEEE operation (reference builds with plain -O3 on baseline x86-64, no FMA
// contraction: /root/reference/CMakeLists.txt:17) is issued through the explicit
// round-to-nearest intrinsics below, which nvcc never contracts into FMAs.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace psm {

constexpr int kBoxK = 8;        // GIF_R_WIN, reference include/ComFunc.h:49 (8x8 box, anchor 4)
constexpr int kBoxAnchor = 4;   // cv::boxFilter default anchor = ksize/2
constexpr float kGifEps = 0.0001f;  // GIF_EPS, include/ComFunc.h:50

// The two disparity-map formats, by element type: uint8_t maps (psm_create, D <= 256) and uint16_t maps
// (psm_create_u16, D <= 4096).  The post-filter packs a map value and the three 6-bit colours of its pixel into one u32,
//   d << kDispShift | R6 << 2 * kColourBits | G6 << kColourBits | B6,
// and its bisection gives the taps outside the window the disparity kSentinel, above every map value.
template <typename T> struct MapFormat;
template <> struct MapFormat<uint8_t> {
    static constexpr int kMaxDisp = 256;
    static constexpr int kDispShift = 24, kColourBits = 8;
    static constexpr uint32_t kSentinel = 256u;
};
template <> struct MapFormat<uint16_t> {
    static constexpr int kMaxDisp = 4096;   // a 12-bit disparity and 18 colour bits fill the packed u32
    static constexpr int kDispShift = 18, kColourBits = 6;
    static constexpr uint32_t kSentinel = 0xffffffffu;
};

__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }

// cv::BORDER_REFLECT_101 (gfedcb|abcdefgh|gfedcba); any overshoot, n >= 1.
__host__ __device__ __forceinline__ int reflect101(int i, int n)
{
    if (n == 1) return 0;
    while (i < 0 || i >= n) {
        if (i < 0) i = -i;
        else i = 2 * (n - 1) - i;
    }
    return i;
}

// Float4 component access with a compile-time index (keeps everything in registers).
template <int J> __device__ __forceinline__ float comp(const float4& v)
{
    if (J == 0) return v.x;
    if (J == 1) return v.y;
    if (J == 2) return v.z;
    return v.w;
}
__device__ __forceinline__ float comp(const float4& v, int j)
{
    return j == 0 ? v.x : (j == 1 ? v.y : (j == 2 ? v.z : v.w));
}

// Load 4 consecutive floats of one image row at columns col..col+3 (col % 4 == 0, row 16B-aligned).
// Groups fully inside [0, W) use one 128-bit read-only load; groups touching a border gather
// with BORDER_REFLECT_101 so that box sums see exactly what cv::boxFilter sees.
__device__ __forceinline__ float4 load_row4(const float* __restrict__ row, int col, int W)
{
    if (col >= 0 && col + 3 < W) return __ldg(reinterpret_cast<const float4*>(row + col));
    float4 v;
    v.x = __ldg(row + reflect101(col, W));
    v.y = __ldg(row + reflect101(col + 1, W));
    v.z = __ldg(row + reflect101(col + 2, W));
    v.w = __ldg(row + reflect101(col + 3, W));
    return v;
}

// Order-preserving float -> uint32 (for packed (cost, d) keys). -0 is canonicalised to +0 first so
// that key order agrees with the reference's `<` on floats (DispSel.cpp:96-102).
__device__ __forceinline__ uint32_t float_order_key(float c)
{
    c = c + 0.0f;  // -0.0f + 0.0f == +0.0f
    uint32_t u = __float_as_uint(c);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// (shared by the guide precompute and the streaming guided filter; the derivation is at the top of psm_cvf_stream.cuh)
// ---- widening into the 2^-896-scaled fp64 domain --------------------------------------------
constexpr double kScaleDown = 0x1p-896;   // what the integer widening multiplies by
constexpr double kMeanScaled = 0x1p890;   // 2^896 / 64
constexpr double kMeanPlain = 0x1p-6;     // 1 / 64

// non-negative finite float (zero / denormal included): one IMAD.WIDE.U32
__device__ __forceinline__ double widen_nn(float f)
{
    unsigned long long r;
    asm("mul.wide.u32 %0, %1, 0x20000000;" : "=l"(r) : "r"(__float_as_uint(f)));
    return __longlong_as_double((long long)r);
}
// any finite float: shift the sign out, widen, put the sign back
__device__ __forceinline__ double widen_sg(float f)
{
    const unsigned u = __float_as_uint(f);
    unsigned long long r;
    asm("mul.wide.u32 %0, %1, 0x10000000;" : "=l"(r) : "r"(u + u));
    const unsigned hi = (unsigned)(r >> 32) | (u & 0x80000000u);
    return __hiloint2double((int)hi, (int)(unsigned)r);
}
// anything (slow path): conversion pipe + exact rescale
__device__ __forceinline__ double widen_any(float f) { return __dmul_rn((double)f, kScaleDown); }

}  // namespace psm
