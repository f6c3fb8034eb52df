// psm_reproject.cuh -- OpenCV's reprojectImageTo3D(disp, xyz, Q, handleMissingValues) on the device, bit for bit
// (psm_reproject_device; the definition and its derivation are in DESIGN.md section 24).
//
// For pixel (x, y) with map value d, in fp64 with every product and sum rounded on its own (no fused multiply-add):
//   h[i] = (((+0.0 + Q[i][0] x) + Q[i][1] y) + Q[i][2] d) + Q[i][3],   r = 1 / h[3] (correctly rounded),
//   X = (float)((double)(float)h[0] * r), Y and Z likewise from h[1] and h[2],
// and with handle_missing Z = 10000 wherever d is the minimum of the view's map.  The output is OpenCV's CV_32FC3 layout:
// X, Y, Z interleaved, 12 bytes per pixel, rows row_step bytes apart.
#pragma once
#include "psm_common.cuh"

namespace psm {

constexpr int kRpThreads = 256;                 // one CTA: kRpPix consecutive pixels of one row of one view
constexpr int kRpPerThread = 4;
constexpr int kRpPix = kRpThreads * kRpPerThread;
constexpr int kRpMinBlocks = 528;               // grid cap of the min-reduction (grid-stride beyond it)
constexpr float kRpMissingZ = 10000.0f;         // reprojectImageTo3D's bigZ

__host__ __device__ __forceinline__ double rp_mul(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ __forceinline__ double rp_add(double a, double b)
{
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}

__host__ __device__ __forceinline__ unsigned long long rp_bits(double x)
{
#ifdef __CUDA_ARCH__
    return (unsigned long long)__double_as_longlong(x);
#else
    unsigned long long u;
    __builtin_memcpy(&u, &x, sizeof u);
    return u;
#endif
}
__host__ __device__ __forceinline__ double rp_double(unsigned long long u)
{
#ifdef __CUDA_ARCH__
    return __longlong_as_double((long long)u);
#else
    double x;
    __builtin_memcpy(&x, &u, sizeof x);
    return x;
#endif
}

// 1 / h, correctly rounded to nearest-even for every double h (+-0 -> +-inf, +-inf -> +-0, NaN -> NaN), with no fused
// multiply-add: nvcc's own fp64 division and reciprocal refine with DFMA.  |h| = M 2^E with M in [2^52, 2^53), so
// 1 / |h| = (2^105 / M) 2^(-105 - E) and 2^105 / M lies in (2^52, 2^53].  The 53-bit quotient (fewer bits where the
// result is subnormal: |h| >= 2^1022) comes from a float seed and two Newton steps in fp64, within a few units; the
// exact remainder, taken modulo 2^64, corrects it to floor(2^k / M), and the remainder rounds it.  The carry of a
// quotient that rounds up to 2^53 moves into the exponent field, which also yields +-inf above the largest double.
// Host and device compute the same bits; the host build exists for the exhaustive checks of the quotient correction.
__host__ __device__ __forceinline__ double rp_rcp(double h)
{
    const unsigned long long b = rp_bits(h);
    const unsigned long long sign = b & 0x8000000000000000ull;
    const int e = (int)((b >> 52) & 0x7ff);
    unsigned long long m = b & 0x000fffffffffffffull;
    if (e == 0x7ff) return m ? h : rp_double(sign);
    if (e == 0 && m == 0) return rp_double(sign | 0x7ff0000000000000ull);
    int E;
    if (e) {
        m |= 1ull << 52;
        E = e - 1075;
    } else {
#ifdef __CUDA_ARCH__
        const int s = __clzll((long long)m) - 11;
#else
        const int s = __builtin_clzll(m) - 11;
#endif
        m <<= s;
        E = -1074 - s;
    }
    const int be = 970 - E;                       // the result's biased exponent for a quotient in [2^52, 2^53)
    if (be >= 2047) return rp_double(sign | 0x7ff0000000000000ull);
    const int sh = be >= 1 ? 0 : 1 - be;          // 0, or 1 / 2 bits fewer for a subnormal result
    const double md = (double)m;                  // exact
#ifdef __CUDA_ARCH__
    float seed;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(seed) : "f"((float)md));
#else
    const float seed = 1.0f / (float)md;
#endif
    double r = (double)seed;
    r = rp_mul(r, rp_add(2.0, -rp_mul(md, r)));
    r = rp_mul(r, rp_add(2.0, -rp_mul(md, r)));
    unsigned long long q = (unsigned long long)rp_mul(r, sh == 0 ? 0x1p105 : (sh == 1 ? 0x1p104 : 0x1p103));
    // 2^k - q M for k >= 64, exact modulo 2^64; the true value is a few M at most, far inside int64
    long long rem = (long long)(0ull - q * m);
    while (rem < 0) { --q; rem += (long long)m; }
    while (rem >= (long long)m) { ++q; rem -= (long long)m; }
    if (2 * rem > (long long)m || (2 * rem == (long long)m && (q & 1))) ++q;
    const unsigned long long mag = sh ? q : ((unsigned long long)(be - 1) << 52) + q;
    return rp_double(sign | mag);
}

// the arguments of one reprojection launch: slot z (blockIdx.z) is one requested view
template <typename T>
struct ReprojArgs {
    const T* map[2];
    float* out[2];
    double q[2][16];
    const unsigned* minv;   // handle_missing: the minimum of each slot's map (reproject_min_kernel), else null
    size_t row_step;        // bytes between output rows (a multiple of 4)
    int W, H;
};

// the minimum of each slot's map into minv[slot], which the caller set to 0xFFFFFFFF: one atomicMin per CTA (atomics on
// one address serialise, so the CTA reduces first)
template <typename T>
__global__ void __launch_bounds__(kRpThreads) reproject_min_kernel(const ReprojArgs<T> a, unsigned* minv)
{
    __shared__ unsigned warp_min[kRpThreads / 32];
    const T* m = blockIdx.z ? a.map[1] : a.map[0];
    const size_t n = (size_t)a.W * a.H, stride = (size_t)gridDim.x * kRpThreads;
    unsigned lo = 0xffffffffu;
#pragma unroll 4
    for (size_t i = (size_t)blockIdx.x * kRpThreads + threadIdx.x; i < n; i += stride) lo = min(lo, (unsigned)__ldg(m + i));
    lo = __reduce_min_sync(0xffffffffu, lo);
    if ((threadIdx.x & 31) == 0) warp_min[threadIdx.x / 32] = lo;
    __syncthreads();
    if (threadIdx.x < 32) {
        lo = __reduce_min_sync(0xffffffffu, threadIdx.x < kRpThreads / 32 ? warp_min[threadIdx.x] : 0xffffffffu);
        if (threadIdx.x == 0) atomicMin(minv + blockIdx.z, lo);
    }
}

// kRpPix pixels of one row of slot blockIdx.z (blockIdx.x = row * segs + segment, segs = ceil(W / kRpPix)): each thread computes four pixels
// kRpThreads apart (coalesced map reads) into the CTA's staging row, which then leaves as 128-bit streaming stores where
// the output row is 16-byte aligned and as coalesced 32-bit stores where it is not
template <typename T>
__global__ void __launch_bounds__(kRpThreads) reproject_kernel(const ReprojArgs<T> a, unsigned segs)
{
    __shared__ float4 stage[kRpPix * 3 / 4];
    float* s = reinterpret_cast<float*>(stage);
    const int z = blockIdx.z, y = (int)(blockIdx.x / segs), x0 = (int)(blockIdx.x % segs) * kRpPix;
    const int n = min(kRpPix, a.W - x0);
    double q[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) q[i] = z ? a.q[1][i] : a.q[0][i];
    const double yd = (double)y;
    double qy[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) qy[i] = rp_mul(q[4 * i + 1], yd);
    const T* row = (z ? a.map[1] : a.map[0]) + (size_t)y * a.W + x0;
    const unsigned miss = a.minv ? a.minv[z] : 0xffffffffu;   // never a map value
#pragma unroll
    for (int k = 0; k < kRpPerThread; ++k) {
        const int i = threadIdx.x + k * kRpThreads;
        if (i < n) {
            const unsigned d = __ldg(row + i);
            const double xd = (double)(x0 + i), dd = (double)d;
            double h[4];
#pragma unroll
            for (int j = 0; j < 4; ++j)
                h[j] = rp_add(rp_add(rp_add(rp_add(0.0, rp_mul(q[4 * j], xd)), qy[j]), rp_mul(q[4 * j + 2], dd)), q[4 * j + 3]);
            const double r = rp_rcp(h[3]);
            float* o = s + 3 * i;
            o[0] = __double2float_rn(rp_mul((double)__double2float_rn(h[0]), r));
            o[1] = __double2float_rn(rp_mul((double)__double2float_rn(h[1]), r));
            o[2] = d == miss ? kRpMissingZ : __double2float_rn(rp_mul((double)__double2float_rn(h[2]), r));
        }
    }
    __syncthreads();
    float* orow = reinterpret_cast<float*>(reinterpret_cast<char*>(z ? a.out[1] : a.out[0]) + (size_t)y * a.row_step) +
                  (size_t)x0 * 3;
    const int nf = 3 * n;
    int tail = 0;
    if ((reinterpret_cast<uintptr_t>(orow) & 15) == 0) {
        float4* o4 = reinterpret_cast<float4*>(orow);
        for (int i = threadIdx.x; i < nf / 4; i += kRpThreads) __stcs(o4 + i, stage[i]);
        tail = nf / 4 * 4;
    }
    for (int i = tail + threadIdx.x; i < nf; i += kRpThreads) __stcs(orow + i, s[i]);
}

}  // namespace psm
