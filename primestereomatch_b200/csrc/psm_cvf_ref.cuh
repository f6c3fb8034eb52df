// psm_cvf_ref.cuh -- the guided filter and the guide precompute in cv::boxFilter's own order of fp64 operations.
//
// cv::boxFilter (CV_32F, K x K, anchor K/2, BORDER_REFLECT_101) keeps RUNNING fp64 sums: RowSum slides one sum along the
// whole row (s += p[i+K] - p[i]; rows of up to 5 taps are summed directly), ColumnSum slides one sum per column down the
// whole column (s0 = SUM + newest, out = (float)(s0 / K^2), SUM = s0 - oldest).  A rounding error, an inf or a NaN that
// enters one of those sums stays in it after its window has passed, so a mean depends on everything left of and above
// its pixel.  The tuned kernels add the same values in other orders (guide_kernel and cvf_stream_kernel restart their
// column sums at every row segment and take each row sum from one window; cvf_window_kernel likewise).  Both orders give
// the same float while every fp64 sum is exact; where one is not, only this order reproduces the reference.
//
// The kernels below repeat the order of the CPU oracle's orc_box operation for operation: one thread per row slides
// along it, then one thread per column slides down it.  They are cooperative launches (grid-wide barriers between the
// passes) over scratch of one slice ([4][H][W] fp64 row sums, [4][H][W] float planes):
//   guide_ref_kernel : CVF::preprocess (CVF.cpp:44-70) + the solve terms of guide_solve_eps, for every view whose ingest
//                      flag says the guide sums may be inexact (kGuideOutside | kGuideInexact);
//   cvf_ref_kernel   : GuidedFilter_cv (CVF.cpp:72-165) of every slice psm_write_cost_slice flagged (a cost that is
//                      negative, -0, inf, NaN or >= 2^63), of every slice of a view whose image is outside the integer
//                      domain or whose solve terms are not finite, of every slice in PSM_CVF_NAIVE, or a, b of one slice
//                      (psm_read_ab_slice).
// Every block reads the same flags, so the choice of slices is uniform over the grid; with nothing flagged every block
// leaves after one parallel read of the flags.  The host launches them only where a flag can be set (float images, a
// non-default window, a flagged slice), so u8 frames at the defaults never pay for them.
// Cost: one thread per row and then per column, and one slice at a time with grid-wide barriers in between -- the rows
// are read one per lane (uncoalesced) -- so a view that takes this pass costs far more than the tuned kernel (not measured
// at 1920 x 1080 x 128; it is meant for inputs outside the image contract, not for real frames).
#pragma once
#include <cooperative_groups.h>

#include "psm_cvf_window.cuh"

namespace psm {

namespace cg = cooperative_groups;

constexpr int kRefThreads = 128;

// cvf_ref_kernel modes
constexpr int kRefFlagged = 0;   // flagged slices and views (after the tuned kernels)
constexpr int kRefAll = 1;       // every slice (PSM_CVF_NAIVE, tiny images)
constexpr int kRefAbOnly = 2;    // a, b of slice one_d of view one_view, left in the float scratch; no q

struct RefParams {
    const float* vol_in[2];
    float* vol_out[2];
    float* guide[2];
    int* guide_flags;     // [2]
    const int* slice_flags;   // [2][Dloc], nonzero: the slice takes this pass
    double* rs;           // scratch [4][H][W]
    float* pl;            // scratch [4][H][W]
    int W, H, Wp, Dloc, K, a;
    double scale;         // 1 / K^2
    float eps;
    int mode, one_view, one_d;
};

// Row pass: rs[q][y][x] = the K-wide row sum of quantity q at (x, y), RowSum<float, double>'s order.  One thread per row.
template <class Tap>
__device__ __forceinline__ void ref_rows(const Tap& tap, double* __restrict__ rs, int W, int H, int K, int a)
{
    const size_t n = (size_t)W * H;
    const int stride = gridDim.x * blockDim.x;
    for (int y = blockIdx.x * blockDim.x + threadIdx.x; y < H; y += stride) {
        double* D = rs + (size_t)y * W;
        double acc[4];
        if (K <= 5) {   // direct: p[x-a] + p[x-a+1] + ... left to right, from the first tap
            for (int x = 0; x < W; ++x) {
#pragma unroll
                for (int q = 0; q < 4; ++q) acc[q] = (double)tap(q, reflect101(x - a, W), y);
                for (int i = 1; i < K; ++i) {
                    const int xx = reflect101(x - a + i, W);
#pragma unroll
                    for (int q = 0; q < 4; ++q) acc[q] = __dadd_rn(acc[q], (double)tap(q, xx, y));
                }
#pragma unroll
                for (int q = 0; q < 4; ++q) D[q * n + x] = acc[q];
            }
        } else {        // sliding: s = 0 + p[-a] + ... + p[K-1-a], then s += p[x+K-a] - p[x-a]
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[q] = 0.0;
            for (int i = 0; i < K; ++i) {
                const int xx = reflect101(i - a, W);
#pragma unroll
                for (int q = 0; q < 4; ++q) acc[q] = __dadd_rn(acc[q], (double)tap(q, xx, y));
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) D[q * n] = acc[q];
            for (int x = 0; x < W - 1; ++x) {
                const int xn = reflect101(x + K - a, W), xo = reflect101(x - a, W);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    acc[q] = __dadd_rn(acc[q], __dsub_rn((double)tap(q, xn, y), (double)tap(q, xo, y)));
                    D[q * n + x + 1] = acc[q];
                }
            }
        }
    }
}

// Column pass: emit(x, y, m) with m[q] = the K x K mean of quantity q at (x, y), ColumnSum<double, float>'s order.  One
// thread per column.  K = 1 is a copy in OpenCV.
template <class Emit>
__device__ __forceinline__ void ref_cols(const double* __restrict__ rs, int W, int H, int K, int a, double scale, const Emit& emit)
{
    const size_t n = (size_t)W * H;
    const int stride = gridDim.x * blockDim.x;
    for (int x = blockIdx.x * blockDim.x + threadIdx.x; x < W; x += stride) {
        double sum[4] = {0.0, 0.0, 0.0, 0.0};
        for (int r = 0; r < K - 1; ++r) {
            const double* S = rs + (size_t)reflect101(r - a, H) * W + x;
#pragma unroll
            for (int q = 0; q < 4; ++q) sum[q] = __dadd_rn(sum[q], S[q * n]);
        }
        for (int y = 0; y < H; ++y) {
            const double* Sp = rs + (size_t)reflect101(y + K - 1 - a, H) * W + x;
            const double* Sm = rs + (size_t)reflect101(y - a, H) * W + x;
            float m[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const double s0 = __dadd_rn(sum[q], Sp[q * n]);
                m[q] = K == 1 ? (float)Sp[q * n] : (float)__dmul_rn(s0, scale);
                sum[q] = __dsub_rn(s0, Sm[q * n]);
            }
            emit(x, y, m);
        }
    }
}

// CVF::preprocess of the flagged views: box of I0, I1, I2 and of the six products (CVF.cpp:49-69) in three rounds of four
// quantities, the means into the mean planes and the product means into the var planes, then guide_solve_eps per pixel.
__global__ void __launch_bounds__(kRefThreads) guide_ref_kernel(const RefParams P)
{
    const bool todo0 = (P.guide_flags[0] & (kGuideOutside | kGuideInexact)) != 0;
    const bool todo1 = (P.guide_flags[1] & (kGuideOutside | kGuideInexact)) != 0;
    if (!todo0 && !todo1) return;   // the same for every block
    cg::grid_group grid = cg::this_grid();
    const int W = P.W, H = P.H, Wp = P.Wp;
    const size_t plane = (size_t)H * Wp;
    constexpr int kA[9] = {0, 1, 2, 0, 0, 0, 1, 1, 2}, kB[9] = {-1, -1, -1, 0, 1, 2, 1, 2, 2};
    for (int view = 0; view < 2; ++view) {
        if (!(view ? todo1 : todo0)) continue;
        float* G = P.guide[view];
        for (int k0 = 0; k0 < 9; k0 += 4) {
            auto tap = [&](int q, int x, int y) -> float {
                const int k = k0 + q;
                if (k >= 9) return 0.f;
                const size_t o = (size_t)y * Wp + x;
                const float u = G[(size_t)kA[k] * plane + o];
                return kB[k] < 0 ? u : fmul(u, G[(size_t)kB[k] * plane + o]);   // CVF.cpp:62
            };
            ref_rows(tap, P.rs, W, H, P.K, P.a);
            grid.sync();
            ref_cols(P.rs, W, H, P.K, P.a, P.scale, [&](int x, int y, const float (&m)[4]) {
                const size_t o = (size_t)y * Wp + x;
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int k = k0 + q;
                    if (k < 3) G[(size_t)(kGuideMean + k) * plane + o] = m[q];
                    else if (k < 9) G[(size_t)(kGuideVar + k - 3) * plane + o] = m[q];
                }
            });
            grid.sync();
        }
        const int stride = gridDim.x * blockDim.x;
        unsigned worst = 0;
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < W * H; i += stride) {
            const size_t o = (size_t)(i / W) * Wp + i % W;
            float m[9];
#pragma unroll
            for (int k = 0; k < 3; ++k) m[k] = G[(size_t)(kGuideMean + k) * plane + o];
#pragma unroll
            for (int k = 0; k < 6; ++k) m[3 + k] = G[(size_t)(kGuideVar + k) * plane + o];
            float v[6], M[6], idet;
            guide_solve_eps(m, P.eps, v, M, idet);
#pragma unroll
            for (int k = 0; k < 6; ++k) {
                G[(size_t)(kGuideAdj + k) * plane + o] = M[k];
                G[(size_t)(kGuideVar + k) * plane + o] = v[k];
                worst = max(worst, __float_as_uint(M[k]) & 0x7fffffffu);
            }
            G[(size_t)kGuideIdet * plane + o] = idet;
#pragma unroll
            for (int k = 0; k < 3; ++k) worst = max(worst, __float_as_uint(m[k]) & 0x7fffffffu);
            worst = max(worst, __float_as_uint(idet) & 0x7fffffffu);
        }
        if (worst >= 0x7f800000u) atomicOr(P.guide_flags + view, kGuideNonFinite);
        grid.sync();   // the scratch is free for the next view
    }
}

// GuidedFilter_cv of one slice: box of p and I_c p -> a, b (gif_coeffs) -> box of a_c, b -> q (CVF.cpp:157-163).
__device__ __forceinline__ void ref_filter_slice(const RefParams& P, cg::grid_group& grid, int view, int dl, bool ab_only)
{
    const int W = P.W, H = P.H, Wp = P.Wp;
    const size_t plane = (size_t)H * Wp, n = (size_t)W * H;
    const float* __restrict__ p = P.vol_in[view] + (size_t)dl * plane;
    const float* __restrict__ g = P.guide[view];
    float* __restrict__ pl = P.pl;
    ref_rows([&](int q, int x, int y) -> float {
        const size_t o = (size_t)y * Wp + x;
        return q == 0 ? p[o] : fmul(g[(size_t)(q - 1) * plane + o], p[o]);   // CVF.cpp:87
    }, P.rs, W, H, P.K, P.a);
    grid.sync();
    ref_cols(P.rs, W, H, P.K, P.a, P.scale, [&](int x, int y, const float (&m)[4]) {
        float a0, a1, a2, b;
        gif_coeffs(m[0], m[1], m[2], m[3], load_guide_pix(g, plane, (size_t)y * Wp + x), a0, a1, a2, b);
        const size_t o = (size_t)y * W + x;
        pl[o] = a0; pl[n + o] = a1; pl[2 * n + o] = a2; pl[3 * n + o] = b;
    });
    grid.sync();
    if (ab_only) return;
    ref_rows([&](int q, int x, int y) -> float { return pl[(size_t)q * n + (size_t)y * W + x]; }, P.rs, W, H, P.K, P.a);
    grid.sync();
    float* __restrict__ out = P.vol_out[view] + (size_t)dl * plane;
    ref_cols(P.rs, W, H, P.K, P.a, P.scale, [&](int x, int y, const float (&m)[4]) {
        const size_t o = (size_t)y * Wp + x;
        float qv = fadd(m[3], fmul(m[0], g[o]));
        qv = fadd(qv, fmul(m[1], g[plane + o]));
        qv = fadd(qv, fmul(m[2], g[2 * plane + o]));
        out[o] = qv;
    });
    grid.sync();   // the scratch is free for the next slice
}

__global__ void __launch_bounds__(kRefThreads) cvf_ref_kernel(const RefParams P)
{
    const int views_all = ((P.guide_flags[0] & (kGuideOutside | kGuideNonFinite)) ? 1 : 0) |
                          ((P.guide_flags[1] & (kGuideOutside | kGuideNonFinite)) ? 2 : 0);
    if (P.mode == kRefFlagged) {
        int any = views_all;
        for (int i = threadIdx.x; i < 2 * P.Dloc; i += blockDim.x) any |= P.slice_flags[i];
        if (!__syncthreads_or(any)) return;   // the same for every block
    }
    cg::grid_group grid = cg::this_grid();
    if (P.mode == kRefAbOnly) {
        ref_filter_slice(P, grid, P.one_view, P.one_d, true);
        return;
    }
    for (int view = 0; view < 2; ++view)
        for (int dl = 0; dl < P.Dloc; ++dl)
            if (P.mode == kRefAll || ((views_all >> view) & 1) || P.slice_flags[view * P.Dloc + dl])
                ref_filter_slice(P, grid, view, dl, false);
}

}  // namespace psm
