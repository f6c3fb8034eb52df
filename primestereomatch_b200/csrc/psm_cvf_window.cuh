// psm_cvf_window.cuh -- the guided filter at a run-time window size and epsilon (psm_set_guided_filter).
//
// The reference fixes its full-resolution guided filter to a GIF_R_WIN x GIF_R_WIN box (anchor GIF_R_WIN/2,
// BORDER_REFLECT_101) and GIF_EPS on the covariance diagonal (include/ComFunc.h:49-50, CVF.cpp:46-128).  The tuned
// kernels (psm_cvf_stream.cuh, guide_kernel) are built around the default 8 x 8 box.  The kernels here take the window
// K (1..kWinMax) and eps at run time and compute the same quantities:
//   guide_window_kernel : the 19-plane guide layout of guide_kernel (mean_I, adjugate of Sigma + eps I, 1/det, var_I)
//   cvf_window_kernel   : the streaming guided filter, p read once and q written once per voxel, a and b never leave the SM
//
// Numerics are those of psm_cvf_stream.cuh: every box sum in fp64 (exact, hence order-independent, unless a window spans
// more than 2^(29 - ceil(log2 K^2)) in magnitude), scaled by 1/K^2 and rounded once; every f32 operation of a, b and q a
// separate round-to-nearest operation in the reference's order (gif_coeffs).  The widening is the plain conversion, so
// negative, -0 and non-finite costs need no separate path.
//
// Streaming kernel, one CTA = one slice x one strip of `tw` output columns x one row segment (tw = kWinThreads - 2K + 2, so
// that every per-column role below fits one thread):
//   stage 1  thread = one (virtual) input column of the strip's a,b columns' windows: fp64 running column sums over the K
//            window rows of p, I0 p, I1 p, I2 p (+ newest row, - oldest row; both read from the volume / guide planes);
//   rows     window sums along the row with the van Herk / Gil-Werman split: per K-column block one prefix and one suffix
//            scan, then sum(i .. i+K-1) = suffix(i) + prefix(i+K-1) -- three fp64 adds per value whatever K is, and every
//            partial sum is a sub-sum of one window, so the exactness bound above is unchanged;
//   a, b     gif_coeffs at the REAL columns the strip's second stage needs (reflected columns are real columns: cv::boxFilter
//            reflects its input, which for the second stage is a, b), kept in a shared-memory ring of the last K+1 rows;
//   stage 2  thread = one virtual column of the output windows: fp64 running column sums of a0, a1, a2, b read from the ring
//            (reflect101 of the virtual column and row), the same row sums, then q = box(b) + sum_c box(a_c) I_c.
// Every column and row index goes through reflect101, so any W, H >= 1 work, and nothing reads the mirrored halo columns.
// A segment starts with a direct K-row sum (warm-up: ~2K rows), after which every row costs the same.
#pragma once
#include "psm_kernels.cuh"

namespace psm {

constexpr int kWinMax = 32;        // largest window psm_set_guided_filter accepts
constexpr int kWinThreads = 256;   // threads per CTA of cvf_window_kernel
constexpr int kWinGuideSegRows = 64;
constexpr int kWinBuf = 2 * kWinThreads;   // doubles per quantity in the row buffers (block-padded layout, see win_pos)

// guide_solve with a run-time eps (CVF.cpp:60-69, 108-120; same operations in the same order)
__device__ __forceinline__ void guide_solve_eps(const float m[9], float eps, float v[6], float M[6], float& idet)
{
    v[0] = fsub(m[3], fmul(m[0], m[0]));
    v[1] = fsub(m[4], fmul(m[0], m[1]));
    v[2] = fsub(m[5], fmul(m[0], m[2]));
    v[3] = fsub(m[6], fmul(m[1], m[1]));
    v[4] = fsub(m[7], fmul(m[1], m[2]));
    v[5] = fsub(m[8], fmul(m[2], m[2]));
    const float a11 = fadd(v[0], eps), a12 = v[1], a13 = v[2];
    const float a21 = v[1], a22 = fadd(v[3], eps), a23 = v[4];
    const float a31 = v[2], a32 = v[4], a33 = fadd(v[5], eps);
    M[0] = fsub(fmul(a33, a22), fmul(a32, a23));
    M[1] = fsub(fmul(a31, a23), fmul(a33, a21));
    M[2] = fsub(fmul(a32, a21), fmul(a31, a22));
    M[3] = fsub(fmul(a33, a11), fmul(a31, a13));
    M[4] = fsub(fmul(a31, a12), fmul(a32, a11));
    M[5] = fsub(fmul(a22, a11), fmul(a21, a12));
    const float t1 = fsub(fmul(a33, a12), fmul(a32, a13));
    const float t2 = fsub(fmul(a23, a12), fmul(a22, a13));
    const float det = fadd(fsub(fmul(a11, M[0]), fmul(a21, t1)), fmul(a31, t2));
    idet = __fdiv_rn(1.0f, det);
}

struct WinGuideParams {
    float* guide[2];
    int* guide_flags;   // [2]: kGuideNonFinite raised when a mean / adjugate / 1/det value is not finite
    int W, H, Wp, K, a, seg_rows;
    double scale;   // 1 / K^2
    float eps;
};

// thread = one column x one row segment of one view (blockIdx.z); fp64 K-wide row sums of the nine planes, fp64 running sums
// down the rows, then the solve.  Writes planes kGuideMean .. kGuidePlanes-1 at columns [0, W).
__global__ void __launch_bounds__(128) guide_window_kernel(const WinGuideParams P)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int view = blockIdx.z;
    if (x >= P.W) return;
    const int W = P.W, H = P.H, K = P.K, a = P.a;
    const int y0 = blockIdx.y * P.seg_rows, y1 = min(H, y0 + P.seg_rows);
    const size_t plane = (size_t)H * P.Wp;
    float* __restrict__ G = P.guide[view];
    double V[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) V[k] = 0.0;
    auto row = [&](int r, double sgn) {   // V += sgn * (K-wide row sums of row r)
        const size_t ro = (size_t)reflect101(r, H) * P.Wp;
        double h[9];
#pragma unroll
        for (int k = 0; k < 9; ++k) h[k] = 0.0;
        for (int dx = -a; dx < K - a; ++dx) {
            const size_t o = ro + reflect101(x + dx, W);
            const float i0 = __ldg(G + o), i1 = __ldg(G + plane + o), i2 = __ldg(G + 2 * plane + o);
            const float t[9] = {i0, i1, i2, fmul(i0, i0), fmul(i0, i1), fmul(i0, i2), fmul(i1, i1), fmul(i1, i2), fmul(i2, i2)};
#pragma unroll
            for (int k = 0; k < 9; ++k) h[k] = __dadd_rn(h[k], (double)t[k]);
        }
#pragma unroll
        for (int k = 0; k < 9; ++k) V[k] = sgn > 0 ? __dadd_rn(V[k], h[k]) : __dsub_rn(V[k], h[k]);
    };
    for (int dy = -a; dy < K - a; ++dy) row(y0 + dy, 1.0);
    for (int y = y0; y < y1; ++y) {
        if (y > y0) { row(y + K - a - 1, 1.0); row(y - a - 1, -1.0); }
        float m[9];
#pragma unroll
        for (int k = 0; k < 9; ++k) m[k] = (float)__dmul_rn(V[k], P.scale);
        float v[6], M[6], idet;
        guide_solve_eps(m, P.eps, v, M, idet);
        const size_t o = (size_t)y * P.Wp + x;
#pragma unroll
        for (int k = 0; k < 3; ++k) G[(size_t)(kGuideMean + k) * plane + o] = m[k];
#pragma unroll
        for (int k = 0; k < 6; ++k) {
            G[(size_t)(kGuideAdj + k) * plane + o] = M[k];
            G[(size_t)(kGuideVar + k) * plane + o] = v[k];
        }
        G[(size_t)kGuideIdet * plane + o] = idet;
        unsigned worst = __float_as_uint(idet) & 0x7fffffffu;
#pragma unroll
        for (int k = 0; k < 6; ++k) worst = max(worst, __float_as_uint(M[k]) & 0x7fffffffu);
#pragma unroll
        for (int k = 0; k < 3; ++k) worst = max(worst, __float_as_uint(m[k]) & 0x7fffffffu);
        if (worst >= 0x7f800000u) atomicOr(P.guide_flags + view, kGuideNonFinite);
    }
}

__device__ __forceinline__ GuidePix load_guide_pix(const float* __restrict__ g, size_t plane, size_t o)
{
    GuidePix q;
    q.mI0 = __ldg(g + (kGuideMean + 0) * plane + o); q.mI1 = __ldg(g + (kGuideMean + 1) * plane + o);
    q.mI2 = __ldg(g + (kGuideMean + 2) * plane + o);
    q.M00 = __ldg(g + (kGuideAdj + 0) * plane + o); q.M01 = __ldg(g + (kGuideAdj + 1) * plane + o);
    q.M02 = __ldg(g + (kGuideAdj + 2) * plane + o); q.M11 = __ldg(g + (kGuideAdj + 3) * plane + o);
    q.M12 = __ldg(g + (kGuideAdj + 4) * plane + o); q.M22 = __ldg(g + (kGuideAdj + 5) * plane + o);
    q.idet = __ldg(g + kGuideIdet * plane + o);
    return q;
}

struct WinParams {
    const float* vol_in[2];
    float* vol_out[2];
    const float* guide[2];
    int W, H, Wp, Dloc, K, a;
    int tw, nstrips, nseg, seg_rows, ring_stride;
    double scale;   // 1 / K^2
};

// shared memory of cvf_window_kernel: three fp64 row buffers [4][kWinBuf] (column sums, block prefixes, block suffixes)
// and the a,b ring [K+1][4][ring_stride] floats
__host__ __device__ inline size_t win_smem_bytes(int K, int ring_stride)
{
    return (size_t)3 * 4 * kWinBuf * sizeof(double) + (size_t)(K + 1) * 4 * ring_stride * sizeof(float);
}

// Row-buffer position of value i: K-blocks are laid out S = K | 1 doubles apart, an odd stride, so that the lanes of a warp
// that scan different blocks hit different banks (with stride K, K = 8 or 16 would be a 16-way conflict).
__device__ __forceinline__ int win_pos(int i, int K, int S) { return i + (i / K) * (S - K); }

// van Herk / Gil-Werman block scans of the m values cs[q][0..m) of the four quantities: F = prefix inside each K-block,
// Gs = suffix inside each K-block.  Called by the whole CTA between two barriers.
__device__ __forceinline__ void win_block_scans(const double* cs, double* F, double* Gs, int m, int K)
{
    const int nb = (m + K - 1) / K, S = K | 1;
    for (int t = threadIdx.x; t < 8 * nb; t += blockDim.x) {
        const int q = t / (2 * nb), rem = t - q * 2 * nb, blk = rem >> 1;
        const int n = min(m - blk * K, K), o = q * kWinBuf + blk * S;   // values blk*K .. blk*K+n-1 at o .. o+n-1
        const double* src = cs + o;
        if ((rem & 1) == 0) {
            double* dst = F + o;
            double s = src[0];
            dst[0] = s;
            for (int i = 1; i < n; ++i) { s = __dadd_rn(s, src[i]); dst[i] = s; }
        } else {
            double* dst = Gs + o;
            double s = src[n - 1];
            dst[n - 1] = s;
            for (int i = n - 2; i >= 0; --i) { s = __dadd_rn(src[i], s); dst[i] = s; }
        }
    }
}

// sum of the K values starting at i (i + K - 1 < m); F, Gs point at one quantity's buffer
__device__ __forceinline__ double win_sum(const double* F, const double* Gs, int i, int K)
{
    const int S = K | 1;
    return (i % K == 0) ? F[win_pos(i + K - 1, K, S)] : __dadd_rn(Gs[win_pos(i, K, S)], F[win_pos(i + K - 1, K, S)]);
}

__global__ void __launch_bounds__(kWinThreads) cvf_window_kernel(const WinParams P)
{
    extern __shared__ double wsm[];
    double* cs = wsm;                    // [4][kWinBuf]
    double* F = cs + 4 * kWinBuf;        // [4][kWinBuf]
    double* Gs = F + 4 * kWinBuf;        // [4][kWinBuf]
    float* ring = reinterpret_cast<float*>(Gs + 4 * kWinBuf);   // [K+1][4][ring_stride]

    int task = blockIdx.x;
    const int strip = task % P.nstrips; task /= P.nstrips;
    const int seg = task % P.nseg; task /= P.nseg;
    const int dl = task % P.Dloc;
    const int view = task / P.Dloc;
    const int W = P.W, H = P.H, Wp = P.Wp, K = P.K, a = P.a, b = K - 1 - a, RING = K + 1, RS = P.ring_stride;
    const int t = threadIdx.x, tpos = win_pos(t, K, K | 1);
    const size_t plane = (size_t)H * Wp;
    const float* __restrict__ pin = P.vol_in[view] + (size_t)dl * plane;
    float* __restrict__ qout = P.vol_out[view] + (size_t)dl * plane;
    const float* __restrict__ g = P.guide[view];

    const int X0 = strip * P.tw, X1 = min(W, X0 + P.tw), nout = X1 - X0;
    const int NO2 = nout + K - 1;             // virtual columns of the output windows
    int rlo = W, rhi = -1;                    // real a,b columns those windows touch
    for (int e = X0 - a; e < X0 - a + NO2; ++e) { const int r = reflect101(e, W); rlo = min(rlo, r); rhi = max(rhi, r); }
    const int NR = rhi - rlo + 1, NP = NR + K - 1;

    // stage-1 role: virtual input column rlo - a + t (real column c1); stage-2 role: virtual column X0 - a + t (ring column c2)
    const bool s1 = t < NP, s2 = t < NO2;
    const int c1 = reflect101(rlo - a + t, W);
    const int c2 = reflect101(X0 - a + t, W) - rlo;

    double S1[4] = {0.0, 0.0, 0.0, 0.0}, S2[4] = {0.0, 0.0, 0.0, 0.0};
    auto feed1 = [&](int r, bool add) {   // S1 +/-= (p, I0 p, I1 p, I2 p) of input row r at column c1
        const size_t o = (size_t)reflect101(r, H) * Wp + c1;
        const float p = __ldg(pin + o);
        const float v[4] = {p, fmul(__ldg(g + o), p), fmul(__ldg(g + plane + o), p), fmul(__ldg(g + 2 * plane + o), p)};
#pragma unroll
        for (int q = 0; q < 4; ++q) S1[q] = add ? __dadd_rn(S1[q], (double)v[q]) : __dsub_rn(S1[q], (double)v[q]);
    };
    auto feed2 = [&](int r, bool add) {   // S2 +/-= (a0, a1, a2, b) of a,b row r at ring column c2
        const float* src = ring + (size_t)(reflect101(r, H) % RING) * 4 * RS + c2;
#pragma unroll
        for (int q = 0; q < 4; ++q) S2[q] = add ? __dadd_rn(S2[q], (double)src[q * RS]) : __dsub_rn(S2[q], (double)src[q * RS]);
    };

    const int y0 = seg * P.seg_rows, y1 = min(H, y0 + P.seg_rows);
    int lo_ab = H, hi0 = -1;   // real a,b rows of the first output row's window
    for (int dy = -a; dy <= b; ++dy) { const int r = reflect101(y0 + dy, H); lo_ab = min(lo_ab, r); hi0 = max(hi0, r); }
    if (s1)
        for (int dy = -a; dy <= b; ++dy) feed1(lo_ab + dy, true);
    int next_ab = lo_ab;   // next a,b row stage 1 produces; S1 holds its window sums

    for (int y = y0; y < y1; ++y) {
        const int need = (y == y0) ? hi0 : reflect101(y + b, H);
        for (; next_ab <= need; ++next_ab) {
            // ---- stage 1: row sums of the column sums -> a, b of row next_ab at real columns rlo .. rhi
            if (s1) {
#pragma unroll
                for (int q = 0; q < 4; ++q) cs[q * kWinBuf + tpos] = S1[q];
            }
            __syncthreads();
            win_block_scans(cs, F, Gs, NP, K);
            __syncthreads();
            if (t < NR) {
                float m[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) m[q] = (float)__dmul_rn(win_sum(F + q * kWinBuf, Gs + q * kWinBuf, t, K), P.scale);
                float a0, a1, a2, bb;
                gif_coeffs(m[0], m[1], m[2], m[3], load_guide_pix(g, plane, (size_t)next_ab * Wp + rlo + t), a0, a1, a2, bb);
                float* dst = ring + (size_t)(next_ab % RING) * 4 * RS + t;
                dst[0] = a0; dst[RS] = a1; dst[2 * RS] = a2; dst[3 * RS] = bb;
            }
            if (s1) { feed1(next_ab + 1 + b, true); feed1(next_ab - a, false); }   // slide to row next_ab + 1
        }
        __syncthreads();   // the ring rows are complete
        // ---- stage 2: column sums of a, b over rows y-a .. y+b (reflected), row sums, q
        if (s2) {
            if (y == y0) {
                for (int dy = -a; dy <= b; ++dy) feed2(y + dy, true);
            } else {
                feed2(y + b, true);
                feed2(y - 1 - a, false);
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) cs[q * kWinBuf + tpos] = S2[q];
        }
        __syncthreads();
        win_block_scans(cs, F, Gs, NO2, K);
        __syncthreads();
        if (t < nout) {
            float m[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) m[q] = (float)__dmul_rn(win_sum(F + q * kWinBuf, Gs + q * kWinBuf, t, K), P.scale);
            const size_t o = (size_t)y * Wp + X0 + t;
            // q = box(b) + box(a0) I0 + box(a1) I1 + box(a2) I2, left to right (CVF.cpp:157-163)
            float qv = fadd(m[3], fmul(m[0], __ldg(g + o)));
            qv = fadd(qv, fmul(m[1], __ldg(g + plane + o)));
            qv = fadd(qv, fmul(m[2], __ldg(g + 2 * plane + o)));
            qout[o] = qv;
        }
    }
}

}  // namespace psm
