// psm_fgf.cuh -- the Fast Guided Filter branch (CostFilter_FGF) on the device.
//
// Reference: FastGuidedFilterColor (/root/reference/src/fastguidedfilter.cpp:121-198) as driven by
// DispEst::CostFilter_FGF (src/DispEst.cpp:281-296): FastGuidedFilter(img, GIF_R_WIN = 8, GIF_EPS, s); every
// slice is NN-subsampled by s, guided-filtered there with a K x K box, K = 2*(8/s)+1 (:206-208), and the four
// coefficient means are bilinearly up-sampled and applied at full resolution.  It is what the reference's CPU
// branch runs today (src/StereoMatch.cpp:214); it is NOT the full-resolution GIF of psm_cvf_stream.cuh.
//
// Numerics follow the CPU restatement orc_fgf_* (test infrastructure, oracle/) (pinned against cv2 with IPP off, tests/golden/
// make_golden_fgf.py): the K x K box is DEFINED as the direct fp64 sum, from 0.0, K taps left to right, then the K row
// sums top to bottom, * 1/(K*K) in double, one rounding (orc_box_k).  That equals cv::blur wherever the fp64 sums are
// exact (OpenCV slides part of its sums); beyond that, at wide-range, outlier or non-finite inputs, the direct order is
// this project's definition, and the device performs the same fp64 operations in the same order at any input.  Every float
// operation a separate IEEE op in source order; the diagonal variance terms (x - y + eps) in double with one
// rounding (cv::addWeighted); true divisions; OpenCV's own INTER_NN / INTER_LINEAR index and weight formulas
// (tables built on the host by the same float / double expressions, see psm_capi.cu).
//
// Work split (nothing like the reference's per-slice Mat pipeline of ~40 OpenCV calls):
//   fgf_guide_kernel : per view, per low-res pixel: channel means, (Sigma + eps I)^-1          (once per frame)
//   fgf_lowres_kernel: per slice tile, both low-res stages in shared memory (separable fp64 box sums): p and I*p box
//                      means -> a (3), b -> their box means                                      (reads 1/s^2 of p)
//   fgf_up_kernel    : per full-res pixel group (4 px, 128-bit store): bilinear up-sampling of the four means and
//                      q = ((ma_r*I_r + ma_g*I_g) + ma_b*I_b) + mb, written over p (p is only read at the sample
//                      points by the earlier kernels, so the filter runs in place)
// HBM traffic per view ~ 4*V written + V/s^2 * 4 read + low-res planes: the pass is write-bound like CVC.
#pragma once
#include "psm_common.cuh"

namespace psm {

struct FgfGeom {
    int W, H, Wp, w2, h2, K, s;
    double ifx, ify;   // 1 / (w2 / W), 1 / (h2 / H): INTER_NN source index = min(floor(x * ifx), W - 1)
};

__device__ __forceinline__ int fgf_nn(int i, double inv, int n)
{
    const int v = (int)floor((double)i * inv);
    return v < n - 1 ? v : n - 1;
}

// low-res planes of one view: Ic[3], m[3], inv[6] (rr rg rb gg gb bb), each h2 x w2, contiguous
__global__ void fgf_guide_kernel(const float* __restrict__ I /* 3 full-res planes, pitch Wp */, size_t plane, FgfGeom g, float eps,
                                 float* __restrict__ lo /* 12 planes */)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= g.w2 || y >= g.h2) return;
    const int a = g.K / 2;
    const size_t n2 = (size_t)g.w2 * g.h2, o = (size_t)y * g.w2 + x;
    // direct box sums in orc_box_k's order: per row, from 0.0, the taps left to right; then the row sums top to bottom
    double sm[3] = {0, 0, 0}, sp[6] = {0, 0, 0, 0, 0, 0};
    for (int dy = -a; dy <= a; ++dy) {
        const int yy = fgf_nn(reflect101(y + dy, g.h2), g.ify, g.H);
        double rm[3] = {0, 0, 0}, rp[6] = {0, 0, 0, 0, 0, 0};
        for (int dx = -a; dx <= a; ++dx) {
            const int xx = fgf_nn(reflect101(x + dx, g.w2), g.ifx, g.W);
            const size_t q = (size_t)yy * g.Wp + xx;
            const float c0 = I[q], c1 = I[plane + q], c2 = I[2 * plane + q];
            rm[0] += (double)c0; rm[1] += (double)c1; rm[2] += (double)c2;
            rp[0] += (double)fmul(c0, c0); rp[1] += (double)fmul(c0, c1); rp[2] += (double)fmul(c0, c2);
            rp[3] += (double)fmul(c1, c1); rp[4] += (double)fmul(c1, c2); rp[5] += (double)fmul(c2, c2);
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) sm[k] += rm[k];
#pragma unroll
        for (int k = 0; k < 6; ++k) sp[k] += rp[k];
    }
    const double scale = 1.0 / ((double)g.K * g.K);
    const float m0 = (float)(sm[0] * scale), m1 = (float)(sm[1] * scale), m2 = (float)(sm[2] * scale);
    float bx[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) bx[k] = (float)(sp[k] * scale);
    // fastguidedfilter.cpp:144-149 (diagonal: addWeighted in double, one rounding)
    const float rr = (float)(((double)bx[0] - (double)fmul(m0, m0)) + (double)eps);
    const float rg = fsub(bx[1], fmul(m0, m1));
    const float rb = fsub(bx[2], fmul(m0, m2));
    const float gg = (float)(((double)bx[3] - (double)fmul(m1, m1)) + (double)eps);
    const float gb = fsub(bx[4], fmul(m1, m2));
    const float bb = (float)(((double)bx[5] - (double)fmul(m2, m2)) + (double)eps);
    const float irr = fsub(fmul(gg, bb), fmul(gb, gb));   // :152-157
    const float irg = fsub(fmul(gb, rb), fmul(rg, bb));
    const float irb = fsub(fmul(rg, gb), fmul(gg, rb));
    const float igg = fsub(fmul(rr, bb), fmul(rb, rb));
    const float igb = fsub(fmul(rb, rg), fmul(rr, gb));
    const float ibb = fsub(fmul(rr, gg), fmul(rg, rg));
    const float det = fadd(fadd(fmul(irr, rr), fmul(irg, rg)), fmul(irb, rb));   // :159
    const int ys = fgf_nn(y, g.ify, g.H), xs = fgf_nn(x, g.ifx, g.W);
    const size_t q = (size_t)ys * g.Wp + xs;
    lo[o] = I[q]; lo[n2 + o] = I[plane + q]; lo[2 * n2 + o] = I[2 * plane + q];
    lo[3 * n2 + o] = m0; lo[4 * n2 + o] = m1; lo[5 * n2 + o] = m2;
    lo[6 * n2 + o] = __fdiv_rn(irr, det); lo[7 * n2 + o] = __fdiv_rn(irg, det); lo[8 * n2 + o] = __fdiv_rn(irb, det);   // :161-166
    lo[9 * n2 + o] = __fdiv_rn(igg, det); lo[10 * n2 + o] = __fdiv_rn(igb, det); lo[11 * n2 + o] = __fdiv_rn(ibb, det);
}

// Both low-resolution stages of one slice tile in ONE kernel (shared-memory tiles, separable fp64 box sums):
//   region R1 = tile + 2h halo (h = K/2): p and I*p at the NN sample points, widened once into shared memory (doubles)
//   horizontal K-sums -> vertical K-sums -> box means on R2 = tile + h halo -> a (3), b there (floats, shared memory)
//   horizontal / vertical K-sums of a, b -> their box means on the tile -> global memory (4 planes per slice)
// Cells outside the low-res image hold the value of the BORDER_REFLECT_101 pixel.  The a, b cells of R2 outside the
// image are computed as the a, b of the pixel they mirror (see the box sums below), so the second stage sees exactly the
// direct box's border handling of the first stage's output.
constexpr int kFgfTX = 32, kFgfTY = 16, kFgfThreads = 256;

__host__ __device__ inline size_t fgf_smem_bytes(int K)
{
    const int h = K / 2;
    // the three regions with odd row strides; this bounds the box the call accepts (K <= 19 in an H100's 227 KB per block)
    const size_t r1 = (size_t)((kFgfTX + 4 * h) | 1) * (kFgfTY + 4 * h);    // inputs (4 planes of doubles)
    const size_t hs = (size_t)((kFgfTX + 2 * h) | 1) * (kFgfTY + 4 * h);    // horizontal sums (4 planes of doubles)
    const size_t r2 = (size_t)((kFgfTX + 2 * h) | 1) * (kFgfTY + 2 * h);    // a, b (4 planes of floats)
    return (r1 + hs) * 4 * sizeof(double) + r2 * 4 * sizeof(float);
}

// Direct fp64 box sums of the four planes (`pstride` apart) at two outputs at once: from 0.0, K taps `step` apart, in
// order.  Eight independent chains, so that the dependent fp64 adds of one thread overlap.
template <typename T>
__device__ __forceinline__ void fgf_sum8(const T* a, const T* b, size_t pstride, int step, int K, double sa[4], double sb[4])
{
#pragma unroll
    for (int k = 0; k < 4; ++k) sa[k] = sb[k] = 0.0;
    for (int t = 0; t < K; ++t) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            sa[k] += (double)a[k * pstride + (size_t)t * step];
            sb[k] += (double)b[k * pstride + (size_t)t * step];
        }
    }
}

__global__ void __launch_bounds__(kFgfThreads) fgf_lowres_kernel(const float* __restrict__ vol, size_t vplane, FgfGeom g,
                                                                 const float* __restrict__ lo, float* __restrict__ mean)
{
    extern __shared__ double fsm[];
    const int h = g.K / 2, K = g.K;
    const int W1n = kFgfTX + 4 * h, H1 = kFgfTY + 4 * h;     // input region (W1n columns used, odd stride W1)
    const int W2n = kFgfTX + 2 * h, H2 = kFgfTY + 2 * h;     // a,b region
    const int W1 = W1n | 1, W2 = W2n | 1;
    constexpr int kTXs = kFgfTX | 1;                          // stage-2 row stride
    double* in = fsm;                                        // [4][H1][W1]
    double* hs = in + (size_t)4 * W1 * H1;                   // [4][H1][W2]  (stage 2 reuses it as [4][H2][kTXs])
    // every sum below runs one thread per output, lanes along a row, so the strides give no bank conflicts either way
    float* ab = reinterpret_cast<float*>(hs + (size_t)4 * W2 * H1);   // [4][H2][W2]
    const int x0 = blockIdx.x * kFgfTX, y0 = blockIdx.y * kFgfTY, dl = blockIdx.z;
    const size_t n2 = (size_t)g.w2 * g.h2;
    const float* p = vol + (size_t)dl * vplane;
    const double scale = 1.0 / ((double)K * K);
    const int tx0 = threadIdx.x & 31, ty0 = threadIdx.x >> 5;   // 32 x 8 thread grid: rows by warps, columns by lanes (no runtime division)
    constexpr int kRowsPerPass = kFgfThreads / 32;
    // ---- inputs: p2 = resize(p, INTER_NN) (:69) and I*p2 (:175-177) on R1, widened once
    for (int ry = ty0; ry < H1; ry += kRowsPerPass) {
        const int ly = reflect101(y0 - 2 * h + ry, g.h2);
        const float* prow = p + (size_t)fgf_nn(ly, g.ify, g.H) * g.Wp;
        for (int rx = tx0; rx < W1n; rx += 32) {
            const int lx = reflect101(x0 - 2 * h + rx, g.w2);
            const float pv = __ldg(prow + fgf_nn(lx, g.ifx, g.W));
            const size_t q = (size_t)ly * g.w2 + lx;
            const int i = ry * W1 + rx;
            in[i] = (double)pv;
            in[(size_t)W1 * H1 + i] = (double)fmul(__ldg(lo + q), pv);
            in[(size_t)2 * W1 * H1 + i] = (double)fmul(__ldg(lo + n2 + q), pv);
            in[(size_t)3 * W1 * H1 + i] = (double)fmul(__ldg(lo + 2 * n2 + q), pv);
        }
    }
    __syncthreads();
    // Box sums are DIRECT fp64 sums in orc_box_k's order: from 0.0, the K taps of a row left to right, then the K row sums
    // top to bottom.  Every R2 cell gets the box of the real pixel it stands for, (reflect101(x), reflect101(y)): its taps
    // are read around that pixel's own position in R1 (R1 cell j holds the value at reflect101(x0 - 2h + j), and
    // reflect101 is idempotent), not around the halo cell, whose taps are the same values in mirrored order.  For every
    // R2 cell a valid output reads, those taps lie inside R1; the others (beyond the image edge by more than h) are
    // clamped into R1 and only feed outputs that are never stored.
    // Each thread takes two outputs at a time and all four planes of each: eight independent chains of dependent adds.
    // ---- stage 1, horizontal: row sums of every R1 row at the R2 columns
    for (int i = threadIdx.x; i < H1 * W2n; i += 2 * kFgfThreads) {
        const bool two = i + kFgfThreads < H1 * W2n;
        const int j = two ? i + kFgfThreads : i;
        const int ry0 = i / W2n, rx0 = i - ry0 * W2n, ry1 = j / W2n, rx1 = j - ry1 * W2n;
        const int bx0 = min(max(reflect101(x0 - h + rx0, g.w2) - x0 + h, 0), W1n - K);   // R1 column of the first tap
        const int bx1 = min(max(reflect101(x0 - h + rx1, g.w2) - x0 + h, 0), W1n - K);
        double s0[4], s1[4];
        fgf_sum8(in + ry0 * W1 + bx0, in + ry1 * W1 + bx1, (size_t)W1 * H1, 1, K, s0, s1);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            hs[((size_t)k * H1 + ry0) * W2 + rx0] = s0[k];
            if (two) hs[((size_t)k * H1 + ry1) * W2 + rx1] = s1[k];
        }
    }
    __syncthreads();
    // ---- stage 1, vertical: K row sums per R2 cell, top to bottom -> box means (floats) into `ab`
    for (int i = threadIdx.x; i < H2 * W2n; i += 2 * kFgfThreads) {
        const bool two = i + kFgfThreads < H2 * W2n;
        const int j = two ? i + kFgfThreads : i;
        const int ry0 = i / W2n, rx0 = i - ry0 * W2n, ry1 = j / W2n, rx1 = j - ry1 * W2n;
        const int by0 = min(max(reflect101(y0 - h + ry0, g.h2) - y0 + h, 0), H1 - K);    // R1 row of the first tap
        const int by1 = min(max(reflect101(y0 - h + ry1, g.h2) - y0 + h, 0), H1 - K);
        double s0[4], s1[4];
        fgf_sum8(hs + by0 * W2 + rx0, hs + by1 * W2 + rx1, (size_t)W2 * H1, W2, K, s0, s1);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            ab[((size_t)k * H2 + ry0) * W2 + rx0] = (float)(s0[k] * scale);
            if (two) ab[((size_t)k * H2 + ry1) * W2 + rx1] = (float)(s1[k] * scale);
        }
    }
    __syncthreads();
    // ---- a, b on R2 from the four means of every cell, in place (fastguidedfilter.cpp:178-186)
    for (int ry = ty0; ry < H2; ry += kRowsPerPass) {
        const int ly = reflect101(y0 - h + ry, g.h2);
        for (int rx = tx0; rx < W2n; rx += 32) {
            const int i = ry * W2 + rx;
            const float mp = ab[i], mIp0 = ab[(size_t)W2 * H2 + i], mIp1 = ab[(size_t)2 * W2 * H2 + i], mIp2 = ab[(size_t)3 * W2 * H2 + i];
            const int lx = reflect101(x0 - h + rx, g.w2);
            const size_t o = (size_t)ly * g.w2 + lx;
            const float m0 = __ldg(lo + 3 * n2 + o), m1 = __ldg(lo + 4 * n2 + o), m2 = __ldg(lo + 5 * n2 + o);
            const float c0 = fsub(mIp0, fmul(m0, mp)), c1 = fsub(mIp1, fmul(m1, mp)), c2 = fsub(mIp2, fmul(m2, mp));
            const float irr = __ldg(lo + 6 * n2 + o), irg = __ldg(lo + 7 * n2 + o), irb = __ldg(lo + 8 * n2 + o);
            const float igg = __ldg(lo + 9 * n2 + o), igb = __ldg(lo + 10 * n2 + o), ibb = __ldg(lo + 11 * n2 + o);
            const float ar = fadd(fadd(fmul(irr, c0), fmul(irg, c1)), fmul(irb, c2));
            const float ag = fadd(fadd(fmul(irg, c0), fmul(igg, c1)), fmul(igb, c2));
            const float ab_ = fadd(fadd(fmul(irb, c0), fmul(igb, c1)), fmul(ibb, c2));
            const float bb = fsub(fsub(fsub(mp, fmul(ar, m0)), fmul(ag, m1)), fmul(ab_, m2));
            ab[i] = ar; ab[(size_t)W2 * H2 + i] = ag; ab[(size_t)2 * W2 * H2 + i] = ab_; ab[(size_t)3 * W2 * H2 + i] = bb;
        }
    }
    __syncthreads();
    // ---- stage 2, horizontal: row sums of every R2 row at the tile's columns (output x reads R2 columns x - x0 .. + K-1)
    for (int i = threadIdx.x; i < H2 * kFgfTX; i += 2 * kFgfThreads) {
        const bool two = i + kFgfThreads < H2 * kFgfTX;
        const int j = two ? i + kFgfThreads : i;
        const int ry0 = i / kFgfTX, rx0 = i % kFgfTX, ry1 = j / kFgfTX, rx1 = j % kFgfTX;
        double s0[4], s1[4];
        fgf_sum8(ab + ry0 * W2 + rx0, ab + ry1 * W2 + rx1, (size_t)W2 * H2, 1, K, s0, s1);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            hs[((size_t)k * H2 + ry0) * kTXs + rx0] = s0[k];
            if (two) hs[((size_t)k * H2 + ry1) * kTXs + rx1] = s1[k];
        }
    }
    __syncthreads();
    // ---- stage 2, vertical -> (mean_a_r, mean_a_g, mean_a_b, mean_b) of the tile, interleaved per pixel, coalesced 128-bit
    // stores (:188-191); the 32 x 16 outputs are exactly two per thread, rows ty0 and ty0 + 8
    static_assert(kFgfTY == 2 * kRowsPerPass, "two output rows per thread");
    {
        double s0[4], s1[4];
        fgf_sum8(hs + ty0 * kTXs + tx0, hs + (ty0 + kRowsPerPass) * kTXs + tx0, (size_t)kTXs * H2, kTXs, K, s0, s1);
        const int x = x0 + tx0;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int y = y0 + ty0 + r * kRowsPerPass;
            const double* sr = r ? s1 : s0;
            if (x < g.w2 && y < g.h2)
                reinterpret_cast<float4*>(mean)[(size_t)dl * n2 + (size_t)y * g.w2 + x] =
                    make_float4((float)(sr[0] * scale), (float)(sr[1] * scale), (float)(sr[2] * scale), (float)(sr[3] * scale));
        }
    }
}

// up-sampling plan (OpenCV's own INTER_LINEAR formula, built on the host): per destination column / row the two source
// indices and the float weight of the second one, 16 bytes each so that one 128-bit load fetches an entry
struct alignas(16) FgfTap { int i0, i1; float f, pad; };
struct FgfPlan { const FgfTap* x; const FgfTap* y; };

__global__ void __launch_bounds__(128) fgf_up_kernel(float* __restrict__ vol, size_t vplane, const float* __restrict__ I, size_t plane,
                                                     FgfGeom g, FgfPlan pl, const float* __restrict__ mean)
{
    const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4, y = blockIdx.y, dl = blockIdx.z;
    if (x4 >= g.W) return;
    const size_t n2 = (size_t)g.w2 * g.h2;
    const float4* m = reinterpret_cast<const float4*>(mean) + (size_t)dl * n2;   // (ma_r, ma_g, ma_b, mb) per low-res pixel
    const FgfTap ty = pl.y[y];
    const float fy = ty.f, b0 = fsub(1.f, fy);
    const float4* row0 = m + (size_t)ty.i0 * g.w2;
    const float4* row1 = m + (size_t)ty.i1 * g.w2;
    const size_t o4 = (size_t)y * g.Wp + x4;
    float i0[4], i1[4], i2[4];
    if (x4 + 3 < g.Wp) {   // rows are padded to a multiple of 4 floats: a full 128-bit read is always inside the row
        const float4 a = __ldg(reinterpret_cast<const float4*>(I + o4)), b = __ldg(reinterpret_cast<const float4*>(I + plane + o4)),
                     c = __ldg(reinterpret_cast<const float4*>(I + 2 * plane + o4));
        i0[0] = a.x; i0[1] = a.y; i0[2] = a.z; i0[3] = a.w; i1[0] = b.x; i1[1] = b.y; i1[2] = b.z; i1[3] = b.w;
        i2[0] = c.x; i2[1] = c.y; i2[2] = c.z; i2[3] = c.w;
    }
    float q[4];
    int c0 = -1, c1 = -1;
    float4 s00 = make_float4(0.f, 0.f, 0.f, 0.f), s01 = s00, s10 = s00, s11 = s00;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int x = x4 + j;
        if (x >= g.W) { q[j] = 0.f; continue; }
        const FgfTap tx = pl.x[x];
        const float fx = tx.f, a0 = fsub(1.f, fx);
        // consecutive pixels share their low-res column pair (s >= 2) or shift it by one: reload only what changed
        if (tx.i0 != c0 || tx.i1 != c1) {
            if (tx.i0 == c1) { s00 = s01; s10 = s11; }
            else { s00 = __ldg(row0 + tx.i0); s10 = __ldg(row1 + tx.i0); }
            s01 = __ldg(row0 + tx.i1); s11 = __ldg(row1 + tx.i1);
            c0 = tx.i0; c1 = tx.i1;
        }
        // rows after columns, like cv::resize: h = S0*(1-fx) + S1*fx per source row, then h0*(1-fy) + h1*fy
#define PSM_FGF_UP(c) fadd(fmul(fadd(fmul(s00.c, a0), fmul(s01.c, fx)), b0), fmul(fadd(fmul(s10.c, a0), fmul(s11.c, fx)), fy))
        const float ur = PSM_FGF_UP(x), ug = PSM_FGF_UP(y), ub = PSM_FGF_UP(z), ubb = PSM_FGF_UP(w);
#undef PSM_FGF_UP
        q[j] = fadd(fadd(fadd(fmul(ur, i0[j]), fmul(ug, i1[j])), fmul(ub, i2[j])), ubb);   // :196
    }
    float* dst = vol + (size_t)dl * vplane + o4;
    if (x4 + 3 < g.W) __stcs(reinterpret_cast<float4*>(dst), make_float4(q[0], q[1], q[2], q[3]));
    else for (int j = 0; j < 4 && x4 + j < g.W; ++j) dst[j] = q[j];
}

}  // namespace psm
