// psm_kernels.cuh -- ingest, cost-volume construction (CVC), guide precompute and WTA.  The fused
// streaming CVF kernel is in psm_cvf_stream.cuh, the reference-order guided filter (PSM_CVF_NAIVE)
// in psm_cvf_ref.cuh.  Layout: every plane / volume row has pitch Wp floats and is stored with a
// column halo: kPadLeft columns before column 0 and at least kPadRight after column W-1 (so a
// pointer to (row, col 0) may be indexed from -kPadLeft .. W+kPadRight-1); pitch and halo are
// multiples of 4 floats, so 4-column groups are 16-byte aligned.  The halos of the cost volumes
// and of the three guide channels hold the BORDER_REFLECT_101 mirror of the row (written by
// pad_cols_kernel), which lets the streaming CVF kernel use plain 128-bit loads everywhere.
// Planes are [H][Wp], volumes [d_local][H][Wp]; "W4" below is W rounded up to 4.
#pragma once
#include <type_traits>

#include "psm_common.cuh"

namespace psm {

constexpr int kPadLeft = 32;   // floats before column 0 (128 B: column 0 of every row is cache-line aligned);
                               // the last 8 of them are the mirrored left halo
constexpr int kPadRight = 12;  // minimum halo columns after column W4-1 (the last strip reads up to W+10)

// Row pitch (floats) for an image of width W: left pad + max(W4 + right halo, one full strip),
// rounded up to a multiple of 32 floats so that every row starts on a 128-byte line.
__host__ __device__ inline int pitch_for_width(int W)
{
    const int w4 = (W + 3) & ~3;
    const int right = (w4 + kPadRight > 120) ? w4 + kPadRight : 120;
    return kPadLeft + ((right + 31) & ~31);
}

// Fill the column halos of `nrows` rows with the BORDER_REFLECT_101 mirror of the row:
// row[-k] = row[k] (k = 1..8), row[W+k] = row[W-2-k] (k = 0..7), zeros beyond.
__global__ void pad_cols_kernel(float* __restrict__ base, size_t nrows, int W, int Wp)
{
    const size_t row = (size_t)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
    if (row >= nrows) return;
    float* r = base + row * (size_t)Wp;
    const int lane = threadIdx.x & 31;
    const int right = Wp - kPadLeft - W;  // halo columns after W-1
    for (int k = lane; k < kPadLeft + right; k += 32) {
        const int x = k < kPadLeft ? -(k + 1) : W + (k - kPadLeft);
        const bool mirrored = (x < 0 && x >= -8) || (x >= W && x < W + 8);
        r[x] = mirrored ? r[reflect101(x, W)] : 0.f;
    }
}

// ------------------------------------------------------------------------------------------
// Ingest: a BGR frame (float or u8) in any PlanesSrc layout, a YUV frame (YuvSrc) or a Bayer frame (BayerSrc); an 8-bit
// frame of any kind may be read through rectification maps (RectifySrc) -> 3 planar channels + x-gradient of the gray image.
// Restates StereoMatch.cpp:193-197 (u8 * (1/255.0f)), CVF.cpp:47 (split) and CVC.cpp:41-46
// (cvtColor RGB2GRAY on the BGR image, Sobel dx=1 ksize=1 with BORDER_REFLECT_101).
// ------------------------------------------------------------------------------------------
// guide_flags bits (per view): raised by ingest_kernel (kGuideOutside, kGuideInexact) and the guide precompute (kGuideNonFinite)
constexpr int kGuideOutside = 1;     // a channel value is negative, -0, inf, NaN or >= 2^61: no integer widening
constexpr int kGuideNonFinite = 2;   // a mean, adjugate or 1/det value is not finite
constexpr int kGuideInexact = 4;     // a nonzero channel value lies outside [2^-12, 1]: the guide's box sums may be inexact

__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(uint8_t v) { return fmul((float)v, 1 / 255.0f); }

// gray of one pixel's channels c0, c1, c2 (B, G, R) in either PSM_OPT_GRAY_MODE
__device__ __forceinline__ float gray_of(float c0, float c1, float c2, int gray_mode)
{
    if (gray_mode == 0) return __fmaf_rn(c2, 0.114f, __fmaf_rn(c0, 0.299f, fmul(c1, 0.587f)));
    return fadd(fadd(fmul(c0, 0.299f), fmul(c1, 0.587f)), fmul(c2, 0.114f));
}

// the guide flags one pixel's channel values raise (see ingest_kernel)
__device__ __forceinline__ void ingest_flags(float v0, float v1, float v2, int* __restrict__ guide_flag)
{
    const unsigned u0 = __float_as_uint(v0), u1 = __float_as_uint(v1), u2 = __float_as_uint(v2);
    if (max(max(u0, u1), u2) >= 0x5e000000u) atomicOr(guide_flag, kGuideOutside | kGuideInexact);
    auto inexact = [](unsigned u) { return u != 0u && u - 0x39800000u > 0x3f800000u - 0x39800000u; };   // outside {0} U [2^-12, 1]
    if (inexact(u0) || inexact(u1) || inexact(u2)) atomicOr(guide_flag, kGuideInexact);
}

// A frame given as three channel pointers (B, G, R) and byte steps: sample (x, y) of channel c at
// ch[c] + y * row_step + x * col_step.  HWC BGR / RGB, BGRA and planar CHW frames all fit.
struct PlanesSrc {
    const char* ch[3];
    size_t row_step, col_step;
};

// the PlanesSrc of an interleaved BGR frame of `elem`-byte samples whose rows lie `step` bytes apart
inline PlanesSrc interleaved_src(const void* p, size_t elem, size_t step)
{
    const char* b = static_cast<const char*>(p);
    return PlanesSrc{{b, b + elem, b + 2 * elem}, step, 3 * elem};
}

// A YUV frame (psm_set_images_yuv / psm_set_images_device_yuv): luma Y(x, y) at p[0] + y * y_row_step + x * y_col_step,
// chroma U and V at (x >> 1, y >> vs) of p[1] / p[2] with the chroma steps; vs = 1 for 4:2:0, 0 for 4:2:2.  NV12 / NV21,
// I420 / YV12 and the packed YUYV / UYVY / YVYU layouts differ only in these offsets and steps (DESIGN.md section 27).
struct YuvSrc {
    const char* p[3];   // Y, U, V
    size_t y_row_step, y_col_step, c_row_step, c_col_step;
    int vs;
};

// A Bayer frame of Wf x Hf (psm_set_images_bayer / psm_set_images_device_bayer): raw sample (x, y) at p + y * row_step +
// x * col_step, one byte per pixel, the colour of each site given by the red site's column and row parity (DESIGN.md
// section 28).  The four patterns differ only in (rx, ry).
struct BayerSrc {
    const char* p;
    size_t row_step, col_step;
    int Wf, Hf;
    int rx, ry;   // the red site's column and row parity: RGGB (0, 0), BGGR (1, 1), GRBG (1, 0), GBRG (0, 1)
    int ea;       // 1: the edge-aware method (COLOR_Bayer*2BGR_EA), 0: bilinear (COLOR_Bayer*2BGR)
};

// A u8 frame of SW x SH, BGR (PlanesSrc), YUV (YuvSrc) or Bayer (BayerSrc), read through the rectification maps of one
// view (psm_set_rectify): output pixel (x, y) of the W x H crop is OpenCV's remap(frame, xy, a, INTER_LINEAR,
// BORDER_CONSTANT 0) with the fixed-point maps of initUndistortRectifyMap(..., CV_16SC2), cropped (DESIGN.md section 25);
// a YUV or Bayer frame is remapped as the BGR frame cvtColor makes of it.  The maps are dense: entry (x, y) at y * W + x.
template <class F>
struct RectifySrc {
    F frame;                   // the source frame, SW x SH
    const short2* xy;          // map[0]: the integer tap (sx, sy)
    const uint16_t* a;         // map[1]: the 5 + 5-bit fraction (fy << 5 | fx); bits above 10 are ignored
    int SW, SH, W;
};

// channel c of the sample at (x, y), as to_f32 sees it
template <typename T>
__device__ __forceinline__ float read_sample(const PlanesSrc& src, size_t row, int c, int x, int)
{
    return to_f32(*reinterpret_cast<const T*>(src.ch[c] + row + (size_t)x * src.col_step));
}

// tap(sx, sy, w) for each tap of rectified pixel (x, y) inside the frame: the four taps' weights w sum to 32768 and a tap
// outside the frame reads 0.  Every tap is bounds-checked before it is read, so any map is memory-safe.
template <class F, class Tap>
__device__ __forceinline__ void remap_taps(const RectifySrc<F>& src, int x, int y, Tap tap)
{
    const size_t i = (size_t)y * src.W + x;
    const short2 p = src.xy[i];
    const int a = src.a[i] & 1023, fx = a & 31, fy = a >> 5;
    const int wx[2] = {32 - fx, fx}, wy[2] = {32 - fy, fy};
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
            const int sx = p.x + dx, sy = p.y + dy;
            if ((unsigned)sx < (unsigned)src.SW && (unsigned)sy < (unsigned)src.SH) tap(sx, sy, wx[dx] * wy[dy] * 32);
        }
}

// channel c of rectified pixel (x, y): the integer sum is rounded like OpenCV's FixedPtCast (+ 2^14, >> 15), so the
// value is the u8 remap writes
template <typename T>
__device__ __forceinline__ float read_sample(const RectifySrc<PlanesSrc>& src, size_t, int c, int x, int y)
{
    static_assert(std::is_same<T, uint8_t>::value, "rectification reads 8-bit frames");
    int acc = 0;
    remap_taps(src, x, y, [&](int sx, int sy, int w) {
        acc += w * *reinterpret_cast<const uint8_t*>(src.frame.ch[c] + (size_t)sy * src.frame.row_step +
                                                     (size_t)sx * src.frame.col_step);
    });
    return to_f32((uint8_t)((acc + 16384) >> 15));
}

// B, G, R of pixel (x, y) of a YUV frame: OpenCV's BT.601 limited-range fixed-point conversion (cvtColor
// COLOR_YUV2BGR_NV12 / NV21 / I420 / YV12 / YUYV / UYVY / YVYU), each value clamped to 0..255.  The sums stay below 2^31.
__device__ __forceinline__ void read_bgr(const YuvSrc& src, int x, int y, int bgr[3])
{
    const size_t co = (size_t)(y >> src.vs) * src.c_row_step + (size_t)(x >> 1) * src.c_col_step;
    const int Y = *reinterpret_cast<const uint8_t*>(src.p[0] + (size_t)y * src.y_row_step + (size_t)x * src.y_col_step);
    const int u = *reinterpret_cast<const uint8_t*>(src.p[1] + co) - 128;
    const int v = *reinterpret_cast<const uint8_t*>(src.p[2] + co) - 128;
    const int yy = max(0, Y - 16) * 1220542 + (1 << 19);
    bgr[0] = min(max((yy + 2116026 * u) >> 20, 0), 255);
    bgr[1] = min(max((yy - 852492 * v - 409993 * u) >> 20, 0), 255);
    bgr[2] = min(max((yy + 1673527 * v) >> 20, 0), 255);
}

// B, G, R of pixel (x, y) of a Bayer frame: OpenCV's demosaicing (cvtColor COLOR_Bayer<PATTERN>2BGR, or _EA), each pixel
// the interior pixel at (clamp(x, 1, Wf - 2), clamp(y, 1, Hf - 2)) and every pixel 0 when Wf < 3 or Hf < 3, as cv2 does.
// At the interior pixel, of colour c: c is its own sample; at an R or B site G is (n4 + 2) >> 2 over the four edge
// neighbours (edge-aware: the horizontal pair's rounded mean when |left - right| <= |up - down|, else the vertical
// pair's) and the opposite colour (d4 + 2) >> 2 over the four diagonal ones; at a G site the colour of its row's other
// sites is the horizontal pair's (a + b + 1) >> 1, the third colour the vertical pair's.  Only samples of the 3 x 3
// neighbourhood of the clamped pixel are read, all inside the frame.
__device__ __forceinline__ void read_bgr(const BayerSrc& src, int x, int y, int bgr[3])
{
    if (src.Wf < 3 || src.Hf < 3) {
        bgr[0] = bgr[1] = bgr[2] = 0;
        return;
    }
    const int cx = min(max(x, 1), src.Wf - 2), cy = min(max(y, 1), src.Hf - 2);
    const char* row[3];
    row[1] = src.p + (size_t)cy * src.row_step + (size_t)cx * src.col_step;
    row[0] = row[1] - src.row_step;
    row[2] = row[1] + src.row_step;
    int s[3][3];   // s[dy + 1][dx + 1] = raw(cx + dx, cy + dy)
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        s[k][0] = *reinterpret_cast<const uint8_t*>(row[k] - src.col_step);
        s[k][1] = *reinterpret_cast<const uint8_t*>(row[k]);
        s[k][2] = *reinterpret_cast<const uint8_t*>(row[k] + src.col_step);
    }
    const int l = s[1][0], r = s[1][2], u = s[0][1], d = s[2][1];
    const int hor = (l + r + 1) >> 1, ver = (u + d + 1) >> 1;
    const bool red_row = ((cy ^ src.ry) & 1) == 0, red_col = ((cx ^ src.rx) & 1) == 0;
    int R, G, B;
    if (red_row == red_col) {   // an R (both) or B (neither) site
        G = !src.ea ? (l + r + u + d + 2) >> 2 : abs(l - r) <= abs(u - d) ? hor : ver;
        const int opp = (s[0][0] + s[0][2] + s[2][0] + s[2][2] + 2) >> 2;
        R = red_row ? s[1][1] : opp;
        B = red_row ? opp : s[1][1];
    } else {   // a G site
        G = s[1][1];
        R = red_row ? hor : ver;
        B = red_row ? ver : hor;
    }
    bgr[0] = B;
    bgr[1] = G;
    bgr[2] = R;
}

// B, G, R of rectified pixel (x, y) of a YUV or Bayer frame: each tap's BGR once, then remap's rounding per channel
template <class F>
__device__ __forceinline__ void read_bgr(const RectifySrc<F>& src, int x, int y, int bgr[3])
{
    int acc[3] = {0, 0, 0};
    remap_taps(src, x, y, [&](int sx, int sy, int w) {
        int t[3];
        read_bgr(src.frame, sx, sy, t);
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[c] += w * t[c];
    });
#pragma unroll
    for (int c = 0; c < 3; ++c) bgr[c] = (acc[c] + 16384) >> 15;
}

// source kinds that convert whole pixels (read_bgr) instead of reading the channels one by one (read_sample)
template <class Src> constexpr bool kPixelSrc = false;
template <> constexpr bool kPixelSrc<YuvSrc> = true;
template <> constexpr bool kPixelSrc<BayerSrc> = true;
template <class F> constexpr bool kPixelSrc<RectifySrc<F>> = kPixelSrc<F>;

// the three channels of pixel (x, y) of a YUV or Bayer source, as to_f32 sees them
template <class Src>
__device__ __forceinline__ void read_pixel(const Src& src, int x, int y, float v[3])
{
    int bgr[3];
    read_bgr(src, x, y, bgr);
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = to_f32((uint8_t)bgr[c]);
}

template <typename T, class Src = PlanesSrc>
__global__ void ingest_kernel(Src src, int W, int H, int Wp,
                              float* __restrict__ I0, float* __restrict__ I1, float* __restrict__ I2,
                              float* __restrict__ grd, int gray_mode, int* __restrict__ guide_flag)
{
    static_assert(!kPixelSrc<Src> || std::is_same<T, uint8_t>::value, "YUV and Bayer frames are 8-bit");
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= ((W + 3) & ~3) || y >= H) return;
    const size_t o = (size_t)y * Wp + x;
    if (x >= W) { I0[o] = 0.f; I1[o] = 0.f; I2[o] = 0.f; grd[o] = 0.f; return; }
    size_t row = 0;
    if constexpr (std::is_same<Src, PlanesSrc>::value) row = (size_t)y * src.row_step;
    // A BGR source reads the channels one by one (sample(c, xx): channel c of pixel (xx, y)); a YUV or Bayer source
    // converts each pixel it reads once (read_pixel).  gray_at(xx): the gray value of pixel (xx, y).
    auto sample = [&](int c, int xx) {
        if constexpr (kPixelSrc<Src>) return 0.f;
        else return read_sample<T>(src, row, c, xx, y);
    };
    auto gray_at = [&](int xx) {
        if constexpr (kPixelSrc<Src>) {
            float p[3];
            read_pixel(src, xx, y, p);
            return gray_of(p[0], p[1], p[2], gray_mode);
        } else {
            return gray_of(sample(0, xx), sample(1, xx), sample(2, xx), gray_mode);
        }
    };
    float v[3];
    if constexpr (kPixelSrc<Src>) read_pixel(src, x, y, v);
    else v[0] = sample(0, x), v[1] = sample(1, x), v[2] = sample(2, x);
    const float v0 = v[0], v1 = v[1], v2 = v[2];
    I0[o] = v0;
    I1[o] = v1;
    I2[o] = v2;
    // the integer widening in guide_kernel / the CVF kernel assumes I >= +0, finite, and I * I finite (images are in
    // [0,1] by contract, DispEst data contract SURVEY 8b); a negative, non-finite or >= 2^61 value raises kGuideOutside
    // and selects their conversion-pipe paths (bit patterns compare like the magnitudes; the sign bit sorts last).
    // Below 2^61 every cost psm_cost_const builds is finite, >= +0 and < 2^63 (|l - r| < 2^61 per channel), so the
    // slices of such a view need no reference-order pass of their own; with kGuideOutside the whole view takes it.
    // The guide's box sums (I_c and the rounded products I_c I_c', CVF.cpp:49-62) are exact in any order when every
    // nonzero value lies in [2^-12, 1]: a product is then 0 or at least 2^-24, a multiple of 2^-47, and a sum of at most
    // 64 such values in [0, 64] needs at most 53 bits.  Any other nonzero value raises kGuideInexact and the guide is
    // recomputed in OpenCV's order (psm_cvf_ref.cuh).  u8 images (0 or 1/255 .. 1) never raise it.
    ingest_flags(v0, v1, v2, guide_flag);
    const int xr = reflect101(x + 1, W), xl = reflect101(x - 1, W);
    const float gr = gray_at(xr);
    const float gl = gray_at(xl);
    grd[o] = fsub(gr, gl);
}

// ------------------------------------------------------------------------------------------
// K1 CVC.  One thread = 4 consecutive pixels of one row of ONE view; it walks the owned
// disparities keeping the matched window of the other image in registers (one new scalar load
// per plane per disparity; GROUPED builds take one 128-bit load per plane per FOUR disparities when
// the shard starts at a multiple of 4 -- same speed, more registers, kept for A/B) and writes one
// 128-bit store per slice.
//   left  volume (SIGN=-1): x >= d     ? cost4(L[x], R[x-d]) : border(L[x])   CVC.cpp:122-149
//   right volume (SIGN=+1): x <  W - d ? cost4(R[x], L[x+d]) : border(R[x])   CVC.cpp:151-179
// cost4 = CVC.cpp:18-27 (float), border = CVC.cpp:30-39 (double intermediates, BC_32F = 1.0).
// ------------------------------------------------------------------------------------------
struct CvcParams {
    const float* self[4];   // planes of the view being built: c0,c1,c2,grd
    const float* other[4];  // planes of the matched view
    float* vol;             // [d_count][H][Wp]
    int W, H, Wp, d_begin, d_count;
    int fold_halo;          // 1: this kernel also writes the mirrored column halo (W >= 32)
};

// The weighting of the colour and gradient differences.  CostFixed is the reference's compiled ALPHA_32F = 0.9f without
// truncation (the shipped kernels); CostParam restores the truncation lines CVC.cpp:24-25, 36-37 with run-time alpha and
// thresholds (psm_set_matching_cost).  Both round every operation separately; (1 - alpha) is one fsub as in CVC.cpp:26.
struct CostFixed {
    __device__ __forceinline__ float operator()(float clr, float grd) const
    {
        return fadd(fmul(0.9f, clr), fmul(fsub(1.0f, 0.9f), grd));
    }
};

struct CvcCost { float alpha, tau_color, tau_grad; };   // psm_set_matching_cost; +inf = no truncation

struct CostParam {
    float alpha, one_minus_alpha, tau_color, tau_grad;
    __device__ __forceinline__ explicit CostParam(const CvcCost& k)
        : alpha(k.alpha), one_minus_alpha(fsub(1.0f, k.alpha)), tau_color(k.tau_color), tau_grad(k.tau_grad) {}
    __device__ __forceinline__ float operator()(float clr, float grd) const
    {
        clr = clr > tau_color ? tau_color : clr;   // a select, not fminf: a NaN difference stays NaN
        grd = grd > tau_grad ? tau_grad : grd;
        return fadd(fmul(alpha, clr), fmul(one_minus_alpha, grd));
    }
};

template <class Weigh>
__device__ __forceinline__ float cost4(float l0, float l1, float l2, float lg,
                                       float r0, float r1, float r2, float rg, const Weigh& weigh)
{
    const float clr = fadd(fadd(fabsf(fsub(l0, r0)), fabsf(fsub(l1, r1))), fabsf(fsub(l2, r2)));
    const float grd = fabsf(fsub(lg, rg));
    return weigh(clr, grd);
}

template <class Weigh>
__device__ __forceinline__ float cost_border(float l0, float l1, float l2, float lg, const Weigh& weigh)
{
    const double s = __dadd_rn(__dadd_rn(fabs(__dsub_rn((double)l0, 1.0)), fabs(__dsub_rn((double)l1, 1.0))),
                               fabs(__dsub_rn((double)l2, 1.0)));
    const float clr = (float)s;
    const float grd = (float)fabs(__dsub_rn((double)lg, 1.0));
    return weigh(clr, grd);
}

template <int SIGN, int GROUPED, class Weigh>
__device__ __forceinline__ void cvc_body(const CvcParams& P, const Weigh& weigh);

// both volumes in ONE launch (blockIdx.z = view): twice the CTAs in flight and no tail between the two views.
// MINB = resident CTAs per SM the register budget is cut for; GROUPED: 0 = shipped (interior fast path + scalar-load window for the
// border warps), 1 = border / all warps use grouped 128-bit window loads when the shard is aligned (A/B), 2 = no fast path (round-1 loop).
// blockIdx.z = chunk * 2 + view: with chunk > 0 (P2.chunk slices per CTA instead of all owned slices) the grid walks the volume
// chunk by chunk -- z is the slowest block index -- so that at any moment the GPU writes a few neighbouring slices instead of one
// 2 KB run in each of 128 slices 8 MB apart (DRAM page locality of the 2.1 GB store stream; DESIGN.md section 10).
// NVIEWS = 1 (PSM_VIEWS_LEFT) builds the left volume alone: blockIdx.z = chunk.
struct CvcParams2 { CvcParams v[2]; int chunk; };
template <int MINB, int GROUPED, int NVIEWS = 2>
__global__ void __launch_bounds__(128, MINB) cvc_both_kernel(const CvcParams2 P2)
{
    const int view = NVIEWS == 2 ? blockIdx.z & 1 : 0, chunk = NVIEWS == 2 ? blockIdx.z >> 1 : blockIdx.z;
    CvcParams P = P2.v[view];
    if (P2.chunk > 0) {
        const int first = chunk * P2.chunk;
        P.vol += (size_t)first * P.H * P.Wp;
        P.d_begin += first;
        P.d_count = min(P2.chunk, P.d_count - first);
    }
    if (view == 0) cvc_body<-1, GROUPED>(P, CostFixed());
    else cvc_body<+1, GROUPED>(P, CostFixed());
}

// The same K1 at any psm_set_matching_cost setting other than the default: the shipped decomposition (interior fast path,
// scalar window loads, all owned slices per CTA; tuning options 106 and 108 do not apply), grid z = view (NVIEWS = 1: the
// left volume alone).
template <int NVIEWS = 2>
__global__ void __launch_bounds__(128, 7) cvc_cost_kernel(const CvcParams2 P2, const CvcCost K)
{
    const int view = NVIEWS == 2 ? blockIdx.z & 1 : 0;
    const CvcParams P = P2.v[view];
    const CostParam weigh(K);
    if (view == 0) cvc_body<-1, 0>(P, weigh);
    else cvc_body<+1, 0>(P, weigh);
}

template <int SIGN, int GROUPED, class Weigh>
__device__ __forceinline__ void cvc_body(const CvcParams& P, const Weigh& weigh)
{
    const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const int y = blockIdx.y;
    if (x4 >= ((P.W + 3) & ~3)) return;
    const int W = P.W;
    const size_t ro = (size_t)y * P.Wp;

    float s[4][4], bord[4];  // [plane][pixel]
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(P.self[c] + ro + x4));
        s[c][0] = v.x; s[c][1] = v.y; s[c][2] = v.z; s[c][3] = v.w;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) bord[j] = cost_border(s[0][j], s[1][j], s[2][j], s[3][j], weigh);

    const float* o0 = P.other[0] + ro;
    const float* o1 = P.other[1] + ro;
    const float* o2 = P.other[2] + ro;
    const float* o3 = P.other[3] + ro;
    auto clampx = [W](int x) { return x < 0 ? 0 : (x >= W ? W - 1 : x); };

    int d = P.d_begin;
    const size_t slice = (size_t)P.H * P.Wp;
    float* out = P.vol + ro + x4;
    // mirrored column halo (see pad_cols_kernel), written here for W >= 32: pixel x in [1,8] also goes to
    // column -x, pixel x in [W-9, W-2] also to column 2(W-1)-x.  Only the edge threads of a row take part.
    int halo_off[4];
    bool edge = false;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int x = x4 + j;
        halo_off[j] = 0;
        if (P.fold_halo && x < W) {
            if (x >= 1 && x <= 8) halo_off[j] = -x - x4;
            else if (x >= W - 9 && x <= W - 2) halo_off[j] = 2 * (W - 1) - x - x4;
        }
        edge |= halo_off[j] != 0;
    }
    const bool full_group = x4 + 3 < W || !P.fold_halo;
    auto emit = [&](int dl, int dd, const float (&m)[4][4]) {   // m[c][j]: matched pixel of plane c for pixel j at disparity dd
        float4 r;
        float* rp = reinterpret_cast<float*>(&r);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int x = x4 + j;
            const bool interior = (SIGN < 0) ? (x >= dd) : (x < W - dd);
            const float c = cost4(s[0][j], s[1][j], s[2][j], s[3][j], m[0][j], m[1][j], m[2][j], m[3][j], weigh);
            rp[j] = (x < W) ? (interior ? c : bord[j]) : 0.f;
        }
        float* o = out + (size_t)dl * slice;
        if (full_group) __stcs(reinterpret_cast<float4*>(o), r);   // streaming store: 2 GB per frame, next touched by the CVF kernel from HBM
        else {  // last, partial group of a row: columns >= W belong to the mirrored halo
#pragma unroll
            for (int j = 0; j < 4; ++j) if (x4 + j < W) o[j] = rp[j];
        }
        if (edge) {
#pragma unroll
            for (int j = 0; j < 4; ++j) if (halo_off[j] != 0) o[halo_off[j]] = rp[j];
        }
    };

    // Interior fast path: a warp whose 128 pixels are matched inside the image for EVERY owned disparity (left volume: x >= the
    // largest d; right volume: x + largest d < W), away from the mirrored-halo columns and the ragged last group -- 13 of the 15
    // warps of a 1920-pixel row at D = 128 -- runs the same arithmetic without the per-pixel interior / x < W selects, the address
    // clamps and the halo branches: ~50 instead of ~98 instructions per 128-bit store.  (The one load past the matched range in
    // the last iteration lands in the row's mirrored halo and is never used.)
    if (GROUPED != 2) {
        const int dmax = P.d_begin + P.d_count - 1;
        const bool all_in = (SIGN < 0) ? (x4 >= dmax) : (x4 + 3 < W - dmax);
        if (__all_sync(0xffffffffu, all_in && !edge && x4 + 3 < W)) {
            const float* q[4] = {o0 + x4, o1 + x4, o2 + x4, o3 + x4};
            float w[4][4];
#pragma unroll
            for (int c = 0; c < 4; ++c)
#pragma unroll
                for (int j = 0; j < 4; ++j) w[c][j] = __ldg(q[c] + j + SIGN * d);
            float* o = out;
#pragma unroll 4
            for (int dl = 0; dl < P.d_count; ++dl, ++d, o += slice) {
                float4 r;
                r.x = cost4(s[0][0], s[1][0], s[2][0], s[3][0], w[0][0], w[1][0], w[2][0], w[3][0], weigh);
                r.y = cost4(s[0][1], s[1][1], s[2][1], s[3][1], w[0][1], w[1][1], w[2][1], w[3][1], weigh);
                r.z = cost4(s[0][2], s[1][2], s[2][2], s[3][2], w[0][2], w[1][2], w[2][2], w[3][2], weigh);
                r.w = cost4(s[0][3], s[1][3], s[2][3], s[3][3], w[0][3], w[1][3], w[2][3], w[3][3], weigh);
                __stcs(reinterpret_cast<float4*>(o), r);
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    if (SIGN < 0) { w[c][3] = w[c][2]; w[c][2] = w[c][1]; w[c][1] = w[c][0]; w[c][0] = __ldg(q[c] - (d + 1)); }
                    else { w[c][0] = w[c][1]; w[c][1] = w[c][2]; w[c][2] = w[c][3]; w[c][3] = __ldg(q[c] + 3 + (d + 1)); }
                }
            }
            return;
        }
    }
    if (GROUPED == 1 && (P.d_begin & 3) == 0) {
        // Aligned shard (every D/N split of the BASELINE configs): four disparities per block.  With d % 4 == 0 the matched
        // positions x4 + j -/+ (d + k), k = 0..3, lie in two ALIGNED 4-column groups of the other view, and the next block
        // needs exactly one new group per plane -- one 128-bit load per plane per four slices instead of four scalar loads.
        // A group that lies wholly outside [0, W) is only ever matched by border pixels (whose cost is bord[j]), so its
        // address is clamped to a valid group and its contents do not matter.
        const int glast = (W - 1) & ~3;
        auto group = [&](const float* base, int g) {
            g = g < 0 ? 0 : (g > glast ? glast : g);
            return __ldg(reinterpret_cast<const float4*>(base + g));
        };
        const float* ob[4] = {o0, o1, o2, o3};
        int mb = x4 + SIGN * d;                       // first matched column of pixel 0 at this block's first disparity
        float4 lo[4], hi[4];                          // columns [g, g+4) and [g+4, g+8) with g = mb - 4 (left) / mb (right)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            lo[c] = group(ob[c], SIGN < 0 ? mb - 4 : mb);
            hi[c] = group(ob[c], SIGN < 0 ? mb : mb + 4);
        }
        for (int dl = 0; dl < P.d_count; dl += 4, d += 4) {
            float4 nx[4];                             // the group the next block adds, loaded ahead of this block's arithmetic
#pragma unroll
            for (int c = 0; c < 4; ++c) nx[c] = group(ob[c], SIGN < 0 ? mb - 8 : mb + 8);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                if (dl + k < P.d_count) {
                    float m[4][4];
#pragma unroll
                    for (int c = 0; c < 4; ++c)
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            // element of the 8-column window [lo | hi]: left j - k + 4 (1..7), right j + k (0..6)
                            const int e = SIGN < 0 ? j - k + 4 : j + k;
                            m[c][j] = e < 4 ? comp(lo[c], e) : comp(hi[c], e - 4);
                        }
                    emit(dl + k, d + k, m);
                }
            }
            mb += 4 * SIGN;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                if (SIGN < 0) { hi[c] = lo[c]; lo[c] = nx[c]; }
                else { lo[c] = hi[c]; hi[c] = nx[c]; }
            }
        }
        return;
    }
    // unaligned shard: window w[c][j] = other[c][x4 + j + SIGN*d], one new scalar load per plane per disparity
    float w[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int xo = clampx(x4 + j + SIGN * d);
        w[0][j] = __ldg(o0 + xo); w[1][j] = __ldg(o1 + xo); w[2][j] = __ldg(o2 + xo); w[3][j] = __ldg(o3 + xo);
    }
#pragma unroll 4
    for (int dl = 0; dl < P.d_count; ++dl, ++d) {
        emit(dl, d, w);
        // slide the window by one disparity
        if (SIGN < 0) {
            const int xo = clampx(x4 - (d + 1));
#pragma unroll
            for (int c = 0; c < 4; ++c) { w[c][3] = w[c][2]; w[c][2] = w[c][1]; w[c][1] = w[c][0]; }
            w[0][0] = __ldg(o0 + xo); w[1][0] = __ldg(o1 + xo); w[2][0] = __ldg(o2 + xo); w[3][0] = __ldg(o3 + xo);
        } else {
            const int xo = clampx(x4 + 3 + (d + 1));
#pragma unroll
            for (int c = 0; c < 4; ++c) { w[c][0] = w[c][1]; w[c][1] = w[c][2]; w[c][2] = w[c][3]; }
            w[0][3] = __ldg(o0 + xo); w[1][3] = __ldg(o1 + xo); w[2][3] = __ldg(o2 + xo); w[3][3] = __ldg(o3 + xo);
        }
    }
}

// ------------------------------------------------------------------------------------------
// K2 guide precompute (CVF::preprocess, CVF.cpp:44-70) + the d-independent part of the 3x3
// solve of GuidedFilter_cv (CVF.cpp:117-126): the symmetric adjugate of (Sigma + eps I) and
// 1/det.  One fused kernel: fp64 horizontal 8-sums of the 9 planes (I_c, I_c*I_c') per row,
// fp64 running sums down the rows of a segment, then mean/var and the solve terms.
// guide planes (each [H][Wp]): 0-2 I, 3-5 mean_I, 6-11 adj (M00,M01,M02,M11,M12,M22), 12 1/det,
// 13-18 var_I (rr,rg,rb,gg,gb,bb; kept for parity reads).
// ------------------------------------------------------------------------------------------
constexpr int kGuideI = 0, kGuideMean = 3, kGuideAdj = 6, kGuideIdet = 12, kGuideVar = 13, kGuidePlanes = 19;

// d-independent per-pixel terms from the nine box means m[0..8] = mean of I0,I1,I2, I0I0,I0I1,I0I2,I1I1,I1I2,I2I2:
// var_I (CVF.cpp:60-69), symmetric adjugate of (Sigma + eps I) and 1/det (CVF.cpp:108-120).
__device__ __forceinline__ void guide_solve(const float m[9], float v[6], float M[6], float& idet)
{
    v[0] = fsub(m[3], fmul(m[0], m[0]));
    v[1] = fsub(m[4], fmul(m[0], m[1]));
    v[2] = fsub(m[5], fmul(m[0], m[2]));
    v[3] = fsub(m[6], fmul(m[1], m[1]));
    v[4] = fsub(m[7], fmul(m[1], m[2]));
    v[5] = fsub(m[8], fmul(m[2], m[2]));
    const float a11 = fadd(v[0], kGifEps), a12 = v[1], a13 = v[2];
    const float a21 = v[1], a22 = fadd(v[3], kGifEps), a23 = v[4];
    const float a31 = v[2], a32 = v[4], a33 = fadd(v[5], kGifEps);
    // cofactors exactly as written at CVF.cpp:117-146 (the adjugate is symmetric bit-for-bit
    // because each mirrored entry is the same two products in commuted order)
    M[0] = fsub(fmul(a33, a22), fmul(a32, a23));  // M00
    M[1] = fsub(fmul(a31, a23), fmul(a33, a21));  // M01
    M[2] = fsub(fmul(a32, a21), fmul(a31, a22));  // M02
    M[3] = fsub(fmul(a33, a11), fmul(a31, a13));  // M11
    M[4] = fsub(fmul(a31, a12), fmul(a32, a11));  // M12
    M[5] = fsub(fmul(a22, a11), fmul(a21, a12));  // M22
    // DET = a11*(a33*a22-a32*a23) - a21*(a33*a12-a32*a13) + a31*(a23*a12-a22*a13)  (CVF.cpp:117-119)
    const float t1 = fsub(fmul(a33, a12), fmul(a32, a13));
    const float t2 = fsub(fmul(a23, a12), fmul(a22, a13));
    const float det = fadd(fsub(fmul(a11, M[0]), fmul(a21, t1)), fmul(a31, t2));
    idet = __fdiv_rn(1.0f, det);  // CVF.cpp:120
}

// 8-wide window sums from the 4 column sums c[0..3] a lane owns:
// h[j] = columns (4l+j) .. (4l+j+7) = suffix_l[j..3] + total_{l+1} + prefix_{l+2}[0..j-1]   (4 fp64 shuffles)
__device__ __forceinline__ void hsum8(const double c[4], double h[4])
{
    const double P1 = c[0], P2 = c[0] + c[1], P3 = P2 + c[2], Tt = P3 + c[3];
    const double S1 = c[3], S2 = c[2] + c[3], S3 = c[1] + S2;
#if defined(PSM_KNOCKOUT) && (PSM_KNOCKOUT & 1)   // diagnostics only, see psm_cvf_stream.cuh
    const double Tn = Tt, Q1 = P1, Q2 = P2, Q3 = P3;
#else
    const double Tn = __shfl_down_sync(0xffffffffu, Tt, 1);
    const double Q1 = __shfl_down_sync(0xffffffffu, P1, 2);
    const double Q2 = __shfl_down_sync(0xffffffffu, P2, 2);
    const double Q3 = __shfl_down_sync(0xffffffffu, P3, 2);
#endif
    h[0] = Tt + Tn;
    h[1] = (S3 + Tn) + Q1;
    h[2] = (S2 + Tn) + Q2;
    h[3] = (S1 + Tn) + Q3;
}

// K2: warp = strip of 128 input columns (120 output columns) x seg_rows rows of one view;
// lane = 4 columns.  fp64 running column sums of the nine planes (newest row added, oldest row
// removed, both re-read from the I planes whose column halo is mirrored), 8-wide row sums by
// hsum8, then guide_solve per pixel; every plane is written with 128-bit stores.
constexpr int kGuideSegRows = 32;
constexpr int kGuideStripOut = 120;

struct GuideParams {
    float* guide[2];
    int* guide_flags;   // [2]: kGuideNonFinite raised when a mean / adjugate / 1/det value is not finite
    int W, H, Wp, nstrips, nseg, seg_rows;
};

__global__ void __launch_bounds__(128) guide_kernel(const GuideParams P)
{
    const int lane = threadIdx.x & 31;
    int task = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int strip = task % P.nstrips; task /= P.nstrips;
    const int seg = task % P.nseg;
    const int view = task / P.nseg;
    if (view >= 2) return;
    const int W = P.W, H = P.H, Wp = P.Wp;
    const size_t plane = (size_t)H * Wp;
    float* __restrict__ G = P.guide[view];
    const int cin = strip * kGuideStripOut - 4 + 4 * lane;  // input columns; outputs are cin+4 .. cin+7
    const int co = cin + 4;
    const bool in_ok = cin <= W + 4;       // beyond: nothing this lane feeds is ever stored (and the halo ends at W+7)
    const bool out_ok = lane <= 29 && co < W;
    const int y0 = seg * P.seg_rows;
    const int y1 = min(H, y0 + P.seg_rows);

    double V[9][4];
#pragma unroll
    for (int k = 0; k < 9; ++k)
#pragma unroll
        for (int j = 0; j < 4; ++j) V[k][j] = 0.0;

    // (widening I and I*I' with the integer trick of the streaming filter was measured here and is 15 % SLOWER, 119 vs 104 us:
    // this kernel has XU slack and the IMAD.WIDEs land on the FMA pipe next to its multiplies -- plain conversions stay)
    auto feed = [&](int r, const bool add) {
        const size_t ro = (size_t)reflect101(r, H) * Wp + cin;
        float4 a4 = make_float4(0.f, 0.f, 0.f, 0.f), b4 = a4, c4 = a4;
        if (in_ok) {
            a4 = __ldg(reinterpret_cast<const float4*>(G + ro));
            b4 = __ldg(reinterpret_cast<const float4*>(G + plane + ro));
            c4 = __ldg(reinterpret_cast<const float4*>(G + 2 * plane + ro));
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float a = comp(a4, j), b = comp(b4, j), c = comp(c4, j);
            const float t[9] = {a, b, c, fmul(a, a), fmul(a, b), fmul(a, c), fmul(b, b), fmul(b, c), fmul(c, c)};  // CVF.cpp:62
#pragma unroll
            for (int k = 0; k < 9; ++k) V[k][j] = add ? __dadd_rn(V[k][j], (double)t[k]) : __dsub_rn(V[k][j], (double)t[k]);
        }
    };

    for (int r = y0 - kBoxAnchor; r < y0 + kBoxK - kBoxAnchor - 1; ++r) feed(r, true);
    for (int y = y0; y < y1; ++y) {
        feed(y + kBoxK - kBoxAnchor - 1, true);
        float m[9][4];
#pragma unroll
        for (int k = 0; k < 9; ++k) {
            double h[4];
            hsum8(V[k], h);
#pragma unroll
            for (int j = 0; j < 4; ++j) m[k][j] = (float)__dmul_rn(h[j], kMeanPlain);
        }
        feed(y - kBoxAnchor, false);
        float o[16][4];  // planes kGuideMean .. kGuidePlanes-1
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float mm[9] = {m[0][j], m[1][j], m[2][j], m[3][j], m[4][j], m[5][j], m[6][j], m[7][j], m[8][j]};
            float v[6], M[6], idet;
            guide_solve(mm, v, M, idet);
            const bool px_ok = co + j < W;  // columns W .. W4-1 of the last group hold zeros
            o[0][j] = px_ok ? mm[0] : 0.f; o[1][j] = px_ok ? mm[1] : 0.f; o[2][j] = px_ok ? mm[2] : 0.f;
#pragma unroll
            for (int k = 0; k < 6; ++k) { o[3 + k][j] = px_ok ? M[k] : 0.f; o[10 + k][j] = px_ok ? v[k] : 0.f; }
            o[9][j] = px_ok ? idet : 0.f;
        }
        if (out_ok) {
            const size_t oo = (size_t)y * Wp + co;
            unsigned worst = 0;
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                *reinterpret_cast<float4*>(G + (size_t)(kGuideMean + k) * plane + oo) = make_float4(o[k][0], o[k][1], o[k][2], o[k][3]);
                if (k < 10) {
#pragma unroll
                    for (int j = 0; j < 4; ++j) worst = max(worst, __float_as_uint(o[k][j]) & 0x7fffffffu);
                }
            }
            if (worst >= 0x7f800000u) atomicOr(P.guide_flags + view, kGuideNonFinite);
        }
    }
}

// Per-voxel coefficient math shared by every CVF kernel: CVF.cpp:92-95 (cov), :121-146 (a),
// :152-155 (b).  mp/mIp are the four stage-1 box means at this voxel.
struct GuidePix { float mI0, mI1, mI2, M00, M01, M02, M11, M12, M22, idet; };

__device__ __forceinline__ void gif_coeffs(float mp, float mIp0, float mIp1, float mIp2, const GuidePix& g,
                                           float& a0, float& a1, float& a2, float& b)
{
    const float c0 = fsub(mIp0, fmul(g.mI0, mp));
    const float c1 = fsub(mIp1, fmul(g.mI1, mp));
    const float c2 = fsub(mIp2, fmul(g.mI2, mp));
    a0 = fmul(g.idet, fadd(fadd(fmul(c0, g.M00), fmul(c1, g.M01)), fmul(c2, g.M02)));
    a1 = fmul(g.idet, fadd(fadd(fmul(c0, g.M01), fmul(c1, g.M11)), fmul(c2, g.M12)));
    a2 = fmul(g.idet, fadd(fadd(fmul(c0, g.M02), fmul(c1, g.M12)), fmul(c2, g.M22)));
    b = fsub(fsub(fsub(mp, fmul(a0, g.mI0)), fmul(a1, g.mI1)), fmul(a2, g.mI2));
}

// ------------------------------------------------------------------------------------------
// K4 WTA (DispSel.cpp:83-109): per pixel argmin over global d in [1, D), strict <, ties -> lowest d,
// minCost starts at +inf, result 0 when nothing compares below +inf.  One thread = 4 pixels.  wta_scan4 (below) is the
// scan of every selection kernel, wta_key the packed (cost, d) key in which every shard, block and rank exchanges its
// minima.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long wta_key(float cost, int d)
{
    return ((unsigned long long)float_order_key(cost) << 32) | (unsigned)d;
}

// ------------------------------------------------------------------------------------------
// The filtered costs beside each winner (PSM_OPT_COSTS): q(m - 1), q(m), q(m + 1) of the volume selection scanned, at the
// selection map's m, copied bit for bit.  An index outside the problem's range [d_lo, D) gives kCostNaN; a pixel without a
// winner (m = 0) gets (kCostNaN, q(0), q(1)) where d_lo = 0, and kCostNaN for each index below d_lo otherwise.
// ------------------------------------------------------------------------------------------
// Planes of H * W floats (row pitch W), per view.  The result: kCostOut planes holding q(m - 1), q(m), q(m + 1); the
// selection stages write them and nothing else does, so they stay the last selection's until the next one.  A blocked
// context's tracking planes, which its walk rewrites block by block: planes 0..2 hold the running winner's costs, then
// kCostLast the cost at the last slice of the block walked last and, on a shard that does not own the problem's first
// slice d_lo, kCostFirst the cost at its first owned slice (read by the shard below it at their seam).
constexpr int kCostOut = 3, kCostLast = 3, kCostFirst = 4;
constexpr unsigned kCostNaNBits = 0x7fc00000u;   // the canonical quiet NaN of an index outside [0, D)

struct CostPlanes {
    float* base;
    size_t npix;   // H * W
    __host__ __device__ float* plane(int k) const { return base + (size_t)k * npix; }
    __host__ __device__ unsigned* uplane(int k) const { return reinterpret_cast<unsigned*>(plane(k)); }
};

// ------------------------------------------------------------------------------------------
// The runner-up away from the winner (PSM_OPT_RUNNER_UP).  The candidates are the arg-min's: d in [1, D) whose cost
// compares below +inf, in the order of wta_key (the cost, -0 equal to +0, then the lowest d).  The runner-up r of a pixel
// with map m is the first candidate with |d - m| >= 2, 0 when there is none; the result planes hold (float)r and q(r)
// bit for bit (kCostNaN where r = 0).
// Every path keeps, per pixel, the list of its four lowest candidates, lowest first, empty entries (+inf, 0) behind them.
// Four are enough: at most three entries lie in {m - 1, m, m + 1}, so the first entry outside them is the lowest
// candidate outside them.  The list is mergeable: the four lowest of a union of disjoint slice ranges are the four
// lowest of the ranges' lists.  So a blocked walk folds each block's list into a running one, and the shards of a
// multi-device context each pick from their own list and the first shard takes the lowest key of the picks.
// ------------------------------------------------------------------------------------------
// Planes of the same shape.  The result: kRunnerUpOut planes, r as a float and q(r) bit for bit (kCostNaN where r = 0);
// only the selection stages write them.  A blocked context's running list (kListPlanes, beside the head's key in its
// running keys): planes kListCost + e hold the cost bits of entries e = 0..3, planes kListD + e - 1 the d of entries
// e = 1..3.  A multi-device context's slots on the first shard (RunnerUpSlots): per shard and pixel, the candidate's key
// and its cost bits.
constexpr int kRunnerUpOut = 2, kListLen = 4, kListCost = 0, kListD = 4, kListPlanes = 7;

struct RunnerUpSlots {
    unsigned char* base;   // [nslots][npix] keys, then [nslots][npix] cost bits
    size_t npix;
    int nslots;
    static size_t bytes(size_t npix, int nslots) { return (size_t)nslots * npix * (sizeof(unsigned long long) + sizeof(float)); }
    __host__ __device__ unsigned long long* key(int k) const { return reinterpret_cast<unsigned long long*>(base) + (size_t)k * npix; }
    __host__ __device__ float* cost(int k) const
    {
        return reinterpret_cast<float*>(base + (size_t)nslots * npix * sizeof(unsigned long long)) + (size_t)k * npix;
    }
};

// c at slice d into entries 1.. of a sorted list whose head (c0, d0) c replaces where `head`; every entry comes from a
// slice below d or costs less: the strict < puts c behind every entry of equal cost, as the arg-min's lowest-d rule does,
// and a +inf or NaN cost never enters
__device__ __forceinline__ void list_insert_tail(float (&lc)[kListLen], int (&ld)[kListLen], float c, int d, bool head, float c0,
                                                 int d0)
{
    const bool b1 = c < lc[1], b2 = c < lc[2], b3 = c < lc[3];
    lc[3] = b2 ? lc[2] : (b3 ? c : lc[3]);  ld[3] = b2 ? ld[2] : (b3 ? d : ld[3]);
    lc[2] = b1 ? lc[1] : (b2 ? c : lc[2]);  ld[2] = b1 ? ld[1] : (b2 ? d : ld[2]);
    lc[1] = head ? c0 : (b1 ? c : lc[1]);   ld[1] = head ? d0 : (b1 ? d : ld[1]);
}

// c at slice d into a whole sorted list
__device__ __forceinline__ void list_insert(float (&lc)[kListLen], int (&ld)[kListLen], float c, int d)
{
    const bool b0 = c < lc[0];
    list_insert_tail(lc, ld, c, d, b0, lc[0], ld[0]);
    lc[0] = b0 ? c : lc[0];                 ld[0] = b0 ? d : ld[0];
}

// pixel i's running list in planes L, whose head's d is in its running key
__device__ __forceinline__ void list_load(const CostPlanes& L, unsigned long long key, size_t i, float (&lc)[kListLen],
                                          int (&ld)[kListLen])
{
    ld[0] = (int)(unsigned)key;
#pragma unroll
    for (int e = 0; e < kListLen; ++e) {
        lc[e] = L.plane(kListCost + e)[i];
        if (e > 0) ld[e] = (int)L.uplane(kListD + e - 1)[i];
    }
}

// the list back into planes L (the head's key is the caller's to write)
__device__ __forceinline__ void list_store(const CostPlanes& L, size_t i, const float (&lc)[kListLen], const int (&ld)[kListLen])
{
#pragma unroll
    for (int e = 0; e < kListLen; ++e) {
        L.plane(kListCost + e)[i] = lc[e];
        if (e > 0) L.uplane(kListD + e - 1)[i] = (unsigned)ld[e];
    }
}

// the runner-up of a pixel with map m from its list: (r, q(r)), or (0, kCostNaN)
__device__ __forceinline__ void runner_up_pick(const float (&lc)[kListLen], const int (&ld)[kListLen], int m, int& r, float& q)
{
    r = 0;
    q = __uint_as_float(kCostNaNBits);
#pragma unroll
    for (int e = kListLen - 1; e >= 0; --e)
        if (ld[e] != 0 && abs(ld[e] - m) >= 2) { r = ld[e]; q = lc[e]; }
}

// ------------------------------------------------------------------------------------------
// The selection scan.  Per pixel j of its four, what wta_scan4 tracks beside the arg-min (mc, md):
//   kCosts: the costs beside the running minimum.  On a new minimum at d, lo = the previous slice's cost (`prev`, seeded
//           with the cost before the range) and hi waits for slice d + 1.  Slice 0 is read but is never a candidate:
//           the no-winner state (md = 0) takes ce = q(0) and, from the md == d - 1 rule, hi = q(1).  `first` and
//           `prev` end as the range's first and last costs.
//   kList:  the list of the four lowest candidates.  Its head is the arg-min itself, so during the scan only entries 1..
//           are kept here; wta_scan4 copies (mc, md) into entry 0 at its end.
// ------------------------------------------------------------------------------------------
template <bool kCosts, bool kList>
struct ScanTrack {
    float lo[4], ce[4], hi[4], prev[4], first[4];
    float lc[4][kListLen];
    int ld[4][kListLen];

    __device__ __forceinline__ ScanTrack()
    {
        const float nan = __uint_as_float(kCostNaNBits);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if constexpr (kCosts) lo[j] = ce[j] = hi[j] = prev[j] = nan;
            if constexpr (kList)
#pragma unroll
                for (int e = 0; e < kListLen; ++e) { lc[j][e] = INFINITY; ld[j][e] = 0; }
        }
    }

    // pixel j's cost c at slice d, the dl-th of the range, before the arg-min (mc, md) sees it
    __device__ __forceinline__ void step(int j, float c, int d, int dl, bool cand, float mc, int md)
    {
        const bool take = cand && c < mc;   // the arg-min's test: c becomes the new minimum
        if constexpr (kCosts) {
            if (md == d - 1) hi[j] = c;
            if (!cand) ce[j] = c;
            else if (take) { lo[j] = prev[j]; ce[j] = c; hi[j] = __uint_as_float(kCostNaNBits); }
            prev[j] = c;
            if (dl == 0) first[j] = c;
        }
        if constexpr (kList)
            if (cand) list_insert_tail(lc[j], ld[j], c, d, take, mc, md);
    }
};

// The scan of slices [d_begin, d_begin + d_count), slice dl at p + dl * plane, into the caller's mc / md (set to +inf / 0;
// returning them in a struct instead changes the kernels' SASS) and t; an inactive lane scans nothing.  Global d = 0 is
// never a candidate (DispSel.cpp:96); only the costs read its slice.  Each pixel's tracker step sees the slice before the
// arg-min, whose strict < keeps the lowest d, takes it.  The four pixels stay four statements on the float4's components:
// a loop over an array of them, or a helper taking mc / md by reference, changes the SASS of the kernels without a
// tracker.
template <bool kCosts, bool kList>
__device__ __forceinline__ void wta_scan4(const float* p, size_t plane, int d_begin, int d_count, bool active, float (&mc)[4],
                                          int (&md)[4], ScanTrack<kCosts, kList>& t)
{
    int dl = (!kCosts && d_begin == 0) ? 1 : 0;
#pragma unroll 8
    for (; active && dl < d_count; ++dl) {
        const float4 c = __ldg(reinterpret_cast<const float4*>(p + (size_t)dl * plane));
        const int d = d_begin + dl;
        const bool cand = !kCosts || d != 0;
        t.step(0, c.x, d, dl, cand, mc[0], md[0]); if (cand && c.x < mc[0]) { mc[0] = c.x; md[0] = d; }
        t.step(1, c.y, d, dl, cand, mc[1], md[1]); if (cand && c.y < mc[1]) { mc[1] = c.y; md[1] = d; }
        t.step(2, c.z, d, dl, cand, mc[2], md[2]); if (cand && c.z < mc[2]) { mc[2] = c.z; md[2] = d; }
        t.step(3, c.w, d, dl, cand, mc[3], md[3]); if (cand && c.w < mc[3]) { mc[3] = c.w; md[3] = d; }
    }
    if constexpr (kList)
#pragma unroll
        for (int j = 0; j < 4; ++j) { t.lc[j][0] = mc[j]; t.ld[j][0] = md[j]; }
}

// The selection of one volume: the map (T = uint8_t or uint16_t) and/or the keys used by the disparity-sharded
// reduction; kList (an unblocked single-device context with the runner-up) also the runner-up into its result planes
// ru, in the same read
template <typename T, bool kList>
__global__ void __launch_bounds__(256) wta_kernel(const float* __restrict__ vol, int W, int H, int Wp, int d_begin, int d_count,
                                                  T* __restrict__ dis /* [H][W] or null */,
                                                  unsigned long long* __restrict__ keys /* [H][W] or null */, const CostPlanes ru)
{
    const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const int y = blockIdx.y;
    if (x4 >= W) return;
    const size_t plane = (size_t)H * Wp;
    const float* p = vol + (size_t)y * Wp + x4;
    float mc[4] = {INFINITY, INFINITY, INFINITY, INFINITY};
    int md[4] = {0, 0, 0, 0};
    ScanTrack<false, kList> t;
    wta_scan4(p, plane, d_begin, d_count, true, mc, md, t);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int x = x4 + j;
        if (x < W) {
            const size_t i = (size_t)y * W + x;
            if (dis) dis[i] = (T)md[j];
            if (keys) keys[i] = wta_key(mc[j], md[j]);
            if constexpr (kList) {
                int r;
                float q;
                runner_up_pick(t.lc[j], t.ld[j], md[j], r, q);
                ru.plane(0)[i] = (float)r;
                ru.plane(1)[i] = q;
            }
        }
    }
}

// WTA of one block of slices of a blocked context (psm_create_blocked), both views in one launch (blockIdx.z = view):
// wta_scan4 over the block's d_count slices starting at global d_begin, then its wta_key is stored (first block) or
// folded into the running key by min.  The min over keys of consecutive blocks is the
// selection over their union: the strict <, the lowest-d tie-break and +inf / NaN costs behave as in one scan.
// kCosts: the costs in track[view] (the tracking planes).  Planes 0..2 hold the running winner's (lo, ce, hi).  A block
// whose key is below the running key replaces them; its lo at its first slice is the previous block's last cost
// (kCostLast).  A running winner on the previous block's last slice takes hi from this block's first slice.  The first
// block starts from the no-winner state and, if write_first, records kCostFirst.
// kList: the running list in list[view] (the head's key stays in the running keys): the block's list folds into it,
// entry by entry, and only a list that changes is written back.
struct FoldParams {
    const float* vol[2];             // the block's filtered volumes [d_count][H][Wp]
    unsigned long long* keys[2];     // running keys [H][W]
    int W, H, Wp, d_begin, d_count, first;
    CostPlanes track[2];             // kCosts
    int write_first;                 // kCosts
    CostPlanes list[2];              // kList
};

template <bool kCosts, bool kList>
__global__ void __launch_bounds__(256) wta_fold_kernel(const FoldParams P)
{
    const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const int y = blockIdx.y, view = blockIdx.z;
    if (x4 >= P.W) return;
    const size_t plane = (size_t)P.H * P.Wp;
    const size_t row = (size_t)y * P.W;
    // views selected, not indexed: a parameter array indexed by a run-time value is copied to the stack
    const float* p = (view ? P.vol[1] : P.vol[0]) + (size_t)y * P.Wp + x4;
    const CostPlanes tr = view ? P.track[1] : P.track[0];
    float mc[4] = {INFINITY, INFINITY, INFINITY, INFINITY};
    int md[4] = {0, 0, 0, 0};
    ScanTrack<kCosts, kList> t;
    if constexpr (kCosts)
        if (!P.first)
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (x4 + j < P.W) t.prev[j] = tr.plane(kCostLast)[row + x4 + j];
    wta_scan4(p, plane, P.d_begin, P.d_count, true, mc, md, t);
    unsigned long long* k = (view ? P.keys[1] : P.keys[0]) + row;
    const CostPlanes L = view ? P.list[1] : P.list[0];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int x = x4 + j;
        if (x >= P.W) continue;
        const size_t i = row + x;
        unsigned long long v = wta_key(mc[j], md[j]);
        if constexpr (!kCosts && !kList) {
            if (!P.first) {
                const unsigned long long old = k[x];
                v = old < v ? old : v;
            }
            k[x] = v;
            continue;
        }
        const unsigned long long old = P.first ? 0ull : k[x];
        if constexpr (kCosts) {
            tr.plane(kCostLast)[i] = t.prev[j];
            bool win = true;
            if (P.first) {
                if (P.write_first) tr.plane(kCostFirst)[i] = t.first[j];
            } else {
                win = v < old;
                if (!win && (int)(unsigned)old == P.d_begin - 1) tr.plane(2)[i] = t.first[j];
            }
            if (win) {
                if constexpr (!kList) k[x] = v;   // with the list, the merged head's key is written below
                tr.plane(0)[i] = t.lo[j]; tr.plane(1)[i] = t.ce[j]; tr.plane(2)[i] = t.hi[j];
            }
        }
        if constexpr (kList) {
            float rc[kListLen];
            int rd[kListLen];
            if (P.first) {
#pragma unroll
                for (int e = 0; e < kListLen; ++e) { rc[e] = t.lc[j][e]; rd[e] = t.ld[j][e]; }
            } else {
                if (!(t.lc[j][0] < L.plane(kListCost + 3)[i])) continue;   // no entry of the block enters the running list
                list_load(L, old, i, rc, rd);
#pragma unroll
                for (int e = 0; e < kListLen; ++e) list_insert(rc, rd, t.lc[j][e], t.ld[j][e]);
            }
            k[x] = wta_key(rc[0], rd[0]);
            list_store(L, i, rc, rd);
        }
    }
}

// The costs of the entries a context owns, from the complete selection map (T) into dst, which may be a peer's planes.
// Entry k of pixel i is q(d), d = m + k - 1.  Its one writer: the owner of slice d, [d_begin, d_begin + d_count), for d
// in the problem's range [d_lo, D), and otherwise (kCostNaN) the owner of m, or of d_lo where m lies below the range (the
// no-winner map 0 of a range starting above 0).  kTracked = false reads q(d) from the resident volume (an unblocked
// context); kTracked = true from the tracking planes of a blocked one: planes 0..2 for its own winners, and at its seams
// kCostFirst (m just below its range) or kCostLast (m just above).
struct CostWriteParams {
    const void* map;      // [H][W] of T
    const float* vol;     // kTracked = false: the filtered volume of slices [d_begin, d_begin + d_count), [d][H][Wp]
    CostPlanes src;       // kTracked = true: the tracking planes
    CostPlanes dst;
    int W, H, Wp, D, d_lo, d_begin, d_count;
};

template <typename T, bool kTracked>
__global__ void __launch_bounds__(256) cost_write_kernel(const CostWriteParams P)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= P.W) return;
    const size_t i = (size_t)y * P.W + x;
    const int m = static_cast<const T*>(P.map)[i];
    const int mo = m < P.d_lo ? P.d_lo : m;   // the slice whose owner holds m's state: its planes 0..2 on a blocked one
    const auto owned = [&](int d) { return d >= P.d_begin && d < P.d_begin + P.d_count; };
#pragma unroll
    for (int k = 0; k < kCostOut; ++k) {
        const int d = m + k - 1;
        float q;
        if (d < P.d_lo || d >= P.D) {
            if (!owned(mo)) continue;
            q = __uint_as_float(kCostNaNBits);
        } else if (!owned(d)) {
            continue;
        } else if (!kTracked) {
            q = P.vol[(size_t)(d - P.d_begin) * P.H * P.Wp + (size_t)y * P.Wp + x];
        } else {
            q = P.src.plane(owned(mo) ? k : (k == 2 ? kCostFirst : kCostLast))[i];
        }
        P.dst.plane(k)[i] = q;
    }
}

// The runner-up of the slices a context owns, from the complete selection map (T): from a list scan of its resident
// volume (kTracked = false: an unblocked shard) or from its running list (kTracked = true: a blocked context).  Into the
// result planes, or, where slots.base is set (a shard of a multi-device context), into slot `slot` of the first shard's
// slots as (key, cost bits), wta_key(+inf, 0) and kCostNaN where it has none.
struct RunnerUpWriteParams {
    const void* map;                    // [H][W] of T
    const float* vol;                   // kTracked = false: the filtered volume of slices [d_begin, d_begin + d_count)
    const unsigned long long* keys;     // kTracked = true: the running keys (the lists' heads) ...
    CostPlanes list;                    // ... and the running lists
    CostPlanes dst;
    RunnerUpSlots slots;
    int slot, W, H, Wp, d_begin, d_count;
};

template <typename T, bool kTracked>
__global__ void __launch_bounds__(256) runner_up_write_kernel(const RunnerUpWriteParams P)
{
    const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const int y = blockIdx.y;
    if (x4 >= P.W) return;
    const size_t row = (size_t)y * P.W;
    ScanTrack<false, true> t;
    if constexpr (!kTracked) {
        float mc[4] = {INFINITY, INFINITY, INFINITY, INFINITY};
        int md[4] = {0, 0, 0, 0};
        wta_scan4(P.vol + (size_t)y * P.Wp + x4, (size_t)P.H * P.Wp, P.d_begin, P.d_count, true, mc, md, t);
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (x4 + j < P.W) list_load(P.list, P.keys[row + x4 + j], row + x4 + j, t.lc[j], t.ld[j]);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int x = x4 + j;
        if (x >= P.W) continue;
        const size_t i = row + x;
        int r;
        float q;
        runner_up_pick(t.lc[j], t.ld[j], static_cast<const T*>(P.map)[i], r, q);
        if (P.slots.base) {
            P.slots.key(P.slot)[i] = r ? wta_key(q, r) : wta_key(INFINITY, 0);
            P.slots.cost(P.slot)[i] = q;
        } else {
            P.dst.plane(0)[i] = (float)r;
            P.dst.plane(1)[i] = q;
        }
    }
}

// The first shard's runner-up: the lowest key of the shards' picks (the first slot on equal keys, which only empty
// picks share) and its cost bits
__global__ void __launch_bounds__(256) runner_up_reduce_kernel(const RunnerUpSlots S, const CostPlanes dst)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= S.npix) return;
    unsigned long long k = S.key(0)[i];
    int best = 0;
    for (int s = 1; s < S.nslots; ++s) {
        const unsigned long long v = S.key(s)[i];
        if (v < k) { k = v; best = s; }
    }
    dst.plane(0)[i] = (float)(unsigned)k;
    dst.plane(1)[i] = S.cost(best)[i];
}

// Sharded WTA fused with its exchange (reduce-scatter + all-gather of a min-reduction, hand-rolled
// over NVLink peer memory).  Pixels are partitioned into `nranks` chunks; rank r is the reducer of
// chunk r.
//   wta_scatter_kernel : wta_scan4 over the filtered volume, then the wta_key minimum of every pixel
//                        is stored into its reducer's exchange block, slot [this rank][pixel-in-chunk]
//                        (peer device memory, plain st.global over NVLink) -- compute + scatter in one kernel;
//                        its last CTA then raises this rank's ARRIVE flag in every peer's block;
//   chunk_reduce_kernel: waits for the ARRIVE flags of all ranks (acquire loads on its own block), takes
//                        the min over the nranks slots of its chunk, stores the winning disparity (u8 or u16)
//                        into EVERY rank's result map -- reduce + gather in one kernel -- and its last CTA
//                        raises this rank's DONE flag in every peer's block;
//   keys_scatter_kernel: the scatter of a blocked shard of a multi-device context, whose minima are already folded
//                        into its running keys; same staged store (p2p_store_row) and ARRIVE flag as wta_scatter_kernel;
//   p2p_wait_done_kernel: spins until all ranks' DONE flags carry this frame's sequence number; after it the local result
//                        maps are complete.  Launched only in front of a consumer of the maps (D2H fetch, post-filter);
//                        the NEXT frame's scatter kernel does the same wait itself before it overwrites the key slots.
// Flags are monotonically increasing frame sequence numbers (never reset), written with release and read
// with acquire semantics at system scope, so the exchange needs NO library collective or host barrier:
// a waiting kernel only ever waits for kernels of other GPUs that do not wait for it.
constexpr int kMaxRanks = 8;
constexpr int kScatterRows = 4;   // image rows per CTA of wta_scatter_kernel

struct P2pPeers {
    unsigned long long* keys[kMaxRanks];  // per rank: exchange block of this view  [nranks][chunk]
    unsigned char* maps[kMaxRanks];       // per rank: result map of this view       [H*W] of the map type
    unsigned* flags[kMaxRanks];           // per rank: flag words of this view: arrive[kMaxRanks], done[kMaxRanks]
    unsigned* counter;                    // device-local CTA counter of the launching rank (zero between launches)
    int nranks, rank;
    unsigned chunk;                       // pixels per chunk (last chunk may be partly unused)
    unsigned seq;                         // frame sequence number (>= 1)
};

__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) { asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p)
{
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// called by every thread of the CTA after its peer stores: the LAST CTA of the launch publishes `seq` in slot
// flag_base[rank] of every peer's flag words
__device__ __forceinline__ void p2p_publish(const P2pPeers& peers, int flag_offset)
{
    __syncthreads();
    if (threadIdx.x == 0 && threadIdx.y == 0) {
        __threadfence_system();                       // this CTA's peer stores are visible system-wide ...
        const unsigned total = gridDim.x * gridDim.y;
        const unsigned prev = atomicAdd(peers.counter, 1u);
        if (prev == total - 1) {                      // ... before the last CTA (which observed every increment) raises the flags
            __threadfence();
            *peers.counter = 0;
            for (int r = 0; r < peers.nranks; ++r) st_release_sys(peers.flags[r] + flag_offset + peers.rank, peers.seq);
        }
    }
}

// called by every thread of a scatter kernel before its peer stores: the key slots it writes were read by the reducers
// of the PREVIOUS frame, so wait for their DONE flags
__device__ __forceinline__ void p2p_wait_reducers(const P2pPeers& peers)
{
    if (peers.seq > 1) {
        if (threadIdx.x < (unsigned)peers.nranks) {
            const unsigned* f = peers.flags[peers.rank] + kMaxRanks + threadIdx.x;
            while ((int)(ld_acquire_sys(f) - (peers.seq - 1)) < 0) __nanosleep(64);
        }
        __syncthreads();
    }
}

// The scatter kernels' store of one row: lane `lane` holds the keys key(0..3) of columns x4 .. x4 + 3, x4 = xw + 4 * lane,
// and every pixel's key goes to slot [this rank][pixel-in-chunk] of its reducer's exchange block (peer or own memory).
// The warp's 128 keys are staged in `stage` (128 shared slots of the warp) and sent out lane-contiguously: every store
// instruction then writes 32 consecutive keys (256 contiguous bytes, whole 32-byte sectors) to one peer, instead of
// 32 lanes x 8 bytes at a 32-byte stride (partial sectors over NVLink).  Every lane of the warp takes part, also those
// whose columns lie past the image.
template <class Key>
__device__ __forceinline__ void p2p_store_row(unsigned long long* stage, const P2pPeers& peers, int W, int y, int xw, int lane,
                                              Key key)
{
    __syncwarp();   // the previous row's staged keys have been sent
#pragma unroll
    for (int j = 0; j < 4; ++j)
        stage[4 * lane + j] = key(j);
    __syncwarp();
#pragma unroll
    for (int s4 = 0; s4 < 4; ++s4) {
        const int idx = 32 * s4 + lane;
        const int x = xw + idx;
        if (x < W) {
            const unsigned pix = (unsigned)y * (unsigned)W + (unsigned)x;
            const unsigned owner = pix / peers.chunk;
            peers.keys[owner][(size_t)peers.rank * peers.chunk + (pix - owner * peers.chunk)] = stage[idx];
        }
    }
}

__global__ void __launch_bounds__(256) wta_scatter_kernel(const float* __restrict__ vol, int W, int H, int Wp, int d_begin, int d_count,
                                                          P2pPeers peers)
{
    // p2p_wait_reducers, spelled out: the call schedules this kernel's instructions differently
    if (peers.seq > 1) {
        if (threadIdx.x < (unsigned)peers.nranks) {
            const unsigned* f = peers.flags[peers.rank] + kMaxRanks + threadIdx.x;
            while ((int)(ld_acquire_sys(f) - (peers.seq - 1)) < 0) __nanosleep(64);
        }
        __syncthreads();
    }
    const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const bool active = x4 < W;  // inactive lanes still take part in the staged store below
    const size_t plane = (size_t)H * Wp;
    __shared__ unsigned long long stage[8][128];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // a CTA handles kScatterRows consecutive rows: four times fewer CTAs have to fence and count in p2p_publish
    for (int y = blockIdx.y * kScatterRows; y < min(H, (int)(blockIdx.y + 1) * kScatterRows); ++y) {
        const float* p = vol + (size_t)y * Wp + (active ? x4 : 0);
        float mc[4] = {INFINITY, INFINITY, INFINITY, INFINITY};
        int md[4] = {0, 0, 0, 0};
        ScanTrack<false, false> none;
        wta_scan4(p, plane, d_begin, d_count, active, mc, md, none);
        p2p_store_row(stage[warp], peers, W, y, x4 - 4 * lane, lane,
                      [&](int j) { return wta_key(mc[j], md[j]); });
    }
    if (peers.seq) p2p_publish(peers, 0);   // ARRIVE
}

// The scatter of a blocked shard of a multi-device context (psm_create_multi): its selection is already folded into the
// running keys (wta_fold_kernel), so each pixel's running key goes to its reducer's slot, with wta_scatter_kernel's
// grid, staged store and ARRIVE flag.
__global__ void __launch_bounds__(256) keys_scatter_kernel(const unsigned long long* __restrict__ keys /* [H][W] */, int W, int H,
                                                           P2pPeers peers)
{
    p2p_wait_reducers(peers);
    const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    __shared__ unsigned long long stage[8][128];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int y = blockIdx.y * kScatterRows; y < min(H, (int)(blockIdx.y + 1) * kScatterRows); ++y) {
        const unsigned long long* k = keys + (size_t)y * W + x4;
        p2p_store_row(stage[warp], peers, W, y, x4 - 4 * lane, lane,
                      [&](int j) { return x4 + j < W ? __ldg(k + j) : 0ull; });
    }
    if (peers.seq) p2p_publish(peers, 0);   // ARRIVE
}

template <typename T>
__global__ void __launch_bounds__(256) chunk_reduce_kernel(P2pPeers peers, unsigned npix)
{
    if (peers.seq) {   // wait until every rank's minima for this frame have landed in this rank's block
        if (threadIdx.x < (unsigned)peers.nranks) {
            const unsigned* f = peers.flags[peers.rank] + threadIdx.x;
            while ((int)(ld_acquire_sys(f) - peers.seq) < 0) __nanosleep(64);
        }
        __syncthreads();
    }
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;   // pixel inside this rank's chunk
    const unsigned pix = (unsigned)peers.rank * peers.chunk + i;
    if (i < peers.chunk && pix < npix) {
        const unsigned long long* mine = peers.keys[peers.rank];
        unsigned long long k = __ldcg(mine + i);   // L2: the slots were written by peer GPUs
        for (int r = 1; r < peers.nranks; ++r) {
            const unsigned long long v = __ldcg(mine + (size_t)r * peers.chunk + i);
            k = v < k ? v : k;
        }
        const T d = (T)k;
        for (int r = 0; r < peers.nranks; ++r) reinterpret_cast<T*>(peers.maps[r])[pix] = d;  // every rank receives the final map
    }
    if (peers.seq) p2p_publish(peers, kMaxRanks);   // DONE
}

__global__ void p2p_wait_done_kernel(const unsigned* flags /* this rank's flag words: [2 views][2 * kMaxRanks] */, int nranks, unsigned seq)
{
    if (threadIdx.x < 2u * (unsigned)nranks) {
        const unsigned view = threadIdx.x / nranks, r = threadIdx.x - view * nranks;
        const unsigned* f = flags + view * 2 * kMaxRanks + kMaxRanks + r;
        while ((int)(ld_acquire_sys(f) - seq) < 0) __nanosleep(64);
    }
}

// Final step of the sharded WTA: min over ranks of the packed keys, low 8 or 16 bits -> the map.
template <typename T>
__global__ void keys_reduce_kernel(const unsigned long long* __restrict__ gathered, int nranks, size_t npix,
                                   T* __restrict__ dis)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix) return;
    unsigned long long k = gathered[i];
    for (int r = 1; r < nranks; ++r) {
        const unsigned long long v = gathered[(size_t)r * npix + i];
        k = v < k ? v : k;
    }
    dis[i] = (T)k;
}

}  // namespace psm
