/*
 * stereo_oracle.h -- CPU ORACLE for the STEREO_GIF hot path (CVC -> CVF -> WTA).
 *
 * THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it.  The product
 * (primestereomatch_b200/) never links, imports or calls anything in oracle/.
 *
 * It is a plain-C restatement of the reference's pthreads CPU path
 * (/root/reference: src/CVC.cpp, src/CVF.cpp, src/DispSel.cpp, driven the way
 * src/DispEst.cpp:222-270 drives CVC).  The reference itself cannot be compiled
 * in this image (include/ComFunc.h:33-38 needs <CL/cl.h> and <opencv2/opencv.hpp>,
 * neither is installed), so there is no oracle/_ref.  The OpenCV primitives the
 * reference calls (cvtColor, Sobel, boxFilter, multiply, split) are un-vendored
 * third-party code; they are restated here from OpenCV's published algorithm and
 * PINNED against python cv2 4.13.0 by tests/golden/make_golden.py + tests/test_oracle.py
 * (box filter, Sobel, multiply: bit-exact; RGB2GRAY: bit-exact vs this cv2 build).
 *
 * The reference fixes the guided filter's window and epsilon (GIF_R_WIN, GIF_EPS) and the matching cost's weight
 * (ALPHA_32F, with the truncation by TAU_1_32F / TAU_2_32F commented out, CVC.cpp:24-25, 36-37) at compile time; the
 * product takes them per context (psm_set_guided_filter, psm_set_matching_cost).  This is the one restatement of those
 * stages: every function takes them as arguments, and the ORC_* constants below are the reference's values.
 *
 * Layouts: images are interleaved 3-channel float (BGR order as cv::imread gives,
 * reference StereoMatch.cpp:557) with an element step; volumes are [d][y][x] float,
 * contiguous; disparity maps are u8 [y][x] (u8 or u16 for orc_wta and orc_wmf, chosen by map_bytes).
 */
#ifndef STEREO_ORACLE_H
#define STEREO_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ORC_GIF_R_WIN 8          /* reference include/ComFunc.h:49 */
#define ORC_GIF_EPS 0.0001f      /* reference include/ComFunc.h:50 */
#define ORC_ALPHA 0.9f           /* reference include/CVC.h:22 ALPHA_32F; no truncation: both thresholds +inf */
#define ORC_MAX_CPU_THREADS 8    /* reference include/ComFunc.h:52 */

/* StereoMatch.cpp:193-197: convertTo(CV_32F, 1/255.0f) */
void orc_u8_to_f32(const uint8_t* src, float* dst, size_t n);

/* CVC.cpp:43  cvtColor(Img, GrdX, CV_RGB2GRAY) on a 3-channel f32 image.
 * gray_mode 0: cv2-4.13(+IPP/AVX2 dispatch) rounding  fma(c2,.114f, fma(c0,.299f, c1*.587f))
 * gray_mode 1: plain left-to-right  (c0*.299f + c1*.587f) + c2*.114f  (non-FMA OpenCV builds) */
void orc_rgb2gray(const float* img3, int W, int H, float* gray, int gray_mode);

/* CVC.cpp:44  Sobel(GrdX, GrdX, CV_32F, 1, 0, 1): G[x+1]-G[x-1], BORDER_REFLECT_101 */
void orc_sobel_x(const float* gray, int W, int H, float* grdx);

/* CVC.cpp:41-46 */
void orc_cvc_preprocess(const float* img3, int W, int H, float* grdx, int gray_mode);

/* CVC.cpp:122-149 (== buildCV_left_thread :48-83): one slice of the left volume, with the reference's signature and so
 * at its constants (ORC_ALPHA, no truncation); orc_cost_const builds the same slices at any setting */
void orc_buildcv_left(const float* lImg, const float* rImg, const float* lGrd, const float* rGrd,
                      int W, int H, int d, float* cost);
/* CVC.cpp:151-179 (== buildCV_right_thread :85-120); called with swapped images
 * exactly as DispEst.cpp:217,260 do */
void orc_buildcv_right(const float* lImg, const float* rImg, const float* lGrd, const float* rGrd,
                       int W, int H, int d, float* cost);

/* The two K x K boxes: normalised, anchor K/2, BORDER_REFLECT_101 with any overshoot, fp64 sums, * 1.0/(K*K) in
 * double, one rounding to float.  src may equal dst for orc_box.
 *
 * orc_box is cv::boxFilter(src, dst, -1, Size(K,K)) as used at CVF.cpp:50,63,82,88,158,160, in OpenCV's own order of
 * operations (RowSum<float,double>: direct sums left to right for K <= 5, one running sum per row above;
 * ColumnSum<double,float>: one running sum per column; K == 1 copies), so it equals cv2 even where the fp64 sums are
 * not exact.
 *
 * orc_box_k is the Fast Guided Filter's box, DEFINED as the direct order: per pixel, from 0.0, the K reflected taps of a
 * row left to right, then the K row sums top to bottom.  cv::blur is orc_box, so the two agree exactly when every fp64
 * sum either order forms is exact.  That holds when all values are integer multiples of 2^q and below 2^Q in magnitude
 * with Q - q + ceil(log2(K*K)) <= 53: every partial sum is then a multiple of 2^q of magnitude at most 2^(q+53).  For
 * normal floats (a float in [2^e, 2^(e+1)) is a multiple of 2^(e-23)) this allows the exponents of the nonzero values
 * to span 29 - ceil(log2(K*K)) binary orders of magnitude: 20 at K = 17, 16 at K = 65.  Beyond that the direct order is
 * this project's definition, not cv::blur's. */
void orc_box(const float* src, int W, int H, int K, float* dst);
void orc_box_k(const float* src, int W, int H, int K, float* dst);

/* CVF.cpp:44-70 with a window x window box.  Planes are H*W each: rgb[3], mean[3], var[6] (contiguous, plane-major) */
void orc_cvf_preprocess(const float* img3, int W, int H, int window, float* rgb, float* mean, float* var);

/* CVF.cpp:72-165 GuidedFilter_cv on one slice, in place (CVF.cpp:38), window x window boxes, eps added in float to the
 * three diagonal terms of the covariance.
 * a_out (3 planes) / b_out (1 plane) may be NULL; when given they receive the
 * coefficient planes (a: CVF.cpp:131-146, b: mean_p after CVF.cpp:152-155). */
void orc_guided_filter(const float* rgb, const float* mean, const float* var, int W, int H, int window, float eps,
                       float* p_inout, float* a_out, float* b_out);

/* DispSel.cpp:83-109: the arg-min over d in [1, D) (strict <, lowest d on ties, 0 when nothing is below +inf) into a
 * u8 map (map_bytes 1, the reference's uchar store: the low byte) or a u16 map (map_bytes 2) */
void orc_wta(const float* vol, int W, int H, int D, void* disp, int map_bytes);

/* DispEst.cpp:222-270 CostConst_CPU: preprocess both, then left volume in batches of
 * `threads` pthreads (one per d), then right volume likewise.  The volumes hold the d_count slices of the disparities
 * [d_begin, d_begin + d_count) (a disparity of W or more leaves no pixel with a match).  lGrd/rGrd (H*W) are outputs.
 * The cost of a pixel is alpha * min(colour difference, tau_color) + (1 - alpha) * min(gradient difference, tau_grad)
 * in float, 1 - alpha in float too, with `if (x > tau) x = tau` as the min: a NaN difference stays NaN, tau = +inf
 * truncates nothing.  Where the other view has no pixel the differences are taken against BC_32F = 1.0 in double and
 * rounded once. */
int orc_cost_const(const float* lImg, const float* rImg, int W, int H, int d_begin, int d_count, int threads,
                   int gray_mode, float alpha, float tau_color, float tau_grad,
                   float* lGrd, float* rGrd, float* lVol, float* rVol);

/* The CostFilter_CPU that DispEst.h:42 declares but never defines, reconstructed on the
 * model of CostConst_CPU with CVF::preprocess (CVF.cpp:44) + CVF::filterCV_thread (CVF.cpp:28). */
int orc_cost_filter(const float* lImg, const float* rImg, int W, int H, int D, int threads, int window, float eps,
                    float* lVol, float* rVol);

/* DispEst.cpp:311-321 DispSelect_CPU */
int orc_disp_select(const float* lVol, const float* rVol, int W, int H, int D,
                    uint8_t* lDis, uint8_t* rDis);

/* Whole path with get_rt()-style per-stage timers (ComFunc.h:67-71); times_ms[3] = cvc,cvf,wta */
int orc_pipeline(const float* lImg, const float* rImg, int W, int H, int D, int threads,
                 int gray_mode, float alpha, float tau_color, float tau_grad, int window, float eps,
                 float* lVol, float* rVol, uint8_t* lDis, uint8_t* rDis, double* times_ms);

/* Fast Guided Filter branch (src/fastguidedfilter.cpp via DispEst::CostFilter_FGF, DispEst.cpp:281-296):
 * FastGuidedFilter(img, window, eps, s), s = sub-sampling rate, orc_box_k boxes of K = 2 * (window / s) + 1 at the
 * sub-sampled resolution, volumes filtered in place.  Pinned against cv2 (IPP off) by tests/golden/make_golden_fgf.py. */
int orc_cost_filter_fgf(const float* lImg, const float* rImg, int W, int H, int D, int threads, int s, int window, float eps,
                        float* lVol, float* rVol);

/* Post-processing (PP::processDM live code, src/PP.cpp:414-422 -> JointWMF::filter): see stereo_oracle.c.
 * PARITY UNPINNED for natural images (cv::kmeans feature clustering is RNG-seeded); this is the un-clustered filter. */
enum { ORC_WMF_EXP = 0, ORC_WMF_IV1 = 1, ORC_WMF_IV2 = 2, ORC_WMF_OFF = 5 };   /* weightType, JointWMF.h:503-508 */
#define ORC_PP_TABLE_MAX (3 * 63 * 63 + 1)   /* largest squared distance between two 6-bit colours, + 1 */

/* The weight table of (sigma, type), 2^-22 fixed point: with s = sigma / 256.0f * 64 and w(k) in float with the
 * operation order of JointWMF.h:620-648 (exp: expf(-(float)k * (1.0f / ((2*s)*s))), iv1: 1.0f / ((float)k + s),
 * iv2: 1.0f / ((float)k + s*s), off: 1.0f), t[k] = lrintf((w(k) / w(0)) * 4194304.0f).  k is the squared distance of
 * the 6-bit colours (exp, iv2), their L1 distance (iv1) or 0 (off).  t has room for ORC_PP_TABLE_MAX entries.
 * -> the number of entries */
int orc_pp_weight_table(float sigma, int type, uint32_t* t);
/* JointWMF::filter(disp, img8, r, sigma, nI, 256, iterations, type) without the colour clustering:
 * out(p) = min { v : 2 * sum_{q in window, I_q <= v} t[k(p,q)] >= sum_{q in window} t[k(p,q)] }, window clipped at the
 * border, u64 sums; each iteration filters the previous output.  disp / out: u8 (map_bytes 1) or u16 (map_bytes 2) maps,
 * may alias; img8: interleaved BGR u8 feature image; rows split over `threads` pthreads.  -> 0, or -1 (out of memory
 * or no thread) */
int orc_wmf(const void* disp, int map_bytes, const uint8_t* img8_bgr, int W, int H, int r, float sigma, int iterations,
            int type, int threads, void* out);
void orc_f32_to_u8x255(const float* src, uint8_t* dst, size_t n);

#ifdef __cplusplus
}
#endif
#endif
