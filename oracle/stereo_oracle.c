/*
 * stereo_oracle.c -- CPU ORACLE (test infrastructure only; see stereo_oracle.h).
 *
 * Plain-C restatement of the reference pthreads path.  Every function cites the
 * reference file:line it follows (paths relative to /root/reference).
 * Build: see oracle/Makefile (-O3 -ffp-contract=off, no -march=native, no fast-math:
 * the reference builds with plain -O3 on baseline x86-64, CMakeLists.txt:17, so no
 * FMA contraction happens there either).
 */
#define _GNU_SOURCE
#include "stereo_oracle.h"

#include <math.h>
#include <pthread.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

/* ------------------------------------------------------------------ utilities */

/* ComFunc.h:67-71 get_rt(): CLOCK_MONOTONIC; kept in double here (the reference
 * truncates to float, which is only a precision loss of the timer itself). */
static double now_ms(void)
{
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (double)ts.tv_sec * 1e3 + (double)ts.tv_nsec * 1e-6;
}

/* cv::BORDER_REFLECT_101 index map (gfedcb|abcdefgh|gfedcba) */
static inline int reflect101(int i, int n)
{
    if (n == 1) return 0;
    while (i < 0 || i >= n) {
        if (i < 0) i = -i;
        else i = 2 * (n - 1) - i;
    }
    return i;
}

/* ------------------------------------------------------------------ a1: input scaling */

/* StereoMatch.cpp:193-197: lFrame.convertTo(lFrame, CV_32F, 1 / 255.0f)
 * OpenCV cvtScale 8u->32f works in float: (float)u * (float)alpha (+0). */
void orc_u8_to_f32(const uint8_t* src, float* dst, size_t n)
{
    const float alpha = 1 / 255.0f;
    for (size_t i = 0; i < n; ++i) dst[i] = (float)src[i] * alpha;
}

/* ------------------------------------------------------------------ a2: CVC::preprocess */

/* CVC.cpp:43 cv::cvtColor(Img, GrdX, CV_RGB2GRAY).  OpenCV RGB2Gray<float>: coefficient
 * 0.299f on channel 0, 0.587f on channel 1, 0.114f on channel 2 (the reference feeds a BGR
 * image, so 0.299 lands on blue -- replicated, not fixed). */
void orc_rgb2gray(const float* img3, int W, int H, float* gray, int gray_mode)
{
    const size_t n = (size_t)W * H;
    if (gray_mode == 0) {
        for (size_t i = 0; i < n; ++i) {
            const float c0 = img3[3 * i], c1 = img3[3 * i + 1], c2 = img3[3 * i + 2];
            gray[i] = fmaf(c2, 0.114f, fmaf(c0, 0.299f, c1 * 0.587f));
        }
    } else {
        for (size_t i = 0; i < n; ++i) {
            const float c0 = img3[3 * i], c1 = img3[3 * i + 1], c2 = img3[3 * i + 2];
            gray[i] = (c0 * 0.299f + c1 * 0.587f) + c2 * 0.114f;
        }
    }
}

/* CVC.cpp:44 cv::Sobel(GrdX, GrdX, CV_32F, 1, 0, 1): ksize=1, dx=1 -> kernel [-1 0 1],
 * BORDER_REFLECT_101 (so columns 0 and W-1 are exactly 0). */
void orc_sobel_x(const float* gray, int W, int H, float* grdx)
{
    for (int y = 0; y < H; ++y) {
        const float* g = gray + (size_t)y * W;
        float* o = grdx + (size_t)y * W;
        for (int x = 0; x < W; ++x) {
            const float r = g[reflect101(x + 1, W)];
            const float l = g[reflect101(x - 1, W)];
            o[x] = r - l;
        }
    }
}

/* CVC.cpp:41-46 */
void orc_cvc_preprocess(const float* img3, int W, int H, float* grdx, int gray_mode)
{
    float* gray = (float*)malloc((size_t)W * H * sizeof(float));
    orc_rgb2gray(img3, W, H, gray, gray_mode);
    orc_sobel_x(gray, W, H, grdx);
    free(gray);
}

/* ------------------------------------------------------------------ a3/a4: myCostGrd */

/* CVC.cpp:24-27 / 36-39 with the truncation the reference leaves commented out restored: a NaN difference is not above
 * any threshold and stays NaN, +inf truncates nothing; every float operation is rounded separately. */
static inline float cost_weigh(float clrDiff, float grdDiff, float alpha, float tau_color, float tau_grad)
{
    if (clrDiff > tau_color) clrDiff = tau_color;
    if (grdDiff > tau_grad) grdDiff = tau_grad;
    return alpha * clrDiff + (1 - alpha) * grdDiff;
}

/* CVC.cpp:18-27: all-float arithmetic (math.h in C++ gives fabs(float) -> float). */
static inline float cost_grd4(const float* lC, const float* rC, const float* lG, const float* rG,
                              float alpha, float tau_color, float tau_grad)
{
    float clrDiff = fabsf(lC[0] - rC[0]) + fabsf(lC[1] - rC[1]) + fabsf(lC[2] - rC[2]);
    float grdDiff = fabsf(*lG - *rG);
    return cost_weigh(clrDiff, grdDiff, alpha, tau_color, tau_grad);
}

/* CVC.cpp:30-39: BC_32F is the double literal 1.0 (CVC.h:12), so the differences, fabs and
 * the three-term sum are evaluated in double and rounded to float once per assignment. */
static inline float cost_grd2(const float* lC, const float* lG, float alpha, float tau_color, float tau_grad)
{
    float clrDiff = (float)(fabs((double)lC[0] - 1.0) + fabs((double)lC[1] - 1.0) + fabs((double)lC[2] - 1.0));
    float grdDiff = (float)fabs((double)*lG - 1.0);
    return cost_weigh(clrDiff, grdDiff, alpha, tau_color, tau_grad);
}

/* ------------------------------------------------------------------ a5/a6: buildCV */

/* CVC.cpp:122-149 */
static void buildcv_left(const float* lImg, const float* rImg, const float* lGrd, const float* rGrd,
                         int W, int H, int d, float alpha, float tau_color, float tau_grad, float* cost)
{
    for (int y = 0; y < H; ++y) {
        const float* lData = lImg + (size_t)y * W * 3;
        const float* rData = rImg + (size_t)y * W * 3;
        const float* lGData = lGrd + (size_t)y * W;
        const float* rGData = rGrd + (size_t)y * W;
        float* c = cost + (size_t)y * W;
        for (int x = d; x < W; ++x)
            c[x] = cost_grd4(lData + 3 * x, rData + 3 * (x - d), lGData + x, rGData + x - d, alpha, tau_color, tau_grad);
        for (int x = 0; x < d && x < W; ++x)
            c[x] = cost_grd2(lData + 3 * x, lGData + x, alpha, tau_color, tau_grad);
    }
}

/* CVC.cpp:151-179 */
static void buildcv_right(const float* lImg, const float* rImg, const float* lGrd, const float* rGrd,
                          int W, int H, int d, float alpha, float tau_color, float tau_grad, float* cost)
{
    int border = W - d;
    if (border < 0) border = 0;
    for (int y = 0; y < H; ++y) {
        const float* lData = lImg + (size_t)y * W * 3;
        const float* rData = rImg + (size_t)y * W * 3;
        const float* lGData = lGrd + (size_t)y * W;
        const float* rGData = rGrd + (size_t)y * W;
        float* c = cost + (size_t)y * W;
        for (int x = 0; x < border; ++x)
            c[x] = cost_grd4(lData + 3 * x, rData + 3 * (x + d), lGData + x, rGData + x + d, alpha, tau_color, tau_grad);
        for (int x = border; x < W; ++x)
            c[x] = cost_grd2(lData + 3 * x, lGData + x, alpha, tau_color, tau_grad);
    }
}

/* the reference's own entry points: its signatures, its constants */
void orc_buildcv_left(const float* lImg, const float* rImg, const float* lGrd, const float* rGrd,
                      int W, int H, int d, float* cost)
{
    buildcv_left(lImg, rImg, lGrd, rGrd, W, H, d, ORC_ALPHA, INFINITY, INFINITY, cost);
}

void orc_buildcv_right(const float* lImg, const float* rImg, const float* lGrd, const float* rGrd,
                       int W, int H, int d, float* cost)
{
    buildcv_right(lImg, rImg, lGrd, rGrd, W, H, d, ORC_ALPHA, INFINITY, INFINITY, cost);
}

/* ------------------------------------------------------------------ a10: cv::boxFilter K x K */

/* OpenCV box filter for CV_32F, normalize=true, ksize K x K, default anchor (K/2, K/2), BORDER_REFLECT_101 with any
 * overshoot (images smaller than the window).  Restates modules/imgproc/src/box_filter.simd.hpp:
 *   K == 1:                 a copy
 *   RowSum<float,double>:   K <= 5: S[i] + S[i+1] + ... + S[i+K-1], left to right;
 *                           above:  s = sum of the first K (double); then s += (double)S[i+K] - (double)S[i]
 *   ColumnSum<double,float>: s0 = SUM + newest; dst = (float)(s0 * (1.0/(K*K))); SUM = s0 - oldest
 * Rows are padded K/2 left / K-1-K/2 right, the column pass sees rows y-K/2 .. y+K-1-K/2 (reflected). */
void orc_box(const float* src, int W, int H, int K, float* dst)
{
    if (K == 1) {
        if (dst != src) memcpy(dst, src, (size_t)W * H * sizeof(float));
        return;
    }
    const int AL = K / 2;
    const double scale = 1.0 / (double)(K * K);
    const int PW = W + K - 1;
    float* prow = (float*)malloc((size_t)PW * sizeof(float));
    double* rs = (double*)malloc((size_t)W * H * sizeof(double)); /* row sums of every source row */
    double* SUM = (double*)calloc((size_t)W, sizeof(double));

    for (int y = 0; y < H; ++y) {
        const float* s = src + (size_t)y * W;
        for (int i = 0; i < PW; ++i) prow[i] = s[reflect101(i - AL, W)];
        double* D = rs + (size_t)y * W;
        if (K <= 5) {
            for (int i = 0; i < W; ++i) {
                double acc = (double)prow[i];
                for (int j = 1; j < K; ++j) acc += (double)prow[i + j];
                D[i] = acc;
            }
            continue;
        }
        double acc = 0;
        for (int i = 0; i < K; ++i) acc += (double)prow[i];
        D[0] = acc;
        for (int i = 0; i < W - 1; ++i) {
            acc += (double)prow[i + K] - (double)prow[i];
            D[i + 1] = acc;
        }
    }
    /* column pass; padded row index r = y' + AL maps to source row reflect101(y', H) */
    for (int r = 0; r < K - 1; ++r) {
        const double* Sp = rs + (size_t)reflect101(r - AL, H) * W;
        for (int i = 0; i < W; ++i) SUM[i] += Sp[i];
    }
    float* out = dst;
    float* tmp = NULL;
    if (src == dst) { tmp = (float*)malloc((size_t)W * H * sizeof(float)); out = tmp; }
    for (int y = 0; y < H; ++y) {
        const double* Sp = rs + (size_t)reflect101(y + K - 1 - AL, H) * W; /* newest */
        const double* Sm = rs + (size_t)reflect101(y - AL, H) * W;         /* oldest */
        float* D = out + (size_t)y * W;
        for (int i = 0; i < W; ++i) {
            double s0 = SUM[i] + Sp[i];
            D[i] = (float)(s0 * scale);
            SUM[i] = s0 - Sm[i];
        }
    }
    if (tmp) { memcpy(dst, tmp, (size_t)W * H * sizeof(float)); free(tmp); }
    free(SUM); free(rs); free(prow);
}

/* ------------------------------------------------------------------ a8: CVF::preprocess */

/* CVF.cpp:44-70 */
void orc_cvf_preprocess(const float* img3, int W, int H, int window, float* rgb, float* mean, float* var)
{
    const size_t n = (size_t)W * H;
    for (size_t i = 0; i < n; ++i)                 /* split(), CVF.cpp:47 */
        for (int c = 0; c < 3; ++c) rgb[c * n + i] = img3[3 * i + c];
    for (int c = 0; c < 3; ++c)                    /* CVF.cpp:49-51 */
        orc_box(rgb + c * n, W, H, window, mean + c * n);
    float* tmp = (float*)malloc(n * sizeof(float));
    int varIdx = 0;
    for (int c = 0; c < 3; ++c) {                  /* CVF.cpp:60-69 */
        for (int cp = c; cp < 3; ++cp) {
            float* v = var + (size_t)varIdx * n;
            for (size_t i = 0; i < n; ++i) tmp[i] = rgb[c * n + i] * rgb[cp * n + i];
            orc_box(tmp, W, H, window, v);
            for (size_t i = 0; i < n; ++i) tmp[i] = mean[c * n + i] * mean[cp * n + i];
            for (size_t i = 0; i < n; ++i) v[i] -= tmp[i];
            ++varIdx;
        }
    }
    free(tmp);
}

/* ------------------------------------------------------------------ a9: GuidedFilter_cv */

/* CVF.cpp:72-165 */
void orc_guided_filter(const float* rgb, const float* mean_I, const float* var_I, int W, int H, int window, float eps,
                       float* p, float* a_out, float* b_out)
{
    const size_t n = (size_t)W * H;
    float* mean_p = (float*)malloc(n * sizeof(float));
    float* tmp = (float*)malloc(n * sizeof(float));
    float* mean_Ip = (float*)malloc(3 * n * sizeof(float)); /* becomes cov_Ip */
    float* a = (float*)malloc(3 * n * sizeof(float));
    float* q = (float*)malloc(n * sizeof(float));

    orc_box(p, W, H, window, mean_p);                                  /* CVF.cpp:81-82 */
    for (int c = 0; c < 3; ++c) {                                /* CVF.cpp:86-89 */
        for (size_t i = 0; i < n; ++i) tmp[i] = rgb[c * n + i] * p[i];
        orc_box(tmp, W, H, window, mean_Ip + c * n);
    }
    for (int c = 0; c < 3; ++c) {                                /* CVF.cpp:92-95 */
        for (size_t i = 0; i < n; ++i) tmp[i] = mean_I[c * n + i] * mean_p[i];
        for (size_t i = 0; i < n; ++i) mean_Ip[c * n + i] = mean_Ip[c * n + i] - tmp[i];
    }
    const float* cov = mean_Ip;
    for (size_t i = 0; i < n; ++i) {                             /* CVF.cpp:102-149 */
        float c0 = cov[i], c1 = cov[n + i], c2 = cov[2 * n + i];
        float a11 = var_I[i] + eps;
        float a12 = var_I[n + i];
        float a13 = var_I[2 * n + i];
        float a21 = var_I[n + i];
        float a22 = var_I[3 * n + i] + eps;
        float a23 = var_I[4 * n + i];
        float a31 = var_I[2 * n + i];
        float a32 = var_I[4 * n + i];
        float a33 = var_I[5 * n + i] + eps;
        float DET = a11 * (a33 * a22 - a32 * a23) -
                    a21 * (a33 * a12 - a32 * a13) +
                    a31 * (a23 * a12 - a22 * a13);
        DET = 1 / DET;
        a[i] = DET * (
            c0 * (a33 * a22 - a32 * a23) +
            c1 * (a31 * a23 - a33 * a21) +
            c2 * (a32 * a21 - a31 * a22));
        a[n + i] = DET * (
            c0 * (a32 * a13 - a33 * a12) +
            c1 * (a33 * a11 - a31 * a13) +
            c2 * (a31 * a12 - a32 * a11));
        a[2 * n + i] = DET * (
            c0 * (a23 * a12 - a22 * a13) +
            c1 * (a21 * a13 - a23 * a11) +
            c2 * (a22 * a11 - a21 * a12));
    }
    for (int c = 0; c < 3; ++c) {                                /* CVF.cpp:152-155 */
        for (size_t i = 0; i < n; ++i) tmp[i] = a[c * n + i] * mean_I[c * n + i];
        for (size_t i = 0; i < n; ++i) mean_p[i] -= tmp[i];
    }
    if (a_out) memcpy(a_out, a, 3 * n * sizeof(float));
    if (b_out) memcpy(b_out, mean_p, n * sizeof(float));

    orc_box(mean_p, W, H, window, q);                                 /* CVF.cpp:157-158 */
    for (int c = 0; c < 3; ++c) {                                /* CVF.cpp:159-163 */
        orc_box(a + c * n, W, H, window, tmp);
        for (size_t i = 0; i < n; ++i) tmp[i] = tmp[i] * rgb[c * n + i];
        for (size_t i = 0; i < n; ++i) q[i] += tmp[i];
    }
    memcpy(p, q, n * sizeof(float));                             /* CVF.cpp:38 in-place */
    free(q); free(a); free(mean_Ip); free(tmp); free(mean_p);
}

/* ------------------------------------------------------------------ a12: WTA */

/* DispSel.cpp:83-109: d from 1, strict <, minCost starts at (float)DBL_MAX = +inf.  The arg-min is an int there; the
 * reference stores it into a uchar (map_bytes 1), a 16-bit map (map_bytes 2) keeps it whole, so the u8 map is the low
 * byte of the u16 one. */
static void wta_rows(const float* vol, int W, int H, int D, void* disp, int map_bytes, int y0, int y1)
{
    const size_t n = (size_t)W * H;
    for (int y = y0; y < y1; ++y) {
        for (int x = 0; x < W; ++x) {
            float minCost = INFINITY;
            int minDis = 0;
            for (int d = 1; d < D; ++d) {
                const float c = vol[(size_t)d * n + (size_t)y * W + x];
                if (c < minCost) { minCost = c; minDis = d; }
            }
            const size_t i = (size_t)y * W + x;
            if (map_bytes == 2) ((uint16_t*)disp)[i] = (uint16_t)minDis;
            else ((uint8_t*)disp)[i] = (uint8_t)minDis;
        }
    }
}

void orc_wta(const float* vol, int W, int H, int D, void* disp, int map_bytes)
{
    wta_rows(vol, W, H, D, disp, map_bytes, 0, H);
}

/* ------------------------------------------------------------------ a7/a11: thread drivers */

typedef struct {
    int kind; /* 0 left cvc, 1 right cvc, 2 filter, 3 wta rows, 4 weighted-median rows */
    const float *lImg, *rImg, *lGrd, *rGrd;
    const float *rgb, *mean, *var;
    const float* vol_in;
    float* slice;
    void* disp;
    int map_bytes;
    const uint16_t* wmf_in;    /* kind 4: map, feature image, weight table, histogram size, output */
    const uint8_t* img8;
    const uint32_t* lut;
    int r, wtype, nbins;
    uint16_t* wmf_out;
    float alpha, tau_color, tau_grad;   /* kinds 0, 1 */
    int window;                         /* kind 2 */
    float eps;
    int W, H, D, d, y0, y1;
} task_t;

static void* wmf_rows(const task_t* t);

static void* task_entry(void* arg)
{
    task_t* t = (task_t*)arg;
    switch (t->kind) {
    case 0: buildcv_left(t->lImg, t->rImg, t->lGrd, t->rGrd, t->W, t->H, t->d, t->alpha, t->tau_color, t->tau_grad, t->slice); break;
    case 1: buildcv_right(t->lImg, t->rImg, t->lGrd, t->rGrd, t->W, t->H, t->d, t->alpha, t->tau_color, t->tau_grad, t->slice); break;
    case 2: orc_guided_filter(t->rgb, t->mean, t->var, t->W, t->H, t->window, t->eps, t->slice, NULL, NULL); break;
    case 3: wta_rows(t->vol_in, t->W, t->H, t->D, t->disp, t->map_bytes, t->y0, t->y1); break;
    case 4: return wmf_rows(t);
    }
    return NULL;
}

/* DispEst.cpp:235-251 batching: for level in 0..=n/threads, block = threads or n%threads,
 * create block pthreads (one per d), join them all, next level.  -> 0, or -1 when a thread could not be created or a
 * task failed */
static int run_batched(task_t* tasks, int n, int threads)
{
    if (threads < 1) threads = 1;
    pthread_t* th = (pthread_t*)malloc((size_t)n * sizeof(pthread_t));
    if (!th) return -1;
    int rc = 0;
    for (int level = 0; level <= n / threads && rc == 0; ++level) {
        int block = (level < n / threads) ? threads : (n % threads);
        int started = 0;
        for (; started < block; ++started)
            if (pthread_create(&th[level * threads + started], NULL, task_entry, &tasks[level * threads + started]) != 0) {
                rc = -1;
                break;
            }
        for (int it = 0; it < started; ++it) {
            void* ret = NULL;
            pthread_join(th[level * threads + it], &ret);
            if (ret) rc = -1;
        }
    }
    free(th);
    return rc;
}

/* rows [0, H) split over `threads` pthreads, one copy of `proto` each (DispSel::CVSelect is "#pragma omp parallel for"
 * over rows, DispSel.cpp:88) */
static int run_rows(task_t proto, int H, int threads)
{
    if (threads < 1) threads = 1;
    if (threads > H) threads = H;
    task_t* tasks = (task_t*)malloc((size_t)threads * sizeof(task_t));
    if (!tasks) return -1;
    for (int t = 0; t < threads; ++t) {
        tasks[t] = proto;
        tasks[t].y0 = (int)((long)H * t / threads);
        tasks[t].y1 = (int)((long)H * (t + 1) / threads);
    }
    int rc = run_batched(tasks, threads, threads);
    free(tasks);
    return rc;
}

/* DispEst.cpp:222-270, the slices of the disparities [d_begin, d_begin + d_count) */
int orc_cost_const(const float* lImg, const float* rImg, int W, int H, int d_begin, int d_count, int threads,
                   int gray_mode, float alpha, float tau_color, float tau_grad,
                   float* lGrd, float* rGrd, float* lVol, float* rVol)
{
    const size_t n = (size_t)W * H;
    orc_cvc_preprocess(lImg, W, H, lGrd, gray_mode);   /* DispEst.cpp:232 */
    orc_cvc_preprocess(rImg, W, H, rGrd, gray_mode);   /* DispEst.cpp:233 */
    task_t* tasks = (task_t*)calloc((size_t)d_count, sizeof(task_t));
    for (int i = 0; i < d_count; ++i) {                /* DispEst.cpp:243 */
        task_t t = {0};
        t.kind = 0; t.lImg = lImg; t.rImg = rImg; t.lGrd = lGrd; t.rGrd = rGrd;
        t.alpha = alpha; t.tau_color = tau_color; t.tau_grad = tau_grad;
        t.W = W; t.H = H; t.d = d_begin + i; t.slice = lVol + (size_t)i * n;
        tasks[i] = t;
    }
    int rc = run_batched(tasks, d_count, threads);
    for (int i = 0; i < d_count && rc == 0; ++i) {     /* DispEst.cpp:260: swapped arguments */
        task_t t = tasks[i];
        t.kind = 1; t.lImg = rImg; t.rImg = lImg; t.lGrd = rGrd; t.rGrd = lGrd;
        t.slice = rVol + (size_t)i * n;
        tasks[i] = t;
    }
    if (rc == 0) rc = run_batched(tasks, d_count, threads);
    free(tasks);
    return rc;
}

/* Reconstructed CostFilter_CPU (declared DispEst.h:42, never defined): CVF::preprocess per
 * view (CVF.cpp:44) then one filterCV_thread per d (CVF.cpp:28-41) in CostConst_CPU batches. */
int orc_cost_filter(const float* lImg, const float* rImg, int W, int H, int D, int threads, int window, float eps,
                    float* lVol, float* rVol)
{
    const size_t n = (size_t)W * H;
    float* g = (float*)malloc(12 * n * sizeof(float));
    float *rgb = g, *mean = g + 3 * n, *var = g + 6 * n;
    task_t* tasks = (task_t*)calloc((size_t)D, sizeof(task_t));
    int rc = 0;
    for (int view = 0; view < 2 && rc == 0; ++view) {
        orc_cvf_preprocess(view == 0 ? lImg : rImg, W, H, window, rgb, mean, var);
        float* vol = view == 0 ? lVol : rVol;
        for (int d = 0; d < D; ++d) {
            task_t t = {0};
            t.kind = 2; t.rgb = rgb; t.mean = mean; t.var = var; t.window = window; t.eps = eps;
            t.W = W; t.H = H; t.d = d; t.slice = vol + (size_t)d * n;
            tasks[d] = t;
        }
        rc = run_batched(tasks, D, threads);
    }
    free(tasks); free(g);
    return rc;
}

/* DispEst.cpp:311-321, rows split over `threads` pthreads */
static int wta_view(const float* vol, int W, int H, int D, uint8_t* dis, int threads)
{
    task_t k = {0};
    k.kind = 3; k.vol_in = vol; k.W = W; k.H = H; k.D = D; k.disp = dis; k.map_bytes = 1;
    return run_rows(k, H, threads);
}

int orc_disp_select(const float* lVol, const float* rVol, int W, int H, int D,
                    uint8_t* lDis, uint8_t* rDis)
{
    orc_wta(lVol, W, H, D, lDis, 1);
    orc_wta(rVol, W, H, D, rDis, 1);
    return 0;
}

int orc_pipeline(const float* lImg, const float* rImg, int W, int H, int D, int threads,
                 int gray_mode, float alpha, float tau_color, float tau_grad, int window, float eps,
                 float* lVol, float* rVol, uint8_t* lDis, uint8_t* rDis, double* times_ms)
{
    const size_t n = (size_t)W * H;
    float* lGrd = (float*)malloc(n * sizeof(float));
    float* rGrd = (float*)malloc(n * sizeof(float));
    double t0 = now_ms();
    int rc = orc_cost_const(lImg, rImg, W, H, 0, D, threads, gray_mode, alpha, tau_color, tau_grad, lGrd, rGrd, lVol, rVol);
    double t1 = now_ms();
    if (rc == 0) rc = orc_cost_filter(lImg, rImg, W, H, D, threads, window, eps, lVol, rVol);
    double t2 = now_ms();
    if (rc == 0) rc = wta_view(lVol, W, H, D, lDis, threads);
    if (rc == 0) rc = wta_view(rVol, W, H, D, rDis, threads);
    double t3 = now_ms();
    if (times_ms) { times_ms[0] = t1 - t0; times_ms[1] = t2 - t1; times_ms[2] = t3 - t2; }
    free(lGrd); free(rGrd);
    return rc;
}


/* ------------------------------------------------------------------------------------------------------------
 * Post-processing: the joint weighted-median filter of the disparity maps (PP::processDM, src/PP.cpp:402-425:
 * img.convertTo(CV_8UC3, 255) then JointWMF::filter(disp, img8UC3, MED_SZ/2 = 9), include/JointWMF.h:81-155).
 *
 * PARITY UNPINNED for natural images: the reference clusters the feature colours with cv::kmeans (k-means++ on
 * cv::theRNG(), JointWMF.h:586-591; un-vendored, RNG-seeded) down to nF = 256 indices and documents the result as an
 * approximation (JointWMF.h:70-72).  This restatement is the filter WITHOUT that approximation -- the weight between
 * two pixels is taken between their own 6-bit colours (what the reference computes when the image has <= 256 distinct
 * 6-bit colours, where every colour is its own cluster) -- with the definition of the output the reference's cut-point
 * search implements (JointWMF.h:257-316):  out = min { v : sum_{I_q <= v} w_q  >=  sum_{I_q > v} w_q }  over the
 * (2r+1)^2 window clipped at the image border (JointWMF.h:207-211, 322-325).
 * Weights: JointWMF.h:620-648's float formulas (see orc_pp_weight_table) held as 2^-22 fixed point so that the sums are
 * exact integers, independent of summation order (the reference's float sums depend on its necklace-table insertion
 * history).  r, sigma, iter and weightType are JointWMF::filter's arguments; PP::processDM passes (9, 25.5, 1, exp).
 * -------------------------------------------------------------------------------------------------------------- */
static float pp_weight(int type, float s, int k)
{
    switch (type) {
    case ORC_WMF_EXP: return expf(-(float)k * (1.0f / ((2 * s) * s)));
    case ORC_WMF_IV1: return 1.0f / ((float)k + s);
    case ORC_WMF_IV2: return 1.0f / ((float)k + s * s);
    default: return 1.0f;
    }
}

int orc_pp_weight_table(float sigma, int type, uint32_t* t)
{
    const float s = sigma / 256.0f * 64;
    const float w0 = pp_weight(type, s, 0);
    const int n = type == ORC_WMF_IV1 ? 3 * 63 + 1 : (type == ORC_WMF_OFF ? 1 : ORC_PP_TABLE_MAX);
    for (int k = 0; k < n; ++k) t[k] = (uint32_t)lrintf((pp_weight(type, s, k) / w0) * 4194304.0f);
    return n;
}

/* one pass over rows [y0, y1): wmf_in -> wmf_out, a histogram over the map values [0, nbins) */
static void* wmf_rows(const task_t* a)
{
    const int W = a->W, H = a->H, r = a->r;
    uint64_t* hist = (uint64_t*)malloc((size_t)a->nbins * sizeof(uint64_t));
    if (!hist) return (void*)1;
    for (int y = a->y0; y < a->y1; ++y) {
        for (int x = 0; x < W; ++x) {
            memset(hist, 0, (size_t)a->nbins * sizeof(uint64_t));
            const uint8_t* cp = a->img8 + ((size_t)y * W + x) * 3;
            const int b = cp[0] >> 2, g = cp[1] >> 2, rr = cp[2] >> 2;
            uint64_t total = 0;
            const int ya = y - r < 0 ? 0 : y - r, yb = y + r > H - 1 ? H - 1 : y + r;
            const int xa = x - r < 0 ? 0 : x - r, xb = x + r > W - 1 ? W - 1 : x + r;
            for (int yy = ya; yy <= yb; ++yy)
                for (int xx = xa; xx <= xb; ++xx) {
                    const uint8_t* cq = a->img8 + ((size_t)yy * W + xx) * 3;
                    const int d0 = b - (cq[0] >> 2), d1 = g - (cq[1] >> 2), d2 = rr - (cq[2] >> 2);
                    const int k = a->wtype == ORC_WMF_IV1 ? abs(d0) + abs(d1) + abs(d2)
                                : a->wtype == ORC_WMF_OFF ? 0 : d0 * d0 + d1 * d1 + d2 * d2;
                    const uint32_t w = a->lut[k];
                    hist[a->wmf_in[(size_t)yy * W + xx]] += w;
                    total += w;
                }
            uint64_t cum = 0;
            int v = 0;
            for (; v < a->nbins - 1; ++v) {
                cum += hist[v];
                if (2 * cum >= total) break;
            }
            a->wmf_out[(size_t)y * W + x] = (uint16_t)v;
        }
    }
    free(hist);
    return NULL;
}

int orc_wmf(const void* disp, int map_bytes, const uint8_t* img8, int W, int H, int r, float sigma, int iterations,
            int type, int threads, void* out)
{
    const size_t n = (size_t)W * H;
    uint32_t* lut = (uint32_t*)malloc(ORC_PP_TABLE_MAX * sizeof(uint32_t));
    uint16_t* cur = (uint16_t*)malloc(n * sizeof(uint16_t));
    uint16_t* next = (uint16_t*)malloc(n * sizeof(uint16_t));
    int rc = lut && cur && next ? 0 : -1;
    if (rc == 0) {
        orc_pp_weight_table(sigma, type, lut);
        int maxv = 0;
        for (size_t i = 0; i < n; ++i) {
            cur[i] = map_bytes == 2 ? ((const uint16_t*)disp)[i] : ((const uint8_t*)disp)[i];
            maxv = cur[i] > maxv ? cur[i] : maxv;
        }
        task_t k = {0};
        k.kind = 4; k.img8 = img8; k.lut = lut; k.W = W; k.H = H; k.r = r; k.wtype = type;
        k.nbins = maxv + 1;   /* the median is a value of the window, so no pass raises the maximum */
        /* JointWMF.h:126-131: each iteration filters the previous output with the original feature image */
        for (int it = 0; it < iterations && rc == 0; ++it) {
            k.wmf_in = cur; k.wmf_out = next;
            rc = run_rows(k, H, threads);
            uint16_t* t = cur; cur = next; next = t;
        }
        for (size_t i = 0; i < n && rc == 0; ++i) {
            if (map_bytes == 2) ((uint16_t*)out)[i] = cur[i];
            else ((uint8_t*)out)[i] = (uint8_t)cur[i];
        }
    }
    free(lut); free(cur); free(next);
    return rc;
}

/* lImg.convertTo(lImg_8UC3, CV_8UC3, 255) (src/PP.cpp:416-417): saturate_cast<uchar>(cvRound(v * 255)).  q = v * 255 is
 * rounded to float; cvRound on x86 is cvtss2si, which returns INT_MIN when q is NaN or outside the int range, and that
 * saturates to 0.  So: 0 if q is NaN or q >= 2^31 (+inf included), else clamp(rint(q), 0, 255), ties to even (pinned
 * against cv2 by tests/golden/golden_image.json). */
void orc_f32_to_u8x255(const float* src, uint8_t* dst, size_t n)
{
    for (size_t i = 0; i < n; ++i) {
        const float q = src[i] * 255.0f;
        if (!(q < 2147483648.0f)) { dst[i] = 0; continue; }   /* NaN, >= 2^31 */
        const float r = rintf(q);
        dst[i] = (uint8_t)(r < 0.0f ? 0 : (r > 255.0f ? 255 : (int)r));
    }
}


/* ------------------------------------------------------------------------------------------------------------
 * Fast Guided Filter branch: FastGuidedFilterColor (src/fastguidedfilter.cpp:121-198) as driven by
 * DispEst::CostFilter_FGF (src/DispEst.cpp:281-296): FastGuidedFilter(img, window, eps, s) -> box size
 * K = 2*(window/s)+1 on the s-times sub-sampled planes (:206-208).
 * OpenCV primitives restated from OpenCV's own implementation and pinned against cv2 4.13 (IPP off) by
 * tests/golden/make_golden_fgf.py: cv::blur == normalised K x K box, anchor K/2, BORDER_REFLECT_101, double
 * accumulation, * (1.0/(K*K)) in double, one rounding; cv::resize INTER_NN: x -> min(floor(x * (1/(w2/W))), W-1);
 * cv::resize INTER_LINEAR: f = (float)((d+0.5)*(sn/dn) - 0.5), i = floor(f), f -= i; horizontally the border clamps
 * with f = 0, vertically the two row indices clamp and f is kept; out = S0*(1-f) + S1*f in float, rows after columns.
 * cv::MatExpr lowering (matop.cpp): a.mul(b) is a rounded product; X - Y + eps -> addWeighted == (X - Y + eps) in DOUBLE, one rounding;
 * /= is a true division.  PARITY NOTE: with IPP, cv::resize INTER_LINEAR differs by up to 1e-4 (build-dependent).
 * -------------------------------------------------------------------------------------------------------------- */
void orc_box_k(const float* src, int W, int H, int K, float* dst)
{
    const int a = K / 2;
    const double scale = 1.0 / ((double)K * K);
    double* rows = (double*)malloc((size_t)W * H * sizeof(double));
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) {
            double sacc = 0.0;
            for (int dx = -a; dx < K - a; ++dx) sacc += (double)src[(size_t)y * W + reflect101(x + dx, W)];
            rows[(size_t)y * W + x] = sacc;
        }
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) {
            double sacc = 0.0;
            for (int dy = -a; dy < K - a; ++dy) sacc += rows[(size_t)reflect101(y + dy, H) * W + x];
            dst[(size_t)y * W + x] = (float)(sacc * scale);
        }
    free(rows);
}

typedef struct {
    int W, H, w2, h2, s, K;
    float* orig[3];   /* full-resolution channels (split) */
    float* Ic[3];     /* sub-sampled channels */
    float* m[3];      /* box means of Ic */
    float* inv[6];    /* rr rg rb gg gb bb of (Sigma + eps I)^-1 */
    int *xs, *ys;     /* NN source indices */
    int *lx0, *lx1, *ly0, *ly1; float *fx, *fy;   /* bilinear up-sampling plan */
} fgf_guide;

static float* fnew(size_t n) { return (float*)malloc(n * sizeof(float)); }

static void fgf_free(fgf_guide* g)
{
    for (int k = 0; k < 3; ++k) { free(g->orig[k]); free(g->Ic[k]); free(g->m[k]); }
    for (int k = 0; k < 6; ++k) free(g->inv[k]);
    free(g->xs); free(g->ys); free(g->lx0); free(g->lx1); free(g->ly0); free(g->ly1); free(g->fx); free(g->fy);
}

static void fgf_build(fgf_guide* g, const float* img3, int W, int H, int s, int window, float eps)
{
    memset(g, 0, sizeof(*g));
    g->W = W; g->H = H; g->s = s; g->w2 = W / s; g->h2 = H / s; g->K = 2 * (window / s) + 1;
    const int w2 = g->w2, h2 = g->h2, K = g->K;
    const size_t n = (size_t)W * H, n2 = (size_t)w2 * h2;
    g->xs = (int*)malloc(w2 * sizeof(int)); g->ys = (int*)malloc(h2 * sizeof(int));
    { const double ifx = 1.0 / ((double)w2 / W), ify = 1.0 / ((double)h2 / H);
      for (int x = 0; x < w2; ++x) { int v = (int)floor(x * ifx); g->xs[x] = v < W - 1 ? v : W - 1; }
      for (int y = 0; y < h2; ++y) { int v = (int)floor(y * ify); g->ys[y] = v < H - 1 ? v : H - 1; } }
    g->lx0 = (int*)malloc(W * sizeof(int)); g->lx1 = (int*)malloc(W * sizeof(int)); g->fx = fnew(W);
    g->ly0 = (int*)malloc(H * sizeof(int)); g->ly1 = (int*)malloc(H * sizeof(int)); g->fy = fnew(H);
    { const double sc = (double)w2 / W;
      for (int x = 0; x < W; ++x) {
          float f = (float)((x + 0.5) * sc - 0.5); int i = (int)floorf(f); f -= (float)i;
          if (i < 0) { f = 0.f; i = 0; }
          if (i >= w2 - 1) { f = 0.f; i = w2 - 1; }
          g->lx0[x] = i; g->lx1[x] = i + 1 < w2 ? i + 1 : w2 - 1; g->fx[x] = f; } }
    { const double sc = (double)h2 / H;
      for (int y = 0; y < H; ++y) {
          float f = (float)((y + 0.5) * sc - 0.5); int i = (int)floorf(f); f -= (float)i;
          int i0 = i < 0 ? 0 : (i > h2 - 1 ? h2 - 1 : i), i1 = i + 1 < 0 ? 0 : (i + 1 > h2 - 1 ? h2 - 1 : i + 1);
          g->ly0[y] = i0; g->ly1[y] = i1; g->fy[y] = f; } }
    for (int k = 0; k < 3; ++k) {
        g->orig[k] = fnew(n); g->Ic[k] = fnew(n2); g->m[k] = fnew(n2);
        for (size_t i = 0; i < n; ++i) g->orig[k][i] = img3[3 * i + k];
        for (int y = 0; y < h2; ++y) for (int x = 0; x < w2; ++x) g->Ic[k][(size_t)y * w2 + x] = g->orig[k][(size_t)g->ys[y] * W + g->xs[x]];
        orc_box_k(g->Ic[k], w2, h2, K, g->m[k]);
    }
    float* var[6]; float* t = fnew(n2);
    static const int pa[6] = {0, 0, 0, 1, 1, 2}, pb[6] = {0, 1, 2, 1, 2, 2};
    for (int v = 0; v < 6; ++v) {
        var[v] = fnew(n2);
        for (size_t i = 0; i < n2; ++i) t[i] = g->Ic[pa[v]][i] * g->Ic[pb[v]][i];
        orc_box_k(t, w2, h2, K, var[v]);
        const int diag = pa[v] == pb[v];
        for (size_t i = 0; i < n2; ++i) {
            const float mm = g->m[pa[v]][i] * g->m[pb[v]][i];
            /* fastguidedfilter.cpp:144-149: 'box - m.mul(m) + eps' lowers to addWeighted(box, 1, mm, -1, eps), which
               evaluates in double and rounds once; the off-diagonal terms are a plain float subtract */
            var[v][i] = diag ? (float)(((double)var[v][i] - (double)mm) + (double)eps) : var[v][i] - mm;
        }
    }
    float *rr = var[0], *rg = var[1], *rb = var[2], *gg = var[3], *gb = var[4], *bb = var[5];
    for (int k = 0; k < 6; ++k) g->inv[k] = fnew(n2);
    for (size_t i = 0; i < n2; ++i) {                                         /* :152-166 */
        const float irr = gg[i] * bb[i] - gb[i] * gb[i];
        const float irg = gb[i] * rb[i] - rg[i] * bb[i];
        const float irb = rg[i] * gb[i] - gg[i] * rb[i];
        const float igg = rr[i] * bb[i] - rb[i] * rb[i];
        const float igb = rb[i] * rg[i] - rr[i] * gb[i];
        const float ibb = rr[i] * gg[i] - rg[i] * rg[i];
        const float det = (irr * rr[i] + irg * rg[i]) + irb * rb[i];
        g->inv[0][i] = irr / det; g->inv[1][i] = irg / det; g->inv[2][i] = irb / det;
        g->inv[3][i] = igg / det; g->inv[4][i] = igb / det; g->inv[5][i] = ibb / det;
    }
    for (int v = 0; v < 6; ++v) free(var[v]);
    free(t);
}

static void fgf_upsample(const fgf_guide* g, const float* lo, float* full, float* tmp /* h2 x W */)
{
    const int W = g->W, H = g->H, w2 = g->w2, h2 = g->h2;
    for (int y = 0; y < h2; ++y)
        for (int x = 0; x < W; ++x)
            tmp[(size_t)y * W + x] = lo[(size_t)y * w2 + g->lx0[x]] * (1.f - g->fx[x]) + lo[(size_t)y * w2 + g->lx1[x]] * g->fx[x];
    for (int y = 0; y < H; ++y) {
        const float b0 = 1.f - g->fy[y], b1 = g->fy[y];
        const float *r0 = tmp + (size_t)g->ly0[y] * W, *r1 = tmp + (size_t)g->ly1[y] * W;
        for (int x = 0; x < W; ++x) full[(size_t)y * W + x] = r0[x] * b0 + r1[x] * b1;
    }
}

static void fgf_filter(const fgf_guide* g, float* p /* in place, full resolution */)
{
    const int W = g->W, H = g->H, w2 = g->w2, h2 = g->h2, K = g->K;
    const size_t n = (size_t)W * H, n2 = (size_t)w2 * h2;
    float *p2 = fnew(n2), *mp = fnew(n2), *t = fnew(n2), *mIp[3], *a[3], *b = fnew(n2), *tmp = fnew((size_t)h2 * W), *up = fnew(n), *q = fnew(n);
    for (int y = 0; y < h2; ++y) for (int x = 0; x < w2; ++x) p2[(size_t)y * w2 + x] = p[(size_t)g->ys[y] * W + g->xs[x]];
    orc_box_k(p2, w2, h2, K, mp);
    for (int k = 0; k < 3; ++k) {
        mIp[k] = fnew(n2); a[k] = fnew(n2);
        for (size_t i = 0; i < n2; ++i) t[i] = g->Ic[k][i] * p2[i];
        orc_box_k(t, w2, h2, K, mIp[k]);
    }
    for (size_t i = 0; i < n2; ++i) {
        const float c0 = mIp[0][i] - g->m[0][i] * mp[i], c1 = mIp[1][i] - g->m[1][i] * mp[i], c2 = mIp[2][i] - g->m[2][i] * mp[i];   /* :178-180 */
        const float ar = (g->inv[0][i] * c0 + g->inv[1][i] * c1) + g->inv[2][i] * c2;      /* :182-184 */
        const float ag = (g->inv[1][i] * c0 + g->inv[3][i] * c1) + g->inv[4][i] * c2;
        const float ab = (g->inv[2][i] * c0 + g->inv[4][i] * c1) + g->inv[5][i] * c2;
        a[0][i] = ar; a[1][i] = ag; a[2][i] = ab;
        b[i] = ((mp[i] - ar * g->m[0][i]) - ag * g->m[1][i]) - ab * g->m[2][i];             /* :186 */
    }
    for (int k = 0; k < 3; ++k) {
        orc_box_k(a[k], w2, h2, K, t);
        fgf_upsample(g, t, up, tmp);
        for (size_t i = 0; i < n; ++i) {
            const float prod = up[i] * g->orig[k][i];
            q[i] = k == 0 ? prod : q[i] + prod;                                              /* :196 (t1 + t2) + t3 */
        }
    }
    orc_box_k(b, w2, h2, K, t);
    fgf_upsample(g, t, up, tmp);
    for (size_t i = 0; i < n; ++i) p[i] = q[i] + up[i];
    for (int k = 0; k < 3; ++k) { free(mIp[k]); free(a[k]); }
    free(p2); free(mp); free(t); free(b); free(tmp); free(up); free(q);
}

typedef struct { const fgf_guide* g; float* slice; } fgf_task;
static void* fgf_thread(void* arg) { fgf_task* k = (fgf_task*)arg; fgf_filter(k->g, k->slice); return NULL; }

/* DispEst::CostFilter_FGF (DispEst.cpp:281-296; OpenMP over d there, `threads` pthreads here), volumes filtered in place */
int orc_cost_filter_fgf(const float* lImg, const float* rImg, int W, int H, int D, int threads, int s, int window, float eps,
                        float* lVol, float* rVol)
{
    if (s < 1 || W / s < 1 || H / s < 1) return -1;
    const float* imgs[2] = {lImg, rImg};
    float* vols[2] = {lVol, rVol};
    if (threads < 1) threads = 1;
    for (int v = 0; v < 2; ++v) {
        fgf_guide g;
        fgf_build(&g, imgs[v], W, H, s, window, eps);
        pthread_t* th = (pthread_t*)malloc((size_t)D * sizeof(pthread_t));
        fgf_task* tk = (fgf_task*)malloc((size_t)D * sizeof(fgf_task));
        for (int d0 = 0; d0 < D; d0 += threads) {
            const int nb = d0 + threads <= D ? threads : D - d0;
            for (int i = 0; i < nb; ++i) { tk[d0 + i].g = &g; tk[d0 + i].slice = vols[v] + (size_t)(d0 + i) * W * H; pthread_create(&th[d0 + i], NULL, fgf_thread, &tk[d0 + i]); }
            for (int i = 0; i < nb; ++i) pthread_join(th[d0 + i], NULL);
        }
        free(th); free(tk);
        fgf_free(&g);
    }
    return 0;
}
