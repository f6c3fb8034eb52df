/* wide_oracle.c -- CPU restatement of the 16-bit-map stages (TEST INFRASTRUCTURE; compiled by tests/wide_oracle.py with
 * -O3 -ffp-contract=off, the flags of the oracle build).
 *
 * orc_wta16: DispSel::CVSelect (src/DispSel.cpp:83-109) with the arg-min kept as an int: over d in [1, D), strict <,
 *   ties -> lowest d, minCost starts at +inf, 0 when nothing compares below +inf.  The reference stores it into a uchar,
 *   so its map is this one's low byte.
 * orc_wmf16: the post-filter of tests/pp_oracle.c (DESIGN.md section 13) on u16 maps at any radius, sigma, iterations
 *   and weight type:
 *   out(p) = min { v : 2 * sum_{q in window, I_q <= v} W >= sum_{q in window} W }, window clipped at the border, u64
 *   sums, a direct histogram over [0, max value]; each iteration filters the previous output with the original
 *   feature image. */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { WMF_EXP = 0, WMF_IV1 = 1, WMF_IV2 = 2, WMF_OFF = 5 };
#define PP_MAXD2 (3 * 63 * 63)

void orc_wta16(const float* vol, int W, int H, int D, uint16_t* dis)
{
    const size_t plane = (size_t)W * H;
    for (size_t i = 0; i < plane; ++i) {
        float mc = INFINITY;
        int md = 0;
        for (int d = 1; d < D; ++d) {
            const float c = vol[(size_t)d * plane + i];
            if (c < mc) { mc = c; md = d; }
        }
        dis[i] = (uint16_t)md;
    }
}

static int table_size(int type) { return type == WMF_IV1 ? 3 * 63 + 1 : (type == WMF_OFF ? 1 : PP_MAXD2 + 1); }

static float wfun(int type, float s, int k)
{
    switch (type) {
    case WMF_EXP: return expf(-(float)k * (1.0f / ((2 * s) * s)));
    case WMF_IV1: return 1.0f / ((float)k + s);
    case WMF_IV2: return 1.0f / ((float)k + s * s);
    default: return 1.0f;
    }
}

typedef struct {
    const uint16_t* disp;
    const uint8_t* img8;
    int W, H, r, type, y0, y1, nbins;
    const uint32_t* lut;
    uint16_t* out;
} pass_args;

static void* pass_rows(void* p)
{
    const pass_args* a = (const pass_args*)p;
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
                    const int k = a->type == WMF_IV1 ? abs(d0) + abs(d1) + abs(d2)
                                : a->type == WMF_OFF ? 0 : d0 * d0 + d1 * d1 + d2 * d2;
                    const uint32_t w = a->lut[k];
                    hist[a->disp[(size_t)yy * W + xx]] += w;
                    total += w;
                }
            uint64_t cum = 0;
            int v = 0;
            for (; v < a->nbins - 1; ++v) {
                cum += hist[v];
                if (2 * cum >= total) break;
            }
            a->out[(size_t)y * W + x] = (uint16_t)v;
        }
    }
    free(hist);
    return NULL;
}

/* img8: interleaved BGR u8 feature image; disp, out: u16 maps (may alias) */
int orc_wmf16(const uint16_t* disp, const uint8_t* img8, int W, int H, int r, float sigma, int iterations, int type,
              int threads, uint16_t* out)
{
    const size_t n = (size_t)W * H;
    uint32_t* lut = (uint32_t*)malloc((PP_MAXD2 + 1) * sizeof(uint32_t));
    uint16_t* src = (uint16_t*)malloc(n * sizeof(uint16_t));
    if (!lut || !src) { free(lut); free(src); return 1; }
    const float s = sigma / 256.0f * 64;
    const float w0 = wfun(type, s, 0);
    for (int k = 0; k < table_size(type); ++k) lut[k] = (uint32_t)lrintf((wfun(type, s, k) / w0) * 4194304.0f);
    memcpy(src, disp, n * sizeof(uint16_t));
    int maxv = 0;
    for (size_t i = 0; i < n; ++i) maxv = src[i] > maxv ? src[i] : maxv;
    if (threads < 1) threads = 1;
    if (threads > 64) threads = 64;
    int rc = 0;
    for (int it = 0; it < iterations; ++it) {
        pthread_t tid[64];
        pass_args args[64];
        for (int t = 0; t < threads; ++t) {
            args[t] = (pass_args){src, img8, W, H, r, type, (int)((long)H * t / threads), (int)((long)H * (t + 1) / threads),
                                  maxv + 1, lut, out};
            pthread_create(&tid[t], NULL, pass_rows, &args[t]);
        }
        for (int t = 0; t < threads; ++t) {
            void* ret = NULL;
            pthread_join(tid[t], &ret);
            if (ret) rc = 1;
        }
        memcpy(src, out, n * sizeof(uint16_t));
    }
    free(lut);
    free(src);
    return rc;
}
