/* pp_oracle.c -- CPU restatement of the post-filter at any psm_set_post_filter setting (TEST INFRASTRUCTURE; compiled
 * by tests/pp_oracle.py with -O3 -ffp-contract=off, the flags of the oracle build).
 *
 * JointWMF::filter(disp, img8UC3, r, sigma, 256, 256, iter, weightType) without the colour clustering, the definition
 * of DESIGN.md section 13:
 *   s = sigma / 256.0f * 64;  w(k) in float with the reference's operation order (JointWMF.h:620-648):
 *     exp: expf(-(float)k * (1.0f / ((2*s)*s)))   k = d0^2+d1^2+d2^2
 *     iv1: 1.0f / ((float)k + s)                  k = |d0|+|d1|+|d2|
 *     iv2: 1.0f / ((float)k + s*s)                k = d0^2+d1^2+d2^2
 *     off: 1.0f
 *   W(k) = lrintf((w(k) / w(0)) * 4194304.0f)
 *   out(p) = min { v : 2 * sum_{q in window, I_q <= v} W >= sum_{q in window} W }, window clipped at the border,
 *   u64 sums; each iteration filters the previous output with the original feature image (JointWMF.h:126-131).
 * At (9, 25.5, 1, exp) this is oracle/stereo_oracle.c's orc_wmf. */
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { WMF_EXP = 0, WMF_IV1 = 1, WMF_IV2 = 2, WMF_OFF = 5 };
#define PP_MAXD2 (3 * 63 * 63)

int pp_table_size(int type)
{
    return type == WMF_IV1 ? 3 * 63 + 1 : (type == WMF_OFF ? 1 : PP_MAXD2 + 1);
}

static float pp_w(int type, float s, int k)
{
    switch (type) {
    case WMF_EXP: return expf(-(float)k * (1.0f / ((2 * s) * s)));
    case WMF_IV1: return 1.0f / ((float)k + s);
    case WMF_IV2: return 1.0f / ((float)k + s * s);
    default: return 1.0f;
    }
}

/* t: room for pp_table_size(type) entries -> that number */
int pp_weight_table(float sigma, int type, uint32_t* t)
{
    const float s = sigma / 256.0f * 64;
    const float w0 = pp_w(type, s, 0);
    const int n = pp_table_size(type);
    for (int k = 0; k < n; ++k) t[k] = (uint32_t)lrintf((pp_w(type, s, k) / w0) * 4194304.0f);
    return n;
}

typedef struct {
    const uint8_t* disp;
    const uint8_t* img8;
    int W, H, r, type, y0, y1;
    const uint32_t* lut;
    uint8_t* out;
} pass_args;

static void* pass_rows(void* p)
{
    const pass_args* a = (const pass_args*)p;
    const int W = a->W, H = a->H, r = a->r;
    for (int y = a->y0; y < a->y1; ++y) {
        for (int x = 0; x < W; ++x) {
            uint64_t hist[256];
            memset(hist, 0, sizeof(hist));
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
            for (; v < 255; ++v) {
                cum += hist[v];
                if (2 * cum >= total) break;
            }
            a->out[(size_t)y * W + x] = (uint8_t)v;
        }
    }
    return NULL;
}

/* img8: interleaved BGR u8 feature image; disp, out: u8 maps (may alias) */
int pp_wmf(const uint8_t* disp, const uint8_t* img8, int W, int H, int r, float sigma, int iterations, int type,
           int threads, uint8_t* out)
{
    uint32_t* lut = (uint32_t*)malloc((PP_MAXD2 + 1) * sizeof(uint32_t));
    uint8_t* src = (uint8_t*)malloc((size_t)W * H);
    if (!lut || !src) { free(lut); free(src); return 1; }
    pp_weight_table(sigma, type, lut);
    memcpy(src, disp, (size_t)W * H);
    if (threads < 1) threads = 1;
    if (threads > 64) threads = 64;
    for (int it = 0; it < iterations; ++it) {
        pthread_t tid[64];
        pass_args args[64];
        for (int t = 0; t < threads; ++t) {
            args[t] = (pass_args){src, img8, W, H, r, type, (int)((long)H * t / threads), (int)((long)H * (t + 1) / threads), lut, out};
            pthread_create(&tid[t], NULL, pass_rows, &args[t]);
        }
        for (int t = 0; t < threads; ++t) pthread_join(tid[t], NULL);
        memcpy(src, out, (size_t)W * H);
    }
    free(lut);
    free(src);
    return 0;
}
