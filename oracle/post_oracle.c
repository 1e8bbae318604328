/*
 * post_oracle.c -- CPU ORACLE for the bloom + tonemap chain (TEST INFRASTRUCTURE ONLY).
 * Restates PathTracer/PostProcessor.cpp:128-246 and PathTracer/Shaders/PostProcess/
 * {BloomDownSample,BloomUpSample,Tonemap}.slang.  Quirks Q14, Q15 kept.
 */
#include "pt_oracle.h"
#include "orc_math.h"
#include <stdlib.h>
#include <string.h>

void orc_default_post_config(OrcPostConfig *c) {                 /* PT/PostProcessor.h:8-21 */
    c->Exposure = 1.0f; c->Gamma = 2.2f; c->BloomThreshold = 2.0f; c->BloomStrength = 1.0f; c->FalloffRange = 5.0f; c->MipCount = 10;
}

/* PT/PostProcessor.cpp:128-158 */
uint32_t orc_bloom_mip_sizes(uint32_t W, uint32_t H, uint32_t *wh) {
    uint32_t w = W, h = H, n = 0;
    for (uint32_t i = 0; i < 10; i++) {
        wh[2 * n] = w; wh[2 * n + 1] = h; n++;
        if (w % 2 != 0) w -= 1;
        if (h % 2 != 0) h -= 1;
        w /= 2; h /= 2;
        if (w < 2 || h < 2) break;
    }
    return n;
}

/* SH/PostProcess/Tonemap.slang:20-55 */
void orc_aces_fitted(const float in[3], float out[3]) {
    static const float I[3][3] = { {0.59719f, 0.35458f, 0.04823f}, {0.07600f, 0.90834f, 0.01566f}, {0.02840f, 0.13383f, 0.83777f} };
    static const float O[3][3] = { {1.60475f, -0.53108f, -0.07367f}, {-0.10208f, 1.10813f, -0.00605f}, {-0.00327f, -0.07276f, 1.07602f} };
    float c[3], r[3];
    for (int k = 0; k < 3; k++) c[k] = I[k][0] * in[0] + I[k][1] * in[1] + I[k][2] * in[2];
    for (int k = 0; k < 3; k++) {
        float v = c[k];
        float a = v * (v + 0.0245786f) - 0.000090537f;
        float b = v * (0.983729f * v + 0.4329510f) + 0.238081f;
        r[k] = a / b;
    }
    for (int k = 0; k < 3; k++) out[k] = orc_saturate(O[k][0] * r[0] + O[k][1] * r[1] + O[k][2] * r[2]);
}

static inline int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

void orc_post_process(const float *hdr, uint32_t W, uint32_t H, const OrcPostConfig *c,
                      uint8_t *ldr_out, float *bloom0_out, int nthreads) {
    (void)nthreads;
    uint32_t wh[20];
    uint32_t levels = orc_bloom_mip_sizes(W, H, wh);
    uint32_t mips = c->MipCount; if (mips < 1) mips = 1; if (mips > levels) mips = levels;   /* :195 */
    float *mip[10] = { 0 };
    for (uint32_t i = 0; i < levels; i++) mip[i] = (float *)calloc((size_t)wh[2 * i] * wh[2 * i + 1] * 4, sizeof(float));
    /* down pass 0: threshold (BloomDownSample.slang:32-45) */
    {
        float start = c->BloomThreshold - c->FalloffRange, end = c->BloomThreshold + c->FalloffRange;
        for (size_t p = 0; p < (size_t)W * H; p++) {
            const float *s = hdr + p * 4; float *d = mip[0] + p * 4;
            float br = s[0] * 0.2126f + s[1] * 0.7152f + s[2] * 0.0722f;
            float f = orc_smoothstep(start, end, br);
            d[0] = s[0] * f; d[1] = s[1] * f; d[2] = s[2] * f; d[3] = 1.0f;
        }
    }
    /* down passes i>=1 (BloomDownSample.slang:46-64) */
    for (uint32_t i = 1; i < mips; i++) {
        int iw = (int)wh[2 * (i - 1)], ih = (int)wh[2 * (i - 1) + 1], ow = (int)wh[2 * i], oh = (int)wh[2 * i + 1];
        const float *src = mip[i - 1]; float *dst = mip[i];
        for (int y = 0; y < oh; y++) for (int x = 0; x < ow; x++) {
            float acc[3] = { 0, 0, 0 };
            for (int a = -2; a < 2; a++) for (int b = -2; b < 2; b++) {
                int sx = clampi(x * 2 + a, 0, iw - 1), sy = clampi(y * 2 + b, 0, ih - 1);
                const float *s = src + ((size_t)sy * iw + sx) * 4;
                acc[0] += s[0]; acc[1] += s[1]; acc[2] += s[2];
            }
            float *d = dst + ((size_t)y * ow + x) * 4;
            for (int k = 0; k < 3; k++) d[k] = (acc[k] / 25.0f) * c->BloomStrength;   /* Q14 */
            d[3] = 1.0f;
        }
    }
    /* up passes (BloomUpSample.slang:21-48) */
    for (int i = (int)mips - 1; i > 0; i--) {
        int iw = (int)wh[2 * i], ih = (int)wh[2 * i + 1], ow = (int)wh[2 * (i - 1)], oh = (int)wh[2 * (i - 1) + 1];
        const float *src = mip[i]; float *dst = mip[i - 1];
        for (int y = 0; y < oh; y++) for (int x = 0; x < ow; x++) {
            float acc[3] = { 0, 0, 0 };
            for (int a = -2; a < 2; a++) for (int b = -2; b < 2; b++) {
                int sx = clampi(x / 2 + a + 1, 0, iw - 1), sy = clampi(y / 2 + b + 1, 0, ih - 1);
                const float *s = src + ((size_t)sy * iw + sx) * 4;
                acc[0] += s[0]; acc[1] += s[1]; acc[2] += s[2];
            }
            float *d = dst + ((size_t)y * ow + x) * 4;
            for (int k = 0; k < 3; k++) d[k] = (acc[k] / 25.0f) * c->BloomStrength + d[k];
            d[3] = 1.0f;
        }
    }
    if (bloom0_out) memcpy(bloom0_out, mip[0], (size_t)W * H * 4 * sizeof(float));
    /* tonemap (Tonemap.slang:159-175): bloom sampled bilinear, CLAMP_TO_EDGE, uv = xy/size (Q15) */
    {
        int iw = (int)W, ih = (int)H; const float *b0 = mip[0];
        float invGamma = 1.0f / c->Gamma;
        for (int y = 0; y < ih; y++) for (int x = 0; x < iw; x++) {
            float u = (float)x / (float)W, v = (float)y / (float)H;
            float fxp = u * (float)W - 0.5f, fyp = v * (float)H - 0.5f;
            float fx = floorf(fxp), fy = floorf(fyp);
            float ax = fxp - fx, ay = fyp - fy;
            int x0 = clampi((int)fx, 0, iw - 1), x1 = clampi((int)fx + 1, 0, iw - 1);
            int y0 = clampi((int)fy, 0, ih - 1), y1 = clampi((int)fy + 1, 0, ih - 1);
            const float *h4 = hdr + ((size_t)y * W + x) * 4;
            float col[3];
            for (int k = 0; k < 3; k++) {
                float t00 = b0[((size_t)y0 * iw + x0) * 4 + k], t10 = b0[((size_t)y0 * iw + x1) * 4 + k];
                float t01 = b0[((size_t)y1 * iw + x0) * 4 + k], t11 = b0[((size_t)y1 * iw + x1) * 4 + k];
                float top = t00 + ax * (t10 - t00), bot = t01 + ax * (t11 - t01);
                float bl = top + ay * (bot - top);
                float cc = h4[k] + bl;
                cc = cc * c->Exposure;
                col[k] = cc > 0.0f ? powf(cc, invGamma) : (cc == 0.0f ? 0.0f : NAN);   /* Q18: exp2(y log2 x): pow(0, y) = 0, pow(x < 0, y) = NaN */
            }
            float outc[3];
            orc_aces_fitted(col, outc);
            uint8_t *o = ldr_out + ((size_t)y * W + x) * 4;
            for (int k = 0; k < 3; k++) {
                float q = outc[k];                       /* RGBA8 UNORM store: saturate, *255, round-half-even */
                if (!(q > 0.0f)) q = 0.0f;               /* NaN -> 0 */
                if (q > 1.0f) q = 1.0f;
                o[k] = (uint8_t)rintf(q * 255.0f);
            }
            o[3] = 255;
        }
    }
    for (uint32_t i = 0; i < levels; i++) free(mip[i]);
}
