/*
 * ggml_oracle.c -- CPU restatement of the reference's quantized-inference hot path (see ggml_oracle.h).
 *
 * TEST INFRASTRUCTURE ONLY: the checker for the CUDA path, never the thing measured or shipped.
 *
 * Written from the reference's behaviour (file:line cited per function, paths under /root/reference);
 * scalar C, no SIMD.  Must be compiled WITHOUT fp contraction / fast-math (oracle/Makefile) because the
 * reference is built with -std=c11, which disables a*b+c fusing, and the codecs are bit-exact contracts.
 */
#include "ggml_oracle.h"
#include <math.h>
#include <float.h>
#include <stdlib.h>
#include <string.h>
#include <pthread.h>

#define QK 32      /* legacy block: QK4_0 .. QK8_1, ggml.c:878-921 */
#define SB 256     /* K-quant super-block: QK_K, k_quants.h:15       */

static inline int imin(int a, int b) { return a < b ? a : b; }
static inline int imax(int a, int b) { return a > b ? a : b; }

/* ------------------------------------------------------------------------------------------------
 * fp16 conversion.  The reference uses F16C (_cvtss_sh(x,0) / _cvtsh_ss) on x86 (ggml.c:349-360):
 * IEEE round-to-nearest-even, subnormals kept, overflow -> inf.
 * ---------------------------------------------------------------------------------------------- */
float orc_f16_to_f32(uint16_t h) {
    uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
    uint32_t exp = (h >> 10) & 0x1f, man = h & 0x3ffu, bits;
    if (exp == 0) {
        if (man == 0) bits = sign;
        else { /* subnormal: normalise */
            int e = -1;
            do { man <<= 1; e++; } while (!(man & 0x400u));
            bits = sign | ((uint32_t)(127 - 15 - e) << 23) | ((man & 0x3ffu) << 13);
        }
    } else if (exp == 31) bits = sign | 0x7f800000u | (man << 13);
    else bits = sign | ((exp + 112) << 23) | (man << 13);
    float f; memcpy(&f, &bits, 4); return f;
}

uint16_t orc_f32_to_f16(float f) {
    uint32_t x; memcpy(&x, &f, 4);
    uint16_t sign = (uint16_t)((x >> 16) & 0x8000u);
    uint32_t ax = x & 0x7fffffffu;
    if (ax >= 0x7f800000u) return (uint16_t)(sign | 0x7c00u | (ax > 0x7f800000u ? (0x200u | ((ax >> 13) & 0x3ffu)) : 0)); /* inf / nan */
    if (ax >= 0x477ff000u) return (uint16_t)(sign | 0x7c00u);            /* >= 65520 rounds to inf */
    if (ax < 0x33000001u) return sign;                                   /* < 2^-25 (or == 2^-25 tie -> 0) */
    int e = (int)(ax >> 23) - 127;
    uint32_t m = (ax & 0x7fffffu) | 0x800000u;
    int shift;                       /* bits to drop from the 24-bit significand */
    uint32_t hexp;
    if (e < -14) { shift = 13 + (-14 - e); hexp = 0; }   /* result subnormal */
    else { shift = 13; hexp = (uint32_t)(e + 15); }
    uint32_t q = m >> shift, rem = m & ((1u << shift) - 1u), half = 1u << (shift - 1);
    if (rem > half || (rem == half && (q & 1u))) q++;
    uint32_t out = (hexp == 0) ? q : ((hexp << 10) + (q - 0x400u));     /* carry propagates into the exponent */
    return (uint16_t)(sign | out);
}

/* ------------------------------------------------------------------------------------------------ */
int orc_block_elems(int t) {
    switch (t) {
        case ORC_F32: case ORC_F16: return 1;
        case ORC_Q4_0: case ORC_Q4_1: case ORC_Q5_0: case ORC_Q5_1: case ORC_Q8_0: case ORC_Q8_1: return QK;
        case ORC_Q2_K: case ORC_Q3_K: case ORC_Q4_K: case ORC_Q5_K: case ORC_Q6_K: case ORC_Q8_K: return SB;
    }
    return 0;
}
size_t orc_block_bytes(int t) {
    switch (t) {
        case ORC_F32: return 4; case ORC_F16: return 2;
        case ORC_Q4_0: return 18; case ORC_Q4_1: return 20; case ORC_Q5_0: return 22; case ORC_Q5_1: return 24;
        case ORC_Q8_0: return 34; case ORC_Q8_1: return 40;
        case ORC_Q2_K: return 84; case ORC_Q3_K: return 110; case ORC_Q4_K: return 144; case ORC_Q5_K: return 176;
        case ORC_Q6_K: return 210; case ORC_Q8_K: return 292;
    }
    return 0;
}
size_t orc_row_bytes(int t, int64_t k) { int e = orc_block_elems(t); return e ? (size_t)(k / e) * orc_block_bytes(t) : 0; }
int orc_vec_dot_type(int t) {
    switch (t) {
        case ORC_Q4_0: case ORC_Q5_0: case ORC_Q8_0: return ORC_Q8_0;
        case ORC_Q4_1: case ORC_Q5_1: return ORC_Q8_1;
        case ORC_Q2_K: case ORC_Q3_K: case ORC_Q4_K: case ORC_Q5_K: case ORC_Q6_K: return ORC_Q8_K;
    }
    return -1;
}

/* byte-level accessors: the block structs are packed (no padding), so plain offsets are used */
static inline uint16_t ld16(const uint8_t *p) { uint16_t v; memcpy(&v, p, 2); return v; }
static inline void     st16(uint8_t *p, uint16_t v) { memcpy(p, &v, 2); }
static inline float    ldf(const uint8_t *p) { float v; memcpy(&v, p, 4); return v; }
static inline void     stf(uint8_t *p, float v) { memcpy(p, &v, 4); }

/* round-half-even to int via the 1.5*2^23 magic constant: nearest_int, k_quants.c:50-55 */
static inline int rne_int(float v) {
    float t = v + 12582912.f; int32_t i; memcpy(&i, &t, 4);
    return (i & 0x007fffff) - 0x00400000;
}

/* =================================== legacy 32-element codecs ================================== */
/* block_q4_0 {f16 d; u8 qs[16]}: ggml.c:879-884, quantize 927-962, dequantize 1509-1527 */
static void q4_0_enc(const float *x, uint8_t *y, int64_t k) {
    for (int64_t b = 0; b < k / QK; b++, x += QK, y += 18) {
        float amax = 0.f, vmax = 0.f;
        for (int j = 0; j < QK; j++) if (amax < fabsf(x[j])) { amax = fabsf(x[j]); vmax = x[j]; }
        const float d = vmax / -8, id = d ? 1.0f / d : 0.0f;
        st16(y, orc_f32_to_f16(d));
        for (int j = 0; j < QK / 2; j++) {
            uint8_t lo = (uint8_t)imin(15, (int8_t)(x[j] * id + 8.5f));
            uint8_t hi = (uint8_t)imin(15, (int8_t)(x[j + QK / 2] * id + 8.5f));
            y[2 + j] = (uint8_t)(lo | (hi << 4));
        }
    }
}
static void q4_0_dec(const uint8_t *x, float *y, int64_t k) {
    for (int64_t b = 0; b < k / QK; b++, x += 18, y += QK) {
        const float d = orc_f16_to_f32(ld16(x));
        for (int j = 0; j < QK / 2; j++) {
            y[j] = ((x[2 + j] & 0x0F) - 8) * d;
            y[j + QK / 2] = ((x[2 + j] >> 4) - 8) * d;
        }
    }
}
/* block_q4_1 {f16 d, m; u8 qs[16]}: ggml.c:886-892, 968-1002, 1529-1547 */
static void q4_1_enc(const float *x, uint8_t *y, int64_t k) {
    for (int64_t b = 0; b < k / QK; b++, x += QK, y += 20) {
        float mn = FLT_MAX, mx = -FLT_MAX;
        for (int j = 0; j < QK; j++) { if (x[j] < mn) mn = x[j]; if (x[j] > mx) mx = x[j]; }
        const float d = (mx - mn) / 15, id = d ? 1.0f / d : 0.0f;
        st16(y, orc_f32_to_f16(d)); st16(y + 2, orc_f32_to_f16(mn));
        for (int j = 0; j < QK / 2; j++) {
            uint8_t lo = (uint8_t)imin(15, (int8_t)((x[j] - mn) * id + 0.5f));
            uint8_t hi = (uint8_t)imin(15, (int8_t)((x[j + QK / 2] - mn) * id + 0.5f));
            y[4 + j] = (uint8_t)(lo | (hi << 4));
        }
    }
}
static void q4_1_dec(const uint8_t *x, float *y, int64_t k) {
    for (int64_t b = 0; b < k / QK; b++, x += 20, y += QK) {
        const float d = orc_f16_to_f32(ld16(x)), m = orc_f16_to_f32(ld16(x + 2));
        for (int j = 0; j < QK / 2; j++) {
            y[j] = (x[4 + j] & 0x0F) * d + m;
            y[j + QK / 2] = (x[4 + j] >> 4) * d + m;
        }
    }
}
/* block_q5_0 {f16 d; u8 qh[4]; u8 qs[16]}: ggml.c:894-900, 1008-1046, 1549-1573 */
static void q5_0_enc(const float *x, uint8_t *y, int64_t k) {
    for (int64_t b = 0; b < k / QK; b++, x += QK, y += 22) {
        float amax = 0.f, vmax = 0.f;
        for (int j = 0; j < QK; j++) if (amax < fabsf(x[j])) { amax = fabsf(x[j]); vmax = x[j]; }
        const float d = vmax / -16, id = d ? 1.0f / d : 0.0f;
        st16(y, orc_f32_to_f16(d));
        uint32_t qh = 0;
        for (int j = 0; j < QK / 2; j++) {
            uint8_t lo = (uint8_t)imin(31, (int8_t)(x[j] * id + 16.5f));
            uint8_t hi = (uint8_t)imin(31, (int8_t)(x[j + QK / 2] * id + 16.5f));
            y[6 + j] = (uint8_t)((lo & 0x0F) | ((hi & 0x0F) << 4));
            qh |= (uint32_t)((lo & 0x10) >> 4) << j;
            qh |= (uint32_t)((hi & 0x10) >> 4) << (j + QK / 2);
        }
        memcpy(y + 2, &qh, 4);
    }
}
static void q5_0_dec(const uint8_t *x, float *y, int64_t k) {
    for (int64_t b = 0; b < k / QK; b++, x += 22, y += QK) {
        const float d = orc_f16_to_f32(ld16(x));
        uint32_t qh; memcpy(&qh, x + 2, 4);
        for (int j = 0; j < QK / 2; j++) {
            int lo = ((x[6 + j] & 0x0F) | (((qh >> j) << 4) & 0x10)) - 16;
            int hi = ((x[6 + j] >> 4) | ((qh >> (j + 12)) & 0x10)) - 16;
            y[j] = lo * d; y[j + QK / 2] = hi * d;
        }
    }
}
/* block_q5_1 {f16 d, m; u8 qh[4]; u8 qs[16]}: ggml.c:902-909, 1052-1090, 1575-1600 */
static void q5_1_enc(const float *x, uint8_t *y, int64_t k) {
    for (int64_t b = 0; b < k / QK; b++, x += QK, y += 24) {
        float mn = FLT_MAX, mx = -FLT_MAX;
        for (int j = 0; j < QK; j++) { if (x[j] < mn) mn = x[j]; if (x[j] > mx) mx = x[j]; }
        const float d = (mx - mn) / 31, id = d ? 1.0f / d : 0.0f;
        st16(y, orc_f32_to_f16(d)); st16(y + 2, orc_f32_to_f16(mn));
        uint32_t qh = 0;
        for (int j = 0; j < QK / 2; j++) {
            uint8_t lo = (uint8_t)((x[j] - mn) * id + 0.5f);
            uint8_t hi = (uint8_t)((x[j + QK / 2] - mn) * id + 0.5f);
            y[8 + j] = (uint8_t)((lo & 0x0F) | ((hi & 0x0F) << 4));
            qh |= (uint32_t)((lo & 0x10) >> 4) << j;
            qh |= (uint32_t)((hi & 0x10) >> 4) << (j + QK / 2);
        }
        memcpy(y + 4, &qh, 4);
    }
}
static void q5_1_dec(const uint8_t *x, float *y, int64_t k) {
    for (int64_t b = 0; b < k / QK; b++, x += 24, y += QK) {
        const float d = orc_f16_to_f32(ld16(x)), m = orc_f16_to_f32(ld16(x + 2));
        uint32_t qh; memcpy(&qh, x + 4, 4);
        for (int j = 0; j < QK / 2; j++) {
            int lo = (x[8 + j] & 0x0F) | (((qh >> j) << 4) & 0x10);
            int hi = (x[8 + j] >> 4) | ((qh >> (j + 12)) & 0x10);
            y[j] = lo * d + m; y[j + QK / 2] = hi * d + m;
        }
    }
}
/* block_q8_0 {f16 d; i8 qs[32]}: ggml.c:911-916; scalar reference 1106-1129 (roundf), dequantize 1602-1619 */
static void q8_0_enc_ref(const float *x, uint8_t *y, int64_t k) {
    for (int64_t b = 0; b < k / QK; b++, x += QK, y += 34) {
        float amax = 0.f;
        for (int j = 0; j < QK; j++) amax = fabsf(x[j]) > amax ? fabsf(x[j]) : amax;
        const float d = amax / 127, id = d ? 1.0f / d : 0.0f;
        st16(y, orc_f32_to_f16(d));
        for (int j = 0; j < QK; j++) ((int8_t *)y)[2 + j] = (int8_t)roundf(x[j] * id);
    }
}
/* the AVX/AVX2 body the mat-mul really runs on x86, ggml.c:1201-1237 */
void orc_quantize_row_q8_0_x86(const float *x, void *vy, int64_t k) {
    uint8_t *y = (uint8_t *)vy;
    for (int64_t b = 0; b < k / QK; b++, x += QK, y += 34) {
        float amax = 0.f;
        for (int j = 0; j < QK; j++) amax = fabsf(x[j]) > amax ? fabsf(x[j]) : amax;
        st16(y, orc_f32_to_f16(amax / 127.f));
        const float id = (amax != 0.0f) ? 127.f / amax : 0.0f;
        for (int j = 0; j < QK; j++) ((int8_t *)y)[2 + j] = (int8_t)rne_int(x[j] * id);  /* |x*id| <= 127: rne_int == cvtps(round) */
    }
}
static void q8_0_dec(const uint8_t *x, float *y, int64_t k) {
    for (int64_t b = 0; b < k / QK; b++, x += 34, y += QK) {
        const float d = orc_f16_to_f32(ld16(x));
        for (int j = 0; j < QK; j++) y[j] = ((const int8_t *)x)[2 + j] * d;
    }
}
/* block_q8_1 {f32 d; f32 s = d*sum(qs); i8 qs[32]}: ggml.c:918-924; scalar reference 1292-1325 */
static void q8_1_enc_ref(const float *x, uint8_t *y, int64_t k) {
    for (int64_t b = 0; b < k / QK; b++, x += QK, y += 40) {
        float amax = 0.f;
        for (int j = 0; j < QK; j++) amax = fabsf(x[j]) > amax ? fabsf(x[j]) : amax;
        const float d = amax / 127, id = d ? 1.0f / d : 0.0f;
        stf(y, d);
        int sum = 0;
        for (int j = 0; j < QK; j++) { int8_t q = (int8_t)roundf(x[j] * id); ((int8_t *)y)[8 + j] = q; sum += q; }
        stf(y + 4, sum * d);
    }
}
/* AVX2 body, ggml.c:1421-1470: id = 127/amax, round-half-even, s = d * sum */
void orc_quantize_row_q8_1_x86(const float *x, void *vy, int64_t k) {
    uint8_t *y = (uint8_t *)vy;
    for (int64_t b = 0; b < k / QK; b++, x += QK, y += 40) {
        float amax = 0.f;
        for (int j = 0; j < QK; j++) amax = fabsf(x[j]) > amax ? fabsf(x[j]) : amax;
        const float d = amax / 127.f, id = (amax != 0.0f) ? 127.f / amax : 0.0f;
        stf(y, d);
        int sum = 0;
        for (int j = 0; j < QK; j++) { int q = rne_int(x[j] * id); ((int8_t *)y)[8 + j] = (int8_t)q; sum += q; }
        stf(y + 4, d * (float)sum);
    }
}

/* =================================== K-quant helpers =========================================== */
/* make_qkx1_quants, k_quants.c:222-262: asymmetric (scale,min) fit of n values to levels 0..nmax */
static float fit_scale_min(int n, int nmax, const float *x, uint8_t *L, float *the_min, int ntry) {
    float mn = x[0], mx = x[0];
    for (int i = 1; i < n; i++) { if (x[i] < mn) mn = x[i]; if (x[i] > mx) mx = x[i]; }
    if (mx == mn) { for (int i = 0; i < n; i++) L[i] = 0; *the_min = 0; return 0.f; }
    if (mn > 0) mn = 0;
    float iscale = nmax / (mx - mn), scale = 1 / iscale;
    for (int t = 0; t < ntry; t++) {
        float sumlx = 0; int suml2 = 0; int changed = 0;
        for (int i = 0; i < n; i++) {
            int l = imax(0, imin(nmax, rne_int(iscale * (x[i] - mn))));
            if (l != L[i]) { L[i] = (uint8_t)l; changed = 1; }
            sumlx += (x[i] - mn) * l; suml2 += l * l;
        }
        scale = sumlx / suml2;
        float sum = 0;
        for (int i = 0; i < n; i++) sum += x[i] - scale * L[i];
        mn = sum / n; if (mn > 0) mn = 0;
        iscale = 1 / scale;
        if (!changed) break;
    }
    *the_min = -mn;
    return scale;
}
/* make_q3_quants (do_rmse = true branch), k_quants.c:163-220 */
static float fit_scale_q3(int n, int nmax, const float *x, int8_t *L) {
    float vmax = 0, amax = 0;
    for (int i = 0; i < n; i++) { float ax = fabsf(x[i]); if (ax > amax) { amax = ax; vmax = x[i]; } }
    if (!amax) { for (int i = 0; i < n; i++) L[i] = 0; return 0.f; }
    float iscale = -nmax / vmax, sumlx = 0, suml2 = 0;
    for (int i = 0; i < n; i++) {
        int l = imax(-nmax, imin(nmax - 1, rne_int(iscale * x[i])));
        L[i] = (int8_t)l;
        float w = x[i] * x[i];
        sumlx += w * x[i] * l; suml2 += w * l * l;
    }
    for (int t = 0; t < 5; t++) {
        int nchg = 0;
        for (int i = 0; i < n; i++) {
            float w = x[i] * x[i];
            float slx = sumlx - w * x[i] * L[i];
            if (slx > 0) {
                float sl2 = suml2 - w * L[i] * L[i];
                int nl = imax(-nmax, imin(nmax - 1, rne_int(x[i] * sl2 / slx)));
                if (nl != L[i]) {
                    slx += w * x[i] * nl; sl2 += w * nl * nl;
                    if (sl2 > 0 && slx * slx * suml2 > sumlx * sumlx * sl2) { L[i] = (int8_t)nl; sumlx = slx; suml2 = sl2; nchg++; }
                }
            }
        }
        if (!nchg) break;
    }
    for (int i = 0; i < n; i++) L[i] = (int8_t)(L[i] + nmax);
    return sumlx / suml2;
}
/* make_qx_quants with rmse_type == 1 (the only mode q6_K uses), k_quants.c:57-161 */
static float fit_scale_sym(int n, int nmax, const float *x, int8_t *L) {
    float vmax = 0, amax = 0;
    for (int i = 0; i < n; i++) { float ax = fabsf(x[i]); if (ax > amax) { amax = ax; vmax = x[i]; } }
    if (!amax) { for (int i = 0; i < n; i++) L[i] = 0; return 0.f; }
    float iscale = -nmax / vmax, sumlx = 0, suml2 = 0;
    for (int i = 0; i < n; i++) {
        int l = imax(-nmax, imin(nmax - 1, rne_int(iscale * x[i])));
        L[i] = (int8_t)(l + nmax);
        float w = x[i] * x[i];
        sumlx += w * x[i] * l; suml2 += w * l * l;
    }
    float scale = sumlx / suml2, best = scale * sumlx;
    for (int t = 0; t < 3; t++) {
        iscale = 1 / scale;
        float slx = 0, sl2 = 0; int changed = 0;
        for (int i = 0; i < n; i++) {
            int l = imax(-nmax, imin(nmax - 1, rne_int(iscale * x[i])));
            if (l + nmax != L[i]) changed = 1;
            float w = x[i] * x[i];
            slx += w * x[i] * l; sl2 += w * l * l;
        }
        if (!changed || sl2 == 0 || slx * slx <= best * sl2) break;
        for (int i = 0; i < n; i++) L[i] = (int8_t)(nmax + imax(-nmax, imin(nmax - 1, rne_int(iscale * x[i]))));
        sumlx = slx; suml2 = sl2; scale = sumlx / suml2; best = scale * sumlx;
    }
    for (int t = 0; t < 5; t++) {
        int nchg = 0;
        for (int i = 0; i < n; i++) {
            float w = x[i] * x[i];
            int l = L[i] - nmax;
            float slx = sumlx - w * x[i] * l;
            if (slx > 0) {
                float sl2 = suml2 - w * l * l;
                int nl = imax(-nmax, imin(nmax - 1, rne_int(x[i] * sl2 / slx)));
                if (nl != l) {
                    slx += w * x[i] * nl; sl2 += w * nl * nl;
                    if (sl2 > 0 && slx * slx * suml2 > sumlx * sumlx * sl2) {
                        L[i] = (int8_t)(nmax + nl); sumlx = slx; suml2 = sl2;
                        scale = sumlx / suml2; best = scale * sumlx; nchg++;
                    }
                }
            }
        }
        if (!nchg) break;
    }
    (void)best;
    return scale;
}
/* 6-bit (scale, min) pair j of the 12-byte packed field: get_scale_min_k4, k_quants.c:264-271 */
static inline void unpack_sm6(int j, const uint8_t *q, uint8_t *sc, uint8_t *mn) {
    if (j < 4) { *sc = q[j] & 63; *mn = q[j + 4] & 63; }
    else { *sc = (uint8_t)((q[j + 4] & 0xF) | ((q[j - 4] >> 6) << 4)); *mn = (uint8_t)((q[j + 4] >> 4) | ((q[j] >> 6) << 4)); }
}
static void pack_sm6(int j, uint8_t *q, uint8_t ls, uint8_t lm) {   /* k_quants.c:565-578 */
    if (j < 4) { q[j] = ls; q[j + 4] = lm; }
    else { q[j + 4] = (uint8_t)((ls & 0xF) | ((lm & 0xF) << 4)); q[j - 4] |= (uint8_t)((ls >> 4) << 6); q[j] |= (uint8_t)((lm >> 4) << 6); }
}
/* the sixteen signed 6-bit scales of q3_K (bias 32 NOT removed): k_quants.c:486-493 */
static void unpack_q3_scales(const uint8_t *packed, int8_t out[16]) {
    uint32_t a[4]; memcpy(a, packed, 12);
    const uint32_t m3 = 0x03030303u, m4 = 0x0f0f0f0fu, t = a[2];
    a[2] = ((a[0] >> 4) & m4) | (((t >> 4) & m3) << 4);
    a[3] = ((a[1] >> 4) & m4) | (((t >> 6) & m3) << 4);
    a[0] = (a[0] & m4) | (((t >> 0) & m3) << 4);
    a[1] = (a[1] & m4) | (((t >> 2) & m3) << 4);
    memcpy(out, a, 16);
}

/* =================================== Q2_K ====================================================== */
/* block_q2_K {u8 scales[16]; u8 qs[64]; f16 d, dmin}: k_quants.h:20-26; quantize k_quants.c:275-342 */
/* make_qkx1_quants (Q2_K, Q4_K, Q5_K) ends its refinement after a round that leaves L unchanged, and its round 0 compares
 * against what L already holds: the reference declares L once per call, so block b starts from block b-1's final codes.  That
 * chaining is restated here.  For block 0 the reference reads uninitialised stack; here it reads zeros.  fresh != 0 zeroes L
 * at every block instead, which is what a quantiser that treats blocks independently computes. */
static void q2_K_enc(const float *x, uint8_t *y, int64_t k, int fresh) {
    uint8_t L[SB] = {0}; float mins[16], scales[16];
    for (int64_t b = 0; b < k / SB; b++, x += SB, y += 84) {
        if (fresh) memset(L, 0, sizeof L);
        uint8_t *sc = y, *qs = y + 16;
        float max_scale = 0, max_min = 0;
        for (int j = 0; j < 16; j++) {
            scales[j] = fit_scale_min(16, 3, x + 16 * j, L + 16 * j, &mins[j], 5);
            if (scales[j] > max_scale) max_scale = scales[j];
            if (mins[j] > max_min) max_min = mins[j];
        }
        if (max_scale > 0) {
            float is = 15.f / max_scale;
            for (int j = 0; j < 16; j++) sc[j] = (uint8_t)rne_int(is * scales[j]);
            st16(y + 80, orc_f32_to_f16(max_scale / 15.f));
        } else { memset(sc, 0, 16); st16(y + 80, orc_f32_to_f16(0.f)); }
        if (max_min > 0) {
            float is = 15.f / max_min;
            for (int j = 0; j < 16; j++) sc[j] |= (uint8_t)(rne_int(is * mins[j]) << 4);
            st16(y + 82, orc_f32_to_f16(max_min / 15.f));
        } else st16(y + 82, orc_f32_to_f16(0.f));
        const float fd = orc_f16_to_f32(ld16(y + 80)), fm = orc_f16_to_f32(ld16(y + 82));
        for (int j = 0; j < 16; j++) {
            const float d = fd * (sc[j] & 0xF);
            if (!d) continue;
            const float dm = fm * (sc[j] >> 4);
            for (int i = 0; i < 16; i++) L[16 * j + i] = (uint8_t)imax(0, imin(3, rne_int((x[16 * j + i] + dm) / d)));
        }
        for (int j = 0; j < SB; j += 128)
            for (int l = 0; l < 32; l++)
                qs[j / 4 + l] = (uint8_t)(L[j + l] | (L[j + l + 32] << 2) | (L[j + l + 64] << 4) | (L[j + l + 96] << 6));
    }
}
/* k_quants.c:344-378 */
static void q2_K_dec(const uint8_t *x, float *y, int64_t k) {
    for (int64_t b = 0; b < k / SB; b++, x += 84) {
        const float d = orc_f16_to_f32(ld16(x + 80)), mn = orc_f16_to_f32(ld16(x + 82));
        const uint8_t *q = x + 16; int is = 0;
        for (int n = 0; n < SB; n += 128, q += 32)
            for (int shift = 0; shift < 8; shift += 2)
                for (int half = 0; half < 2; half++) {
                    uint8_t s = x[is++];
                    float dl = d * (s & 0xF), ml = mn * (s >> 4);
                    for (int l = 0; l < 16; l++) *y++ = dl * ((int8_t)((q[l + 16 * half] >> shift) & 3)) - ml;
                }
    }
}
/* =================================== Q3_K ====================================================== */
/* block_q3_K {u8 hmask[32]; u8 qs[64]; u8 scales[12]; f16 d}: k_quants.h:32-37; quantize k_quants.c:396-470 */
static void q3_K_enc(const float *x, uint8_t *y, int64_t k) {
    int8_t L[SB]; float scales[16];
    for (int64_t b = 0; b < k / SB; b++, x += SB, y += 110) {
        uint8_t *hm = y, *qs = y + 32, *sc = y + 96;
        float max_scale = 0, amax = 0;
        for (int j = 0; j < 16; j++) {
            scales[j] = fit_scale_q3(16, 4, x + 16 * j, L + 16 * j);
            float a = fabsf(scales[j]);
            if (a > amax) { amax = a; max_scale = scales[j]; }
        }
        memset(sc, 0, 12);
        if (max_scale) {
            float is = -32.f / max_scale;
            for (int j = 0; j < 16; j++) {
                int8_t l = (int8_t)rne_int(is * scales[j]);
                l = (int8_t)(imax(-32, imin(31, l)) + 32);
                if (j < 8) sc[j] = (uint8_t)(l & 0xF); else sc[j - 8] |= (uint8_t)((l & 0xF) << 4);
                l >>= 4;
                sc[j % 4 + 8] |= (uint8_t)(l << (2 * (j / 4)));
            }
            st16(y + 108, orc_f32_to_f16(1 / is));
        } else st16(y + 108, orc_f32_to_f16(0.f));
        const float fd = orc_f16_to_f32(ld16(y + 108));
        for (int j = 0; j < 16; j++) {
            int8_t s = (int8_t)(j < 8 ? sc[j] & 0xF : sc[j - 8] >> 4);
            s = (int8_t)((s | (((sc[8 + j % 4] >> (2 * (j / 4))) & 3) << 4)) - 32);
            float d = fd * s;
            if (!d) continue;
            for (int i = 0; i < 16; i++) L[16 * j + i] = (int8_t)(imax(-4, imin(3, rne_int(x[16 * j + i] / d))) + 4);
        }
        memset(hm, 0, 32);
        for (int j = 0; j < SB; j++) if (L[j] > 3) { hm[j % 32] |= (uint8_t)(1u << (j / 32)); L[j] -= 4; }
        for (int j = 0; j < SB; j += 128)
            for (int l = 0; l < 32; l++)
                qs[j / 4 + l] = (uint8_t)(L[j + l] | (L[j + l + 32] << 2) | (L[j + l + 64] << 4) | (L[j + l + 96] << 6));
    }
}
/* k_quants.c:472-521 */
static void q3_K_dec(const uint8_t *x, float *y, int64_t k) {
    int8_t sc[16];
    for (int64_t b = 0; b < k / SB; b++, x += 110) {
        const float d_all = orc_f16_to_f32(ld16(x + 108));
        const uint8_t *hm = x, *q = x + 32;
        unpack_q3_scales(x + 96, sc);
        int is = 0; uint8_t m = 1;
        for (int n = 0; n < SB; n += 128, q += 32)
            for (int shift = 0; shift < 8; shift += 2, m <<= 1)
                for (int half = 0; half < 2; half++) {
                    float dl = d_all * (sc[is++] - 32);
                    for (int l = 16 * half; l < 16 * half + 16; l++)
                        *y++ = dl * ((int8_t)((q[l] >> shift) & 3) - ((hm[l] & m) ? 0 : 4));
                }
    }
}
/* =================================== Q4_K / Q5_K =============================================== */
/* block_q4_K {f16 d, dmin; u8 scales[12]; u8 qs[128]}: k_quants.h:44-49; quantize k_quants.c:542-605
 * block_q5_K {f16 d, dmin; u8 scales[12]; u8 qh[32]; u8 qs[128]}: k_quants.h:56-63; quantize k_quants.c:652-732 */
static void q45_K_enc(const float *x, uint8_t *y, int64_t k, int bits, int fresh) {   /* L chained as in q2_K_enc */
    const int nmax = (1 << bits) - 1; const size_t bsz = bits == 4 ? 144 : 176;
    uint8_t L[SB] = {0}; float mins[8], scales[8];
    for (int64_t b = 0; b < k / SB; b++, x += SB, y += bsz) {
        if (fresh) memset(L, 0, sizeof L);
        uint8_t *sc = y + 4;
        float max_scale = 0, max_min = 0;
        for (int j = 0; j < 8; j++) {
            scales[j] = fit_scale_min(32, nmax, x + 32 * j, L + 32 * j, &mins[j], 5);
            if (scales[j] > max_scale) max_scale = scales[j];
            if (mins[j] > max_min) max_min = mins[j];
        }
        float inv_s = max_scale > 0 ? 63.f / max_scale : 0.f, inv_m = max_min > 0 ? 63.f / max_min : 0.f;
        for (int j = 0; j < 8; j++) {
            uint8_t ls = (uint8_t)rne_int(inv_s * scales[j]), lm = (uint8_t)rne_int(inv_m * mins[j]);
            pack_sm6(j, sc, (uint8_t)imin(63, ls), (uint8_t)imin(63, lm));
        }
        st16(y, orc_f32_to_f16(max_scale / 63.f)); st16(y + 2, orc_f32_to_f16(max_min / 63.f));
        const float fd = orc_f16_to_f32(ld16(y)), fm = orc_f16_to_f32(ld16(y + 2));
        for (int j = 0; j < 8; j++) {
            uint8_t s, m; unpack_sm6(j, sc, &s, &m);
            const float d = fd * s;
            if (!d) continue;
            const float dm = fm * m;
            for (int i = 0; i < 32; i++) L[32 * j + i] = (uint8_t)imax(0, imin(nmax, rne_int((x[32 * j + i] + dm) / d)));
        }
        if (bits == 4) {
            uint8_t *q = y + 16;
            for (int j = 0; j < SB; j += 64) for (int l = 0; l < 32; l++) *q++ = (uint8_t)(L[j + l] | (L[j + l + 32] << 4));
        } else {
            uint8_t *qh = y + 16, *ql = y + 48;
            memset(qh, 0, 32);
            uint8_t m1 = 1, m2 = 2;
            for (int n = 0; n < SB; n += 64, m1 <<= 2, m2 <<= 2, ql += 32)
                for (int j = 0; j < 32; j++) {
                    int l1 = L[n + j], l2 = L[n + j + 32];
                    if (l1 > 15) { l1 -= 16; qh[j] |= m1; }
                    if (l2 > 15) { l2 -= 16; qh[j] |= m2; }
                    ql[j] = (uint8_t)(l1 | (l2 << 4));
                }
        }
    }
}
/* k_quants.c:607-631 */
static void q4_K_dec(const uint8_t *x, float *y, int64_t k) {
    for (int64_t b = 0; b < k / SB; b++, x += 144) {
        const float d = orc_f16_to_f32(ld16(x)), mn = orc_f16_to_f32(ld16(x + 2));
        const uint8_t *q = x + 16;
        for (int p = 0; p < 4; p++, q += 32) {
            uint8_t s, m;
            unpack_sm6(2 * p, x + 4, &s, &m);     const float d1 = d * s, m1 = mn * m;
            unpack_sm6(2 * p + 1, x + 4, &s, &m); const float d2 = d * s, m2 = mn * m;
            for (int l = 0; l < 32; l++) *y++ = d1 * (q[l] & 0xF) - m1;
            for (int l = 0; l < 32; l++) *y++ = d2 * (q[l] >> 4) - m2;
        }
    }
}
/* k_quants.c:734-760 */
static void q5_K_dec(const uint8_t *x, float *y, int64_t k) {
    for (int64_t b = 0; b < k / SB; b++, x += 176) {
        const float d = orc_f16_to_f32(ld16(x)), mn = orc_f16_to_f32(ld16(x + 2));
        const uint8_t *qh = x + 16, *ql = x + 48;
        uint8_t u1 = 1, u2 = 2;
        for (int p = 0; p < 4; p++, ql += 32, u1 <<= 2, u2 <<= 2) {
            uint8_t s, m;
            unpack_sm6(2 * p, x + 4, &s, &m);     const float d1 = d * s, m1 = mn * m;
            unpack_sm6(2 * p + 1, x + 4, &s, &m); const float d2 = d * s, m2 = mn * m;
            for (int l = 0; l < 32; l++) *y++ = d1 * ((ql[l] & 0xF) + ((qh[l] & u1) ? 16 : 0)) - m1;
            for (int l = 0; l < 32; l++) *y++ = d2 * ((ql[l] >> 4) + ((qh[l] & u2) ? 16 : 0)) - m2;
        }
    }
}
/* =================================== Q6_K ====================================================== */
/* block_q6_K {u8 ql[128]; u8 qh[64]; i8 scales[16]; f16 d}: k_quants.h:69-74; quantize k_quants.c:781-843 */
static void q6_K_enc(const float *x, uint8_t *y, int64_t k) {
    int8_t L[SB]; float scales[16];
    for (int64_t b = 0; b < k / SB; b++, x += SB, y += 210) {
        int8_t *sc = (int8_t *)(y + 192);
        float max_scale = 0, max_abs = 0;
        for (int j = 0; j < 16; j++) {
            scales[j] = fit_scale_sym(16, 32, x + 16 * j, L + 16 * j);
            float a = fabsf(scales[j]);
            if (a > max_abs) { max_abs = a; max_scale = scales[j]; }
        }
        float is = -128.f / max_scale;
        st16(y + 208, orc_f32_to_f16(1 / is));
        for (int j = 0; j < 16; j++) sc[j] = (int8_t)imin(127, rne_int(is * scales[j]));
        const float fd = orc_f16_to_f32(ld16(y + 208));
        for (int j = 0; j < 16; j++) {
            float d = fd * sc[j];
            if (!d) continue;
            for (int i = 0; i < 16; i++) L[16 * j + i] = (int8_t)(imax(-32, imin(31, rne_int(x[16 * j + i] / d))) + 32);
        }
        uint8_t *ql = y, *qh = y + 128;
        for (int j = 0; j < SB; j += 128, ql += 64, qh += 32)
            for (int l = 0; l < 32; l++) {
                const uint8_t q1 = L[j + l] & 0xF, q2 = L[j + l + 32] & 0xF, q3 = L[j + l + 64] & 0xF, q4 = L[j + l + 96] & 0xF;
                ql[l] = (uint8_t)(q1 | (q3 << 4)); ql[l + 32] = (uint8_t)(q2 | (q4 << 4));
                qh[l] = (uint8_t)((L[j + l] >> 4) | ((L[j + l + 32] >> 4) << 2) | ((L[j + l + 64] >> 4) << 4) | ((L[j + l + 96] >> 4) << 6));
            }
    }
}
/* k_quants.c:845-877 */
static void q6_K_dec(const uint8_t *x, float *y, int64_t k) {
    for (int64_t b = 0; b < k / SB; b++, x += 210) {
        const float d = orc_f16_to_f32(ld16(x + 208));
        const uint8_t *ql = x, *qh = x + 128; const int8_t *sc = (const int8_t *)(x + 192);
        for (int n = 0; n < SB; n += 128, y += 128, ql += 64, qh += 32, sc += 8)
            for (int l = 0; l < 32; l++) {
                int is = l / 16;
                const int8_t q1 = (int8_t)((int8_t)((ql[l] & 0xF) | (((qh[l] >> 0) & 3) << 4)) - 32);
                const int8_t q2 = (int8_t)((int8_t)((ql[l + 32] & 0xF) | (((qh[l] >> 2) & 3) << 4)) - 32);
                const int8_t q3 = (int8_t)((int8_t)((ql[l] >> 4) | (((qh[l] >> 4) & 3) << 4)) - 32);
                const int8_t q4 = (int8_t)((int8_t)((ql[l + 32] >> 4) | (((qh[l] >> 6) & 3) << 4)) - 32);
                y[l] = d * sc[is] * q1; y[l + 32] = d * sc[is + 2] * q2; y[l + 64] = d * sc[is + 4] * q3; y[l + 96] = d * sc[is + 6] * q4;
            }
    }
}
/* =================================== Q8_K ====================================================== */
/* block_q8_K {f32 d; i8 qs[256]; i16 bsums[16]}: k_quants.h:77-82; quantize k_quants.c:899-934 */
static void q8_K_enc(const float *x, uint8_t *y, int64_t k) {
    for (int64_t b = 0; b < k / SB; b++, x += SB, y += 292) {
        int8_t *qs = (int8_t *)(y + 4);
        float vmax = 0, amax = 0;
        for (int j = 0; j < SB; j++) { float ax = fabsf(x[j]); if (ax > amax) { amax = ax; vmax = x[j]; } }
        if (!amax) { stf(y, 0.f); memset(qs, 0, SB); continue; }   /* NB: bsums left untouched, as in the reference */
        const float is = -128.f / vmax;
        for (int j = 0; j < SB; j++) qs[j] = (int8_t)imin(127, rne_int(is * x[j]));
        for (int j = 0; j < 16; j++) {
            int s = 0;
            for (int i = 0; i < 16; i++) s += qs[16 * j + i];
            int16_t s16 = (int16_t)s; memcpy(y + 260 + 2 * j, &s16, 2);
        }
        stf(y, 1 / is);
    }
}
static void q8_K_dec(const uint8_t *x, float *y, int64_t k) {   /* k_quants.c:936-945 */
    for (int64_t b = 0; b < k / SB; b++, x += 292) {
        const float d = ldf(x);
        for (int j = 0; j < SB; j++) *y++ = d * ((const int8_t *)x)[4 + j];
    }
}

/* ------------------------------------------------------------------------------------------------ */
int orc_quantize_row(int type, const float *x, void *y, int64_t k) {
    uint8_t *o = (uint8_t *)y;
    switch (type) {
        case ORC_F32: memcpy(y, x, (size_t)k * 4); return 0;
        case ORC_F16: for (int64_t i = 0; i < k; i++) st16(o + 2 * i, orc_f32_to_f16(x[i])); return 0;
        case ORC_Q4_0: q4_0_enc(x, o, k); return 0;
        case ORC_Q4_1: q4_1_enc(x, o, k); return 0;
        case ORC_Q5_0: q5_0_enc(x, o, k); return 0;
        case ORC_Q5_1: q5_1_enc(x, o, k); return 0;
        case ORC_Q8_0: q8_0_enc_ref(x, o, k); return 0;
        case ORC_Q8_1: q8_1_enc_ref(x, o, k); return 0;
        case ORC_Q2_K: q2_K_enc(x, o, k, 0); return 0;
        case ORC_Q3_K: q3_K_enc(x, o, k); return 0;
        case ORC_Q4_K: q45_K_enc(x, o, k, 4, 0); return 0;
        case ORC_Q5_K: q45_K_enc(x, o, k, 5, 0); return 0;
        case ORC_Q6_K: q6_K_enc(x, o, k); return 0;
        case ORC_Q8_K: q8_K_enc(x, o, k); return 0;
    }
    return -1;
}
int orc_quantize_row_fresh_codes(int type, const float *x, void *y, int64_t k) {
    uint8_t *o = (uint8_t *)y;
    switch (type) {
        case ORC_Q2_K: q2_K_enc(x, o, k, 1); return 0;
        case ORC_Q4_K: q45_K_enc(x, o, k, 4, 1); return 0;
        case ORC_Q5_K: q45_K_enc(x, o, k, 5, 1); return 0;
    }
    return orc_quantize_row(type, x, y, k);
}
int orc_dequantize_row(int type, const void *x, float *y, int64_t k) {
    const uint8_t *i = (const uint8_t *)x;
    switch (type) {
        case ORC_F32: memcpy(y, x, (size_t)k * 4); return 0;
        case ORC_F16: for (int64_t j = 0; j < k; j++) y[j] = orc_f16_to_f32(ld16(i + 2 * j)); return 0;
        case ORC_Q4_0: q4_0_dec(i, y, k); return 0;
        case ORC_Q4_1: q4_1_dec(i, y, k); return 0;
        case ORC_Q5_0: q5_0_dec(i, y, k); return 0;
        case ORC_Q5_1: q5_1_dec(i, y, k); return 0;
        case ORC_Q8_0: q8_0_dec(i, y, k); return 0;
        case ORC_Q2_K: q2_K_dec(i, y, k); return 0;
        case ORC_Q3_K: q3_K_dec(i, y, k); return 0;
        case ORC_Q4_K: q4_K_dec(i, y, k); return 0;
        case ORC_Q5_K: q5_K_dec(i, y, k); return 0;
        case ORC_Q6_K: q6_K_dec(i, y, k); return 0;
        case ORC_Q8_K: q8_K_dec(i, y, k); return 0;
    }
    return -1;
}

/* =================================== dot products ============================================== */
/* integer code of element e (0..31) of a legacy block, before scaling */
static inline int q5_code(const uint8_t *qs, uint32_t qh, int j, int hi) {
    return hi ? ((qs[j] >> 4) | ((qh >> (j + 12)) & 0x10)) : ((qs[j] & 0x0F) | (((qh >> j) << 4) & 0x10));
}
static float dot_legacy(int wt, int64_t k, const uint8_t *w, const uint8_t *a) {
    float sumf = 0.0f;
    const size_t wb = orc_block_bytes(wt), ab = (wt == ORC_Q4_1 || wt == ORC_Q5_1) ? 40 : 34;
    for (int64_t b = 0; b < k / QK; b++, w += wb, a += ab) {
        int sumi = 0;
        if (wt == ORC_Q4_0) {            /* ggml.c:2591-2609 */
            const int8_t *q8 = (const int8_t *)a + 2;
            for (int j = 0; j < 16; j++) sumi += ((w[2 + j] & 0x0F) - 8) * q8[j] + ((w[2 + j] >> 4) - 8) * q8[j + 16];
            sumf += sumi * orc_f16_to_f32(ld16(w)) * orc_f16_to_f32(ld16(a));
        } else if (wt == ORC_Q4_1) {     /* ggml.c:2716-2733 */
            const int8_t *q8 = (const int8_t *)a + 8;
            for (int j = 0; j < 16; j++) sumi += (w[4 + j] & 0x0F) * q8[j] + (w[4 + j] >> 4) * q8[j + 16];
            sumf += (orc_f16_to_f32(ld16(w)) * ldf(a)) * sumi + orc_f16_to_f32(ld16(w + 2)) * ldf(a + 4);
        } else if (wt == ORC_Q5_0) {     /* ggml.c:2952-2974 */
            const int8_t *q8 = (const int8_t *)a + 2; uint32_t qh; memcpy(&qh, w + 2, 4);
            for (int j = 0; j < 16; j++) sumi += (q5_code(w + 6, qh, j, 0) - 16) * q8[j] + (q5_code(w + 6, qh, j, 1) - 16) * q8[j + 16];
            sumf += (orc_f16_to_f32(ld16(w)) * orc_f16_to_f32(ld16(a))) * sumi;
        } else if (wt == ORC_Q5_1) {     /* ggml.c:3208-3230 */
            const int8_t *q8 = (const int8_t *)a + 8; uint32_t qh; memcpy(&qh, w + 4, 4);
            for (int j = 0; j < 16; j++) sumi += q5_code(w + 8, qh, j, 0) * q8[j] + q5_code(w + 8, qh, j, 1) * q8[j + 16];
            sumf += (orc_f16_to_f32(ld16(w)) * ldf(a)) * sumi + orc_f16_to_f32(ld16(w + 2)) * ldf(a + 4);
        } else {                         /* Q8_0, ggml.c:3321-3333 */
            const int8_t *q8 = (const int8_t *)a + 2, *qw = (const int8_t *)w + 2;
            for (int j = 0; j < 32; j++) sumi += qw[j] * q8[j];
            sumf += sumi * (orc_f16_to_f32(ld16(w)) * orc_f16_to_f32(ld16(a)));
        }
    }
    return sumf;
}

/* expand one super-block of weight codes to int8 in element order (what the scalar paths call aux8) */
static void kq_codes(int wt, const uint8_t *w, int8_t *c) {
    if (wt == ORC_Q4_K || wt == ORC_Q5_K) {     /* k_quants.c:2013-2021, 2354-2366 */
        const uint8_t *q = w + (wt == ORC_Q4_K ? 16 : 48), *hm = w + 16; uint8_t m = 1;
        for (int p = 0; p < 4; p++, q += 32) {
            for (int l = 0; l < 32; l++) c[l] = (int8_t)((q[l] & 0xF) + ((wt == ORC_Q5_K && (hm[l] & m)) ? 16 : 0));
            c += 32; m <<= 1;
            for (int l = 0; l < 32; l++) c[l] = (int8_t)((q[l] >> 4) + ((wt == ORC_Q5_K && (hm[l] & m)) ? 16 : 0));
            c += 32; m <<= 1;
        }
    } else if (wt == ORC_Q3_K) {                /* k_quants.c:1710-1726 */
        const uint8_t *hm = w, *q = w + 32; uint8_t m = 1;
        for (int n = 0; n < SB; n += 128, q += 32)
            for (int shift = 0; shift < 8; shift += 2, m <<= 1, c += 32)
                for (int l = 0; l < 32; l++) c[l] = (int8_t)(((q[l] >> shift) & 3) - ((hm[l] & m) ? 0 : 4));
    } else if (wt == ORC_Q6_K) {                /* k_quants.c:2762-2773 */
        const uint8_t *ql = w, *qh = w + 128;
        for (int n = 0; n < SB; n += 128, c += 128, ql += 64, qh += 32)
            for (int l = 0; l < 32; l++) {
                c[l]      = (int8_t)((int8_t)((ql[l] & 0xF) | (((qh[l] >> 0) & 3) << 4)) - 32);
                c[l + 32] = (int8_t)((int8_t)((ql[l + 32] & 0xF) | (((qh[l] >> 2) & 3) << 4)) - 32);
                c[l + 64] = (int8_t)((int8_t)((ql[l] >> 4) | (((qh[l] >> 4) & 3) << 4)) - 32);
                c[l + 96] = (int8_t)((int8_t)((ql[l + 32] >> 4) | (((qh[l] >> 6) & 3) << 4)) - 32);
            }
    } else {                                    /* Q2_K: codes 0..3, k_quants.c:1287-1302 */
        const uint8_t *q = w + 16;
        for (int n = 0; n < SB; n += 128, q += 32)
            for (int shift = 0; shift < 8; shift += 2, c += 32)
                for (int l = 0; l < 32; l++) c[l] = (int8_t)((q[l] >> shift) & 3);
    }
}

static float dot_kquant(int wt, int64_t k, const uint8_t *w, const uint8_t *a) {
    const size_t wb = orc_block_bytes(wt);
    int8_t c[SB]; float lanes[8] = {0}; float sumf = 0;
    for (int64_t b = 0; b < k / SB; b++, w += wb, a += 292) {
        const float ad = ldf(a); const int8_t *q8 = (const int8_t *)a + 4;
        int16_t bs[16]; memcpy(bs, a + 260, 32);
        kq_codes(wt, w, c);
        if (wt == ORC_Q2_K) {                   /* k_quants.c:1271-1304: single int sum, no lanes */
            int summs = 0, isum = 0;
            for (int j = 0; j < 16; j++) summs += bs[j] * (w[j] >> 4);
            for (int j = 0; j < 16; j++) {
                int part = 0;
                for (int l = 0; l < 16; l++) part += q8[16 * j + l] * c[16 * j + l];
                isum += (w[j] & 0xF) * part;
            }
            sumf += (ad * orc_f16_to_f32(ld16(w + 80))) * isum - (ad * orc_f16_to_f32(ld16(w + 82))) * summs;
            continue;
        }
        int32_t acc[8] = {0};
        if (wt == ORC_Q4_K || wt == ORC_Q5_K) { /* k_quants.c:2023-2052 / 2368-2397 */
            int mins_dot = 0;
            for (int j = 0; j < 8; j++) {
                uint8_t s, m; unpack_sm6(j, w + 4, &s, &m);
                mins_dot += (bs[2 * j] + bs[2 * j + 1]) * m;
                for (int i = 0; i < 32; i++) acc[i & 7] += (int32_t)s * (int16_t)(q8[32 * j + i] * c[32 * j + i]);
            }
            const float d = orc_f16_to_f32(ld16(w)) * ad;
            for (int l = 0; l < 8; l++) lanes[l] += d * acc[l];
            sumf -= (orc_f16_to_f32(ld16(w + 2)) * ad) * mins_dot;
        } else {                                /* Q3_K k_quants.c:1727-1742, Q6_K k_quants.c:2774-2785 */
            int8_t s3[16]; const int8_t *sc;
            if (wt == ORC_Q3_K) { unpack_q3_scales(w + 96, s3); for (int j = 0; j < 16; j++) s3[j] -= 32; sc = s3; }
            else sc = (const int8_t *)(w + 192);
            for (int j = 0; j < 16; j++)
                for (int i = 0; i < 16; i++) acc[i & 7] += (int32_t)sc[j] * (int16_t)(q8[16 * j + i] * c[16 * j + i]);
            const float d = orc_f16_to_f32(ld16(w + (wt == ORC_Q3_K ? 108 : 208))) * ad;
            for (int l = 0; l < 8; l++) lanes[l] += d * acc[l];
        }
    }
    for (int l = 0; l < 8; l++) sumf += lanes[l];
    return sumf;
}

float orc_vec_dot(int wt, int64_t k, const void *w, const void *aq) {
    switch (wt) {
        case ORC_Q4_0: case ORC_Q4_1: case ORC_Q5_0: case ORC_Q5_1: case ORC_Q8_0: return dot_legacy(wt, k, (const uint8_t *)w, (const uint8_t *)aq);
        case ORC_Q2_K: case ORC_Q3_K: case ORC_Q4_K: case ORC_Q5_K: case ORC_Q6_K: return dot_kquant(wt, k, (const uint8_t *)w, (const uint8_t *)aq);
    }
    return NAN;
}

/* =================================== mat-mul =================================================== */
typedef struct { int wt; const uint8_t *W; int64_t K, M, N; const float *X; const uint8_t *Xq; size_t xq_row; float *Y; int64_t r0, r1; } mm_job;
static void *mm_worker(void *p) {
    mm_job *j = (mm_job *)p;
    const size_t wrow = orc_row_bytes(j->wt, j->K);
    for (int64_t m = j->r0; m < j->r1; m++) {
        const uint8_t *w = j->W + (size_t)m * wrow;
        for (int64_t n = 0; n < j->N; n++) {
            float s;
            if (j->wt == ORC_F32) {
                const float *wf = (const float *)w, *x = j->X + n * j->K; double acc = 0;  /* reference uses SIMD fp32 lanes; double here = tighter */
                for (int64_t i = 0; i < j->K; i++) acc += (double)wf[i] * x[i];
                s = (float)acc;
            } else if (j->wt == ORC_F16) {
                const float *x = j->X + n * j->K; double acc = 0;
                for (int64_t i = 0; i < j->K; i++) acc += (double)orc_f16_to_f32(ld16(w + 2 * i)) * orc_f16_to_f32(orc_f32_to_f16(x[i]));
                s = (float)acc;
            } else s = orc_vec_dot(j->wt, j->K, w, j->Xq + (size_t)n * j->xq_row);
            j->Y[n * j->M + m] = s;
        }
    }
    return NULL;
}
void orc_mul_mat(int wt, const void *W, int64_t K, int64_t M, const float *X, int64_t N, float *Y, int nthreads) {
    uint8_t *xq = NULL; size_t xq_row = 0;
    const int at = orc_vec_dot_type(wt);
    if (at >= 0) {       /* INIT pass: ggml.c:11462-11476 */
        xq_row = orc_row_bytes(at, K);
        xq = (uint8_t *)malloc(xq_row * (size_t)N);
        for (int64_t n = 0; n < N; n++) {
            if (at == ORC_Q8_0) orc_quantize_row_q8_0_x86(X + n * K, xq + n * xq_row, K);
            else if (at == ORC_Q8_1) orc_quantize_row_q8_1_x86(X + n * K, xq + n * xq_row, K);
            else q8_K_enc(X + n * K, xq + n * xq_row, K);
        }
    }
    if (nthreads < 1) nthreads = 1;
    if (nthreads > 64) nthreads = 64;
    if ((int64_t)nthreads > M) nthreads = (int)M;
    pthread_t th[64]; mm_job jobs[64];
    const int64_t per = (M + nthreads - 1) / nthreads;     /* rows per thread, ggml.c:11484-11487 */
    for (int t = 0; t < nthreads; t++) {
        mm_job j = { wt, (const uint8_t *)W, K, M, N, X, xq, xq_row, Y, t * per, (t + 1) * per < M ? (t + 1) * per : M };
        jobs[t] = j;
        if (t > 0) pthread_create(&th[t], NULL, mm_worker, &jobs[t]);
    }
    mm_worker(&jobs[0]);
    for (int t = 1; t < nthreads; t++) pthread_join(th[t], NULL);
    free(xq);
}

/* =================================== elementwise / attention ops =============================== */
void orc_norm(const float *x, float *y, int64_t n) {       /* ggml.c:10568-10595 */
    double sum = 0.0;
    for (int64_t i = 0; i < n; i++) sum += (double)x[i];
    float mean = (float)(sum / n);
    double sum2 = 0.0;
    for (int64_t i = 0; i < n; i++) { float v = x[i] - mean; y[i] = v; sum2 += (double)(v * v); }
    float variance = (float)(sum2 / n);
    const float scale = 1.0f / sqrtf(variance + 1e-5f);
    for (int64_t i = 0; i < n; i++) y[i] *= scale;
}
void orc_layernorm(const float *x, const float *g, const float *b, float *y, int64_t n) {
    orc_norm(x, y, n);
    for (int64_t i = 0; i < n; i++) y[i] = y[i] * g[i] + b[i];   /* separate fp32 mul then add: libfalcon.cpp:2168-2173 (no fma: -ffp-contract=off) */
}

static uint16_t g_gelu_lut[65536], g_exp_lut[65536];
static pthread_once_t g_lut_once = PTHREAD_ONCE_INIT;
static void build_luts(void) {     /* ggml.c:4277-4295 */
    for (uint32_t i = 0; i < 65536; i++) {
        float f = orc_f16_to_f32((uint16_t)i);
        g_gelu_lut[i] = orc_f32_to_f16(0.5f * f * (1.0f + tanhf(0.79788456080286535587989211986876f * f * (1.0f + 0.044715f * f * f))));
        g_exp_lut[i] = orc_f32_to_f16(expf(f));
    }
}
void orc_gelu(const float *x, float *y, int64_t n) {        /* ggml.c:3476-3484 */
    pthread_once(&g_lut_once, build_luts);
    for (int64_t i = 0; i < n; i++) y[i] = orc_f16_to_f32(g_gelu_lut[orc_f32_to_f16(x[i])]);
}
void orc_soft_max(const float *x, float *y, int64_t n) {    /* ggml.c:12427-12449 */
    pthread_once(&g_lut_once, build_luts);
    float mx = -INFINITY;
    for (int64_t i = 0; i < n; i++) if (x[i] > mx) mx = x[i];
    double sum = 0.0;
    for (int64_t i = 0; i < n; i++) {
        if (x[i] == -INFINITY) y[i] = 0.0f;
        else { float v = orc_f16_to_f32(g_exp_lut[orc_f32_to_f16(x[i] - mx)]); sum += (double)v; y[i] = v; }
    }
    const float inv = (float)(1.0 / sum);
    for (int64_t i = 0; i < n; i++) y[i] *= inv;
}

float orc_rope_theta_scale(int head_dim, int n_ctx_rope, int dynamic_mode, float ntk_alpha, int freq_base) {
    /* ggml.c:12875-12898 */
    const float fb = (float)(freq_base ? freq_base : 10000);
    float alpha = 1.0f;
    if (dynamic_mode) {
        if (n_ctx_rope >= 2048) alpha = powf(((n_ctx_rope / 2048) - 1) * ntk_alpha + 1, head_dim / (head_dim - 2.0));
    } else if (ntk_alpha != 0.0f) alpha = powf(ntk_alpha, head_dim / (head_dim - 2.0));
    return powf(alpha * fb, -2.0f / head_dim);
}
void orc_rope_neox(float *x, int n_tok, int n_head, int head_dim, int64_t tok_stride, int n_past, int n_ctx_rope,
                   int dynamic_mode, float ntk_alpha, int freq_base) {
    /* ggml.c:12957-12979 with n_dims == head_dim */
    const float theta_scale = orc_rope_theta_scale(head_dim, n_ctx_rope, dynamic_mode, ntk_alpha, freq_base);
    for (int t = 0; t < n_tok; t++)
        for (int h = 0; h < n_head; h++) {
            float *v = x + t * tok_stride + (int64_t)h * head_dim;
            float theta = (float)(n_past + t);
            for (int i = 0; i < head_dim / 2; i++) {
                const float c = cosf(theta), s = sinf(theta);
                theta *= theta_scale;
                const float x0 = v[i], x1 = v[i + head_dim / 2];
                v[i] = x0 * c - x1 * s;
                v[i + head_dim / 2] = x0 * s + x1 * c;
            }
        }
}

/* =================================== whole-model eval ========================================== */
static void get_row(const orc_tensor *t, int64_t row, float *out) {    /* ggml_get_rows, ggml.c:11975-12002 */
    orc_dequantize_row(t->type, (const uint8_t *)t->data + (size_t)row * orc_row_bytes(t->type, t->ne0), out, t->ne0);
}
static const float *as_f32(const orc_tensor *t) { return (const float *)t->data; }

int orc_falcon_eval(orc_model *m, const int32_t *tokens, int N, int n_past, int n_ctx_rope,
                    float *logits, int all_logits, int nthreads) {
    return orc_falcon_eval_range(m, tokens, N, n_past, n_ctx_rope, logits, all_logits, nthreads, 0, m->n_layer, NULL, NULL);
}

/* The same eval restricted to layers [layer_first, layer_last): the unit of the layer-range pipeline.
 * layer_first > 0: the residual stream [N][n_embd] comes from resid_in instead of the embedding lookup;
 * layer_last < n_layer: no final norm / lm_head, the residual stream is written to resid_out instead. */
int orc_falcon_eval_range(orc_model *m, const int32_t *tokens, int N, int n_past, int n_ctx_rope,
                          float *logits, int all_logits, int nthreads, int layer_first, int layer_last,
                          const float *resid_in, float *resid_out) {
    const int E = m->n_embd, H = m->n_head, HKV = m->n_head_kv, D = E / H, QKV = (H + 2 * HKV) * D, FF = 4 * E;
    const int group = H / HKV, T = n_past + N;
    if (T > m->n_ctx) return -1;
    float *inp = (float *)malloc(sizeof(float) * (size_t)N * E), *xa = (float *)malloc(sizeof(float) * (size_t)N * E),
          *xm = (float *)malloc(sizeof(float) * (size_t)N * E), *qkv = (float *)malloc(sizeof(float) * (size_t)N * QKV),
          *att = (float *)malloc(sizeof(float) * (size_t)N * E), *ao = (float *)malloc(sizeof(float) * (size_t)N * E),
          *up = (float *)malloc(sizeof(float) * (size_t)N * FF), *dn = (float *)malloc(sizeof(float) * (size_t)N * E),
          *sc = (float *)malloc(sizeof(float) * (size_t)T);
    if (layer_first == 0) for (int t = 0; t < N; t++) get_row(&m->tok_embeddings, tokens[t], inp + (size_t)t * E);   /* libfalcon.cpp:2120 */
    else memcpy(inp, resid_in, sizeof(float) * (size_t)N * E);
    const float kq_scale = 1.0f / sqrtf((float)D);           /* libfalcon.cpp:2313-2317 */
    for (int il = layer_first; il < layer_last; il++) {
        const orc_layer *L = &m->layers[il];
        for (int t = 0; t < N; t++) {                        /* libfalcon.cpp:2166-2188 */
            orc_layernorm(inp + (size_t)t * E, as_f32(&L->ln_mlp_g), as_f32(&L->ln_mlp_b), xm + (size_t)t * E, E);
            if (m->falcon_type == 40) orc_layernorm(inp + (size_t)t * E, as_f32(&L->ln_attn_g), as_f32(&L->ln_attn_b), xa + (size_t)t * E, E);
        }
        const float *attn_in = m->falcon_type == 40 ? xa : xm;
        orc_mul_mat(L->wqkv.type, L->wqkv.data, E, QKV, attn_in, N, qkv, nthreads);      /* :2192 */
        orc_rope_neox(qkv, N, H, D, QKV, n_past, n_ctx_rope, 1, 2.0f, 0);                 /* Q, :2229-2234 */
        orc_rope_neox(qkv + (size_t)H * D, N, HKV, D, QKV, n_past, n_ctx_rope, 1, 2.0f, 0); /* K */
        float *kc = m->k_cache + (size_t)il * m->n_ctx * HKV * D, *vc = m->v_cache + (size_t)il * m->n_ctx * HKV * D;
        for (int t = 0; t < N; t++) {                        /* KV store, :2238-2281 */
            memcpy(kc + (size_t)(n_past + t) * HKV * D, qkv + (size_t)t * QKV + (size_t)H * D, sizeof(float) * HKV * D);
            memcpy(vc + (size_t)(n_past + t) * HKV * D, qkv + (size_t)t * QKV + (size_t)(H + HKV) * D, sizeof(float) * HKV * D);
        }
        for (int t = 0; t < N; t++)                          /* attention, :2285-2366; GQA map h / group: ggml.c:11074 */
            for (int h = 0; h < H; h++) {
                const int kvh = h / group;
                const float *q = qkv + (size_t)t * QKV + (size_t)h * D;
                for (int p = 0; p < T; p++) {
                    if (p > n_past + t) { sc[p] = -INFINITY; continue; }       /* ggml.c:12342-12348 */
                    const float *kk = kc + ((size_t)p * HKV + kvh) * D;
                    float dot = 0; for (int i = 0; i < D; i++) dot += kk[i] * q[i];
                    sc[p] = dot * kq_scale;
                }
                orc_soft_max(sc, sc, T);
                float *o = att + (size_t)t * E + (size_t)h * D;
                for (int i = 0; i < D; i++) {
                    float acc = 0; for (int p = 0; p < T; p++) acc += vc[((size_t)p * HKV + kvh) * D + i] * sc[p];
                    o[i] = acc;
                }
            }
        orc_mul_mat(L->wo.type, L->wo.data, E, E, att, N, ao, nthreads);                 /* :2370 */
        orc_mul_mat(L->ffn_up.type, L->ffn_up.data, E, FF, xm, N, up, nthreads);         /* :2389 */
        orc_gelu(up, up, (int64_t)N * FF);                                                /* :2392 */
        orc_mul_mat(L->ffn_down.type, L->ffn_down.data, FF, E, up, N, dn, nthreads);      /* :2394 */
        for (size_t i = 0; i < (size_t)N * E; i++) { float c = dn[i] + ao[i]; inp[i] = c + inp[i]; }   /* :2399-2400 */
    }
    const int first = all_logits ? 0 : N - 1;
    if (layer_last < m->n_layer) memcpy(resid_out, inp, sizeof(float) * (size_t)N * E);
    else for (int t = first; t < N; t++) orc_layernorm(inp + (size_t)t * E, as_f32(&m->ln_f_g), as_f32(&m->ln_f_b), xa + (size_t)t * E, E);  /* :2422-2431 */
    if (layer_last >= m->n_layer) orc_mul_mat(m->lm_head.type, m->lm_head.data, E, m->n_vocab, xa + (size_t)first * E, N - first, logits, nthreads);  /* :2440 */
    free(inp); free(xa); free(xm); free(qkv); free(att); free(ao); free(up); free(dn); free(sc);
    return 0;
}
