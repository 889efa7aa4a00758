// quant_gpu.cu -- fp32 -> GGML weight blocks on the device, bit for bit what the reference's quantisers write (SURVEY section 8f-3):
// b200_quantize_weights(_rows), and b200_quantize_chunks, ggml_quantize_chunk over falcon_quantize's chunks for every output type.
//   Q4_0  quantize_row_q4_0_reference, ggml.c:927-962;  Q4_1 / Q5_0 / Q5_1 / Q8_0 / F16 at their block functions
//   Q2_K  quantize_row_q2_K_reference, k_quants.c:275-342     (make_qkx1_quants :222-262 on 16 sub-blocks of 16, 4-bit scales / mins)
//   Q3_K  quantize_row_q3_K_reference, k_quants.c:396-470     (make_q3_quants :163-220, 6-bit signed scales, high-bit mask)
//   Q4_K  quantize_row_q4_K_reference, k_quants.c:542-605     (make_qkx1_quants on 8 sub-blocks of 32, 6-bit scales / mins)
//   Q5_K  quantize_row_q5_K_reference, k_quants.c:652-732     (the same, levels 0..31, qh plane)
//   Q6_K  quantize_row_q6_K_reference, k_quants.c:781-843     (make_qx_quants rmse_type 1 :57-161, int8 scales)
// One thread per block, except Q2_K / Q4_K / Q5_K: one thread per row, walking its blocks in order and carrying make_qkx1_quants's
// codes from block to block (quantize_rows_kernel says why).  The arithmetic is the scalar C code's, in its order.  THIS FILE IS
// COMPILED WITH --fmad=false (csrc/Makefile): every a * b + c below is a separately rounded multiply and add, divisions are IEEE, so
// each intermediate equals the CPU's (the reference is built without fp contraction).  Blocks are written in the file layout, ready
// for b200_weight_upload or a GGCC file.
// A Falcon-40B ffn_up (32768 rows of 8192) takes 1-6 ms per type on an H100 80GB (tools/quantise_bench.py).
#include "kernels.h"
#include <algorithm>
#include <cfloat>

namespace {

__device__ __forceinline__ int rne_int(float v) {                     // nearest_int, k_quants.c:50-55: the 1.5 * 2^23 magic constant
    const float t = v + 12582912.f;
    if (t != t) return 0;                                             // x86's default NaN 0x7fc00000 gives 0 by the formula below; CUDA's NaN is 0x7fffffff
    return (__float_as_int(t) & 0x007fffff) - 0x00400000;
}
// (every block size is even and every fp16 field sits at an even offset, so the fields are 2-byte aligned; a byte-wise store of
//  `(uint8_t) bits` was compiled into a NUMERIC half -> u8 conversion by nvcc 12.9, F2I.U8.F16 in the SASS -- hence the single 16-bit store)
__device__ __forceinline__ void st16(uint8_t * p, uint16_t v) { *reinterpret_cast<uint16_t *>(p) = v; }

// make_qkx1_quants: asymmetric (scale, min) fit of n values to levels 0..nmax, up to 5 refinement rounds.  Round 0 compares against
// what L holds on entry: the same sub-block's codes in the row's previous block, zeros in block 0.
__device__ float fit_scale_min(int n, int nmax, const float * x, uint8_t * L, float & the_min) {
    float mn = x[0], mx = x[0];
    for (int i = 1; i < n; i++) { if (x[i] < mn) mn = x[i]; if (x[i] > mx) mx = x[i]; }
    if (mx == mn) { for (int i = 0; i < n; i++) L[i] = 0; the_min = 0.f; return 0.f; }
    if (mn > 0.f) mn = 0.f;
    float iscale = nmax / (mx - mn), scale = 1 / iscale;
    for (int t = 0; t < 5; t++) {
        float sumlx = 0.f; int suml2 = 0; bool changed = false;
        for (int i = 0; i < n; i++) {
            const int l = max(0, min(nmax, rne_int(iscale * (x[i] - mn))));
            if (l != L[i]) { L[i] = (uint8_t) l; changed = true; }
            sumlx += (x[i] - mn) * l; suml2 += l * l;
        }
        scale = sumlx / suml2;
        float sum = 0.f;
        for (int i = 0; i < n; i++) sum += x[i] - scale * L[i];
        mn = sum / n; if (mn > 0.f) mn = 0.f;
        iscale = 1 / scale;
        if (!changed) break;
    }
    the_min = -mn;
    return scale;
}
// make_q3_quants, do_rmse branch: symmetric fit to levels -nmax..nmax-1 with weights x^2, greedy per-element refinement
__device__ float fit_scale_q3(int n, int nmax, const float * x, int8_t * L) {
    float vmax = 0.f, amax = 0.f;
    for (int i = 0; i < n; i++) { const float ax = fabsf(x[i]); if (ax > amax) { amax = ax; vmax = x[i]; } }
    if (!amax) { for (int i = 0; i < n; i++) L[i] = 0; return 0.f; }
    const float iscale = -nmax / vmax;
    float sumlx = 0.f, suml2 = 0.f;
    for (int i = 0; i < n; i++) {
        const int l = max(-nmax, min(nmax - 1, rne_int(iscale * x[i])));
        L[i] = (int8_t) l;
        const float w = x[i] * x[i];
        sumlx += w * x[i] * l; suml2 += w * l * l;
    }
    for (int t = 0; t < 5; t++) {
        int nchg = 0;
        for (int i = 0; i < n; i++) {
            const float w = x[i] * x[i];
            float slx = sumlx - w * x[i] * L[i];
            if (slx > 0.f) {
                float sl2 = suml2 - w * L[i] * L[i];
                const int nl = max(-nmax, min(nmax - 1, rne_int(x[i] * sl2 / slx)));
                if (nl != L[i]) {
                    slx += w * x[i] * nl; sl2 += w * nl * nl;
                    if (sl2 > 0.f && slx * slx * suml2 > sumlx * sumlx * sl2) { L[i] = (int8_t) nl; sumlx = slx; suml2 = sl2; nchg++; }
                }
            }
        }
        if (!nchg) break;
    }
    for (int i = 0; i < n; i++) L[i] = (int8_t) (L[i] + nmax);
    return sumlx / suml2;
}
// make_qx_quants with rmse_type 1: scale refits (<= 3) then greedy per-element refinement (<= 5 rounds)
__device__ float fit_scale_sym(int n, int nmax, const float * x, int8_t * L) {
    float vmax = 0.f, amax = 0.f;
    for (int i = 0; i < n; i++) { const float ax = fabsf(x[i]); if (ax > amax) { amax = ax; vmax = x[i]; } }
    if (!amax) { for (int i = 0; i < n; i++) L[i] = 0; return 0.f; }
    float iscale = -nmax / vmax, sumlx = 0.f, suml2 = 0.f;
    for (int i = 0; i < n; i++) {
        const int l = max(-nmax, min(nmax - 1, rne_int(iscale * x[i])));
        L[i] = (int8_t) (l + nmax);
        const float w = x[i] * x[i];
        sumlx += w * x[i] * l; suml2 += w * l * l;
    }
    float scale = sumlx / suml2, best = scale * sumlx;
    for (int t = 0; t < 3; t++) {
        iscale = 1 / scale;
        float slx = 0.f, sl2 = 0.f; bool changed = false;
        for (int i = 0; i < n; i++) {
            const int l = max(-nmax, min(nmax - 1, rne_int(iscale * x[i])));
            if (l + nmax != L[i]) changed = true;
            const float w = x[i] * x[i];
            slx += w * x[i] * l; sl2 += w * l * l;
        }
        if (!changed || sl2 == 0.f || slx * slx <= best * sl2) break;
        for (int i = 0; i < n; i++) L[i] = (int8_t) (nmax + max(-nmax, min(nmax - 1, rne_int(iscale * x[i]))));
        sumlx = slx; suml2 = sl2; scale = sumlx / suml2; best = scale * sumlx;
    }
    for (int t = 0; t < 5; t++) {
        int nchg = 0;
        for (int i = 0; i < n; i++) {
            const float w = x[i] * x[i];
            const int l = L[i] - nmax;
            float slx = sumlx - w * x[i] * l;
            if (slx > 0.f) {
                float sl2 = suml2 - w * l * l;
                const int nl = max(-nmax, min(nmax - 1, rne_int(x[i] * sl2 / slx)));
                if (nl != l) {
                    slx += w * x[i] * nl; sl2 += w * nl * nl;
                    if (sl2 > 0.f && slx * slx * suml2 > sumlx * sumlx * sl2) {
                        L[i] = (int8_t) (nmax + nl); sumlx = slx; suml2 = sl2;
                        scale = sumlx / suml2; best = scale * sumlx; nchg++;
                    }
                }
            }
        }
        if (!nchg) break;
    }
    return scale;
}

// ---- one block each, xb -> yb.  The legacy types in their C functions' order and rounding:
//   Q4_1 quantize_row_q4_1_reference ggml.c:968-1002     Q5_0 :1008-1046     Q5_1 :1052-1090     Q8_0 :1106-1129
__device__ void quantize_q4_0_block(const float * __restrict__ xb, uint8_t * __restrict__ yb) {
    float amax = 0.f, vmax = 0.f;
    for (int j = 0; j < 32; j++) { const float v = xb[j]; if (amax < fabsf(v)) { amax = fabsf(v); vmax = v; } }
    const float d = __fdiv_rn(vmax, -8.f), id = d != 0.f ? __fdiv_rn(1.0f, d) : 0.0f;
    st16(yb, f32_to_f16_bits(d));
    for (int j = 0; j < 16; j++) {
        const int lo = min(15, (int) (int8_t) __float2int_rz(__fadd_rn(__fmul_rn(xb[j], id), 8.5f)));
        const int hi = min(15, (int) (int8_t) __float2int_rz(__fadd_rn(__fmul_rn(xb[j + 16], id), 8.5f)));
        yb[2 + j] = (uint8_t) ((lo & 0xff) | (hi << 4));
    }
}

__device__ void quantize_q4_1_block(const float * __restrict__ xb, uint8_t * __restrict__ yb) {
    float mn = FLT_MAX, mx = -FLT_MAX;
    for (int j = 0; j < 32; j++) { const float v = xb[j]; if (v < mn) mn = v; if (v > mx) mx = v; }
    const float d = __fdiv_rn(__fsub_rn(mx, mn), 15.f), id = d != 0.f ? __fdiv_rn(1.0f, d) : 0.0f;
    st16(yb, f32_to_f16_bits(d)); st16(yb + 2, f32_to_f16_bits(mn));
    for (int j = 0; j < 16; j++) {
        const int lo = min(15, (int) (int8_t) __float2int_rz(__fadd_rn(__fmul_rn(__fsub_rn(xb[j], mn), id), 0.5f)));
        const int hi = min(15, (int) (int8_t) __float2int_rz(__fadd_rn(__fmul_rn(__fsub_rn(xb[j + 16], mn), id), 0.5f)));
        yb[4 + j] = (uint8_t) ((lo & 0xff) | (hi << 4));
    }
}

// Q5_0 (ASYM false) and Q5_1 (ASYM true): 4 low bits in qs, the fifth bit of value j in bit j of qh
template <bool ASYM>
__device__ void quantize_q5_block(const float * __restrict__ xb, uint8_t * __restrict__ yb) {
    float d, mn = 0.f;
    if (ASYM) {
        float mx = -FLT_MAX; mn = FLT_MAX;
        for (int j = 0; j < 32; j++) { const float v = xb[j]; if (v < mn) mn = v; if (v > mx) mx = v; }
        d = __fdiv_rn(__fsub_rn(mx, mn), 31.f);
        st16(yb, f32_to_f16_bits(d)); st16(yb + 2, f32_to_f16_bits(mn));
    } else {
        float amax = 0.f, vmax = 0.f;
        for (int j = 0; j < 32; j++) { const float v = xb[j]; if (amax < fabsf(v)) { amax = fabsf(v); vmax = v; } }
        d = __fdiv_rn(vmax, -16.f);
        st16(yb, f32_to_f16_bits(d));
    }
    const float id = d != 0.f ? __fdiv_rn(1.0f, d) : 0.0f;
    uint8_t * qs = yb + (ASYM ? 8 : 6);
    uint32_t qh = 0;
    for (int j = 0; j < 16; j++) {
        int lo, hi;
        if (ASYM) {                                                   // (uint8_t)(x0 + 0.5f), no clamp
            lo = (uint8_t) __float2int_rz(__fadd_rn(__fmul_rn(__fsub_rn(xb[j], mn), id), 0.5f));
            hi = (uint8_t) __float2int_rz(__fadd_rn(__fmul_rn(__fsub_rn(xb[j + 16], mn), id), 0.5f));
        } else {                                                      // MIN(31, (int8_t)(x0 + 16.5f))
            lo = (uint8_t) min(31, (int) (int8_t) __float2int_rz(__fadd_rn(__fmul_rn(xb[j], id), 16.5f)));
            hi = (uint8_t) min(31, (int) (int8_t) __float2int_rz(__fadd_rn(__fmul_rn(xb[j + 16], id), 16.5f)));
        }
        qs[j] = (uint8_t) ((lo & 0x0F) | ((hi & 0x0F) << 4));
        qh |= (uint32_t) ((lo & 0x10) >> 4) << j;
        qh |= (uint32_t) ((hi & 0x10) >> 4) << (j + 16);
    }
    st16(yb + (ASYM ? 4 : 2), (uint16_t) qh); st16(yb + (ASYM ? 6 : 4), (uint16_t) (qh >> 16));
}

__device__ void quantize_q8_0_block(const float * __restrict__ xb, uint8_t * __restrict__ yb) {
    float amax = 0.f;
    for (int j = 0; j < 32; j++) { const float a = fabsf(xb[j]); amax = amax > a ? amax : a; }      // MAX(amax, fabsf(v))
    const float d = __fdiv_rn(amax, 127.f), id = d != 0.f ? __fdiv_rn(1.0f, d) : 0.0f;
    st16(yb, f32_to_f16_bits(d));
    for (int j = 0; j < 32; j++) yb[2 + j] = (uint8_t) (int8_t) __float2int_rz(roundf(__fmul_rn(xb[j], id)));
}

__device__ void quantize_q6_K_block(const float * __restrict__ xb, uint8_t * __restrict__ yb) {
    int8_t L[256]; float scales[16]; int8_t sc[16];
    float max_scale = 0.f, max_abs = 0.f;
    for (int j = 0; j < 16; j++) {
        scales[j] = fit_scale_sym(16, 32, xb + 16 * j, L + 16 * j);
        const float a = fabsf(scales[j]);
        if (a > max_abs) { max_abs = a; max_scale = scales[j]; }
    }
    const float is = -128.f / max_scale;
    const uint16_t hd = f32_to_f16_bits(1 / is);
    st16(yb + 208, hd);
    for (int j = 0; j < 16; j++) { sc[j] = (int8_t) min(127, rne_int(is * scales[j])); yb[192 + j] = (uint8_t) sc[j]; }
    const float fd = f16_bits_to_f32(hd);
    for (int j = 0; j < 16; j++) {
        const float d = fd * sc[j];
        if (!d) continue;
        for (int i = 0; i < 16; i++) L[16 * j + i] = (int8_t) (max(-32, min(31, rne_int(xb[16 * j + i] / d))) + 32);
    }
    uint8_t * ql = yb, * qh = yb + 128;
    for (int j = 0; j < 256; j += 128, ql += 64, qh += 32)
        for (int l = 0; l < 32; l++) {
            const uint8_t q1 = L[j + l] & 0xF, q2 = L[j + l + 32] & 0xF, q3 = L[j + l + 64] & 0xF, q4 = L[j + l + 96] & 0xF;
            ql[l] = (uint8_t) (q1 | (q3 << 4)); ql[l + 32] = (uint8_t) (q2 | (q4 << 4));
            qh[l] = (uint8_t) ((L[j + l] >> 4) | ((L[j + l + 32] >> 4) << 2) | ((L[j + l + 64] >> 4) << 4) | ((L[j + l + 96] >> 4) << 6));
        }
}

// ---- the make_qkx1_quants types, one block each: L holds the codes of the row's previous block on entry (zeros for block 0) and
// this block's on exit
__device__ void quantize_q2_K_block(const float * __restrict__ xb, uint8_t * __restrict__ yb, uint8_t * L) {
    float mins[16], scales[16]; uint8_t sc[16];
    float max_scale = 0.f, max_min = 0.f;
    for (int j = 0; j < 16; j++) {
        scales[j] = fit_scale_min(16, 3, xb + 16 * j, L + 16 * j, mins[j]);
        if (scales[j] > max_scale) max_scale = scales[j];
        if (mins[j] > max_min) max_min = mins[j];
    }
    uint16_t hd, hm;
    if (max_scale > 0.f) {
        const float is = 15.f / max_scale;
        for (int j = 0; j < 16; j++) sc[j] = (uint8_t) rne_int(is * scales[j]);
        hd = f32_to_f16_bits(max_scale / 15.f);
    } else { for (int j = 0; j < 16; j++) sc[j] = 0; hd = f32_to_f16_bits(0.f); }
    if (max_min > 0.f) {
        const float is = 15.f / max_min;
        for (int j = 0; j < 16; j++) sc[j] |= (uint8_t) (rne_int(is * mins[j]) << 4);
        hm = f32_to_f16_bits(max_min / 15.f);
    } else hm = f32_to_f16_bits(0.f);
    for (int j = 0; j < 16; j++) yb[j] = sc[j];
    st16(yb + 80, hd); st16(yb + 82, hm);
    const float fd = f16_bits_to_f32(hd), fm = f16_bits_to_f32(hm);
    for (int j = 0; j < 16; j++) {
        const float d = fd * (sc[j] & 0xF);
        if (!d) continue;
        const float dm = fm * (sc[j] >> 4);
        for (int i = 0; i < 16; i++) L[16 * j + i] = (uint8_t) max(0, min(3, rne_int((xb[16 * j + i] + dm) / d)));
    }
    uint8_t * qs = yb + 16;
    for (int j = 0; j < 256; j += 128)
        for (int l = 0; l < 32; l++)
            qs[j / 4 + l] = (uint8_t) (L[j + l] | (L[j + l + 32] << 2) | (L[j + l + 64] << 4) | (L[j + l + 96] << 6));
}

// Q4_K (NMAX 15) and Q5_K (NMAX 31) up to their code packing: the fit of the eight sub-blocks of 32, the 6-bit scales and mins, d / dmin
// and the scales written to yb[0..15], then every code re-quantised into L against what was written
template <int NMAX>
__device__ void quantize_k_sub_blocks(const float * __restrict__ xb, uint8_t * __restrict__ yb, uint8_t * L) {
    float mins[8], scales[8]; uint8_t sc[12];
    for (int i = 0; i < 12; i++) sc[i] = 0;
    float max_scale = 0.f, max_min = 0.f;
    for (int j = 0; j < 8; j++) {
        scales[j] = fit_scale_min(32, NMAX, xb + 32 * j, L + 32 * j, mins[j]);
        if (scales[j] > max_scale) max_scale = scales[j];
        if (mins[j] > max_min) max_min = mins[j];
    }
    const float inv_s = max_scale > 0.f ? 63.f / max_scale : 0.f, inv_m = max_min > 0.f ? 63.f / max_min : 0.f;
    for (int j = 0; j < 8; j++) {
        const uint8_t ls = (uint8_t) rne_int(inv_s * scales[j]), lm = (uint8_t) rne_int(inv_m * mins[j]);
        pack_sm6(j, sc, (uint8_t) min(63, (int) ls), (uint8_t) min(63, (int) lm));
    }
    const uint16_t hd = f32_to_f16_bits(max_scale / 63.f), hm = f32_to_f16_bits(max_min / 63.f);
    st16(yb, hd); st16(yb + 2, hm);
    for (int i = 0; i < 12; i++) yb[4 + i] = sc[i];
    const float fd = f16_bits_to_f32(hd), fm = f16_bits_to_f32(hm);
    for (int j = 0; j < 8; j++) {
        int s, m; unpack_sm6(j, sc, s, m);
        const float d = fd * s;
        if (!d) continue;
        const float dm = fm * m;
        for (int i = 0; i < 32; i++) L[32 * j + i] = (uint8_t) max(0, min(NMAX, rne_int((xb[32 * j + i] + dm) / d)));
    }
}

__device__ void quantize_q4_K_block(const float * __restrict__ xb, uint8_t * __restrict__ yb, uint8_t * L) {
    quantize_k_sub_blocks<15>(xb, yb, L);
    uint8_t * q = yb + 16;
    for (int j = 0; j < 256; j += 64) for (int l = 0; l < 32; l++) *q++ = (uint8_t) (L[j + l] | (L[j + l + 32] << 4));
}

__device__ void quantize_q5_K_block(const float * __restrict__ xb, uint8_t * __restrict__ yb, uint8_t * L) {
    quantize_k_sub_blocks<31>(xb, yb, L);
    uint8_t qh[32];
    for (int i = 0; i < 32; i++) qh[i] = 0;
    uint8_t * ql = yb + 48;
    uint8_t m1 = 1, m2 = 2;
    for (int n = 0; n < 256; n += 64, m1 <<= 2, m2 <<= 2, ql += 32)
        for (int j = 0; j < 32; j++) {
            int l1 = L[n + j], l2 = L[n + j + 32];
            if (l1 > 15) { l1 -= 16; qh[j] |= m1; }
            if (l2 > 15) { l2 -= 16; qh[j] |= m2; }
            ql[j] = (uint8_t) (l1 | (l2 << 4));
        }
    for (int i = 0; i < 32; i++) yb[16 + i] = qh[i];
}

// CTA size of the one-thread-per-block kernels: 256 for the 32-value types, 64 for Q3_K / Q6_K (each thread keeps 256 codes)
constexpr int blocks_cta(int type) { return type_spec(type).blk_elems == 32 ? 256 : 64; }

template <void (*quantize_block)(const float *, uint8_t *), int TYPE>
__global__ void __launch_bounds__(blocks_cta(TYPE)) quantize_blocks_kernel(const float * __restrict__ x, uint8_t * __restrict__ y,
                                                                           int64_t nblocks) {
    constexpr TypeSpec ts = type_spec(TYPE);
    const int64_t b = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    quantize_block(x + b * ts.blk_elems, y + b * ts.blk_bytes);
}

// Q3_K is quantize_blocks_kernel written out: as a block function inlined into the template, nvcc 12.9 lays out its local arrays
// differently (the mask loop through generic addresses, a 4-byte spill), and the kernel runs 1% slower on an H100
__global__ void __launch_bounds__(blocks_cta(T_Q3_K)) quantize_q3_K_kernel(const float * __restrict__ x, uint8_t * __restrict__ y,
                                                                            int64_t nblocks) {
    constexpr TypeSpec ts = type_spec(T_Q3_K);
    const int64_t b = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    const float * xb = x + b * ts.blk_elems; uint8_t * yb = y + b * ts.blk_bytes;
    int8_t L[256]; float scales[16]; uint8_t sc[12], hmk[32];
    float max_scale = 0.f, amax = 0.f;
    for (int j = 0; j < 16; j++) {
        scales[j] = fit_scale_q3(16, 4, xb + 16 * j, L + 16 * j);
        const float a = fabsf(scales[j]);
        if (a > amax) { amax = a; max_scale = scales[j]; }
    }
    for (int i = 0; i < 12; i++) sc[i] = 0;
    uint16_t hd;
    if (max_scale) {
        const float is = -32.f / max_scale;
        for (int j = 0; j < 16; j++) {
            int8_t l = (int8_t) rne_int(is * scales[j]);
            l = (int8_t) (max(-32, min(31, (int) l)) + 32);
            if (j < 8) sc[j] = (uint8_t) (l & 0xF); else sc[j - 8] |= (uint8_t) ((l & 0xF) << 4);
            l >>= 4;
            sc[j % 4 + 8] |= (uint8_t) (l << (2 * (j / 4)));
        }
        hd = f32_to_f16_bits(1 / is);
    } else hd = f32_to_f16_bits(0.f);
    const float fd = f16_bits_to_f32(hd);
    for (int j = 0; j < 16; j++) {
        int8_t s = (int8_t) (j < 8 ? sc[j] & 0xF : sc[j - 8] >> 4);
        s = (int8_t) ((s | (((sc[8 + j % 4] >> (2 * (j / 4))) & 3) << 4)) - 32);
        const float d = fd * s;
        if (!d) continue;
        for (int i = 0; i < 16; i++) L[16 * j + i] = (int8_t) (max(-4, min(3, rne_int(xb[16 * j + i] / d))) + 4);
    }
    for (int i = 0; i < 32; i++) hmk[i] = 0;
    for (int j = 0; j < 256; j++) if (L[j] > 3) { hmk[j % 32] |= (uint8_t) (1u << (j / 32)); L[j] -= 4; }
    for (int i = 0; i < 32; i++) yb[i] = hmk[i];
    uint8_t * qs = yb + 32;
    for (int j = 0; j < 256; j += 128)
        for (int l = 0; l < 32; l++)
            qs[j / 4 + l] = (uint8_t) (L[j + l] | (L[j + l + 32] << 2) | (L[j + l + 64] << 4) | (L[j + l + 96] << 6));
    for (int i = 0; i < 12; i++) yb[96 + i] = sc[i];
    st16(yb + 108, hd);
}

// make_qkx1_quants stops refining after a round that leaves L unchanged, and its round 0 compares against whatever L held before:
// quantize_row_q4_K_reference (and _q2_K / _q5_K) declares L once per call (k_quants.c:546), so block b of a row starts from block
// b-1's final codes.  Whenever a sub-block's round-0 codes equal the ones 256 values earlier -- a repeated or rescaled sub-block does
// it -- the CPU stops after round 0 where fresh codes would refine further.  So one thread walks a whole row and carries L; block 0
// starts from zeros (the CPU reads uninitialised stack there).
template <void (*quantize_block)(const float *, uint8_t *, uint8_t *), int TYPE>
__global__ void __launch_bounds__(32) quantize_rows_kernel(const float * __restrict__ x, uint8_t * __restrict__ y, int64_t nrows,
                                                           int64_t row_blocks) {
    constexpr TypeSpec ts = type_spec(TYPE);
    const int64_t r = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nrows) return;
    uint8_t L[256];
    for (int i = 0; i < 256; i++) L[i] = 0;
    for (int64_t b = r * row_blocks; b < (r + 1) * row_blocks; b++) quantize_block(x + b * ts.blk_elems, y + b * ts.blk_bytes, L);
}

// F16: ggml_fp32_to_fp16_row as the x86-64-v3 (F16C) build runs it: round to nearest even, NaN quietened with its payload kept
__device__ __forceinline__ uint16_t f32_to_f16_f16c(float f) {
    const uint32_t u = __float_as_uint(f);
    if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t) (((u >> 16) & 0x8000u) | 0x7e00u | ((u >> 13) & 0x3ffu));  // vcvtps2ph; CUDA's NaN is 0x7fff
    return f32_to_f16_bits(f);
}
__global__ void f32_to_f16_row_kernel(const float * __restrict__ x, uint16_t * __restrict__ y, int64_t n) {
    for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) y[i] = f32_to_f16_f16c(x[i]);
}

// The 16-bin code histograms ggml_quantize_q4_0 / q4_1 / q5_0 / q5_1 / q8_0 add (ggml.c:19352-19477), from the written blocks of
// block_bytes each.  For Q5_0 / Q5_1 the C loop runs j = 0, 2, .., 30: value j/2's low nibble is binned with bit j of qh, and the high
// nibble with (qh & (1u << (j + 16))) >> (j + 12), shift counts of 32 and more for j >= 16.  The compiled reference (x86, -O3) uses the
// count modulo 32, as x86's shifts do: that is what is reproduced here (tests/test_quantize_file.py pins it against the reference binary).
__global__ void legacy_hist_kernel(int type, int block_bytes, const uint8_t * __restrict__ y, int64_t nblocks, unsigned long long * __restrict__ hist) {
    __shared__ unsigned sh[16];
    if (threadIdx.x < 16) sh[threadIdx.x] = 0;
    __syncthreads();
    for (int64_t b = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; b < nblocks; b += (int64_t) gridDim.x * blockDim.x) {
        const uint8_t * yb = y + b * block_bytes;
        if (type == T_Q8_0) {
            for (int j = 0; j < 32; j++) atomicAdd(&sh[(int8_t) yb[2 + j] / 16 + 8], 1u);
        } else if (type == T_Q4_0 || type == T_Q4_1) {
            const uint8_t * qs = yb + (type == T_Q4_0 ? 2 : 4);
            for (int j = 0; j < 16; j++) { atomicAdd(&sh[qs[j] & 0x0F], 1u); atomicAdd(&sh[qs[j] >> 4], 1u); }
        } else {
            const int qo = type == T_Q5_0 ? 2 : 4;
            const uint32_t qh = (uint32_t) yb[qo] | ((uint32_t) yb[qo + 1] << 8) | ((uint32_t) yb[qo + 2] << 16) | ((uint32_t) yb[qo + 3] << 24);
            const uint8_t * qs = yb + qo + 4;
            for (int j = 0; j < 32; j += 2) {
                const uint8_t vh0 = (uint8_t) (((qh & (1u << j)) >> j) << 4);
                const uint8_t vh1 = (uint8_t) ((qh & (1u << ((j + 16) & 31))) >> ((j + 12) & 31));
                atomicAdd(&sh[(uint8_t) ((qs[j / 2] & 0x0F) | vh0) / 2], 1u);
                atomicAdd(&sh[(uint8_t) ((qs[j / 2] >> 4) | vh1) / 2], 1u);
            }
        }
    }
    __syncthreads();
    if (threadIdx.x < 16 && sh[threadIdx.x]) atomicAdd(&hist[threadIdx.x], (unsigned long long) sh[threadIdx.x]);
}

} // namespace

int64_t launch_quantize_chunks(int ggml_type, const float * x, void * dst, int64_t n, int64_t chunk, unsigned long long * hist_dev,
                               cudaStream_t s) {
    void (*blocks)(const float *, uint8_t *, int64_t) = nullptr;             // one thread per block
    void (*rows)(const float *, uint8_t *, int64_t, int64_t) = nullptr;      // one thread per chunk
    switch (ggml_type) {
        case T_F16: break;
        case T_Q4_0: blocks = quantize_blocks_kernel<quantize_q4_0_block, T_Q4_0>; break;
        case T_Q4_1: blocks = quantize_blocks_kernel<quantize_q4_1_block, T_Q4_1>; break;
        case T_Q5_0: blocks = quantize_blocks_kernel<quantize_q5_block<false>, T_Q5_0>; break;
        case T_Q5_1: blocks = quantize_blocks_kernel<quantize_q5_block<true>, T_Q5_1>; break;
        case T_Q8_0: blocks = quantize_blocks_kernel<quantize_q8_0_block, T_Q8_0>; break;
        case T_Q3_K: blocks = quantize_q3_K_kernel; break;
        case T_Q6_K: blocks = quantize_blocks_kernel<quantize_q6_K_block, T_Q6_K>; break;
        case T_Q2_K: rows = quantize_rows_kernel<quantize_q2_K_block, T_Q2_K>; break;
        case T_Q4_K: rows = quantize_rows_kernel<quantize_q4_K_block, T_Q4_K>; break;
        case T_Q5_K: rows = quantize_rows_kernel<quantize_q5_K_block, T_Q5_K>; break;
        default: return 0;
    }
    const TypeSpec ts = type_spec(ggml_type);
    if (n < 0 || n % ts.blk_elems != 0 || chunk <= 0 || chunk % ts.blk_elems != 0) return -1;
    if (n == 0) return 0;
    uint8_t * y = (uint8_t *) dst;
    const int64_t nb = n / ts.blk_elems;
    if (blocks) {
        const int cta = blocks_cta(ggml_type);
        blocks<<<(unsigned) ((nb + cta - 1) / cta), cta, 0, s>>>(x, y, nb);
    } else if (rows) {                                                  // one chain per full chunk, and the short tail a second launch
        const int64_t full = n / chunk, chain = chunk / 256, tail = (n - full * chunk) / 256;
        if (full) rows<<<(unsigned) ((full + 31) / 32), 32, 0, s>>>(x, y, full, chain);
        if (tail) rows<<<1, 32, 0, s>>>(x + full * chunk, y + full * chain * ts.blk_bytes, 1, tail);
    } else f32_to_f16_row_kernel<<<ew_grid(n), 256, 0, s>>>(x, (uint16_t *) y, n);
    B200_CUDA_CHECK(cudaGetLastError());
    if (hist_dev && ts.blk_elems == 32) {
        legacy_hist_kernel<<<(unsigned) std::min<int64_t>((nb + 255) / 256, 132 * 8), 256, 0, s>>>(ggml_type, ts.blk_bytes, y, nb, hist_dev);
        B200_CUDA_CHECK(cudaGetLastError());
    }
    return nb * ts.blk_bytes;
}

extern "C" int64_t b200_quantize_chunks(int ggml_type, const float * x_dev, void * dst_dev, int64_t n_elems, int64_t chunk_elems,
                                        int64_t * hist16) {
    cudaStream_t s = b200_current_stream();
    unsigned long long * hd = nullptr;
    if (hist16) { B200_CUDA_CHECK(cudaMallocAsync(&hd, 16 * 8, s)); B200_CUDA_CHECK(cudaMemsetAsync(hd, 0, 16 * 8, s)); }
    const int64_t r = launch_quantize_chunks(ggml_type, x_dev, dst_dev, n_elems, chunk_elems, hd, s);
    if (hist16) {
        unsigned long long h[16];
        B200_CUDA_CHECK(cudaMemcpyAsync(h, hd, sizeof(h), cudaMemcpyDeviceToHost, s));
        B200_CUDA_CHECK(cudaFreeAsync(hd, s));
        B200_CUDA_CHECK(cudaStreamSynchronize(s));
        if (r > 0) for (int i = 0; i < 16; i++) hist16[i] += (int64_t) h[i];
    }
    return r;
}

// x_dev: n_elems fp32 values, rows of row_len; blocks_dev: n_elems / block_elems blocks in the file layout.  Returns 1 on success
// (n_elems == 0 launches nothing), 0 if the type has no device quantiser (callers quantise on the host then), -1 if row_len is not a
// positive multiple of the type's block or n_elems not a non-negative multiple of row_len.  Each row is one chunk.
extern "C" int b200_quantize_weights_rows(int ggml_type, const float * x_dev, void * blocks_dev, int64_t n_elems, int64_t row_len) {
    if (ggml_type != T_Q4_0 && !(ggml_type >= T_Q2_K && ggml_type <= T_Q6_K)) return 0;
    const int64_t qk = type_spec(ggml_type).blk_elems;
    if (row_len <= 0 || row_len % qk != 0 || n_elems < 0 || n_elems % row_len != 0) return -1;
    if (n_elems == 0) return 1;
    launch_quantize_chunks(ggml_type, x_dev, blocks_dev, n_elems, row_len, nullptr, b200_current_stream());
    return 1;
}

// the whole buffer as ONE row: one call of quantize_row_q*_reference over n_elems values (what ggml_quantize_chunk does with a
// chunk), so Q2_K / Q4_K / Q5_K carry their codes across the whole buffer on one thread -- for a matrix use the _rows entry point
extern "C" int b200_quantize_weights(int ggml_type, const float * x_dev, void * blocks_dev, int64_t n_elems) {
    return n_elems == 0 ? b200_quantize_weights_rows(ggml_type, x_dev, blocks_dev, 0, 256)
                        : b200_quantize_weights_rows(ggml_type, x_dev, blocks_dev, n_elems, n_elems);
}
