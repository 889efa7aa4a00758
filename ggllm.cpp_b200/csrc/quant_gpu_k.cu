// quant_gpu_k.cu -- fp32 -> Q2_K / Q3_K / Q5_K / Q6_K weight blocks on the device, bit for bit what the reference's quantisers write
// (SURVEY section 8f-3; Q4_0 / Q4_K live in quant_gpu.cu):
//   Q2_K  quantize_row_q2_K_reference, k_quants.c:275-342     (make_qkx1_quants :222-262 on 16 sub-blocks of 16, 4-bit scales / mins)
//   Q3_K  quantize_row_q3_K_reference, k_quants.c:396-470     (make_q3_quants :163-220, 6-bit signed scales, high-bit mask)
//   Q5_K  quantize_row_q5_K_reference, k_quants.c:652-732     (make_qkx1_quants on 8 sub-blocks of 32, 6-bit scales / mins, qh plane)
//   Q6_K  quantize_row_q6_K_reference, k_quants.c:781-843     (make_qx_quants rmse_type 1 :57-161, int8 scales)
// Q3_K / Q6_K: one thread per 256-value block.  Q2_K / Q5_K: one thread per row, walking its blocks in order and carrying
// make_qkx1_quants's codes from block to block (quant_gpu.cu, quantize_q4_K_kernel, says why).  The arithmetic is the scalar C
// code's, in its order.  THIS FILE IS COMPILED WITH --fmad=false (csrc/Makefile): every a * b + c below is a separately rounded multiply and add, divisions are IEEE, so each intermediate equals
// the CPU's (the reference is built without fp contraction).  Blocks are written in the file layout (84 / 110 / 176 / 210 bytes).
// A Falcon-40B ffn_up (32768 rows of 8192) takes 1-6 ms per type on an H100 80GB (tools/quantise_bench.py).
#include "kernels.h"

cudaStream_t b200_current_stream();

namespace {

__device__ __forceinline__ int rne_int(float v) {                     // nearest_int, k_quants.c:50-55: the 1.5 * 2^23 magic constant
    const float t = v + 12582912.f;
    if (t != t) return 0;                                             // x86's default NaN 0x7fc00000 gives 0 by the formula below; CUDA's NaN is 0x7fffffff
    return (__float_as_int(t) & 0x007fffff) - 0x00400000;
}
__device__ __forceinline__ void st16(uint8_t * p, uint16_t v) { *reinterpret_cast<uint16_t *>(p) = v; }      // all fp16 fields sit at even offsets of even-sized blocks
__device__ __forceinline__ int imin(int a, int b) { return a < b ? a : b; }
__device__ __forceinline__ int imax(int a, int b) { return a > b ? a : b; }

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
            const int l = imax(0, imin(nmax, rne_int(iscale * (x[i] - mn))));
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
        const int l = imax(-nmax, imin(nmax - 1, rne_int(iscale * x[i])));
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
                const int nl = imax(-nmax, imin(nmax - 1, rne_int(x[i] * sl2 / slx)));
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
        const int l = imax(-nmax, imin(nmax - 1, rne_int(iscale * x[i])));
        L[i] = (int8_t) (l + nmax);
        const float w = x[i] * x[i];
        sumlx += w * x[i] * l; suml2 += w * l * l;
    }
    float scale = sumlx / suml2, best = scale * sumlx;
    for (int t = 0; t < 3; t++) {
        iscale = 1 / scale;
        float slx = 0.f, sl2 = 0.f; bool changed = false;
        for (int i = 0; i < n; i++) {
            const int l = imax(-nmax, imin(nmax - 1, rne_int(iscale * x[i])));
            if (l + nmax != L[i]) changed = true;
            const float w = x[i] * x[i];
            slx += w * x[i] * l; sl2 += w * l * l;
        }
        if (!changed || sl2 == 0.f || slx * slx <= best * sl2) break;
        for (int i = 0; i < n; i++) L[i] = (int8_t) (nmax + imax(-nmax, imin(nmax - 1, rne_int(iscale * x[i]))));
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
                const int nl = imax(-nmax, imin(nmax - 1, rne_int(x[i] * sl2 / slx)));
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

// one block each; L carries the previous block's codes in and this block's out
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
        for (int i = 0; i < 16; i++) L[16 * j + i] = (uint8_t) imax(0, imin(3, rne_int((xb[16 * j + i] + dm) / d)));
    }
    uint8_t * qs = yb + 16;
    for (int j = 0; j < 256; j += 128)
        for (int l = 0; l < 32; l++)
            qs[j / 4 + l] = (uint8_t) (L[j + l] | (L[j + l + 32] << 2) | (L[j + l + 64] << 4) | (L[j + l + 96] << 6));
}

__global__ void __launch_bounds__(64) quantize_q3_K_kernel(const float * __restrict__ x, uint8_t * __restrict__ y, int64_t nblocks) {
    const int64_t b = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    const float * xb = x + b * 256; uint8_t * yb = y + b * 110;
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
            l = (int8_t) (imax(-32, imin(31, (int) l)) + 32);
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
        for (int i = 0; i < 16; i++) L[16 * j + i] = (int8_t) (imax(-4, imin(3, rne_int(xb[16 * j + i] / d))) + 4);
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

__device__ __forceinline__ void pack_sm6(int j, uint8_t * q, uint8_t ls, uint8_t lm) {      // k_quants.c:565-578 / 681-690
    if (j < 4) { q[j] = ls; q[j + 4] = lm; }
    else { q[j + 4] = (uint8_t) ((ls & 0xF) | ((lm & 0xF) << 4)); q[j - 4] |= (uint8_t) ((ls >> 4) << 6); q[j] |= (uint8_t) ((lm >> 4) << 6); }
}

__device__ void quantize_q5_K_block(const float * __restrict__ xb, uint8_t * __restrict__ yb, uint8_t * L) {
    float mins[8], scales[8]; uint8_t sc[12], qh[32];
    for (int i = 0; i < 12; i++) sc[i] = 0;
    float max_scale = 0.f, max_min = 0.f;
    for (int j = 0; j < 8; j++) {
        scales[j] = fit_scale_min(32, 31, xb + 32 * j, L + 32 * j, mins[j]);
        if (scales[j] > max_scale) max_scale = scales[j];
        if (mins[j] > max_min) max_min = mins[j];
    }
    const float inv_s = max_scale > 0.f ? 63.f / max_scale : 0.f, inv_m = max_min > 0.f ? 63.f / max_min : 0.f;
    for (int j = 0; j < 8; j++) {
        const uint8_t ls = (uint8_t) rne_int(inv_s * scales[j]), lm = (uint8_t) rne_int(inv_m * mins[j]);
        pack_sm6(j, sc, (uint8_t) imin(63, (int) ls), (uint8_t) imin(63, (int) lm));
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
        for (int i = 0; i < 32; i++) L[32 * j + i] = (uint8_t) imax(0, imin(31, rne_int((xb[32 * j + i] + dm) / d)));
    }
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

// one thread per row: the blocks in order, L carried from each to the next and zero at the row's start
template <void (*quantize_block)(const float *, uint8_t *, uint8_t *), int BLOCK_BYTES>
__global__ void __launch_bounds__(32) quantize_rows_kernel(const float * __restrict__ x, uint8_t * __restrict__ y, int64_t nrows,
                                                           int64_t row_blocks) {
    const int64_t r = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nrows) return;
    uint8_t L[256];
    for (int i = 0; i < 256; i++) L[i] = 0;
    for (int64_t b = r * row_blocks; b < (r + 1) * row_blocks; b++) quantize_block(x + b * 256, y + b * BLOCK_BYTES, L);
}

__global__ void __launch_bounds__(64) quantize_q6_K_kernel(const float * __restrict__ x, uint8_t * __restrict__ y, int64_t nblocks) {
    const int64_t b = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    const float * xb = x + b * 256; uint8_t * yb = y + b * 210;
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
    for (int j = 0; j < 16; j++) { sc[j] = (int8_t) imin(127, rne_int(is * scales[j])); yb[192 + j] = (uint8_t) sc[j]; }
    const float fd = f16_bits_to_f32(hd);
    for (int j = 0; j < 16; j++) {
        const float d = fd * sc[j];
        if (!d) continue;
        for (int i = 0; i < 16; i++) L[16 * j + i] = (int8_t) (imax(-32, imin(31, rne_int(xb[16 * j + i] / d))) + 32);
    }
    uint8_t * ql = yb, * qh = yb + 128;
    for (int j = 0; j < 256; j += 128, ql += 64, qh += 32)
        for (int l = 0; l < 32; l++) {
            const uint8_t q1 = L[j + l] & 0xF, q2 = L[j + l + 32] & 0xF, q3 = L[j + l + 64] & 0xF, q4 = L[j + l + 96] & 0xF;
            ql[l] = (uint8_t) (q1 | (q3 << 4)); ql[l + 32] = (uint8_t) (q2 | (q4 << 4));
            qh[l] = (uint8_t) ((L[j + l] >> 4) | ((L[j + l + 32] >> 4) << 2) | ((L[j + l + 64] >> 4) << 4) | ((L[j + l + 96] >> 4) << 6));
        }
}

} // namespace

// nrows rows of row_blocks 256-value blocks, nrows > 0; returns false for a type this file does not cover
bool launch_quantize_kquant(int ggml_type, const float * x_dev, void * blocks_dev, int64_t nrows, int64_t row_blocks, cudaStream_t s) {
    const int64_t nb = nrows * row_blocks;
    const unsigned grid = (unsigned) ((nb + 63) / 64), row_grid = (unsigned) ((nrows + 31) / 32);
    uint8_t * y = (uint8_t *) blocks_dev;
    switch (ggml_type) {
        case T_Q2_K: quantize_rows_kernel<quantize_q2_K_block, 84><<<row_grid, 32, 0, s>>>(x_dev, y, nrows, row_blocks); break;
        case T_Q3_K: quantize_q3_K_kernel<<<grid, 64, 0, s>>>(x_dev, y, nb); break;
        case T_Q5_K: quantize_rows_kernel<quantize_q5_K_block, 176><<<row_grid, 32, 0, s>>>(x_dev, y, nrows, row_blocks); break;
        case T_Q6_K: quantize_q6_K_kernel<<<grid, 64, 0, s>>>(x_dev, y, nb); break;
        default: return false;
    }
    B200_CUDA_CHECK(cudaGetLastError());
    return true;
}
