// quant_gpu.cu -- fp32 -> GGML weight blocks on the device, bit for bit what the reference's quantisers write
// (SURVEY section 8f-3), and b200_quantize_chunks, ggml_quantize_chunk over falcon_quantize's chunks for every output type.
//   Q4_0: quantize_row_q4_0_reference, ggml.c:927-962;  Q4_1 / Q5_0 / Q5_1 / Q8_0 / F16 further down
//   Q4_K: quantize_row_q4_K_reference, k_quants.c:542-605, with make_qkx1_quants (:222-262) and nearest_int (:50-55)
// Q4_0: one thread per block.  Q4_K: one thread per row, walking its blocks in order (make_qkx1_quants carries codes from block
// to block, see quantize_q4_K_kernel).  The arithmetic is the CPU's, in its order, with explicitly rounded fp32 operations (no FMA
// contraction), so that every intermediate equals the scalar C code's; blocks are written in the file layout (18 / 144 bytes),
// ready for b200_weight_upload or a GGCC file.
#include "kernels.h"
#include <algorithm>
#include <cfloat>

cudaStream_t b200_current_stream();
bool launch_quantize_kquant(int ggml_type, const float * x_dev, void * blocks_dev, int64_t nrows, int64_t row_blocks, cudaStream_t s);

__device__ __forceinline__ int rne_int_dev(float v) {                 // nearest_int: the 1.5 * 2^23 magic constant
    const float t = __fadd_rn(v, 12582912.f);
    if (t != t) return 0;                                             // x86 propagates the default NaN 0x7fc00000 -> 0 by the formula below; CUDA's NaN is 0x7fffffff
    return (__float_as_int(t) & 0x007fffff) - 0x00400000;
}
// (block sizes 18 and 144 are even, so the fp16 fields are 2-byte aligned; a byte-wise store of `(uint8_t) bits` was compiled into a
//  NUMERIC half -> u8 conversion by nvcc 12.9, F2I.U8.F16 in the SASS -- hence the single 16-bit store)
__device__ __forceinline__ void st16_dev(uint8_t * p, uint16_t v) { *reinterpret_cast<uint16_t *>(p) = v; }

__global__ void quantize_q4_0_kernel(const float * __restrict__ x, uint8_t * __restrict__ y, int64_t nblocks) {
    const int64_t b = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    const float * xb = x + b * 32; uint8_t * yb = y + b * 18;
    float amax = 0.f, vmax = 0.f;
    for (int j = 0; j < 32; j++) { const float v = xb[j]; if (amax < fabsf(v)) { amax = fabsf(v); vmax = v; } }
    const float d = __fdiv_rn(vmax, -8.f), id = d != 0.f ? __fdiv_rn(1.0f, d) : 0.0f;
    st16_dev(yb, f32_to_f16_bits(d));
    for (int j = 0; j < 16; j++) {
        const int lo = min(15, (int) (int8_t) __float2int_rz(__fadd_rn(__fmul_rn(xb[j], id), 8.5f)));
        const int hi = min(15, (int) (int8_t) __float2int_rz(__fadd_rn(__fmul_rn(xb[j + 16], id), 8.5f)));
        yb[2 + j] = (uint8_t) ((lo & 0xff) | (hi << 4));
    }
}

// make_qkx1_quants: asymmetric (scale, min) fit of 32 values to levels 0..15, five refinement rounds
__device__ float fit_scale_min_dev(const float * x, uint8_t * L, float & the_min) {
    float mn = x[0], mx = x[0];
    for (int i = 1; i < 32; i++) { if (x[i] < mn) mn = x[i]; if (x[i] > mx) mx = x[i]; }
    if (mx == mn) { for (int i = 0; i < 32; i++) L[i] = 0; the_min = 0.f; return 0.f; }
    if (mn > 0.f) mn = 0.f;
    float iscale = __fdiv_rn(15.f, __fsub_rn(mx, mn)), scale = __fdiv_rn(1.f, iscale);
    for (int t = 0; t < 5; t++) {
        float sumlx = 0.f; int suml2 = 0; bool changed = false;
        for (int i = 0; i < 32; i++) {
            const float xm = __fsub_rn(x[i], mn);
            const int l = max(0, min(15, rne_int_dev(__fmul_rn(iscale, xm))));
            if (l != L[i]) { L[i] = (uint8_t) l; changed = true; }
            sumlx = __fadd_rn(sumlx, __fmul_rn(xm, (float) l)); suml2 += l * l;
        }
        scale = __fdiv_rn(sumlx, (float) suml2);
        float sum = 0.f;
        for (int i = 0; i < 32; i++) sum = __fadd_rn(sum, __fsub_rn(x[i], __fmul_rn(scale, (float) L[i])));
        mn = __fdiv_rn(sum, 32.f); if (mn > 0.f) mn = 0.f;
        iscale = __fdiv_rn(1.f, scale);
        if (!changed) break;
    }
    the_min = -mn;
    return scale;
}
__device__ __forceinline__ void pack_sm6_dev(int j, uint8_t * q, uint8_t ls, uint8_t lm) {      // k_quants.c:565-578
    if (j < 4) { q[j] = ls; q[j + 4] = lm; }
    else { q[j + 4] = (uint8_t) ((ls & 0xF) | ((lm & 0xF) << 4)); q[j - 4] |= (uint8_t) ((ls >> 4) << 6); q[j] |= (uint8_t) ((lm >> 4) << 6); }
}

// one Q4_K block.  L holds the codes of the row's previous block on entry (zeros for block 0) and this block's on exit.
__device__ void quantize_q4_K_block(const float * __restrict__ xb, uint8_t * __restrict__ yb, uint8_t * L) {
    float mins[8], scales[8];
    uint8_t sc[12];
    for (int i = 0; i < 12; i++) sc[i] = 0;
    float max_scale = 0.f, max_min = 0.f;
    for (int j = 0; j < 8; j++) {
        scales[j] = fit_scale_min_dev(xb + 32 * j, L + 32 * j, mins[j]);
        if (scales[j] > max_scale) max_scale = scales[j];
        if (mins[j] > max_min) max_min = mins[j];
    }
    const float inv_s = max_scale > 0.f ? __fdiv_rn(63.f, max_scale) : 0.f, inv_m = max_min > 0.f ? __fdiv_rn(63.f, max_min) : 0.f;
    for (int j = 0; j < 8; j++) {
        const uint8_t ls = (uint8_t) rne_int_dev(__fmul_rn(inv_s, scales[j])), lm = (uint8_t) rne_int_dev(__fmul_rn(inv_m, mins[j]));
        pack_sm6_dev(j, sc, (uint8_t) min(63, (int) ls), (uint8_t) min(63, (int) lm));
    }
    const uint16_t hd = f32_to_f16_bits(__fdiv_rn(max_scale, 63.f)), hm = f32_to_f16_bits(__fdiv_rn(max_min, 63.f));
    st16_dev(yb, hd); st16_dev(yb + 2, hm);
    for (int i = 0; i < 12; i++) yb[4 + i] = sc[i];
    const float fd = f16_bits_to_f32(hd), fm = f16_bits_to_f32(hm);
    for (int j = 0; j < 8; j++) {
        int s, m; unpack_sm6(j, sc, s, m);
        const float d = __fmul_rn(fd, (float) s);
        if (d == 0.f) continue;
        const float dm = __fmul_rn(fm, (float) m);
        for (int i = 0; i < 32; i++) L[32 * j + i] = (uint8_t) max(0, min(15, rne_int_dev(__fdiv_rn(__fadd_rn(xb[32 * j + i], dm), d))));
    }
    uint8_t * q = yb + 16;
    for (int j = 0; j < 256; j += 64) for (int l = 0; l < 32; l++) *q++ = (uint8_t) (L[j + l] | (L[j + l + 32] << 4));
}

// make_qkx1_quants stops refining after a round that leaves L unchanged, and its round 0 compares against whatever L held before:
// quantize_row_q4_K_reference declares L once per call (k_quants.c:546), so block b of a row starts from block b-1's final codes.  Whenever a
// sub-block's round-0 codes equal the ones 256 values earlier -- a repeated or rescaled sub-block does it -- the CPU stops after
// round 0 where fresh codes would refine further.  So one thread walks a whole row and carries L; block 0 starts from zeros (the
// CPU reads uninitialised stack there).
__global__ void __launch_bounds__(32) quantize_q4_K_kernel(const float * __restrict__ x, uint8_t * __restrict__ y, int64_t nrows,
                                                           int64_t row_blocks) {
    const int64_t r = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nrows) return;
    uint8_t L[256];
    for (int i = 0; i < 256; i++) L[i] = 0;
    for (int64_t b = r * row_blocks; b < (r + 1) * row_blocks; b++) quantize_q4_K_block(x + b * 256, y + b * 144, L);
}

// x_dev: n_elems fp32 values, rows of row_len; blocks_dev: n_elems / block_elems blocks in the file layout.  Returns 1 on success
// (n_elems == 0 launches nothing), 0 if the type has no device quantiser (callers quantise on the host then), -1 if row_len is not a
// positive multiple of the type's block or n_elems not a non-negative multiple of row_len.
extern "C" int b200_quantize_weights_rows(int ggml_type, const float * x_dev, void * blocks_dev, int64_t n_elems, int64_t row_len) {
    const int64_t qk = ggml_type == T_Q4_0 ? 32 : 256;
    if (ggml_type != T_Q4_0 && ggml_type != T_Q2_K && ggml_type != T_Q3_K && ggml_type != T_Q4_K && ggml_type != T_Q5_K &&
        ggml_type != T_Q6_K) return 0;
    if (row_len <= 0 || row_len % qk != 0 || n_elems < 0 || n_elems % row_len != 0) return -1;
    if (n_elems == 0) return 1;
    cudaStream_t s = b200_current_stream();
    if (ggml_type == T_Q4_0) {
        const int64_t nb = n_elems / 32;
        quantize_q4_0_kernel<<<(unsigned) ((nb + 255) / 256), 256, 0, s>>>(x_dev, (uint8_t *) blocks_dev, nb);
    } else if (ggml_type == T_Q4_K) {
        const int64_t nrows = n_elems / row_len;
        quantize_q4_K_kernel<<<(unsigned) ((nrows + 31) / 32), 32, 0, s>>>(x_dev, (uint8_t *) blocks_dev, nrows, row_len / 256);
    } else launch_quantize_kquant(ggml_type, x_dev, blocks_dev, n_elems / row_len, row_len / 256, s);      // quant_gpu_k.cu
    B200_CUDA_CHECK(cudaGetLastError());
    return 1;
}

// the whole buffer as ONE row: one call of quantize_row_q*_reference over n_elems values (what ggml_quantize_chunk does with a
// chunk), so Q2_K / Q4_K / Q5_K carry their codes across the whole buffer on one thread -- for a matrix use the _rows entry point
extern "C" int b200_quantize_weights(int ggml_type, const float * x_dev, void * blocks_dev, int64_t n_elems) {
    return n_elems == 0 ? b200_quantize_weights_rows(ggml_type, x_dev, blocks_dev, 0, 256)
                        : b200_quantize_weights_rows(ggml_type, x_dev, blocks_dev, n_elems, n_elems);
}

// ---- the remaining falcon_quantize output types, one thread per block (or value), each in its C function's order and rounding:
//   Q4_1 quantize_row_q4_1_reference ggml.c:968-1002     Q5_0 :1008-1046     Q5_1 :1052-1090     Q8_0 :1106-1129
//   F16  ggml_fp32_to_fp16_row as the x86-64-v3 (F16C) build runs it: round to nearest even, NaN quietened with its payload kept
__device__ __forceinline__ uint16_t f32_to_f16_f16c(float f) {
    const uint32_t u = __float_as_uint(f);
    if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t) (((u >> 16) & 0x8000u) | 0x7e00u | ((u >> 13) & 0x3ffu));  // vcvtps2ph; CUDA's NaN is 0x7fff
    return f32_to_f16_bits(f);
}
__global__ void f32_to_f16_row_kernel(const float * __restrict__ x, uint16_t * __restrict__ y, int64_t n) {
    for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) y[i] = f32_to_f16_f16c(x[i]);
}

__global__ void quantize_q4_1_kernel(const float * __restrict__ x, uint8_t * __restrict__ y, int64_t nblocks) {
    const int64_t b = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    const float * xb = x + b * 32; uint8_t * yb = y + b * 20;
    float mn = FLT_MAX, mx = -FLT_MAX;
    for (int j = 0; j < 32; j++) { const float v = xb[j]; if (v < mn) mn = v; if (v > mx) mx = v; }
    const float d = __fdiv_rn(__fsub_rn(mx, mn), 15.f), id = d != 0.f ? __fdiv_rn(1.0f, d) : 0.0f;
    st16_dev(yb, f32_to_f16_bits(d)); st16_dev(yb + 2, f32_to_f16_bits(mn));
    for (int j = 0; j < 16; j++) {
        const int lo = min(15, (int) (int8_t) __float2int_rz(__fadd_rn(__fmul_rn(__fsub_rn(xb[j], mn), id), 0.5f)));
        const int hi = min(15, (int) (int8_t) __float2int_rz(__fadd_rn(__fmul_rn(__fsub_rn(xb[j + 16], mn), id), 0.5f)));
        yb[4 + j] = (uint8_t) ((lo & 0xff) | (hi << 4));
    }
}

// Q5_0 (ASYM false) and Q5_1 (ASYM true): 4 low bits in qs, the fifth bit of value j in bit j of qh
template <bool ASYM>
__global__ void quantize_q5_kernel(const float * __restrict__ x, uint8_t * __restrict__ y, int64_t nblocks) {
    const int64_t b = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    const float * xb = x + b * 32; uint8_t * yb = y + b * (ASYM ? 24 : 22);
    float d, mn = 0.f;
    if (ASYM) {
        float mx = -FLT_MAX; mn = FLT_MAX;
        for (int j = 0; j < 32; j++) { const float v = xb[j]; if (v < mn) mn = v; if (v > mx) mx = v; }
        d = __fdiv_rn(__fsub_rn(mx, mn), 31.f);
        st16_dev(yb, f32_to_f16_bits(d)); st16_dev(yb + 2, f32_to_f16_bits(mn));
    } else {
        float amax = 0.f, vmax = 0.f;
        for (int j = 0; j < 32; j++) { const float v = xb[j]; if (amax < fabsf(v)) { amax = fabsf(v); vmax = v; } }
        d = __fdiv_rn(vmax, -16.f);
        st16_dev(yb, f32_to_f16_bits(d));
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
    st16_dev(yb + (ASYM ? 4 : 2), (uint16_t) qh); st16_dev(yb + (ASYM ? 6 : 4), (uint16_t) (qh >> 16));
}

__global__ void quantize_q8_0_kernel(const float * __restrict__ x, uint8_t * __restrict__ y, int64_t nblocks) {
    const int64_t b = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nblocks) return;
    const float * xb = x + b * 32; uint8_t * yb = y + b * 34;
    float amax = 0.f;
    for (int j = 0; j < 32; j++) { const float a = fabsf(xb[j]); amax = amax > a ? amax : a; }      // MAX(amax, fabsf(v))
    const float d = __fdiv_rn(amax, 127.f), id = d != 0.f ? __fdiv_rn(1.0f, d) : 0.0f;
    st16_dev(yb, f32_to_f16_bits(d));
    for (int j = 0; j < 32; j++) yb[2 + j] = (uint8_t) (int8_t) __float2int_rz(roundf(__fmul_rn(xb[j], id)));
}

// The 16-bin code histograms ggml_quantize_q4_0 / q4_1 / q5_0 / q5_1 / q8_0 add (ggml.c:19352-19477), from the written blocks.  For
// Q5_0 / Q5_1 the C loop runs j = 0, 2, .., 30: value j/2's low nibble is binned with bit j of qh, and the high nibble with
// (qh & (1u << (j + 16))) >> (j + 12), shift counts of 32 and more for j >= 16.  The compiled reference (x86, -O3) uses the count
// modulo 32, as x86's shifts do: that is what is reproduced here (tests/test_quantize_file.py pins it against the reference binary).
__global__ void legacy_hist_kernel(int type, const uint8_t * __restrict__ y, int64_t nblocks, unsigned long long * __restrict__ hist) {
    __shared__ unsigned sh[16];
    if (threadIdx.x < 16) sh[threadIdx.x] = 0;
    __syncthreads();
    const int bb = type == T_Q4_0 ? 18 : type == T_Q4_1 ? 20 : type == T_Q5_0 ? 22 : type == T_Q5_1 ? 24 : 34;
    for (int64_t b = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; b < nblocks; b += (int64_t) gridDim.x * blockDim.x) {
        const uint8_t * yb = y + b * bb;
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

static bool is_legacy(int t) { return t == T_Q4_0 || t == T_Q4_1 || t == T_Q5_0 || t == T_Q5_1 || t == T_Q8_0; }

int64_t quantize_out_bytes(int ggml_type, int64_t n_elems) {
    switch (ggml_type) {
        case T_F16: return n_elems * 2;
        case T_Q4_0: return n_elems / 32 * 18; case T_Q4_1: return n_elems / 32 * 20; case T_Q5_0: return n_elems / 32 * 22;
        case T_Q5_1: return n_elems / 32 * 24; case T_Q8_0: return n_elems / 32 * 34;
        case T_Q2_K: return n_elems / 256 * 84; case T_Q3_K: return n_elems / 256 * 110; case T_Q4_K: return n_elems / 256 * 144;
        case T_Q5_K: return n_elems / 256 * 176; case T_Q6_K: return n_elems / 256 * 210;
    }
    return 0;
}

// ggml_quantize_chunk (ggml.c:19479-19560) over consecutive chunks of chunk_elems values, the last one shorter, enqueued on `s`.
// Only the carried types (make_qkx1_quants: Q2_K, Q4_K, Q5_K) see the chunks: one chain per full chunk, and the short tail a second
// launch; every other type is one launch over the whole buffer.  hist_dev (16 counters, or null) accumulates the legacy histograms.
// Returns the bytes written, 0 for a type outside falcon_quantize's outputs, -1 for a bad shape.
int64_t launch_quantize_chunks(int ggml_type, const float * x, void * dst, int64_t n, int64_t chunk, unsigned long long * hist_dev,
                               cudaStream_t s) {
    if (ggml_type != T_F16 && !is_legacy(ggml_type) && !(ggml_type >= T_Q2_K && ggml_type <= T_Q6_K)) return 0;
    const int64_t out = quantize_out_bytes(ggml_type, n);
    const int64_t qk = ggml_type == T_F16 ? 1 : is_legacy(ggml_type) ? 32 : 256;
    if (n < 0 || n % qk != 0 || chunk <= 0 || chunk % qk != 0) return -1;
    if (n == 0) return 0;
    uint8_t * y = (uint8_t *) dst;
    const int64_t nb = n / qk;
    const unsigned grid = (unsigned) ((nb + 255) / 256);
    switch (ggml_type) {
        case T_F16: f32_to_f16_row_kernel<<<(unsigned) std::min<int64_t>((n + 255) / 256, 132 * 16), 256, 0, s>>>(x, (uint16_t *) y, n); break;
        case T_Q4_0: quantize_q4_0_kernel<<<grid, 256, 0, s>>>(x, y, nb); break;
        case T_Q4_1: quantize_q4_1_kernel<<<grid, 256, 0, s>>>(x, y, nb); break;
        case T_Q5_0: quantize_q5_kernel<false><<<grid, 256, 0, s>>>(x, y, nb); break;
        case T_Q5_1: quantize_q5_kernel<true><<<grid, 256, 0, s>>>(x, y, nb); break;
        case T_Q8_0: quantize_q8_0_kernel<<<grid, 256, 0, s>>>(x, y, nb); break;
        case T_Q3_K: case T_Q6_K: launch_quantize_kquant(ggml_type, x, y, 1, nb, s); break;
        default: {                                                      // Q2_K, Q4_K, Q5_K: one chain per chunk
            const int64_t full = n / chunk, chain = chunk / 256, tail = (n - full * chunk) / 256, bb = out / nb;
            auto chains = [&](const float * xc, uint8_t * yc, int64_t nrows, int64_t row_blocks) {
                if (ggml_type == T_Q4_K) quantize_q4_K_kernel<<<(unsigned) ((nrows + 31) / 32), 32, 0, s>>>(xc, yc, nrows, row_blocks);
                else launch_quantize_kquant(ggml_type, xc, yc, nrows, row_blocks, s);
            };
            if (full) chains(x, y, full, chain);
            if (tail) chains(x + full * chunk, y + full * chain * bb, 1, tail);
        }
    }
    B200_CUDA_CHECK(cudaGetLastError());
    if (hist_dev && is_legacy(ggml_type)) {
        legacy_hist_kernel<<<(unsigned) std::min<int64_t>((nb + 255) / 256, 132 * 8), 256, 0, s>>>(ggml_type, y, nb, hist_dev);
        B200_CUDA_CHECK(cudaGetLastError());
    }
    return out;
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
