// quant_gpu.cu -- fp32 -> GGML weight blocks on the device, bit for bit what the reference's quantisers write
// (SURVEY section 8f-3, first two types: the ones BASELINE's models use).
//   Q4_0: quantize_row_q4_0_reference, ggml.c:927-962
//   Q4_K: quantize_row_q4_K_reference, k_quants.c:542-605, with make_qkx1_quants (:222-262) and nearest_int (:50-55)
// Q4_0: one thread per block.  Q4_K: one thread per row, walking its blocks in order (make_qkx1_quants carries codes from block
// to block, see quantize_q4_K_kernel).  The arithmetic is the CPU's, in its order, with explicitly rounded fp32 operations (no FMA
// contraction), so that every intermediate equals the scalar C code's; blocks are written in the file layout (18 / 144 bytes),
// ready for b200_weight_upload or a GGCC file.
#include "kernels.h"

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
