// formats.cuh -- device-side layout of GGML block-quantised weights and of quantised activations.
//
// Weights arrive in the reference's array-of-structs block formats (block_q4_0 .. block_q6_K,
// ggml.c:879-916, k_quants.h:20-74) whose block sizes (18, 20, 22, 24, 34, 84, 110, 144, 176, 210 bytes) give
// rows that are only 2-byte aligned.  The backend owns the device copy (ggml_cuda_transform_tensor,
// ggml-cuda.cu:3030-3073), so at upload every matrix is split into PLANES: per row, all quant bytes of all
// blocks contiguous, then (separate plane) all scales, etc.  Every plane row starts 16-byte aligned, so the
// mat-vec kernels issue fully coalesced 16-byte loads and the GEMM producer can fetch rectangular tiles.
// The repack is a pure byte permutation: dequantisation stays bit-exact (tests/test_codecs_gpu.py).
#pragma once
#include "common.cuh"

#define B200_MAX_PLANES 4

// where a plane's bytes come from inside one source block.  kind 0: `bytes` copied verbatim from src_off;
// kind 1 (Q4_K/Q5_K scales): the 12-byte packed 6-bit (scale,min) field at src_off is expanded losslessly into
// 16 bytes, {sc[2p], sc[2p+1], min[2p], min[2p+1]} for p = 0..3 (get_scale_min_k4, k_quants.c:264-271), so that a
// lane fetches the four values of its sub-block pair with one 32-bit load and feeds them straight to dp2a.
// kind 2 (Q3_K scales): the 12-byte packed 6-bit field -> 16 SIGNED bytes (scale - 32, k_quants.c:486-493 + :646), ordered so that
// the four scales of a 16-byte qs piece are one 32-bit word: byte 4 * (2n + c) + quad = scale of elements 128n + 32 quad + 16c ..+15.
struct PlaneSpec { int src_off; int bytes; int kind; };
struct TypeSpec {
    int blk_elems;      // weights per block (32 legacy, 256 K-quants, 1 for f16/f32)
    int blk_bytes;      // bytes per source block
    int n_planes;
    PlaneSpec plane[B200_MAX_PLANES];
};

// plane 0 is always the main quant plane
static constexpr TypeSpec type_spec(int t) {
    switch (t) {
        case T_F32:  return {1, 4, 1, {{0, 4}}};
        case T_F16:  return {1, 2, 1, {{0, 2}}};
        case T_Q4_0: return {32, 18, 2, {{2, 16}, {0, 2}}};                          // qs | d
        case T_Q4_1: return {32, 20, 2, {{4, 16}, {0, 4}}};                          // qs | d,m
        case T_Q5_0: return {32, 22, 3, {{6, 16}, {2, 4}, {0, 2}}};                  // qs | qh | d
        case T_Q5_1: return {32, 24, 3, {{8, 16}, {4, 4}, {0, 4}}};                  // qs | qh | d,m
        case T_Q8_0: return {32, 34, 2, {{2, 32}, {0, 2}}};                          // qs | d
        case T_Q2_K: return {256, 84, 3, {{16, 64}, {0, 16}, {80, 4}}};              // qs | scales | d,dmin
        case T_Q3_K: return {256, 110, 4, {{32, 64}, {0, 32}, {96, 16, 2}, {108, 2}}}; // qs | hmask | scales (expanded, signed) | d
        case T_Q4_K: return {256, 144, 3, {{16, 128}, {4, 16, 1}, {0, 4}}};          // qs | scales+mins (expanded) | d,dmin
        case T_Q5_K: return {256, 176, 4, {{48, 128}, {16, 32}, {4, 16, 1}, {0, 4}}}; // qs | qh | scales+mins (expanded) | d,dmin
        case T_Q6_K: return {256, 210, 4, {{0, 128}, {128, 64}, {192, 16}, {208, 2}}}; // ql | qh | scales | d
    }
    return {0, 0, 0, {}};
}

// device-resident weight matrix: M rows of K weights (ggml: ne0 = K contiguous, ne1 = M)
struct WPlanes {
    int type, K, M, nb;                       // nb = blocks per row
    uint8_t * p[B200_MAX_PLANES];             // plane base pointers (one allocation, p[0] owns it)
    uint32_t stride[B200_MAX_PLANES];         // bytes per row of each plane (multiple of 16)
    size_t bytes;                             // total allocation
};

// quantised activations ("vec_dot_type" of the weight type, ggml.c:1627-1718), N rows of K values, planar:
//   q  int8 [N][K]        codes
//   d  f32  [N][K/blk]    scale  (Q8_0: the fp16-rounded value, widened)
//   s  f32  [N][K/32]     Q8_1 only: d * sum(q)
//   bs i16  [N][K/16]     Q8_K: sums of 16 codes (block_q8_K.bsums); Q8_0/Q8_1: [N][K/32] sum of the block's codes
//   h  f16  [N][K]        optional: the dequantised value d * q rounded to fp16 -- the B operand of the tensor-core GEMM -- written by the
//                         same kernel that produces the codes (prompt path), so no separate conversion pass runs
struct ActQ {
    int type, K, N;
    int8_t * q; float * d; float * s; int16_t * bs;
    __half * h;
};
static inline int act_block(int t) { return t == T_Q8_K ? 256 : 32; }
static inline int act_type_for(int wtype) {
    switch (wtype) {
        case T_Q4_0: case T_Q5_0: case T_Q8_0: return T_Q8_0;
        case T_Q4_1: case T_Q5_1: return T_Q8_1;
        case T_Q2_K: case T_Q3_K: case T_Q4_K: case T_Q5_K: case T_Q6_K: return T_Q8_K;
    }
    return -1;
}

#ifdef __CUDACC__
// ------------------------------------------------------------------------------------------------
// Bit-exact element dequantisation from the planar layout.  All arithmetic uses explicit _rn
// intrinsics so that nvcc cannot fuse the multiply with the subtract (the CPU reference is built
// without contraction; see oracle/ggml_oracle.c header).  e = element index inside the row.
// Formulas: ggml.c:1509-1619 (legacy), k_quants.c:344-377, 472-521, 607-631, 734-760, 845-877.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void unpack_sm6(int j, const uint8_t * s, int & sc, int & mn) {   // get_scale_min_k4, k_quants.c:264-271
    if (j < 4) { sc = s[j] & 63; mn = s[j + 4] & 63; }
    else { sc = (s[j + 4] & 0xF) | ((s[j - 4] >> 6) << 4); mn = (s[j + 4] >> 4) | ((s[j] >> 6) << 4); }
}
__device__ __forceinline__ void pack_sm6(int j, uint8_t * q, uint8_t ls, uint8_t lm) {     // its inverse (k_quants.c:565-578), for j = 0..7 in order
    if (j < 4) { q[j] = ls; q[j + 4] = lm; }
    else { q[j + 4] = (uint8_t) ((ls & 0xF) | ((lm & 0xF) << 4)); q[j - 4] |= (uint8_t) ((ls >> 4) << 6); q[j] |= (uint8_t) ((lm >> 4) << 6); }
}
__device__ __forceinline__ int q3_scale(const uint8_t * s, int j) {   // 6-bit scale j of the 12-byte q3_K field, bias kept (k_quants.c:486-493)
    const int lo = j < 8 ? (s[j] & 0xF) : (s[j - 8] >> 4);
    const int hi = (s[8 + (j & 3)] >> (2 * (j >> 2))) & 3;
    return lo | (hi << 4);
}

// scale j (already minus 32) from the expanded 16-byte field of the device layout (PlaneSpec kind 2)
__device__ __forceinline__ int q3_scale16(const uint8_t * s16, int j) { return reinterpret_cast<const int8_t *>(s16)[4 * (2 * (j >> 3) + (j & 1)) + ((j >> 1) & 3)]; }

__device__ inline float dequant_elem(const WPlanes & W, size_t row, int e) {
    const int t = W.type;
    if (t == T_F32) return reinterpret_cast<const float *>(W.p[0] + row * W.stride[0])[e];
    if (t == T_F16) return f16_bits_to_f32(reinterpret_cast<const uint16_t *>(W.p[0] + row * W.stride[0])[e]);
    if (t == T_Q4_0 || t == T_Q4_1 || t == T_Q5_0 || t == T_Q5_1 || t == T_Q8_0) {
        const int b = e >> 5, i = e & 31, j = i & 15, hi = i >> 4;
        if (t == T_Q8_0) {
            const int8_t q = reinterpret_cast<const int8_t *>(W.p[0] + row * W.stride[0])[e];
            const float d = f16_bits_to_f32(reinterpret_cast<const uint16_t *>(W.p[1] + row * W.stride[1])[b]);
            return __fmul_rn((float) q, d);
        }
        const uint8_t byte = (W.p[0] + row * W.stride[0])[b * 16 + j];
        int code = hi ? (byte >> 4) : (byte & 0xF);
        if (t == T_Q4_0) {
            const float d = f16_bits_to_f32(reinterpret_cast<const uint16_t *>(W.p[1] + row * W.stride[1])[b]);
            return __fmul_rn((float) (code - 8), d);
        }
        if (t == T_Q4_1) {
            const uint16_t * dm = reinterpret_cast<const uint16_t *>(W.p[1] + row * W.stride[1]) + 2 * b;
            return __fadd_rn(__fmul_rn((float) code, f16_bits_to_f32(dm[0])), f16_bits_to_f32(dm[1]));
        }
        const uint32_t qh = reinterpret_cast<const uint32_t *>(W.p[1] + row * W.stride[1])[b];
        code |= ((qh >> i) & 1) << 4;       // bit j (low half) / bit j+16 (high half)
        if (t == T_Q5_0) {
            const float d = f16_bits_to_f32(reinterpret_cast<const uint16_t *>(W.p[2] + row * W.stride[2])[b]);
            return __fmul_rn((float) (code - 16), d);
        }
        const uint16_t * dm = reinterpret_cast<const uint16_t *>(W.p[2] + row * W.stride[2]) + 2 * b;
        return __fadd_rn(__fmul_rn((float) code, f16_bits_to_f32(dm[0])), f16_bits_to_f32(dm[1]));
    }
    const int b = e >> 8, i = e & 255;
    if (t == T_Q4_K || t == T_Q5_K) {
        const int ps = t == T_Q4_K ? 1 : 2;                       // plane of the expanded scales; d,dmin follow in the next plane
        const uint8_t * sm = W.p[ps] + row * W.stride[ps] + b * 16;
        const uint16_t * dd = reinterpret_cast<const uint16_t *>(W.p[ps + 1] + row * W.stride[ps + 1] + b * 4);
        const float d = f16_bits_to_f32(dd[0]), dmin = f16_bits_to_f32(dd[1]);
        const int sub = i >> 5, l = i & 31, pair = sub >> 1;
        const int sc = sm[4 * pair + (sub & 1)], mn = sm[4 * pair + 2 + (sub & 1)];
        const uint8_t byte = (W.p[0] + row * W.stride[0])[b * 128 + pair * 32 + l];
        int code = (sub & 1) ? (byte >> 4) : (byte & 0xF);
        if (t == T_Q5_K) code += (((W.p[1] + row * W.stride[1])[b * 32 + l] >> sub) & 1) ? 16 : 0;
        return __fsub_rn(__fmul_rn(__fmul_rn(d, (float) sc), (float) code), __fmul_rn(dmin, (float) mn));
    }
    if (t == T_Q6_K) {
        const int n = i >> 7, r = i & 127, l = r & 31, quad = r >> 5;     // element = 128n + 32*quad + l
        const uint8_t * ql = W.p[0] + row * W.stride[0] + b * 128 + n * 64;
        const uint8_t qhb = (W.p[1] + row * W.stride[1])[b * 64 + n * 32 + l];
        const uint8_t qlb = ql[l + ((quad & 1) ? 32 : 0)];
        const int lo = (quad >> 1) ? (qlb >> 4) : (qlb & 0xF);
        const int code = (int) (int8_t) (lo | (((qhb >> (2 * quad)) & 3) << 4)) - 32;
        const int sc = reinterpret_cast<const int8_t *>(W.p[2] + row * W.stride[2])[b * 16 + n * 8 + (l >> 4) + 2 * quad];
        const float d = f16_bits_to_f32(reinterpret_cast<const uint16_t *>(W.p[3] + row * W.stride[3])[b]);
        return __fmul_rn(__fmul_rn(d, (float) sc), (float) code);
    }
    if (t == T_Q3_K) {
        const int n = i >> 7, r = i & 127, l = r & 31, quad = r >> 5;
        const uint8_t qb = (W.p[0] + row * W.stride[0])[b * 64 + n * 32 + l];
        const uint8_t hb = (W.p[1] + row * W.stride[1])[b * 32 + l];
        const int code = ((qb >> (2 * quad)) & 3) - (((hb >> (4 * n + quad)) & 1) ? 0 : 4);
        const int sc = q3_scale16(W.p[2] + row * W.stride[2] + b * 16, i >> 4);
        const float d = f16_bits_to_f32(reinterpret_cast<const uint16_t *>(W.p[3] + row * W.stride[3])[b]);
        return __fmul_rn(__fmul_rn(d, (float) sc), (float) code);
    }
    if (t == T_Q2_K) {
        const int n = i >> 7, r = i & 127, l = r & 31, quad = r >> 5;
        const uint8_t qb = (W.p[0] + row * W.stride[0])[b * 64 + n * 32 + l];
        const int code = (qb >> (2 * quad)) & 3;
        const uint8_t s = (W.p[1] + row * W.stride[1])[b * 16 + (i >> 4)];
        const uint16_t * dm = reinterpret_cast<const uint16_t *>(W.p[2] + row * W.stride[2]) + 2 * b;
        return __fsub_rn(__fmul_rn(__fmul_rn(f16_bits_to_f32(dm[0]), (float) (s & 0xF)), (float) code),
                         __fmul_rn(f16_bits_to_f32(dm[1]), (float) (s >> 4)));
    }
    return 0.f;
}
#endif
