// mmv.cu -- decode mat-vec: y[m] = sum_k W[m][k] * x[k] for block-quantised W and a Q8-quantised x.
//
// Replaces dequantize_mul_mat_vec<> / dequantize_mul_mat_vec_q{2..6}_k (ggml-cuda.cu:475-845, 1121-1171, one warp
// per row, 2-4 byte scalar loads, fp32 activations) and follows the arithmetic of the CPU twin instead
// (ggml_vec_dot_q*_q8_*, ggml.c:2342-3340 and k_quants.c:1005-2790): int8 x int4..6 block dots in int32 (dp4a),
// one fp32 multiply-accumulate per (sub-)block.  The integer part is exact; only the fp32 summation order
// differs from the CPU (which itself differs between its scalar and AVX2 bodies).
//
// Shape of the kernel (HBM-bound; see DESIGN.md "mmv"):
//   * one persistent CTA of 16 warps per SM; CTA c owns a contiguous, balanced range of rows, its warps pull rows
//     from a shared-memory counter (results do not depend on which warp computes a row: deterministic)
//   * weights never touch registers on their way in: lane 0 of every warp keeps a ring of S "units" (CH blocks of
//     a row, ~3-5 KB over all planes) in flight with 1-D TMA bulk copies (cp.async.bulk + mbarrier complete_tx);
//     16 warps x S stages = 100-200 KB of HBM reads in flight per SM
//   * the activation codes (K bytes) are staged once per CTA by another TMA bulk copy; scales / block sums (tiny)
//     by ordinary loads
//   * a lane reads 16-byte pieces of the unit from shared memory (consecutive lanes -> consecutive 16 B, conflict
//     free), dp4a against the activation codes, one fp32 multiply-accumulate per (sub-)block
//   * one warp-shuffle reduction per row, lane 0 stores (+ fused GELU / residual epilogue)
#include "kernels.h"

#define MMV_THREADS 512
__host__ __device__ constexpr size_t round_up16(size_t v) { return (v + 15) / 16 * 16; }

struct XS {                 // activation row in shared memory
    const int8_t * q; const float * d; const float * s; const int16_t * bs;
};

__device__ __forceinline__ uint4 lds16(const int8_t * p) { return *reinterpret_cast<const uint4 *>(p); }

template <int TYPE> struct MV;

// ---------------------------------------------------------------- Q4_K  (k_quants.c:1999-2055)
// sum_j sc_j * (q4 . q8)_j and sum_j min_j * bsums_j as two dp2a over the expanded scale plane {sc0, sc1, m0, m1}
__device__ __forceinline__ int pack16(int lo, int hi) { return (lo & 0xffff) | (hi << 16); }

template <> struct MV<T_Q4_K> {
    static constexpr int PPB = 8;                // 16-byte pieces per 256-weight block
    static constexpr int CH = 32, NPL = 3;       // blocks per unit, planes
    __host__ __device__ static constexpr int pb(int p) { return p == 0 ? 128 : p == 1 ? 16 : p == 2 ? 4 : 0; }
    static constexpr int O1 = CH * 128, O2 = O1 + CH * 16;
    struct Regs { uint4 q; uint32_t sm, dd; };
    __device__ static Regs load(const uint8_t * sb, int b, int pc) {
        Regs r;
        r.q = *reinterpret_cast<const uint4 *>(sb + b * 128 + pc * 16);
        r.sm = *reinterpret_cast<const uint32_t *>(sb + O1 + b * 16 + (pc >> 1) * 4);
        r.dd = *reinterpret_cast<const uint32_t *>(sb + O2 + b * 4);
        return r;
    }
    __device__ static float finish(int il, int ih, uint32_t sm, uint32_t dd, int b, int pc, const XS & x) {
        const int p = pc >> 1, half = pc & 1;
        const int isum = dp2a_lo_us(pack16(il, ih), sm, 0);
        const int msum = dp2a_hi_us(pack16(x.bs[b * 16 + 4 * p + half], x.bs[b * 16 + 4 * p + 2 + half]), sm, 0);
        const float xd = x.d[b];
        const float2 dm = __half22float2(*reinterpret_cast<const __half2 *>(&dd));
        return (dm.x * xd) * (float) isum - (dm.y * xd) * (float) msum;
    }
    __device__ static float dot(const Regs & r, int b, int pc, const XS & x) {
        const int e0 = b * 256 + 64 * (pc >> 1) + 16 * (pc & 1);          // low nibbles: e0.., high nibbles: e0+32..
        const uint4 xl = lds16(x.q + e0), xh = lds16(x.q + e0 + 32);
        const int il = dot16(r.q.x & 0x0F0F0F0F, r.q.y & 0x0F0F0F0F, r.q.z & 0x0F0F0F0F, r.q.w & 0x0F0F0F0F, xl);
        // high nibbles stay in place (x16): the dot is an exact multiple of 16
        const int ih = dot16(r.q.x & 0xF0F0F0F0, r.q.y & 0xF0F0F0F0, r.q.z & 0xF0F0F0F0, r.q.w & 0xF0F0F0F0, xh) >> 4;
        return finish(il, ih, r.sm, r.dd, b, pc, x);
    }
};

// ---------------------------------------------------------------- Q5_K  (k_quants.c:2340-2400)
template <> struct MV<T_Q5_K> {
    static constexpr int PPB = 8;
    static constexpr int CH = 16, NPL = 4;
    __host__ __device__ static constexpr int pb(int p) { return p == 0 ? 128 : p == 1 ? 32 : p == 2 ? 16 : 4; }
    static constexpr int O1 = CH * 128, O2 = O1 + CH * 32, O3 = O2 + CH * 16;
    struct Regs { uint4 q, qh; uint32_t sm, dd; };
    __device__ static Regs load(const uint8_t * sb, int b, int pc) {
        Regs r;
        r.q = *reinterpret_cast<const uint4 *>(sb + b * 128 + pc * 16);
        r.qh = *reinterpret_cast<const uint4 *>(sb + O1 + b * 32 + (pc & 1) * 16);
        r.sm = *reinterpret_cast<const uint32_t *>(sb + O2 + b * 16 + (pc >> 1) * 4);
        r.dd = *reinterpret_cast<const uint32_t *>(sb + O3 + b * 4);
        return r;
    }
    __device__ static float dot(const Regs & r, int b, int pc, const XS & x) {
        const int p = pc >> 1, half = pc & 1;
        const int e0 = b * 256 + 64 * p + 16 * half;
        const uint4 xl = lds16(x.q + e0), xh = lds16(x.q + e0 + 32);
        const int s0 = 2 * p, s1 = 2 * p + 1;
#define LO5(w, hw) (((w) & 0x0F0F0F0F) | ((((hw) >> s0) & 0x01010101) << 4))
#define HI5(w, hw) ((((w) >> 4) & 0x0F0F0F0F) | ((((hw) >> s1) & 0x01010101) << 4))
        const int il = dot16(LO5(r.q.x, r.qh.x), LO5(r.q.y, r.qh.y), LO5(r.q.z, r.qh.z), LO5(r.q.w, r.qh.w), xl);
        const int ih = dot16(HI5(r.q.x, r.qh.x), HI5(r.q.y, r.qh.y), HI5(r.q.z, r.qh.z), HI5(r.q.w, r.qh.w), xh);
#undef LO5
#undef HI5
        // 5-bit codes: |il| can reach 16*31*127 > int16, so the scale products are plain 32-bit multiplies here
        const int isum = (int) (r.sm & 0xff) * il + (int) ((r.sm >> 8) & 0xff) * ih;
        const int msum = dp2a_hi_us(pack16(x.bs[b * 16 + 4 * p + half], x.bs[b * 16 + 4 * p + 2 + half]), r.sm, 0);
        const float xd = x.d[b];
        const float2 dm = __half22float2(*reinterpret_cast<const __half2 *>(&r.dd));
        return (dm.x * xd) * (float) isum - (dm.y * xd) * (float) msum;
    }
};

// ---------------------------------------------------------------- Q6_K  (k_quants.c:2748-2789)
template <> struct MV<T_Q6_K> {
    static constexpr int PPB = 8;
    static constexpr int CH = 16, NPL = 4;
    __host__ __device__ static constexpr int pb(int p) { return p == 0 ? 128 : p == 1 ? 64 : p == 2 ? 16 : 2; }
    static constexpr int O1 = CH * 128, O2 = O1 + CH * 64, O3 = O2 + CH * 16;
    struct Regs { uint4 ql, qh, sc; uint32_t d; };
    __device__ static Regs load(const uint8_t * sb, int b, int pc) {
        Regs r;
        r.ql = *reinterpret_cast<const uint4 *>(sb + b * 128 + pc * 16);                          // = n*64 + c*16
        r.qh = *reinterpret_cast<const uint4 *>(sb + O1 + b * 64 + (pc >> 2) * 32 + (pc & 1) * 16);
        r.sc = *reinterpret_cast<const uint4 *>(sb + O2 + b * 16);
        r.d = *reinterpret_cast<const uint16_t *>(sb + O3 + b * 2);
        return r;
    }
    __device__ static float dot(const Regs & r, int b, int pc, const XS & x) {
        const int n = pc >> 2, c = pc & 3;
        const int el = 128 * n + ((c & 2) ? 32 : 0) + 16 * (c & 1);      // element offset (in block) of the low-nibble group; high-nibble group = el + 64
        const int ls = (c & 2) ? 2 : 0, hs = ls + 4;
        const uint4 xl = lds16(x.q + b * 256 + el), xh = lds16(x.q + b * 256 + el + 64);
#define LO6(w, hw) (((w) & 0x0F0F0F0F) | ((((hw) >> ls) & 0x03030303) << 4))
#define HI6(w, hw) ((((w) >> 4) & 0x0F0F0F0F) | ((((hw) >> hs) & 0x03030303) << 4))
        int il = dot16(LO6(r.ql.x, r.qh.x), LO6(r.ql.y, r.qh.y), LO6(r.ql.z, r.qh.z), LO6(r.ql.w, r.qh.w), xl);
        int ih = dot16(HI6(r.ql.x, r.qh.x), HI6(r.ql.y, r.qh.y), HI6(r.ql.z, r.qh.z), HI6(r.ql.w, r.qh.w), xh);
#undef LO6
#undef HI6
        il -= 32 * x.bs[b * 16 + (el >> 4)];                             // codes are stored +32
        ih -= 32 * x.bs[b * 16 + ((el + 64) >> 4)];
        const int8_t * sc = reinterpret_cast<const int8_t *>(&r.sc);
        const int isum = (int) sc[el >> 4] * il + (int) sc[(el + 64) >> 4] * ih;
        return (f16_bits_to_f32((uint16_t) r.d) * x.d[b]) * (float) isum;
    }
};

// ---------------------------------------------------------------- Q3_K  (k_quants.c:1684-1745)
template <> struct MV<T_Q3_K> {
    static constexpr int PPB = 4;                // 16 bytes of qs = 64 weights
    static constexpr int CH = 32, NPL = 4;
    __host__ __device__ static constexpr int pb(int p) { return p == 0 ? 64 : p == 1 ? 32 : p == 2 ? 16 : 2; }
    static constexpr int O1 = CH * 64, O2 = O1 + CH * 32, O3 = O2 + CH * 16;
    struct Regs { uint4 q, hm; uint32_t sc, d; };                  // sc: the piece's four signed scales (expanded device layout)
    __device__ static Regs load(const uint8_t * sb, int b, int pc) {
        Regs r;
        r.q = *reinterpret_cast<const uint4 *>(sb + b * 64 + pc * 16);                            // = n*32 + c*16
        r.hm = *reinterpret_cast<const uint4 *>(sb + O1 + b * 32 + (pc & 1) * 16);
        r.sc = reinterpret_cast<const uint32_t *>(sb + O2 + b * 16)[pc];
        r.d = *reinterpret_cast<const uint16_t *>(sb + O3 + b * 2);
        return r;
    }
    __device__ static float dot(const Regs & r, int b, int pc, const XS & x) {
        const int n = pc >> 1, c = pc & 1;
        int isum = 0;
#pragma unroll
        for (int quad = 0; quad < 4; quad++) {
            const int el = 128 * n + 32 * quad + 16 * c;
            const uint4 xv = lds16(x.q + b * 256 + el);
            const int hb = 4 * n + quad;
#define C3(w, hw) ((((w) >> (2 * quad)) & 0x03030303) | ((((hw) >> hb) & 0x01010101) << 2))
            int i = dot16(C3(r.q.x, r.hm.x), C3(r.q.y, r.hm.y), C3(r.q.z, r.hm.z), C3(r.q.w, r.hm.w), xv);
#undef C3
            i -= 4 * x.bs[b * 16 + (el >> 4)];                          // code = (q2 | hbit<<2) - 4
            isum += (int) (int8_t) (r.sc >> (8 * quad)) * i;
        }
        return (f16_bits_to_f32((uint16_t) r.d) * x.d[b]) * (float) isum;
    }
};

// ---------------------------------------------------------------- Q2_K  (k_quants.c:1267-1305)
template <> struct MV<T_Q2_K> {
    static constexpr int PPB = 4;
    static constexpr int CH = 32, NPL = 3;
    __host__ __device__ static constexpr int pb(int p) { return p == 0 ? 64 : p == 1 ? 16 : p == 2 ? 4 : 0; }
    static constexpr int O1 = CH * 64, O2 = O1 + CH * 16;
    struct Regs { uint4 q, sc; uint32_t dm; };
    __device__ static Regs load(const uint8_t * sb, int b, int pc) {
        Regs r;
        r.q = *reinterpret_cast<const uint4 *>(sb + b * 64 + pc * 16);
        r.sc = *reinterpret_cast<const uint4 *>(sb + O1 + b * 16);
        r.dm = *reinterpret_cast<const uint32_t *>(sb + O2 + b * 4);
        return r;
    }
    __device__ static float dot(const Regs & r, int b, int pc, const XS & x) {
        const int n = pc >> 1, c = pc & 1;
        const uint8_t * sc = reinterpret_cast<const uint8_t *>(&r.sc);
        int isum = 0, msum = 0;
#pragma unroll
        for (int quad = 0; quad < 4; quad++) {
            const int el = 128 * n + 32 * quad + 16 * c;
            const uint4 xv = lds16(x.q + b * 256 + el);
#define C2(w) (((w) >> (2 * quad)) & 0x03030303)
            const int i = dot16(C2(r.q.x), C2(r.q.y), C2(r.q.z), C2(r.q.w), xv);
#undef C2
            const int s = sc[el >> 4];
            isum += (s & 0xF) * i;
            msum += (s >> 4) * x.bs[b * 16 + (el >> 4)];
        }
        const float xd = x.d[b];
        return (xd * f16_bits_to_f32((uint16_t) (r.dm & 0xffff))) * (float) isum - (xd * f16_bits_to_f32((uint16_t) (r.dm >> 16))) * (float) msum;
    }
};

// ---------------------------------------------------------------- legacy 32-weight blocks (ggml.c:2591-2609, 2716-2733, 2952-2974, 3208-3230, 3321-3333)
__device__ __forceinline__ uint32_t spread4(uint32_t bits4) { return ((bits4 & 0xF) * 0x00204081u) & 0x01010101u; }   // bit i -> byte i

template <> struct MV<T_Q4_0> {
    static constexpr int PPB = 1;
    static constexpr int CH = 256, NPL = 2;
    __host__ __device__ static constexpr int pb(int p) { return p == 0 ? 16 : p == 1 ? 2 : p == 2 ? 0 : 0; }
    static constexpr int O1 = CH * 16;
    struct Regs { uint4 q; uint32_t d; };
    __device__ static Regs load(const uint8_t * sb, int b, int) {
        Regs r;
        r.q = *reinterpret_cast<const uint4 *>(sb + b * 16);
        r.d = *reinterpret_cast<const uint16_t *>(sb + O1 + b * 2);
        return r;
    }
    __device__ static float dot(const Regs & r, int b, int, const XS & x) {
        const uint4 xl = lds16(x.q + b * 32), xh = lds16(x.q + b * 32 + 16);
        int s = dot16(r.q.x & 0x0F0F0F0F, r.q.y & 0x0F0F0F0F, r.q.z & 0x0F0F0F0F, r.q.w & 0x0F0F0F0F, xl);
        s += dot16((r.q.x >> 4) & 0x0F0F0F0F, (r.q.y >> 4) & 0x0F0F0F0F, (r.q.z >> 4) & 0x0F0F0F0F, (r.q.w >> 4) & 0x0F0F0F0F, xh);
        s -= 8 * x.bs[b];
        return ((float) s * f16_bits_to_f32((uint16_t) r.d)) * x.d[b];
    }
};
template <> struct MV<T_Q4_1> {
    static constexpr int PPB = 1;
    static constexpr int CH = 256, NPL = 2;
    __host__ __device__ static constexpr int pb(int p) { return p == 0 ? 16 : p == 1 ? 4 : p == 2 ? 0 : 0; }
    static constexpr int O1 = CH * 16;
    struct Regs { uint4 q; uint32_t dm; };
    __device__ static Regs load(const uint8_t * sb, int b, int) {
        Regs r;
        r.q = *reinterpret_cast<const uint4 *>(sb + b * 16);
        r.dm = *reinterpret_cast<const uint32_t *>(sb + O1 + b * 4);
        return r;
    }
    __device__ static float dot(const Regs & r, int b, int, const XS & x) {
        const uint4 xl = lds16(x.q + b * 32), xh = lds16(x.q + b * 32 + 16);
        int s = dot16(r.q.x & 0x0F0F0F0F, r.q.y & 0x0F0F0F0F, r.q.z & 0x0F0F0F0F, r.q.w & 0x0F0F0F0F, xl);
        s += dot16((r.q.x >> 4) & 0x0F0F0F0F, (r.q.y >> 4) & 0x0F0F0F0F, (r.q.z >> 4) & 0x0F0F0F0F, (r.q.w >> 4) & 0x0F0F0F0F, xh);
        return (f16_bits_to_f32((uint16_t) (r.dm & 0xffff)) * x.d[b]) * (float) s + f16_bits_to_f32((uint16_t) (r.dm >> 16)) * x.s[b];
    }
};
template <> struct MV<T_Q5_0> {
    static constexpr int PPB = 1;
    static constexpr int CH = 128, NPL = 3;
    __host__ __device__ static constexpr int pb(int p) { return p == 0 ? 16 : p == 1 ? 4 : p == 2 ? 2 : 0; }
    static constexpr int O1 = CH * 16, O2 = O1 + CH * 4;
    struct Regs { uint4 q; uint32_t qh, d; };
    __device__ static Regs load(const uint8_t * sb, int b, int) {
        Regs r;
        r.q = *reinterpret_cast<const uint4 *>(sb + b * 16);
        r.qh = *reinterpret_cast<const uint32_t *>(sb + O1 + b * 4);
        r.d = *reinterpret_cast<const uint16_t *>(sb + O2 + b * 2);
        return r;
    }
    __device__ static int idot(const uint4 q, uint32_t qh, int b, const XS & x) {
        const uint4 xl = lds16(x.q + b * 32), xh = lds16(x.q + b * 32 + 16);
        int s = dot16((q.x & 0x0F0F0F0F) | (spread4(qh) << 4), (q.y & 0x0F0F0F0F) | (spread4(qh >> 4) << 4),
                      (q.z & 0x0F0F0F0F) | (spread4(qh >> 8) << 4), (q.w & 0x0F0F0F0F) | (spread4(qh >> 12) << 4), xl);
        s += dot16(((q.x >> 4) & 0x0F0F0F0F) | (spread4(qh >> 16) << 4), ((q.y >> 4) & 0x0F0F0F0F) | (spread4(qh >> 20) << 4),
                   ((q.z >> 4) & 0x0F0F0F0F) | (spread4(qh >> 24) << 4), ((q.w >> 4) & 0x0F0F0F0F) | (spread4(qh >> 28) << 4), xh);
        return s;
    }
    __device__ static float dot(const Regs & r, int b, int, const XS & x) {
        const int s = idot(r.q, r.qh, b, x) - 16 * x.bs[b];
        return (f16_bits_to_f32((uint16_t) r.d) * x.d[b]) * (float) s;
    }
};
template <> struct MV<T_Q5_1> {
    static constexpr int PPB = 1;
    static constexpr int CH = 128, NPL = 3;
    __host__ __device__ static constexpr int pb(int p) { return p == 0 ? 16 : p == 1 ? 4 : p == 2 ? 4 : 0; }
    static constexpr int O1 = CH * 16, O2 = O1 + CH * 4;
    struct Regs { uint4 q; uint32_t qh, dm; };
    __device__ static Regs load(const uint8_t * sb, int b, int) {
        Regs r;
        r.q = *reinterpret_cast<const uint4 *>(sb + b * 16);
        r.qh = *reinterpret_cast<const uint32_t *>(sb + O1 + b * 4);
        r.dm = *reinterpret_cast<const uint32_t *>(sb + O2 + b * 4);
        return r;
    }
    __device__ static float dot(const Regs & r, int b, int, const XS & x) {
        const int s = MV<T_Q5_0>::idot(r.q, r.qh, b, x);
        return (f16_bits_to_f32((uint16_t) (r.dm & 0xffff)) * x.d[b]) * (float) s + f16_bits_to_f32((uint16_t) (r.dm >> 16)) * x.s[b];
    }
};
template <> struct MV<T_Q8_0> {
    static constexpr int PPB = 2;                // 16 int8 weights per piece
    static constexpr int CH = 128, NPL = 2;
    __host__ __device__ static constexpr int pb(int p) { return p == 0 ? 32 : p == 1 ? 2 : p == 2 ? 0 : 0; }
    static constexpr int O1 = CH * 32;
    struct Regs { uint4 q; uint32_t d; };
    __device__ static Regs load(const uint8_t * sb, int b, int pc) {
        Regs r;
        r.q = *reinterpret_cast<const uint4 *>(sb + b * 32 + pc * 16);
        r.d = *reinterpret_cast<const uint16_t *>(sb + O1 + b * 2);
        return r;
    }
    __device__ static float dot(const Regs & r, int b, int pc, const XS & x) {
        const uint4 xv = lds16(x.q + b * 32 + pc * 16);
        int s = dp4a_ss((int) r.q.x, (int) xv.x, 0); s = dp4a_ss((int) r.q.y, (int) xv.y, s);
        s = dp4a_ss((int) r.q.z, (int) xv.z, s); s = dp4a_ss((int) r.q.w, (int) xv.w, s);
        return (float) s * (f16_bits_to_f32((uint16_t) r.d) * x.d[b]);
    }
};

// ------------------------------------------------------------------------------------------------ the kernel
// Work unit = CH consecutive blocks of one weight row (about 4-5 KB over all planes).  Every warp owns a ring of
// `S` unit buffers in shared memory; its lane 0 keeps S units in flight with 1-D TMA bulk copies (one per plane)
// that complete on the stage's mbarrier.  With 16 warps x 2-3 stages an SM has 100-200 KB of weight bytes in
// flight without spending a single register on them -- that, not occupancy, is what hides HBM latency here.
template <int TYPE> struct UnitGeom {
    static constexpr int NPL = MV<TYPE>::NPL;
    __host__ __device__ static constexpr int plane_bytes(int p) { return MV<TYPE>::pb(p); }
    __host__ __device__ static constexpr int off(int p) {            // byte offset of plane p inside a stage
        int o = 0;
        for (int q = 0; q < p; q++) o += (MV<TYPE>::CH * MV<TYPE>::pb(q) + 15) / 16 * 16;
        return o;
    }
    static constexpr int META = off(NPL);                        // (row, chunk) of the unit a stage holds
    static constexpr int STAGE = META + 16;
};

template <int TYPE>
__global__ void __launch_bounds__(MMV_THREADS, 1) mmv_kernel(const WPlanes W, const ActQ A, float * __restrict__ y, int64_t y_stride,
                                                             const MmvEpilogue epi, const int S) {
    using T = MV<TYPE>;
    using G = UnitGeom<TYPE>;
    constexpr int WARPS = MMV_THREADS / 32;
    extern __shared__ __align__(128) uint8_t smem[];
    const int n = blockIdx.y;                                   // activation row (column of Y)
    const int K = W.K, ablk = TYPE >= T_Q2_K ? 256 : 32;
    const int nd = K / ablk, nbs = TYPE >= T_Q2_K ? K / 16 : K / 32;
    // layout: [x barrier + next-row counter | stage barriers (WARPS*S) | x codes | x scales | stages]
    uint64_t * xbar = reinterpret_cast<uint64_t *>(smem);
    int * next_row = reinterpret_cast<int *>(smem + 8);
    uint64_t * bars = reinterpret_cast<uint64_t *>(smem + 16);
    int8_t * xq = reinterpret_cast<int8_t *>(smem + 16 + round_up16(WARPS * S * 8));
    float * xd = reinterpret_cast<float *>(xq + K);
    float * xs = xd + nd;                                       // Q8_1 only (nd entries)
    int16_t * xbs = reinterpret_cast<int16_t *>((TYPE == T_Q4_1 || TYPE == T_Q5_1) ? (xs + nd) : xs);
    uint8_t * stages = reinterpret_cast<uint8_t *>(xbs) + round_up16(nbs * 2);
    stages = smem + (((stages - smem) + 127) / 128) * 128;

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint64_t * my_bars = bars + warp * S;
    uint8_t * my_stages = stages + (size_t) warp * S * G::STAGE;

    // rows [row0, row1) belong to this CTA (balanced to +-1 row); warps pull rows from a shared-memory counter
    const int per = W.M / gridDim.x, rem = W.M % gridDim.x;
    const int row0 = blockIdx.x * per + min((int) blockIdx.x, rem), row1 = row0 + per + ((int) blockIdx.x < rem ? 1 : 0);
    const int UPR = (W.nb + T::CH - 1) / T::CH;                 // units per row

    if (threadIdx.x == 0) { mbar_init(xbar, 1); *next_row = row0; }
    if (lane == 0) for (int s = 0; s < S; s++) mbar_init(my_bars + s, 1);
    mbar_fence_init();
    __syncthreads();

    // producer state (lane 0 only): the row/chunk of the next unit to issue
    int p_row = -1, p_chunk = 0, issued = 0;
    // consumer state: what the ring holds, in issue order (all lanes track it identically through shuffles)
    auto issue = [&]() -> bool {                                // lane 0: claim + issue the next unit; false when out of rows
        if (p_row < 0 || p_chunk == UPR) { p_row = atomicAdd(next_row, 1); p_chunk = 0; }
        if (p_row >= row1) { p_row = row1; p_chunk = UPR; return false; }
        const int st = issued % S;
        const int b0 = p_chunk * T::CH, nblk = min(T::CH, W.nb - b0);
        uint32_t bytes = 0;
#pragma unroll
        for (int p = 0; p < G::NPL; p++) bytes += (uint32_t) ((nblk * G::plane_bytes(p) + 15) / 16 * 16);
        // (row, chunk) for the consumer side: written before the arrive so that its release ordering covers it
        reinterpret_cast<int *>(my_stages + (size_t) st * G::STAGE + G::META)[0] = p_row;
        reinterpret_cast<int *>(my_stages + (size_t) st * G::STAGE + G::META)[1] = p_chunk;
        mbar_expect_tx(my_bars + st, bytes);
#pragma unroll
        for (int p = 0; p < G::NPL; p++)
            tma_load_1d(my_stages + (size_t) st * G::STAGE + G::off(p), W.p[p] + (size_t) p_row * W.stride[p] + (size_t) b0 * G::plane_bytes(p),
                        (uint32_t) ((nblk * G::plane_bytes(p) + 15) / 16 * 16), my_bars + st);
        p_chunk++; issued++;
        return true;
    };
    if (lane == 0) for (int s = 0; s < S; s++) if (!issue()) break;      // weights start streaming before x is even staged

    // activation tile: codes by TMA, scales / block sums (tiny) by ordinary loads
    if (threadIdx.x == 0) { mbar_expect_tx(xbar, (uint32_t) K); tma_load_1d(xq, A.q + (size_t) n * K, (uint32_t) K, xbar); }
    for (int i = threadIdx.x; i < nd; i += MMV_THREADS) {
        xd[i] = A.d[(size_t) n * nd + i];
        if (TYPE == T_Q4_1 || TYPE == T_Q5_1) xs[i] = A.s[(size_t) n * nd + i];
    }
    for (int i = threadIdx.x; i < nbs; i += MMV_THREADS) xbs[i] = A.bs[(size_t) n * nbs + i];
    __syncthreads();
    mbar_wait(xbar, 0);
    const XS x = { xq, xd, xs, xbs };

    int n_issued = __shfl_sync(0xffffffffu, issued, 0);
    float acc = 0.f;
    for (int u = 0; u < n_issued; u++) {
        const int st = u % S;
        mbar_wait(my_bars + st, (uint32_t) ((u / S) & 1));
        const uint8_t * sb = my_stages + (size_t) st * G::STAGE;
        const int row = reinterpret_cast<const int *>(sb + G::META)[0], chunk = reinterpret_cast<const int *>(sb + G::META)[1];
        const int b0 = chunk * T::CH, nblk = min(T::CH, W.nb - b0);
        const int P = nblk * T::PPB;
#pragma unroll 4
        for (int g = lane; g < P; g += 32) {
            const typename T::Regs r = T::load(sb, g / T::PPB, g % T::PPB);
            acc += T::dot(r, b0 + g / T::PPB, g % T::PPB, x);
        }
        __syncwarp();                                           // every lane is done with this stage
        int more = 0;
        if (lane == 0) more = issue() ? 1 : 0;                  // refill it
        n_issued += __shfl_sync(0xffffffffu, more, 0);
        if (chunk == UPR - 1) {
            const float v0 = warp_sum(acc);
            if (lane == 0) {
                float v = v0;
                if (epi.kind == EPI_GELU) v = gelu_f16lut(v);
                else if (epi.kind == EPI_ADD2) v = (v + epi.r1[(size_t) n * y_stride + row]) + epi.r2[(size_t) n * y_stride + row];
                y[(size_t) n * y_stride + row] = v;
            }
            acc = 0.f;
        }
    }
}

template <int TYPE>
static void launch_typed(const WPlanes & W, const ActQ & A, float * y, int64_t y_stride, MmvEpilogue epi, cudaStream_t stream) {
    using G = UnitGeom<TYPE>;
    constexpr int WARPS = MMV_THREADS / 32;
    const int K = W.K, ablk = TYPE >= T_Q2_K ? 256 : 32;
    const size_t xbytes = (size_t) K + (size_t) (K / ablk) * 4 * ((TYPE == T_Q4_1 || TYPE == T_Q5_1) ? 2 : 1) + round_up16((size_t) (TYPE >= T_Q2_K ? K / 16 : K / 32) * 2);
    int S = 4;                                                  // deepest ring that fits next to the activation tile
    size_t smem = 0;
    for (; S >= 1; S--) {
        smem = 16 + round_up16((size_t) WARPS * S * 8) + xbytes + 256 + (size_t) WARPS * S * G::STAGE;
        if (smem <= 220 * 1024) break;
    }
    B200_ASSERT(S >= 1);
    static bool attr_set = false;
    if (!attr_set) { B200_CUDA_CHECK(cudaFuncSetAttribute(mmv_kernel<TYPE>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024)); attr_set = true; }
    int ctas = num_sms();                                       // one persistent CTA per SM
    if (ctas > W.M) ctas = W.M;
    dim3 grid((unsigned) ctas, (unsigned) A.N);
    mmv_kernel<TYPE><<<grid, MMV_THREADS, smem, stream>>>(W, A, y, y_stride, epi, S);
    B200_CUDA_CHECK(cudaGetLastError());
}

void launch_mmv(const WPlanes & W, const ActQ & A, float * y, int64_t y_stride, MmvEpilogue epi, cudaStream_t stream) {
    B200_ASSERT(A.K == W.K && A.type == act_type_for(W.type));
    if (!getenv("B200_MMV_GENERIC") && launch_mmv_fast(W, A, y, y_stride, epi, stream)) return;
    B200_ASSERT(W.K % 32 == 0 && W.K <= 96 * 1024);
    switch (W.type) {
        case T_Q4_K: launch_typed<T_Q4_K>(W, A, y, y_stride, epi, stream); break;
        case T_Q5_K: launch_typed<T_Q5_K>(W, A, y, y_stride, epi, stream); break;
        case T_Q6_K: launch_typed<T_Q6_K>(W, A, y, y_stride, epi, stream); break;
        case T_Q3_K: launch_typed<T_Q3_K>(W, A, y, y_stride, epi, stream); break;
        case T_Q2_K: launch_typed<T_Q2_K>(W, A, y, y_stride, epi, stream); break;
        case T_Q4_0: launch_typed<T_Q4_0>(W, A, y, y_stride, epi, stream); break;
        case T_Q4_1: launch_typed<T_Q4_1>(W, A, y, y_stride, epi, stream); break;
        case T_Q5_0: launch_typed<T_Q5_0>(W, A, y, y_stride, epi, stream); break;
        case T_Q5_1: launch_typed<T_Q5_1>(W, A, y, y_stride, epi, stream); break;
        case T_Q8_0: launch_typed<T_Q8_0>(W, A, y, y_stride, epi, stream); break;
        default: B200_ASSERT(!"launch_mmv: unsupported weight type");
    }
}

// ---- f16 / f32 weights with fp32 activations (ggml.c:10911-11102, 11104-11316): one warp per row, 16-byte loads
template <bool F16>
__global__ void __launch_bounds__(256) mmv_f_kernel(const WPlanes W, const float * __restrict__ x, int64_t x_stride, float * __restrict__ y, int64_t y_stride) {
    const int n = blockIdx.y, lane = threadIdx.x & 31;
    const int gw = blockIdx.x * 8 + (threadIdx.x >> 5), nw = gridDim.x * 8;
    const float * xr = x + (size_t) n * x_stride;
    for (int row = gw; row < W.M; row += nw) {
        float acc = 0.f;
        const uint8_t * wr = W.p[0] + (size_t) row * W.stride[0];
        if (F16) {
            for (int k = lane * 8; k < W.K; k += 256) {
                if (k + 8 <= W.K) {
                    const uint4 w = ldg_stream_v4(wr + (size_t) k * 2);
                    const __half2 * h = reinterpret_cast<const __half2 *>(&w);
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        const float2 f = __half22float2(h[j]);
                        // the CPU path rounds the activations to fp16 first (ggml.c:11232-11251)
                        acc += f.x * __half2float(__float2half_rn(xr[k + 2 * j])) + f.y * __half2float(__float2half_rn(xr[k + 2 * j + 1]));
                    }
                } else for (int j = k; j < W.K; j++) acc += f16_bits_to_f32(reinterpret_cast<const uint16_t *>(wr)[j]) * __half2float(__float2half_rn(xr[j]));
            }
        } else {
            for (int k = lane * 4; k < W.K; k += 128) {
                if (k + 4 <= W.K) {
                    const uint4 w = ldg_stream_v4(wr + (size_t) k * 4);
                    acc += __uint_as_float(w.x) * xr[k] + __uint_as_float(w.y) * xr[k + 1] + __uint_as_float(w.z) * xr[k + 2] + __uint_as_float(w.w) * xr[k + 3];
                } else for (int j = k; j < W.K; j++) acc += reinterpret_cast<const float *>(wr)[j] * xr[j];
            }
        }
        acc = warp_sum(acc);
        if (lane == 0) y[(size_t) n * y_stride + row] = acc;
    }
}
void launch_mmv_f(const WPlanes & W, const float * x, int64_t x_stride, int N, float * y, int64_t y_stride, cudaStream_t stream) {
    int ctas = num_sms() * 4; const int need = (W.M + 7) / 8; if (ctas > need) ctas = need;
    dim3 grid((unsigned) ctas, (unsigned) N);
    if (W.type == T_F16) mmv_f_kernel<true><<<grid, 256, 0, stream>>>(W, x, x_stride, y, y_stride);
    else if (W.type == T_F32) mmv_f_kernel<false><<<grid, 256, 0, stream>>>(W, x, x_stride, y, y_stride);
    else B200_ASSERT(!"launch_mmv_f: f16/f32 only");
    B200_CUDA_CHECK(cudaGetLastError());
}
