// mmv_fast.cuh -- per-type pieces of the register-resident decode mat-vec (used by mmv_fast.cu)
#pragma once
#include "kernels.h"
#include "actquant.cuh"

struct Epi { int kind; const float * r1; const float * r2; unsigned long long * trace; ActQ qA; unsigned * qctr; int late_wait; };

// Where the activation row comes from (FastX, kernels.h):
//   mode 0: already quantised (ActQ, written by quantize_act / layernorm_q)
//   mode 1: fp32 row x[K]; every CTA quantises it itself while its first weight rows are in flight
//   mode 2: fp32 row -> [x = (ra + rb) + x] -> LayerNorm(gamma, beta) -> quantise, all in the prologue (J == 1 only):
//           the residual adds that close the previous layer (libfalcon.cpp:2399-2400), the LayerNorm
//           (ggml.c:10568-10595 + libfalcon.cpp:2166-2185) and the mat-mul's INIT pass (ggml.c:11462-11476) without a
//           kernel of their own.  CTA 0 writes the updated residual row to x_out.
// In modes 1/2 the 8 threads that share a Q8_K block hold exactly its 256 values (32 each), so the block maximum is
// three shuffles away and the int8 codes are produced directly in the registers the dot products read.

__device__ __forceinline__ int dot16(const uint32_t w0, const uint32_t w1, const uint32_t w2, const uint32_t w3, const uint4 x) {
    int s = dp4a_us(w0, (int) x.x, 0); s = dp4a_us(w1, (int) x.y, s); s = dp4a_us(w2, (int) x.z, s); return dp4a_us(w3, (int) x.w, s);
}
__device__ __forceinline__ int dp2a_lo_su(int pair16, uint32_t bytes) { int d; asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(pair16), "r"(bytes), "r"(0)); return d; }
__device__ __forceinline__ int dp2a_hi_su(int pair16, uint32_t bytes) { int d; asm("dp2a.hi.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(pair16), "r"(bytes), "r"(0)); return d; }
__device__ __forceinline__ int dp2a_lo_ss(int pair16, uint32_t bytes, int c) { int d; asm("dp2a.lo.s32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(pair16), "r"(bytes), "r"(c)); return d; }
__device__ __forceinline__ int dp2a_hi_ss(int pair16, uint32_t bytes, int c) { int d; asm("dp2a.hi.s32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(pair16), "r"(bytes), "r"(c)); return d; }
__device__ __forceinline__ float gelu_lut(float v) {      // fp16-LUT semantics, ggml.c:3461-3484
    const float f = __half2float(__float2half_rn(v));
    const float g = 0.5f * f * (1.0f + tanhf(0.79788456080286535587989211986876f * f * (1.0f + 0.044715f * f * f)));
    return __half2float(__float2half_rn(g));
}

struct WP { const uint8_t * b0, * b1, * b2, * b3; uint32_t s0, s1, s2, s3; };
// keeps the compiler from splitting a per-thread plane pointer back into (uniform base) + (thread offset): with an opaque
// 64-bit register the row address is a single IMAD.WIDE.U32 instead of IMAD.WIDE + IADD3 + IADD3.X
__device__ __forceinline__ const uint8_t * opaque_ptr(const uint8_t * p) { unsigned long long v = (unsigned long long) p; asm volatile("" : "+l"(v)); return (const uint8_t *) v; }

template <int TYPE> struct FX;

template <> struct FX<T_Q4_K> {
    static constexpr int PPB = 8;                                   // pieces per block
    static constexpr bool HAS_PROLOGUE_QUANT = true;                // modes 1 / 2 (fp32 row quantised in the prologue)
    static constexpr int D256 = 8;                                  // ring depth of the J = 1 shapes
    struct XR { uint4 xl, xh; int bs; float xd; };                  // activation state of one piece position (all zero: contributes 0)
    struct WR { uint4 q; uint32_t sm, dd; };
    __device__ static XR load_x(const int8_t * xq, const ActQ & A, int n, int g) {
        const int b = g >> 3, pc = g & 7, p = pc >> 1, half = pc & 1;
        XR r;
        const int e0 = b * 256 + 64 * p + 16 * half;
        r.xl = *reinterpret_cast<const uint4 *>(xq + e0);
        r.xh = *reinterpret_cast<const uint4 *>(xq + e0 + 32);
        const int16_t * bs = A.bs + (size_t) n * (A.K / 16) + b * 16 + 4 * p + half;
        r.bs = ((int) bs[0] & 0xffff) | ((int) bs[2] << 16);
        r.xd = A.d[(size_t) n * (A.K / 256) + b];
        return r;
    }
    // element offsets (in the row) of the two 16-value segments piece g multiplies
    __device__ static void seg(int g, int & ea, int & eb) { const int b = g >> 3, pc = g & 7; ea = b * 256 + 64 * (pc >> 1) + 16 * (pc & 1); eb = ea + 32; }
    // v[0..16) = segment a, v[16..32) = segment b of this thread's piece; the 8 lanes of a block quantise it together
    // (quantize_row_q8_K_reference, k_quants.c:899-934: signed value of largest magnitude, first one on ties)
    __device__ static XR quant_x(const float (&v)[32], int g, int lane) {
        int ea, eb; seg(g, ea, eb);
        float amax = 0.f, vmax = 0.f; int imax = 0;
#pragma unroll
        for (int i = 0; i < 32; i++) { const float ax = fabsf(v[i]); const int idx = (i < 16 ? ea : eb - 16) + i; if (ax > amax || (ax == amax && ax > 0.f && idx < imax)) { amax = ax; vmax = v[i]; imax = idx; } }
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) {
            const float oa = __shfl_xor_sync(0xffffffffu, amax, o), ov = __shfl_xor_sync(0xffffffffu, vmax, o);
            const int oi = __shfl_xor_sync(0xffffffffu, imax, o);
            if (oa > amax || (oa == amax && oi < imax)) { amax = oa; vmax = ov; imax = oi; }
        }
        XR r;
        const bool zero = amax == 0.f;
        const float iscale = zero ? 0.f : __fdiv_rn(-128.f, vmax);
        r.xd = zero ? 0.f : __fdiv_rn(1.f, iscale);
        int s0 = 0, s1 = 0;
        uint32_t w[8];
#pragma unroll
        for (int i = 0; i < 8; i++) {                                         // codes are packed as they are produced: nothing but v[] stays live
            uint32_t pk = 0;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const int q = zero ? 0 : min(127, __float2int_rn(__fmul_rn(iscale, v[4 * i + k])));
                if (i < 4) s0 += q; else s1 += q;
                pk |= (uint32_t) (q & 0xff) << (8 * k);
            }
            w[i] = pk;
        }
        r.xl = make_uint4(w[0], w[1], w[2], w[3]); r.xh = make_uint4(w[4], w[5], w[6], w[7]);
        r.bs = (s0 & 0xffff) | (s1 << 16);
        (void) lane;
        return r;
    }
    // per-thread plane pointers of piece position g; a row's address is then ONE 32x32+64 multiply-add per plane
    __device__ static WP wp(const WPlanes & W, int g) {
        WP r; r.b0 = opaque_ptr(W.p[0] + (size_t) g * 16); r.b1 = opaque_ptr(W.p[1] + (size_t) (g >> 1) * 4); r.b2 = opaque_ptr(W.p[2] + (size_t) (g >> 3) * 4);
        r.s0 = W.stride[0]; r.s1 = W.stride[1]; r.s2 = W.stride[2];
        return r;
    }
    __device__ static WR load_w(const WP & p, uint32_t row) {
        WR r;
        r.q = ldg_stream_v4(p.b0 + (uint64_t) row * p.s0);
        r.sm = ldg_u32(p.b1 + (uint64_t) row * p.s1);
        r.dd = ldg_u32(p.b2 + (uint64_t) row * p.s2);
        return r;
    }
    __device__ static float dot(const WR & w, const XR & x) {
        const int il = dot16(w.q.x & 0x0F0F0F0F, w.q.y & 0x0F0F0F0F, w.q.z & 0x0F0F0F0F, w.q.w & 0x0F0F0F0F, x.xl);
        const int ih = dot16(w.q.x & 0xF0F0F0F0, w.q.y & 0xF0F0F0F0, w.q.z & 0xF0F0F0F0, w.q.w & 0xF0F0F0F0, x.xh) >> 4;
        const int isum = dp2a_lo_su((il & 0xffff) | (ih << 16), w.sm);       // sc0*il + sc1*ih   (|il|,|ih| <= 16*15*127 < 2^15)
        const int msum = dp2a_hi_su(x.bs, w.sm);                             // m0*bs_lo + m1*bs_hi
        const float2 dm = __half22float2(*reinterpret_cast<const __half2 *>(&w.dd));
        return (dm.x * x.xd) * (float) isum - (dm.y * x.xd) * (float) msum;
    }
};

template <> struct FX<T_Q4_0> {
    static constexpr int PPB = 1;
    static constexpr bool HAS_PROLOGUE_QUANT = true;
    static constexpr int D256 = 8;
    struct XR { uint4 xl, xh; int bs; float xd; };
    struct WR { uint4 q; uint32_t d; };
    __device__ static XR load_x(const int8_t * xq, const ActQ & A, int n, int g) {
        XR r;
        r.xl = *reinterpret_cast<const uint4 *>(xq + g * 32);
        r.xh = *reinterpret_cast<const uint4 *>(xq + g * 32 + 16);
        r.bs = A.bs[(size_t) n * (A.K / 32) + g];
        r.xd = A.d[(size_t) n * (A.K / 32) + g];
        return r;
    }
    __device__ static void seg(int g, int & ea, int & eb) { ea = g * 32; eb = ea + 16; }
    // a piece is a whole 32-value block: the x86 body of quantize_row_q8_0 (ggml.c:1201-1237), thread-local
    __device__ static XR quant_x(const float (&v)[32], int, int) {
        float amax = 0.f;
#pragma unroll
        for (int i = 0; i < 32; i++) amax = fmaxf(amax, fabsf(v[i]));
        const float id = amax != 0.f ? __fdiv_rn(127.f, amax) : 0.f;
        XR r;
        r.xd = __half2float(__float2half_rn(__fdiv_rn(amax, 127.f)));
        int s = 0;
        uint32_t w[8];
#pragma unroll
        for (int i = 0; i < 8; i++) {
            uint32_t pk = 0;
#pragma unroll
            for (int k = 0; k < 4; k++) { const int q = __float2int_rn(__fmul_rn(v[4 * i + k], id)); s += q; pk |= (uint32_t) (q & 0xff) << (8 * k); }
            w[i] = pk;
        }
        r.xl = make_uint4(w[0], w[1], w[2], w[3]); r.xh = make_uint4(w[4], w[5], w[6], w[7]);
        r.bs = s;
        return r;
    }
    __device__ static WP wp(const WPlanes & W, int g) {
        WP r; r.b0 = opaque_ptr(W.p[0] + (size_t) g * 16); r.b1 = opaque_ptr(W.p[1] + (size_t) g * 2); r.b2 = nullptr;
        r.s0 = W.stride[0]; r.s1 = W.stride[1]; r.s2 = 0;
        return r;
    }
    __device__ static WR load_w(const WP & p, uint32_t row) {
        WR r;
        r.q = ldg_stream_v4(p.b0 + (uint64_t) row * p.s0);
        r.d = ldg_u16(p.b1 + (uint64_t) row * p.s1);
        return r;
    }
    __device__ static float dot(const WR & w, const XR & x) {
        int s = dot16(w.q.x & 0x0F0F0F0F, w.q.y & 0x0F0F0F0F, w.q.z & 0x0F0F0F0F, w.q.w & 0x0F0F0F0F, x.xl);
        s += dot16(w.q.x & 0xF0F0F0F0, w.q.y & 0xF0F0F0F0, w.q.z & 0xF0F0F0F0, w.q.w & 0xF0F0F0F0, x.xh) >> 4;
        s -= 8 * x.bs;                                                       // codes are stored +8
        return ((float) s * f16_bits_to_f32((uint16_t) w.d)) * x.xd;
    }
};

// -------------------------------------------------------------------------------------------------- Q3_K x Q8_K
// piece g = 16 bytes of the 2-bit plane: block b = g / 4, half n = (g % 4) / 2, c = g % 2; bit pair `quad` of byte l holds
// element 128 n + 32 quad + 16 c + l, its high bit is bit 4 n + quad of hmask[16 c + l] (k_quants.c:1684-1745, 646-692).
// code = (q2 | hbit << 2) - 4, scale - 32 comes pre-expanded (PlaneSpec kind 2): the piece's four scales are one word.
template <> struct FX<T_Q3_K> {
    static constexpr int PPB = 4;
    static constexpr bool HAS_PROLOGUE_QUANT = false;               // mode 0 only (the decode path hands over quantised rows)
    static constexpr int D256 = 4;                                  // 10 registers per ring slot, 19 for the activation piece
    struct XR { uint4 x[4]; int bsA, bsB; float xd; };              // the four 16-code segments, their sums (4 x s16), Q8_K scale
    struct WR { uint4 q, hm; uint32_t sc, d; };
    __device__ static XR load_x(const int8_t * xq, const ActQ & A, int n, int g) {
        const int b = g >> 2, pc = g & 3, hn = pc >> 1, c = pc & 1;
        XR r;
        const int16_t * bs = A.bs + (size_t) n * (A.K / 16) + b * 16 + 8 * hn + c;
#pragma unroll
        for (int quad = 0; quad < 4; quad++) r.x[quad] = *reinterpret_cast<const uint4 *>(xq + b * 256 + 128 * hn + 32 * quad + 16 * c);
        r.bsA = ((int) bs[0] & 0xffff) | ((int) bs[2] << 16);
        r.bsB = ((int) bs[4] & 0xffff) | ((int) bs[6] << 16);
        r.xd = A.d[(size_t) n * (A.K / 256) + b];
        return r;
    }
    __device__ static void seg(int, int & ea, int & eb) { ea = 0; eb = 0; }
    __device__ static XR quant_x(const float (&)[32], int, int) { return XR{}; }      // never instantiated on a live path
    __device__ static WP wp(const WPlanes & W, int g) {
        WP r;
        r.b0 = opaque_ptr(W.p[0] + (size_t) g * 16); r.b1 = opaque_ptr(W.p[1] + (size_t) (g >> 2) * 32 + (g & 1) * 16);
        r.b2 = opaque_ptr(W.p[2] + (size_t) g * 4);  r.b3 = opaque_ptr(W.p[3] + (size_t) (g >> 2) * 2);
        r.s0 = W.stride[0]; r.s1 = W.stride[1]; r.s2 = W.stride[2]; r.s3 = W.stride[3];
        return r;
    }
    __device__ static WR load_w(const WP & p, uint32_t row) {
        WR r;
        r.q = ldg_stream_v4(p.b0 + (uint64_t) row * p.s0);
        r.hm = ldg_v4(p.b1 + (uint64_t) row * p.s1);                     // shared by the block's two halves n: second reader hits L1
        r.sc = ldg_u32(p.b2 + (uint64_t) row * p.s2);
        r.d = ldg_u16(p.b3 + (uint64_t) row * p.s3);
        return r;
    }
    // hsh = 4 n: the per-thread shift into its half of the high-bit plane (piece_aux).
    // The 2-bit field of quad j and the high bit are dotted IN PLACE (as the high nibbles of Q4_K are): a masked byte holds
    // 4^j * q2 (<= 192) resp. 2^(hsh+j) * hbit, dp4a is linear, so one exact shift per quad undoes the factor after the 16-value sum --
    // 2 LOP3 + 2 dp4a per word instead of 2 shifts + 2 masks + or + dp4a (this kernel is issue-bound, not HBM-bound).
    __device__ static float dot(const WR & w, const XR & x, int hsh) {
        const uint32_t q[4] = { w.q.x, w.q.y, w.q.z, w.q.w }, hm[4] = { w.hm.x, w.hm.y, w.hm.z, w.hm.w };
        const uint32_t hbase = 0x01010101u << hsh;
        int i[4];
#pragma unroll
        for (int quad = 0; quad < 4; quad++) {
            const uint32_t qm = 0x03030303u << (2 * quad), hmk = hbase << quad;
            const int dq = dot16(q[0] & qm, q[1] & qm, q[2] & qm, q[3] & qm, x.x[quad]);          // 4^quad * sum q2 x   (< 2^19)
            const int dh = dot16(hm[0] & hmk, hm[1] & hmk, hm[2] & hmk, hm[3] & hmk, x.x[quad]);   // 2^(hsh+quad) * sum hbit x   (< 2^19)
            i[quad] = (dq >> (2 * quad)) + ((dh >> (hsh + quad)) << 2);                            // exact: both are multiples; <= 16 * 7 * 127 < 2^15
        }
        int isum = dp2a_lo_ss((i[0] & 0xffff) | (i[1] << 16), w.sc, 0);
        isum = dp2a_hi_ss((i[2] & 0xffff) | (i[3] << 16), w.sc, isum);
        int bsum = dp2a_lo_ss(x.bsA, w.sc, 0);                              // the -4 of every code: - 4 * sum_quad sc * bsum
        bsum = dp2a_hi_ss(x.bsB, w.sc, bsum);
        return (f16_bits_to_f32((uint16_t) w.d) * x.xd) * (float) (isum - 4 * bsum);
    }
};

// G row sums per lane -> the total of row r in every lane of the 8-lane group r (G == 4), 16-lane group (G == 2) or warp
template <int G> __device__ __forceinline__ float transpose_reduce(const float (&acc)[G], int lane, int & row_of_lane) {
    float w;
    if (G == 4) {
        const bool hi = lane & 16;
        float v0 = hi ? acc[2] : acc[0], v1 = hi ? acc[3] : acc[1];
        v0 += __shfl_xor_sync(0xffffffffu, hi ? acc[0] : acc[2], 16);
        v1 += __shfl_xor_sync(0xffffffffu, hi ? acc[1] : acc[3], 16);
        const bool mid = lane & 8;
        w = mid ? v1 : v0;
        w += __shfl_xor_sync(0xffffffffu, mid ? v0 : v1, 8);
        w += __shfl_xor_sync(0xffffffffu, w, 4);
        row_of_lane = (hi ? 2 : 0) + (mid ? 1 : 0);
    } else if (G == 2) {
        const bool hi = lane & 16;
        w = hi ? acc[G - 1] : acc[0];
        w += __shfl_xor_sync(0xffffffffu, hi ? acc[0] : acc[G - 1], 16);
        w += __shfl_xor_sync(0xffffffffu, w, 8);
        w += __shfl_xor_sync(0xffffffffu, w, 4);
        row_of_lane = hi ? 1 : 0;
    } else {
        w = acc[0];
        w += __shfl_xor_sync(0xffffffffu, w, 16);
        w += __shfl_xor_sync(0xffffffffu, w, 8);
        w += __shfl_xor_sync(0xffffffffu, w, 4);
        row_of_lane = 0;
    }
    w += __shfl_xor_sync(0xffffffffu, w, 2);
    w += __shfl_xor_sync(0xffffffffu, w, 1);
    return w;
}


// HBM -> L2 prefetch of whole rows, `dist` rows ahead of the register ring.  The ring alone keeps 64 KB per SM in flight,
// which the loaded HBM latency turns into a cap on the stream (stalls sit on the first use of a ring slot); one bulk-prefetch instruction per plane and pass, issued by a single
// thread, moves the latency the ring has to cover from HBM to L2.
struct L2PF { const uint8_t * p[3]; uint32_t s[3]; int dist; };
__device__ __forceinline__ void l2_prefetch_rows(const L2PF & pf, int a, int b) {       // rows [a, b) of every plane
    if (b <= a) return;
#pragma unroll
    for (int i = 0; i < 3; i++) {
        if (!pf.p[i]) continue;
        const uint8_t * src = pf.p[i] + (size_t) a * pf.s[i];
        const uint32_t bytes = (uint32_t) (b - a) * pf.s[i];
        asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" :: "l"(src), "r"(bytes) : "memory");
    }
}
__device__ __forceinline__ L2PF l2pf_of(const WPlanes & W, int dist) {
    L2PF r; r.dist = dist;
#pragma unroll
    for (int i = 0; i < 3; i++) { r.p[i] = W.p[i]; r.s[i] = W.stride[i]; }
    return r;
}

__device__ __forceinline__ void named_sync(int id, int n) { asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(n) : "memory"); }

// per-thread constant some types need in their dot (Q3_K: the shift of its half of the high-bit plane)
template <int TYPE> __device__ __forceinline__ int piece_aux(int g) { return TYPE == T_Q3_K ? 4 * ((g & 3) >> 1) : 0; }
template <int TYPE> __device__ __forceinline__ float piece_dot(const typename FX<TYPE>::WR & w, const typename FX<TYPE>::XR & x, int aux) {
    if constexpr (TYPE == T_Q3_K) return FX<TYPE>::dot(w, x, aux); else return FX<TYPE>::dot(w, x);
}
template <int TYPE> __device__ __forceinline__ typename FX<TYPE>::XR zero_xr() {
    typename FX<TYPE>::XR r{}; return r;
}

// ---------------------------------------------------------------------------------------------------------------
// The row loop of mmv_fast.cu.  A group of NTG threads (a CTA, or half of one) owns rows
// [r0, r1) of a matrix; every thread keeps D rows x J pieces of weights in flight in registers (D * J = 8).
template <int TYPE, int J, int D>
__device__ __forceinline__ void ring_fill(typename FX<TYPE>::WR (&w)[D][J], const WP (&wp)[J], int r0, int r1) {
    if (r1 <= r0) return;
#pragma unroll
    for (int s = 0; s < D; s++) {
        const uint32_t row = (uint32_t) min(r0 + s, r1 - 1);
#pragma unroll
        for (int j = 0; j < J; j++) w[s][j] = FX<TYPE>::load_w(wp[j], row);
    }
}

// one pass over the D ring slots starting at relative row `base`.  CHECKED == false: every refill (rows base+D ..
// base+2D-1) is known to be inside the matrix, so the pass is straight-line code.
template <int TYPE, int NTG, int J, int D, bool CHECKED, bool HASNEXT, class Store>
__device__ __forceinline__ void ring_pass(typename FX<TYPE>::WR (&w)[D][J], const WP (&wp)[J], const int r0, const int nrows, const int npad, const int base,
                                          const WP (&wpn)[J], const int n0, const int n1,
                                          const typename FX<TYPE>::XR (&xr)[J], const int (&aux)[J], float * partial, int & gcount, const int bar_id, const int tg, Store & store) {
    using T = FX<TYPE>;
    constexpr int NWG = NTG / 32, G = (D % 4 == 0) ? 4 : (D % 2 == 0) ? 2 : 1;
    const int lane = tg & 31, warp = tg >> 5;
    float acc[G];
#pragma unroll
    for (int s = 0; s < D; s++) {
        float a = piece_dot<TYPE>(w[s][0], xr[0], aux[0]);
#pragma unroll
        for (int j = 1; j < J; j++) a += piece_dot<TYPE>(w[s][j], xr[j], aux[j]);
        acc[s % G] = a;
        const int nxt = base + D + s;                                        // refill this slot D rows ahead
        if (!CHECKED || nxt < nrows) {
#pragma unroll
            for (int j = 0; j < J; j++) w[s][j] = T::load_w(wp[j], (uint32_t) (r0 + nxt));
        } else if (HASNEXT && nxt >= npad && n1 > n0) {
            const uint32_t k = (uint32_t) min(n0 + nxt - npad, n1 - 1);
#pragma unroll
            for (int j = 0; j < J; j++) w[s][j] = T::load_w(wpn[j], k);
        }
        if ((s % G) == G - 1) {
            const int gi = (base + s) / G;
            int rl;
            const float v0 = transpose_reduce<G>(acc, lane, rl);
            float * part = partial + (gcount & 1) * NWG * G;
            gcount++;
            if ((lane & (G == 4 ? 7 : G == 2 ? 15 : 31)) == 0) part[warp * G + rl] = v0;
            named_sync(bar_id, NTG);
            if (tg < G) {
                const int row = r0 + gi * G + tg;
                if (!CHECKED || row < r0 + nrows) {
                    float v = 0.f;
#pragma unroll
                    for (int wi = 0; wi < NWG; wi++) v += part[wi * G + tg];          // fixed order: deterministic
                    store(row, v);
                }
            }
        }
    }
}

// Rows [r0, r1) of the matrix behind wp (ring already filled by ring_fill).  While the last D rows are consumed the
// freed slots are refilled with rows [n0, n1) of the NEXT matrix (wpn, same K), so the HBM stream does not drain
// between two matrices.  `gcount` numbers the reduction groups across calls (double-buffered partial sums);
// `before_tail` runs once when only the checked passes are left (the PDL trigger of the stand-alone kernels).
template <int TYPE, int NTG, int J, int D, bool HASNEXT, class Store, class Tail>
__device__ __forceinline__ void ring_run(typename FX<TYPE>::WR (&w)[D][J], const WP (&wp)[J], const int r0, const int r1,
                                         const WP (&wpn)[J], const int n0, const int n1,
                                         const typename FX<TYPE>::XR (&xr)[J], const int (&aux)[J], float * partial, int & gcount, const int bar_id, const int tg,
                                         Store store, Tail before_tail, const L2PF pf = L2PF{ { nullptr, nullptr, nullptr }, { 0, 0, 0 }, 0 }) {
    const int nrows = r1 - r0, npad = (nrows + D - 1) / D * D;
    if (npad == 0) { before_tail(); if (HASNEXT) ring_fill<TYPE, J, D>(w, wpn, n0, n1); return; }
    int base = 0;
    for (; base + 2 * D <= nrows; base += D) {
        if (pf.dist > 0 && tg == 0) l2_prefetch_rows(pf, min(r0 + base + D + pf.dist, r1), min(r0 + base + 2 * D + pf.dist, r1));
        ring_pass<TYPE, NTG, J, D, false, false>(w, wp, r0, nrows, npad, base, wpn, n0, n1, xr, aux, partial, gcount, bar_id, tg, store);
    }
    before_tail();
    for (; base < npad; base += D)
        ring_pass<TYPE, NTG, J, D, true, HASNEXT>(w, wp, r0, nrows, npad, base, wpn, n0, n1, xr, aux, partial, gcount, bar_id, tg, store);
}
