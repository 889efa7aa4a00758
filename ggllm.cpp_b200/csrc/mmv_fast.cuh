// mmv_fast.cuh -- per-type pieces of the register-resident decode mat-vec (used by mmv_fast.cu)
#pragma once
#include "kernels.h"
#include "actquant.cuh"

struct Epi { int kind; const float * r1; const float * r2; ActQ qA; unsigned * qctr; int late_wait; };

struct WP { const uint8_t * b0, * b1, * b2, * b3; uint32_t s0, s1, s2, s3; };
// keeps the compiler from splitting a per-thread plane pointer back into (uniform base) + (thread offset): with an opaque
// 64-bit register the row address is a single IMAD.WIDE.U32 instead of IMAD.WIDE + IADD3 + IADD3.X
__device__ __forceinline__ const uint8_t * opaque_ptr(const uint8_t * p) { unsigned long long v = (unsigned long long) p; asm volatile("" : "+l"(v)); return (const uint8_t *) v; }

template <int TYPE> struct FX;

template <> struct FX<T_Q4_K> {
    static constexpr int PPB = 8;                                   // pieces per block
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
        const int isum = dp2a_lo_us((il & 0xffff) | (ih << 16), w.sm, 0);    // sc0*il + sc1*ih   (|il|,|ih| <= 16*15*127 < 2^15)
        const int msum = dp2a_hi_us(x.bs, w.sm, 0);                          // m0*bs_lo + m1*bs_hi
        const float2 dm = __half22float2(*reinterpret_cast<const __half2 *>(&w.dd));
        return (dm.x * x.xd) * (float) isum - (dm.y * x.xd) * (float) msum;
    }
};

template <> struct FX<T_Q4_0> {
    static constexpr int PPB = 1;
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
// The row loop of mmv_fast.cu.  The NT threads of a CTA own rows [r0, r1) of the matrix; every thread keeps D rows x J pieces
// of weights in flight in registers (D * J = 8).
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
// base+2D-1) is known to be inside the matrix, so the pass is straight-line code.  `gcount` numbers the reduction groups
// (double-buffered partial sums).
template <int TYPE, int NT, int J, int D, bool CHECKED, class Store>
__device__ __forceinline__ void ring_pass(typename FX<TYPE>::WR (&w)[D][J], const WP (&wp)[J], const int r0, const int nrows, const int base,
                                          const typename FX<TYPE>::XR (&xr)[J], const int (&aux)[J], float * partial, int & gcount, const int tid, Store & store) {
    using T = FX<TYPE>;
    constexpr int NW = NT / 32, G = (D % 4 == 0) ? 4 : (D % 2 == 0) ? 2 : 1;
    const int lane = tid & 31, warp = tid >> 5;
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
        }
        if ((s % G) == G - 1) {
            const int gi = (base + s) / G;
            int rl;
            const float v0 = transpose_reduce<G>(acc, lane, rl);
            float * part = partial + (gcount & 1) * NW * G;
            gcount++;
            if ((lane & (G == 4 ? 7 : G == 2 ? 15 : 31)) == 0) part[warp * G + rl] = v0;
            named_sync(0, NT);
            if (tid < G) {
                const int row = r0 + gi * G + tid;
                if (!CHECKED || row < r0 + nrows) {
                    float v = 0.f;
#pragma unroll
                    for (int wi = 0; wi < NW; wi++) v += part[wi * G + tid];          // fixed order: deterministic
                    store(row, v);
                }
            }
        }
    }
}

// Rows [r0, r1) (ring already filled by ring_fill).  `before_tail` runs once when only the checked passes are left (the
// PDL trigger).
template <int TYPE, int NT, int J, int D, class Store, class Tail>
__device__ __forceinline__ void ring_run(typename FX<TYPE>::WR (&w)[D][J], const WP (&wp)[J], const int r0, const int r1,
                                         const typename FX<TYPE>::XR (&xr)[J], const int (&aux)[J], float * partial, const int tid,
                                         Store store, Tail before_tail) {
    const int nrows = r1 - r0, npad = (nrows + D - 1) / D * D;
    if (npad == 0) { before_tail(); return; }
    int base = 0, gcount = 0;
    for (; base + 2 * D <= nrows; base += D)
        ring_pass<TYPE, NT, J, D, false>(w, wp, r0, nrows, base, xr, aux, partial, gcount, tid, store);
    before_tail();
    for (; base < npad; base += D)
        ring_pass<TYPE, NT, J, D, true>(w, wp, r0, nrows, base, xr, aux, partial, gcount, tid, store);
}
