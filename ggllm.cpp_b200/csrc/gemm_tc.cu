// gemm_tc.cu -- prompt mat-mat on the Hopper tensor cores (wgmma): Y[n][m] = sum_k fp16(W[m][k]) * X[n][k].
//
// Replaces the reference's prompt path (ggml-cuda.cu:2353-2403): dequantise the WHOLE weight matrix to an fp16
// temporary (to_fp16_cuda, 2 B/weight written and re-read = 4.6x the quantised bytes), convert activations
// (float_to_half + stream sync), cublasGemmEx, per call.  Here the quantised blocks are the only thing read from
// HBM; a tile is dequantised once, straight into the shared-memory operand layout of wgmma, and used for BN tokens.
//
// One CTA = one 128-row tile of W x one tile of BN <= 256 tokens (BN = 64, 128 or 256: the accumulator lives in registers,
// 64 x BN fp32 per consumer warpgroup) over its share of K:
//   warpgroup 0    : dequant producers, one thread per weight row, 64 weights per 64-wide K block written as 8 halves per
//                    16-byte chunk into the K-major SWIZZLE_128B layout (chunk c of row r at c ^ (r & 7)), fence.proxy.async,
//                    mbarrier arrive; thread 0 also streams the activation tile B[BN x 64] fp16 with TMA
//                    (cp.async.bulk.tensor.2d, SWIZZLE_128B).  Ring of ST stages, A and B of a stage released together.
//   warpgroups 1, 2: wgmma.mma_async m64nBNk16, rows [64 (g - 1), +64) of the tile, both operands from shared memory; one
//                    wgmma group stays in flight while the next stage is awaited.  Epilogue straight from the accumulator
//                    registers: (GELU) -> fp32 stores.
// Token tiles of the same weight tile are neighbours in the grid (blockIdx.x), so their quantised blocks come from L2.
#include "kernels.h"
#include "wgmma.cuh"
#include <cuda.h>
#include <cudaTypedefs.h>

namespace {

constexpr int BM = 128, BK = 64, ST = 4;
constexpr int N_MAX = 512;
constexpr int THREADS = 384;                               // producer warpgroup + two consumer warpgroups
constexpr int A_STAGE = BM * BK * 2;                       // 16 KB

__device__ __forceinline__ void mbar_arrive(uint64_t * bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void tma_load_2d(void * smem_dst, const CUtensorMap * map, int c0, int c1, uint64_t * bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 :: "r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t *>(&h);
}

// ---- dequantisation of one thread's share of a 64-wide K block: segments [8h, 8h+8) and [32+8h, 32+8h+8) of the block (h = 0..3),
//      returned as 2 chunks of 8 halves
struct Chunks { uint4 c[2]; };      // 8 halves each: elements 8h .. 8h+7 and 32 + 8h .. 32 + 8h+7 of the K block

// generic: element-wise through the bit-exact dequantiser (any type)
__device__ __forceinline__ Chunks dequant_generic(const WPlanes & W, size_t row, int k0, int h) {
    Chunks o;
#pragma unroll
    for (int s = 0; s < 2; s++) {
        const int e = k0 + 32 * s + 8 * h;
        float v[8];
#pragma unroll
        for (int i = 0; i < 8; i++) v[i] = dequant_elem(W, row, e + i);
        o.c[s] = make_uint4(pack_h2(v[0], v[1]), pack_h2(v[2], v[3]), pack_h2(v[4], v[5]), pack_h2(v[6], v[7]));
    }
    return o;
}
// ---- per-type producers.  Prod<TYPE>::Raw = the bytes one thread needs for its 16 weights of a K block (loaded two blocks ahead),
//      ptr / next / load walk the planes, deq turns them into the two fp16 chunks.  Every variant produces the SAME bits as
//      "dequantize_row_* in fp32, then one rounding to fp16" (checked against dequant_elem by tests/test_kernels_gpu.py).
template <int TYPE> struct Prod { static constexpr bool FAST = false; struct Raw {}; struct Ptr {}; };

// Q4_K: w = (d*sc)*q - dmin*m with the fp32 roundings of dequantize_row_q4_K (k_quants.c:607-631), then one rounding to fp16.
// d*sc and dmin*m are exact in fp32 (11-bit x 6-bit significands) and so is (d*sc)*q (17 x 4 bits), hence fma(d*sc, q, -dmin*m) rounds
// exactly once where the CPU's fmul + fsub rounds exactly once: same bits, one instruction less per weight (the producers bound this kernel).
template <> struct Prod<T_Q4_K> {
    static constexpr bool FAST = true;
    struct Raw { uint2 q; uint32_t sm, dd; };
    // K block kb (64 weights) of a row: quant bytes at 32 kb + 8 h, the (sc, sc, min, min) word at 4 kb, (d, dmin) at 4 (kb / 4): running pointers
    struct Ptr { const uint8_t * q, * sm, * dd; };
    static __device__ __forceinline__ Ptr ptr(const WPlanes & W, size_t row, int kb, int h) {      // h = 0..3: bytes 8h .. 8h+7 of the 32
        return { W.p[0] + row * W.stride[0] + (size_t) kb * 32 + h * 8, W.p[1] + row * W.stride[1] + (size_t) kb * 4, W.p[2] + row * W.stride[2] };
    }
    static __device__ __forceinline__ void next(Ptr & p) { p.q += 32; p.sm += 4; }
    static __device__ __forceinline__ Raw load(const Ptr & p, int kb, int) {
        Raw r;
        r.q = ldg_stream_v2(p.q); r.sm = ldg_u32(p.sm); r.dd = ldg_u32(p.dd + (size_t) (kb >> 2) * 4);
        return r;
    }
    static __device__ __forceinline__ Chunks deq(const Raw & r, int, int) {
        const float2 dm = __half22float2(*reinterpret_cast<const __half2 *>(&r.dd));
        const float d0 = __fmul_rn(dm.x, (float) (r.sm & 0xff)), d1 = __fmul_rn(dm.x, (float) ((r.sm >> 8) & 0xff));
        const float m0 = __fmul_rn(dm.y, (float) ((r.sm >> 16) & 0xff)), m1 = __fmul_rn(dm.y, (float) (r.sm >> 24));
        const uint32_t w[2] = { r.q.x, r.q.y };
        float lo[8], hi[8];
#pragma unroll
        for (int i = 0; i < 2; i++)
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const uint32_t byte = (w[i] >> (8 * j)) & 0xff;
                lo[4 * i + j] = __fmaf_rn(d0, (float) (byte & 0xF), -m0);
                hi[4 * i + j] = __fmaf_rn(d1, (float) (byte >> 4), -m1);
            }
        Chunks o;
        o.c[0] = make_uint4(pack_h2(lo[0], lo[1]), pack_h2(lo[2], lo[3]), pack_h2(lo[4], lo[5]), pack_h2(lo[6], lo[7]));
        o.c[1] = make_uint4(pack_h2(hi[0], hi[1]), pack_h2(hi[2], hi[3]), pack_h2(hi[4], hi[5]), pack_h2(hi[6], hi[7]));
        return o;
    }
};

// The legacy and 3-bit types dequantise in HALF arithmetic without losing a bit: code (and code * scale) are small integers, exact in
// fp16, and one fp16 multiply by the fp16 block scale d rounds the exact product once -- which is what "fp32 product (exact: <= 20
// significant bits), then round to fp16" does.  Four codes of a 32-bit word come out of two LOP3s as the halves 1024 + code of bytes
// (0, 2) and (1, 3) (the 0x6400 exponent trick); two PRMTs put them back in element order.
__device__ __forceinline__ uint32_t h2_sub(uint32_t a, uint32_t b) { uint32_t r; asm("sub.rn.f16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
__device__ __forceinline__ uint32_t h2_mul(uint32_t a, uint32_t b) { uint32_t r; asm("mul.rn.f16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
__device__ __forceinline__ uint32_t h2_dup(uint32_t two_halves, bool high) { return __byte_perm(two_halves, 0, high ? 0x3232 : 0x1010); }
// a = halves of elements (0, 2), b = halves of elements (1, 3)  ->  (0, 1) and (2, 3)
__device__ __forceinline__ void h2_order(uint32_t a, uint32_t b, uint32_t & e01, uint32_t & e23) { e01 = __byte_perm(a, b, 0x5410); e23 = __byte_perm(a, b, 0x7632); }

// Q4_0: w = (q - 8) * d (ggml.c:1509-1527); element j of a block sits in the low nibble of qs[j], j + 16 in the high nibble.  The K block
// holds two blocks; thread h owns elements 8h .. 8h+7 of each: low (h < 2) or high nibbles of qs[8 (h & 1) .. +7].
template <> struct Prod<T_Q4_0> {
    static constexpr bool FAST = true;
    struct Raw { uint2 qa, qb; uint32_t dd; };
    struct Ptr { const uint8_t * q, * d; };
    static __device__ __forceinline__ Ptr ptr(const WPlanes & W, size_t row, int kb, int h) {
        return { W.p[0] + row * W.stride[0] + (size_t) kb * 32 + (h & 1) * 8, W.p[1] + row * W.stride[1] + (size_t) kb * 4 };
    }
    static __device__ __forceinline__ void next(Ptr & p) { p.q += 32; p.d += 4; }
    static __device__ __forceinline__ Raw load(const Ptr & p, int, int) {
        Raw r;
        r.qa = ldg_stream_v2(p.q); r.qb = ldg_stream_v2(p.q + 16); r.dd = ldg_u32(p.d);
        return r;
    }
    static __device__ __forceinline__ uint4 block(uint2 q, uint32_t d2, int sh) {
        uint32_t o[4];
#pragma unroll
        for (int i = 0; i < 2; i++) {
            const uint32_t w = (i ? q.y : q.x) >> sh;
            const uint32_t a = h2_mul(h2_sub((w & 0x000F000Fu) | 0x64006400u, 0x64086408u), d2);          // (1024 + q) - 1032 = q - 8
            const uint32_t b = h2_mul(h2_sub(((w >> 8) & 0x000F000Fu) | 0x64006400u, 0x64086408u), d2);
            h2_order(a, b, o[2 * i], o[2 * i + 1]);
        }
        return make_uint4(o[0], o[1], o[2], o[3]);
    }
    static __device__ __forceinline__ Chunks deq(const Raw & r, int, int h) {
        const int sh = (h >> 1) * 4;
        Chunks o;
        o.c[0] = block(r.qa, h2_dup(r.dd, false), sh);
        o.c[1] = block(r.qb, h2_dup(r.dd, true), sh);
        return o;
    }
};

// Q3_K: w = d * (sc - 32) * (q2 + 4 hbit - 4) (k_quants.c:472-521).  K block kb is quarter c = kb % 4 of super-block kb / 4: half n = c / 2,
// 2-bit fields j0 = 2 (c % 2) and j0 + 1 of qs[32 n + l], high bits 4 n + j of hmask[l]; thread h owns l = 8h .. 8h+7 for both fields; their
// two scales are bytes j0, j0 + 1 of one word of the expanded scale plane (formats.cuh: q3_scale16).
template <> struct Prod<T_Q3_K> {
    static constexpr bool FAST = true;
    struct Raw { uint2 q, hm; uint32_t sc; uint16_t d; };
    struct Ptr { const uint8_t * q, * hm, * sc, * d; };
    static __device__ __forceinline__ Ptr ptr(const WPlanes & W, size_t row, int, int h) {
        return { W.p[0] + row * W.stride[0] + h * 8, W.p[1] + row * W.stride[1] + h * 8, W.p[2] + row * W.stride[2] + (h >> 1) * 4, W.p[3] + row * W.stride[3] };
    }
    static __device__ __forceinline__ void next(Ptr &) {}
    static __device__ __forceinline__ Raw load(const Ptr & p, int kb, int) {
        const int b = kb >> 2, n = (kb >> 1) & 1;
        Raw r;
        r.q = ldg_stream_v2(p.q + (size_t) b * 64 + n * 32); r.hm = ldg_stream_v2(p.hm + (size_t) b * 32);
        r.sc = ldg_u32(p.sc + (size_t) b * 16 + n * 8); r.d = __ldg(reinterpret_cast<const uint16_t *>(p.d) + b);
        return r;
    }
    static __device__ __forceinline__ uint4 field(uint2 q, uint2 hm, int qsh, int hsh, uint32_t sc2, uint32_t d2) {
        uint32_t o[4];
#pragma unroll
        for (int i = 0; i < 2; i++) {
            const uint32_t w = (i ? q.y : q.x) >> qsh, m = (i ? hm.y : hm.x) >> hsh;
            // q2 | hbit << 2 = q2 + 4 hbit in 0..7; minus 4 = the signed code; times the scale: |.| <= 128, exact in fp16
            const uint32_t va = (w & 0x00030003u) | ((m & 0x00010001u) << 2) | 0x64006400u;
            const uint32_t vb = ((w >> 8) & 0x00030003u) | (((m >> 8) & 0x00010001u) << 2) | 0x64006400u;
            const uint32_t a = h2_mul(h2_mul(h2_sub(va, 0x64046404u), sc2), d2), b = h2_mul(h2_mul(h2_sub(vb, 0x64046404u), sc2), d2);
            h2_order(a, b, o[2 * i], o[2 * i + 1]);
        }
        return make_uint4(o[0], o[1], o[2], o[3]);
    }
    static __device__ __forceinline__ Chunks deq(const Raw & r, int kb, int) {
        const int n = (kb >> 1) & 1, j0 = 2 * (kb & 1);
        const uint32_t d2 = (uint32_t) r.d | ((uint32_t) r.d << 16);
        const int s0 = (int) (int8_t) (r.sc >> (8 * j0)), s1 = (int) (int8_t) (r.sc >> (8 * j0 + 8));
        const __half2 h0 = __float2half2_rn((float) s0), h1 = __float2half2_rn((float) s1);
        Chunks o;
        o.c[0] = field(r.q, r.hm, 2 * j0, 4 * n + j0, *reinterpret_cast<const uint32_t *>(&h0), d2);
        o.c[1] = field(r.q, r.hm, 2 * j0 + 2, 4 * n + j0 + 1, *reinterpret_cast<const uint32_t *>(&h1), d2);
        return o;
    }
};

struct GemmArgs {
    WPlanes W;
    float * Y; int64_t y_stride;
    int N;                // tokens
    int epi_gelu;
    int ksplit;           // K is split over gridDim.z CTAs; > 1: partial tiles are added into a zeroed Y with atomics
                          // (ksplit == 2 keeps the result deterministic: 0 + a + b is the same in either order)
};

template <int TYPE, int BN>
__global__ void __launch_bounds__(THREADS, 1) gemm_tc_kernel(const __grid_constant__ CUtensorMap xmap, const GemmArgs a) {
    constexpr int B_STAGE = BN * 128;                                      // BN token rows of 64 halves
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t * smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t) 1023);
    uint8_t * sA = smem;                                                   // ST stages of 16 KB
    uint8_t * sB = smem + ST * A_STAGE;                                    // ST stages of BN x 128 B
    uint64_t * bars = reinterpret_cast<uint64_t *>(sB + ST * B_STAGE);
    uint64_t * a_full = bars, * b_full = bars + ST, * empty = bars + 2 * ST;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n0 = blockIdx.x * BN, m0 = blockIdx.y * BM;
    const int KBT = a.W.K / BK;                                            // K blocks in total; this CTA owns [kb0, kb0 + KB)
    const int kb0 = (int) ((int64_t) KBT * blockIdx.z / a.ksplit), KB = (int) ((int64_t) KBT * (blockIdx.z + 1) / a.ksplit) - kb0;

    if (threadIdx.x == 0) {
        for (int s = 0; s < ST; s++) { mbar_init(a_full + s, 128); mbar_init(b_full + s, 1); mbar_init(empty + s, 8); }   // empty: one arrival per consumer warp
        mbar_fence_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ===== dequant producers (one thread per weight row) + the TMA of the activation tile =====
        const int r = threadIdx.x;
        const size_t row = (size_t) min(m0 + r, a.W.M - 1);                // rows past M are computed from row M-1 and never stored
        using P = Prod<TYPE>;
        typename P::Raw raw[4], raw1[4];                                   // the bytes of K blocks kb and kb + 1: two loads in flight per chunk pair
        typename P::Ptr pq[4];
        if constexpr (P::FAST) {
#pragma unroll
            for (int h = 0; h < 4; h++) {
                const typename P::Ptr p0 = P::ptr(a.W, row, kb0, h);
                pq[h] = P::ptr(a.W, row, kb0 + (KB > 1 ? 1 : 0), h);
                raw[h] = P::load(p0, kb0, h); raw1[h] = P::load(pq[h], kb0 + (KB > 1 ? 1 : 0), h);
            }
        }
        const int sw = r & 7;
        const uint32_t st_row = smem_u32(sA) + (uint32_t) (r * 128);
        for (int kb = 0; kb < KB; kb++) {
            const int s = kb % ST;
            if (kb >= ST) mbar_wait(empty + s, (uint32_t) ((kb / ST - 1) & 1));
            if (r == 0) {
                mbar_expect_tx(b_full + s, (uint32_t) B_STAGE);            // rows past N are zero-filled by TMA and still counted
                tma_load_2d(sB + (size_t) s * B_STAGE, &xmap, (kb0 + kb) * BK, n0, b_full + s);
            }
#pragma unroll
            for (int h = 0; h < 4; h++) {
                Chunks ch;
                if constexpr (P::FAST) {
                    ch = P::deq(raw[h], kb0 + kb, h);
                    raw[h] = raw1[h];
                    P::next(pq[h]);                                        // -> K block kb0 + kb + 2
                    if (kb + 2 < KB) raw1[h] = P::load(pq[h], kb0 + kb + 2, h);
                } else ch = dequant_generic(a.W, row, (kb0 + kb) * BK, h);
                const uint32_t st = st_row + (uint32_t) s * A_STAGE;
                asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" :: "r"(st + (uint32_t) ((h ^ sw) << 4)), "r"(ch.c[0].x), "r"(ch.c[0].y), "r"(ch.c[0].z), "r"(ch.c[0].w) : "memory");         // elements 8h .. 8h+7
                asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" :: "r"(st + (uint32_t) (((4 + h) ^ sw) << 4)), "r"(ch.c[1].x), "r"(ch.c[1].y), "r"(ch.c[1].z), "r"(ch.c[1].w) : "memory");   // elements 32+8h .. 32+8h+7
            }
            fence_proxy_async();                                           // generic-proxy stores -> visible to the tensor core (async proxy)
            mbar_arrive(a_full + s);
        }
    } else {
        // ===== consumers: warpgroup g = 1, 2 owns weight rows [64 (g - 1), +64) of the tile =====
        const int g = warp / 4 - 1, wq = warp & 3;
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; i++) acc[i] = 0.f;
        for (int kb = 0; kb < KB; kb++) {
            const int s = kb % ST;
            mbar_wait(a_full + s, (uint32_t) ((kb / ST) & 1));
            mbar_wait(b_full + s, (uint32_t) ((kb / ST) & 1));
            const uint32_t a_addr = smem_u32(sA + (size_t) s * A_STAGE) + g * 64 * 128, b_addr = smem_u32(sB + (size_t) s * B_STAGE);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BK / 16; k++) Wgmma<BN>::mma(acc, wgmma_desc(a_addr + k * 32), wgmma_desc(b_addr + k * 32), 1);
            wgmma_commit();
            wgmma_wait<1>();                                               // the previous stage's MMAs are done: release it
            if (kb > 0 && lane == 0) mbar_arrive(empty + (kb - 1) % ST);
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        // ===== epilogue: accumulator registers -> global =====
        const int mr = m0 + g * 64 + wq * 16 + (lane >> 2);
#pragma unroll
        for (int j = 0; j < BN / 8; j++) {
#pragma unroll
            for (int i = 0; i < 2; i++) {
                const int m = mr + 8 * i;
                if (m >= a.W.M) continue;
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const int n = n0 + 8 * j + 2 * (lane & 3) + e;
                    if (n >= a.N) continue;
                    float y = acc[4 * j + 2 * i + e];
                    if (a.epi_gelu) y = gelu_f16lut(y);
                    if (a.ksplit > 1) atomicAdd(a.Y + (size_t) n * a.y_stride + m, y);
                    else a.Y[(size_t) n * a.y_stride + m] = y;
                }
            }
        }
    }
}

PFN_cuTensorMapEncodeTiled_v12000 get_encode() {
    static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
    if (!fn) {
        cudaDriverEntryPointQueryResult q;
        void * p = nullptr;
        B200_CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
        B200_ASSERT(q == cudaDriverEntryPointSuccess && p);
        fn = (PFN_cuTensorMapEncodeTiled_v12000) p;
    }
    return fn;
}

template <int TYPE, int BN>
void launch_typed(const CUtensorMap & map, const GemmArgs & a, cudaStream_t stream) {
    const size_t smem = 1024 + (size_t) ST * (A_STAGE + BN * 128) + 256;
    static bool set = false;
    if (!set) { B200_CUDA_CHECK(cudaFuncSetAttribute(gemm_tc_kernel<TYPE, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem)); set = true; }
    const dim3 grid((unsigned) ((a.N + BN - 1) / BN), (unsigned) ((a.W.M + BM - 1) / BM), (unsigned) a.ksplit);
    gemm_tc_kernel<TYPE, BN><<<grid, THREADS, smem, stream>>>(map, a);
    B200_CUDA_CHECK(cudaGetLastError());
}

template <int BN>
void launch_bn(int producer, const CUtensorMap & map, const GemmArgs & a, cudaStream_t stream) {
    switch (producer) {
        case T_Q4_K: launch_typed<T_Q4_K, BN>(map, a, stream); break;
        case T_Q4_0: launch_typed<T_Q4_0, BN>(map, a, stream); break;
        case T_Q3_K: launch_typed<T_Q3_K, BN>(map, a, stream); break;
        default:     launch_typed<-1, BN>(map, a, stream); break;           // generic element-wise dequantiser
    }
}

} // namespace

GemmTcShape gemm_tc_pick_shape(int type, int64_t K, int64_t M, int N, int64_t x_stride, bool x_aligned, int epi_gelu) {
    if (N < 1 || N > N_MAX || K % BK != 0 || (x_stride % 8) != 0 || !x_aligned) return {};
    GemmTcShape s;
    s.bn = N <= 64 ? 64 : N <= 128 ? 128 : 256;
    // fewer than ~100 tiles cannot fill the 132 SMs of an H100: split K in two (deterministic, see GemmArgs::ksplit)
    const int64_t tiles = (M + BM - 1) / BM * ((N + s.bn - 1) / s.bn);
    s.ksplit = (tiles < 100 && !epi_gelu && K / BK >= 8) ? 2 : 1;
    s.producer = (type == T_Q4_K || type == T_Q4_0 || type == T_Q3_K) ? type : -1;
    return s;
}

// X: fp16 [N][x_stride] (x_stride >= K, multiple of 8), Y: fp32 [N][y_stride].  N <= 512, K % 64 == 0.
bool launch_gemm_tc(const WPlanes & W, const __half * X, int64_t x_stride, int N, float * Y, int64_t y_stride, int epi_gelu, cudaStream_t stream) {
    const GemmTcShape s = gemm_tc_pick_shape(W.type, W.K, W.M, N, x_stride, ((uintptr_t) X & 15) == 0, epi_gelu);
    if (!s.bn) return false;
    GemmArgs a;
    a.W = W; a.Y = Y; a.y_stride = y_stride; a.N = N; a.epi_gelu = epi_gelu; a.ksplit = s.ksplit;
    const int BN = s.bn;
    // the two halves add into Y: clear the N rows of M outputs, and only those (columns M .. y_stride-1 belong to the caller)
    if (a.ksplit > 1) B200_CUDA_CHECK(cudaMemset2DAsync(Y, (size_t) y_stride * sizeof(float), 0, (size_t) W.M * sizeof(float), (size_t) N, stream));
    CUtensorMap map;
    const cuuint64_t gdim[2] = { (cuuint64_t) W.K, (cuuint64_t) N };
    const cuuint64_t gstr[1] = { (cuuint64_t) x_stride * 2 };
    const cuuint32_t box[2] = { (cuuint32_t) BK, (cuuint32_t) BN };
    const cuuint32_t estr[2] = { 1, 1 };
    const CUresult rc = get_encode()(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void *) X, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (rc != CUDA_SUCCESS) { fprintf(stderr, "b200: cuTensorMapEncodeTiled failed (%d)\n", (int) rc); exit(1); }
    if (BN == 64) launch_bn<64>(s.producer, map, a, stream);
    else if (BN == 128) launch_bn<128>(s.producer, map, a, stream);
    else launch_bn<256>(s.producer, map, a, stream);
    return true;
}
