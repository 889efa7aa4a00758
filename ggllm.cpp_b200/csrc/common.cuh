// common.cuh -- shared device/host helpers for the sm_90a (H100) backend.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>

// Error convention of the reference backend (ggml-cuda.cu:22-51): print and exit(1); no return codes.
#define B200_CUDA_CHECK(expr)                                                                        \
    do {                                                                                             \
        cudaError_t err_ = (expr);                                                                   \
        if (err_ != cudaSuccess) {                                                                   \
            fprintf(stderr, "b200: CUDA error %d (%s) at %s:%d: %s\n", (int) err_,                   \
                    cudaGetErrorString(err_), __FILE__, __LINE__, #expr);                            \
            exit(1);                                                                                 \
        }                                                                                            \
    } while (0)

// contract violations abort like GGML_ASSERT (ggml.h:204-210)
#define B200_ASSERT(x)                                                                               \
    do {                                                                                             \
        if (!(x)) {                                                                                  \
            fprintf(stderr, "B200_ASSERT: %s:%d: %s\n", __FILE__, __LINE__, #x);                     \
            abort();                                                                                 \
        }                                                                                            \
    } while (0)

// enum ggml_type values (ggml.h:241-262); the C ABI passes them as plain ints
enum : int {
    T_F32 = 0, T_F16 = 1, T_Q4_0 = 2, T_Q4_1 = 3, T_Q5_0 = 6, T_Q5_1 = 7, T_Q8_0 = 8, T_Q8_1 = 9,
    T_Q2_K = 10, T_Q3_K = 11, T_Q4_K = 12, T_Q5_K = 13, T_Q6_K = 14, T_Q8_K = 15,
};

static inline size_t round_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// A device buffer that only grows.  get(need) returns at least `need` bytes; to grow, it waits for `stream` (the buffer's user), frees,
// and allocates the size rounded up to 1 MB, zeroed.
struct DevScratch {
    void * p = nullptr; size_t bytes = 0;
    void * get(size_t need, cudaStream_t stream) {
        if (need > bytes) {
            if (p) { B200_CUDA_CHECK(cudaStreamSynchronize(stream)); B200_CUDA_CHECK(cudaFree(p)); }
            bytes = round_up(need, 1 << 20);
            B200_CUDA_CHECK(cudaMalloc(&p, bytes));
            B200_CUDA_CHECK(cudaMemsetAsync(p, 0, bytes, stream));
        }
        return p;
    }
    void release() { if (p) B200_CUDA_CHECK(cudaFree(p)); p = nullptr; bytes = 0; }
};

// One L1/shared-memory split (percent of shared) for every kernel of the decode step.  An SM cannot host kernels that
// ask for different carve-outs at the same time, so without this the small attention kernels wait for the big
// mat-vec of the other stream to drain.  25 % of the H100's 228 KB = 57 KB shared, rest L1.
#define B200_CARVEOUT 25

// multiprocessors of the current device (queried once): the persistent kernels size their grids by it
inline int num_sms() {
    static int n = 0;
    if (!n) { int dev; B200_CUDA_CHECK(cudaGetDevice(&dev)); B200_CUDA_CHECK(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev)); }
    return n;
}

#ifdef __CUDACC__

// streaming 16-byte load of weight data: read-only path, do not allocate in L1 (each byte is used once)
__device__ __forceinline__ uint4 ldg_stream_v4(const void * p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ uint2 ldg_stream_v2(const void * p) {
    uint2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}
__device__ __forceinline__ uint32_t ldg_stream_u32(const void * p) {
    uint32_t r;
    asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}
// small shared-by-neighbours metadata (block headers): read-only path, normal caching
__device__ __forceinline__ uint4 ldg_v4(const void * p) { return __ldg(reinterpret_cast<const uint4 *>(p)); }
__device__ __forceinline__ uint32_t ldg_u32(const void * p) { return __ldg(reinterpret_cast<const uint32_t *>(p)); }
__device__ __forceinline__ uint16_t ldg_u16(const void * p) { return __ldg(reinterpret_cast<const uint16_t *>(p)); }

__device__ __forceinline__ float f16_bits_to_f32(uint16_t h) { return __half2float(__ushort_as_half(h)); }
__device__ __forceinline__ uint16_t f32_to_f16_bits(float f) { return __half_as_ushort(__float2half_rn(f)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ int dp4a_ss(int a, int b, int c) { return __dp4a(a, b, c); }                       // s8 x s8
__device__ __forceinline__ int dp4a_us(unsigned a, int b, int c) {                                            // u8 x s8
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
// u8 x s8 dot of 16 weight bytes (four words) with 16 activation codes
__device__ __forceinline__ int dot16(const uint32_t w0, const uint32_t w1, const uint32_t w2, const uint32_t w3, const uint4 x) {
    int s = dp4a_us(w0, (int) x.x, 0); s = dp4a_us(w1, (int) x.y, s); s = dp4a_us(w2, (int) x.z, s); return dp4a_us(w3, (int) x.w, s);
}
// c + the two s16 halves of pair16 times the low (lo) or high (hi) two bytes of `bytes`, unsigned (us) or signed (ss)
__device__ __forceinline__ int dp2a_lo_us(int pair16, uint32_t bytes, int c) { int d; asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(pair16), "r"(bytes), "r"(c)); return d; }
__device__ __forceinline__ int dp2a_hi_us(int pair16, uint32_t bytes, int c) { int d; asm("dp2a.hi.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(pair16), "r"(bytes), "r"(c)); return d; }
__device__ __forceinline__ int dp2a_lo_ss(int pair16, uint32_t bytes, int c) { int d; asm("dp2a.lo.s32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(pair16), "r"(bytes), "r"(c)); return d; }
__device__ __forceinline__ int dp2a_hi_ss(int pair16, uint32_t bytes, int c) { int d; asm("dp2a.hi.s32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(pair16), "r"(bytes), "r"(c)); return d; }

// fp16-LUT GELU (ggml.c:3461-3484, table 4281-4290): table_gelu_f16[f16(v)] = f16 of the fp32 formula at the fp16 input
__device__ __forceinline__ float gelu_f16lut(float v) {
    const float f = __half2float(__float2half_rn(v));
    const float g = 0.5f * f * (1.0f + tanhf(0.79788456080286535587989211986876f * f * (1.0f + 0.044715f * f * f)));
    return __half2float(__float2half_rn(g));
}
// table_exp_f16[f16(v)] (ggml.c:4281-4290), the softmax exponential of every attention kernel but the wgmma one
__device__ __forceinline__ float exp_f16lut(float v) {
    return __half2float(__float2half_rn(expf(__half2float(__float2half_rn(v)))));
}

// NeoX RoPE (ggml.c:12819-12983).  Pair i of a head at position p: theta = p * theta_scale^i built by repeated fp32 products, as the
// CPU loop does, then (x0, x1) -> (x0 c - x1 s, x0 s + x1 c) with every product and sum rounded on its own.
__device__ __forceinline__ float rope_theta(int p, int i, float theta_scale) {
    float theta = (float) p;
    for (int k = 0; k < i; k++) theta = __fmul_rn(theta, theta_scale);
    return theta;
}
__device__ __forceinline__ float2 rope_rotate(float x0, float x1, float c, float s) {
    return make_float2(__fsub_rn(__fmul_rn(x0, c), __fmul_rn(x1, s)), __fadd_rn(__fmul_rn(x0, s), __fmul_rn(x1, c)));
}

// ---- mbarrier + 1-D bulk (TMA) copy global -> shared: used to stage activation tiles ----
__device__ __forceinline__ uint32_t smem_u32(const void * p) { return (uint32_t) __cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t * bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t * bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t * bar, uint32_t phase) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}"
        :: "r"(smem_u32(bar)), "r"(phase) : "memory");
}
// size must be a multiple of 16 bytes; src/dst 16-byte aligned
__device__ __forceinline__ void tma_load_1d(void * smem_dst, const void * gmem_src, uint32_t bytes, uint64_t * bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

#endif // __CUDACC__
