// attention_ws.cu -- causal grouped-query attention for a batch of N > 8 new tokens (prompt processing): warp-specialised
// Hopper kernel (TMA + wgmma) over an fp16 shadow of the KV cache.
//
// Contract (libfalcon.cpp:2285-2366, ggml.c:12389-12458): scores scaled by 1/sqrt(64), the row's GLOBAL maximum subtracted before
// the fp16-LUT exp, probabilities normalised by 1/sum.  The global maximum makes it a TWO-PASS kernel: pass 1 runs S = Q K^T on
// the tensor cores only to find the row maxima, pass 2 recomputes each S tile, turns it into e = LUT(s - max) -- an fp16 value by
// construction, so the fp16 A operand of the second product is EXACT -- and accumulates O += e V in registers.
//
//   * K and V^T live in HBM as fp16 shadows written ONCE, by the kernel that appends a token to the fp32 cache
//     (rope_kv_append_kernel / kv_shadow_refresh_kernel), in exactly the layouts the MMA operands want:
//       k16  [n_ctx][n_head_kv][64]       a key row is 128 bytes = one SWIZZLE_128B row of the K-major B operand of Q K^T
//       vt16 [n_head_kv][64][ctx_pad]     V transposed: a row of the K-major B operand of P V is 64 consecutive keys of one dim
//   * warp 0 streams the tiles with TMA (cp.async.bulk.tensor, 3-D maps) into a 3-deep K ring and a 2-deep V^T ring
//   * two consumer warpgroups own 64 query rows each: S = Q K^T (wgmma m64n128k16, Q and K from shared memory) lands in registers,
//     the softmax works on the accumulator fragment in place (a row lives in one quad of lanes), and P, packed to fp16, is the
//     REGISTER A operand of O += P V (wgmma m64n64k16), so P never goes through shared memory.  While one warpgroup runs its
//     softmax the other one's MMAs keep the tensor core busy.
// One CTA = 128 query rows of one KV head (row = token * G + head_in_group: the G query heads that share the KV head are stacked,
// a K / V tile serves all of them) x all visible keys in tiles of 128; CTAs with the most key tiles are scheduled first.
// Shared memory 97 KB.
// Precision: Q, K, V rounded to fp16, fp32 accumulation, P exact; the row sum is an fp32 sum of the fp16 probabilities (the CPU's is
// double).  Keys >= T are never loaded (the tensor maps end at T), so stale cache rows cannot reach the P V product.
// Tolerance: tests/test_attention_exact_gpu.py holds the kernel to an exact restatement of these roundings (tests/attn_exact.py)
// within a per-element bound; logits inside the GEMM-path bound.
#include "kernels.h"
#include "wgmma.cuh"
#include <cuda.h>
#include <cudaTypedefs.h>

namespace {

constexpr int M = 128, NK = 128, D = 64;
constexpr int KST = 3, VST = 2;
constexpr int V_SUB = 8192;                         // one 64-key half of a V^T stage: 64 dims x 128 B
constexpr int V_STAGE = 2 * V_SUB;
constexpr int SQ = 0, SK = 16384, SV = SK + KST * 16384, SBAR = SV + VST * V_STAGE;
constexpr size_t SMEM_BYTES = 1024 + SBAR + 256;
constexpr int THREADS = 384;                        // warpgroup 0: TMA (warp 0); warpgroups 1, 2: MMA + softmax

__device__ __forceinline__ void mbar_arrive(uint64_t * bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void tma_load_3d(void * smem_dst, const CUtensorMap * map, int c0, int c1, int c2, uint64_t * bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 :: "r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t *>(&h);
}
// e^x for x <= 0 as the LUT computes it up to the final fp16 rounding: ex2.approx.ftz (2 ulp fp32); results below 2^-126 flush to zero,
// which the fp16 rounding would do anyway (the plain __expf wraps the same instruction in denormal rescaling: 3 extra instructions)
__device__ __forceinline__ float exp_fast(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x * 1.4426950408889634f));
    return y;
}

struct WsArgs {
    const float * qkv; float * out;
    int n_head_kv, G, n_tok, n_past, T, rows;            // T = n_past + n_tok; rows = G * n_tok per KV head
    int64_t qkv_stride, out_stride;
};

// 16 fp32 values (quarter h of a 64-value row, or zeros) -> a quarter of one 128-byte row of a K-major SWIZZLE_128B tile
__device__ __forceinline__ void store_quarter_row_f16(uint8_t * tile, int r, const float * src, bool valid, int h) {
    uint8_t * row = tile + r * 128;
    const int sw = r & 7;
#pragma unroll
    for (int cc = 0; cc < 2; cc++) {
        const int c = 2 * h + cc;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (valid) {
            const float4 a = __ldg(reinterpret_cast<const float4 *>(src) + 2 * c), b = __ldg(reinterpret_cast<const float4 *>(src) + 2 * c + 1);
            v = make_uint4(pack_h2(a.x, a.y), pack_h2(a.z, a.w), pack_h2(b.x, b.y), pack_h2(b.z, b.w));
        }
        *reinterpret_cast<uint4 *>(row + ((c ^ sw) << 4)) = v;
    }
}

__global__ void __launch_bounds__(THREADS, 1) attention_ws_kernel(const __grid_constant__ CUtensorMap kmap, const __grid_constant__ CUtensorMap vmap, const WsArgs a) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t * smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t) 1023);
    uint64_t * bars = reinterpret_cast<uint64_t *>(smem + SBAR);
    uint64_t * k_full = bars, * k_empty = k_full + KST, * v_full = k_empty + KST, * v_empty = v_full + VST;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = blockIdx.y, r0 = ((int) gridDim.x - 1 - (int) blockIdx.x) * M;      // latest rows (most key tiles) first
    const int t_last = (min(r0 + M, a.rows) - 1) / a.G;
    const int kmax = a.n_past + t_last + 1, nt = (kmax + NK - 1) / NK;

    if (threadIdx.x == 0) {
        for (int s = 0; s < KST; s++) { mbar_init(k_full + s, 1); mbar_init(k_empty + s, 8); }      // empty: one arrival per consumer warp
        for (int s = 0; s < VST; s++) { mbar_init(v_full + s, 1); mbar_init(v_empty + s, 8); }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ================================================================ TMA producer
        if (warp == 0 && lane == 0) {
            for (int j = 0; j < 2 * nt; j++) {
                const int kt = j < nt ? j : j - nt, s = j % KST;
                if (j >= KST) mbar_wait(k_empty + s, (uint32_t) ((j / KST - 1) & 1));
                mbar_expect_tx(k_full + s, 16384);
                tma_load_3d(smem + SK + s * 16384, &kmap, 0, g, kt * NK, k_full + s);
                if (j >= nt) {
                    const int i = j - nt, vs = i % VST;
                    if (i >= VST) mbar_wait(v_empty + vs, (uint32_t) ((i / VST - 1) & 1));
                    mbar_expect_tx(v_full + vs, 16384);
                    tma_load_3d(smem + SV + vs * V_STAGE, &vmap, kt * NK, 0, g, v_full + vs);
                    tma_load_3d(smem + SV + vs * V_STAGE + V_SUB, &vmap, kt * NK + 64, 0, g, v_full + vs);
                }
            }
        }
        return;
    }

    // ==================================================================== consumer warpgroup wg = 0, 1: query rows [64 wg, +64) of the tile
    const int ct = threadIdx.x - 128, wg = ct >> 7, wq = (ct >> 5) & 3;
    {   // Q tile: two threads per row, 32 values each, fp32 -> fp16 into the swizzled A-operand layout
        const int t = ct >> 1, row = r0 + t;
        const bool ok = row < a.rows;
        const float * src = a.qkv + (size_t) (ok ? row / a.G : 0) * a.qkv_stride + (size_t) (g * a.G + (ok ? row % a.G : 0)) * D;
        store_quarter_row_f16(smem + SQ, t, src, ok, 2 * (ct & 1));
        store_quarter_row_f16(smem + SQ, t, src, ok, 2 * (ct & 1) + 1);
        fence_proxy_async();                                                // generic-proxy stores -> visible to the tensor core
        asm volatile("bar.sync %0, 128;" :: "r"(1 + wg) : "memory");        // this warpgroup's 64 rows are written
    }
    // this thread's two rows of the accumulator fragments: i = 0, 1 -> tile row 64 wg + 16 wq + lane / 4 + 8 i
    int tok[2], head[2], vis[2];
    bool row_ok[2];
#pragma unroll
    for (int i = 0; i < 2; i++) {
        const int row = r0 + 64 * wg + 16 * wq + (lane >> 2) + 8 * i;
        row_ok[i] = row < a.rows;
        tok[i] = row / a.G; head[i] = g * a.G + row % a.G;
        vis[i] = row_ok[i] ? a.n_past + tok[i] + 1 : 0;                     // causal: keys < vis (ggml.c:12342-12348)
    }
    const int vis_min = r0 + M <= a.rows ? a.n_past + r0 / a.G + 1 : 0;     // keys visible to EVERY row of the tile (0 if it has padding rows)
    const float scale = 0.125f;                                             // 1 / sqrt(64), a power of two: s * scale is exact
    const int col = 2 * (lane & 3);                                         // column of fragment element 4 c + 2 i + e: 8 c + col + e
    const uint32_t q_addr = smem_u32(smem + SQ) + wg * 64 * 128;

    float mraw[2] = { -INFINITY, -INFINITY }, neg_m[2] = { 0.f, 0.f }, lsum[2] = { 0.f, 0.f };
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; i++) o[i] = 0.f;
    for (int j = 0; j < 2 * nt; j++) {
        const int s = j % KST, kt = j < nt ? j : j - nt, k0 = kt * NK;
        mbar_wait(k_full + s, (uint32_t) ((j / KST) & 1));
        float sc[64];
        const uint32_t k_addr = smem_u32(smem + SK + s * 16384);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < D / 16; k++) Wgmma<128>::mma(sc, wgmma_desc(q_addr + k * 32), wgmma_desc(k_addr + k * 32), k != 0);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(sc);
        if (lane == 0) mbar_arrive(k_empty + s);                            // the scores are in registers: the K stage may be refilled
        const bool full = k0 + NK <= vis_min;
        if (j < nt) {
            // ---- pass 1: the row maximum of the raw scores (scale > 0: max(scale * s) = scale * max(s))
#pragma unroll
            for (int c = 0; c < 16; c++)
#pragma unroll
                for (int i = 0; i < 2; i++)
#pragma unroll
                    for (int e = 0; e < 2; e++)
                        if (full || k0 + 8 * c + col + e < vis[i]) mraw[i] = fmaxf(mraw[i], sc[4 * c + 2 * i + e]);
            if (j == nt - 1) {
#pragma unroll
                for (int i = 0; i < 2; i++) {
                    float m = fmaxf(mraw[i], __shfl_xor_sync(0xffffffffu, mraw[i], 1));
                    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
                    neg_m[i] = -__fmul_rn(m, scale);
                }
            }
            continue;
        }
        // ---- pass 2: e = table_exp_f16[f16(s - max)] (ggml.c:12427-12440), P = e as fp16 (exact), packed into the A fragments of P V
        uint32_t p[8][4];
#pragma unroll
        for (int c = 0; c < 16; c++)
#pragma unroll
            for (int i = 0; i < 2; i++) {
                // s - max with ONE rounding: the product with 0.125 is exact, so fma(s, 0.125, -max) == (s * 0.125) - max
                const float x0 = __fmaf_rn(sc[4 * c + 2 * i], scale, neg_m[i]), x1 = __fmaf_rn(sc[4 * c + 2 * i + 1], scale, neg_m[i]);
                const float2 xr = __half22float2(__floats2half2_rn(x0, x1));   // the LUT index: f16(s - max)
                float e0 = exp_fast(xr.x), e1 = exp_fast(xr.y);
                if (!full) { const int key = k0 + 8 * c + col; if (key >= vis[i]) e0 = 0.f; if (key + 1 >= vis[i]) e1 = 0.f; }
                const uint32_t pk = pack_h2(e0, e1);                         // table_exp_f16 value: exact as fp16
                const float2 ef = __half22float2(*reinterpret_cast<const __half2 *>(&pk));
                lsum[i] += ef.x + ef.y;
                p[c >> 1][(c & 1) * 2 + i] = pk;
            }
        const int i = j - nt, vs = i % VST;
        mbar_wait(v_full + vs, (uint32_t) ((i / VST) & 1));
        const uint32_t v_addr = smem_u32(smem + SV + vs * V_STAGE);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < NK / 16; kk++) wgmma_rs_n64(o, p[kk], wgmma_desc(v_addr + (kk >> 2) * V_SUB + (kk & 3) * 32));
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(o);
        if (lane == 0) mbar_arrive(v_empty + vs);
    }

    // ---- epilogue: O / sum -> out[tok][head * 64 + ...]
#pragma unroll
    for (int i = 0; i < 2; i++) {
        float l = lsum[i];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        const float inv = (float) (1.0 / (double) l);                       // ggml.c:12427-12449
        if (!row_ok[i]) continue;
        float * dst = a.out + (size_t) tok[i] * a.out_stride + (size_t) head[i] * D + col;
#pragma unroll
        for (int c = 0; c < 8; c++)
            *reinterpret_cast<float2 *>(dst + 8 * c) = make_float2(__fmul_rn(o[4 * c + 2 * i], inv), __fmul_rn(o[4 * c + 2 * i + 1], inv));
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

// cache rows [pos, pos + n) -> the fp16 planes the prompt kernel reads (used when a cache was filled by something other than
// rope_kv_append: session restore, kv_write, the per-operator C ABI).  f32 cache (E = float): k16 and vt16; fp16 cache: vt16 only
template <typename E>
__global__ void kv_shadow_refresh_kernel(const KvCache c, int n_head_kv, int pos, int n) {
    const int64_t total = (int64_t) n * n_head_kv * 64;
    for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t) gridDim.x * blockDim.x) {
        const int d = (int) (i % 64), h = (int) ((i / 64) % n_head_kv), p = pos + (int) (i / (64 * n_head_kv));
        const size_t src = ((size_t) p * n_head_kv + h) * 64 + d;
        if (sizeof(E) == 4) c.k16[src] = __float2half_rn(c.k[src]);
        c.vt16[((size_t) h * 64 + d) * c.ctx_pad + p] = __float2half_rn(kv_ld(kv_v<E>(c) + src));
    }
}

} // namespace

int attention_ctx_pad(int n_ctx) { return (n_ctx + 63) / 64 * 64; }
size_t attention_shadow_halves(int n_head_kv, int n_ctx) { return (size_t) n_head_kv * 64 * attention_ctx_pad(n_ctx); }     // per layer, for K and for V^T each

void launch_kv_shadow_refresh(const KvCache & c, int n_head_kv, int pos, int n, cudaStream_t stream) {
    if (n <= 0 || !c.vt16) return;           // no shadow (an f32 cache's k16 exists exactly when vt16 does)
    const int64_t total = (int64_t) n * n_head_kv * 64;
    const unsigned grid = (unsigned) (total / 256 + 1 > 132 * 8 ? 132 * 8 : total / 256 + 1);
    if (kv_f16(c)) kv_shadow_refresh_kernel<__half><<<grid, 256, 0, stream>>>(c, n_head_kv, pos, n);
    else kv_shadow_refresh_kernel<float><<<grid, 256, 0, stream>>>(c, n_head_kv, pos, n);
    B200_CUDA_CHECK(cudaGetLastError());
}

// the shapes this kernel takes: an fp16 shadow, head_dim 64, a host n_past, more than MMV_MAX_N tokens (B200_ATTN_TC: also fewer)
bool attention_ws_covers(const AttnParams & p) {
    if (!p.kv.k16 || !p.kv.vt16 || p.head_dim != D || p.n_past_dev != nullptr || (p.qkv_stride % 4) != 0 || getenv("B200_ATTN_SIMT")) return false;
    return p.n_tok > MMV_MAX_N || getenv("B200_ATTN_TC");     // small batches keep fp32 attention (reassociation-level parity)
}
void launch_attention_ws(const float * qkv, float * out, int64_t out_stride, const AttnParams & p, cudaStream_t stream) {
    B200_ASSERT(out_stride % 4 == 0);
    WsArgs a;
    a.qkv = qkv; a.out = out;
    a.n_head_kv = p.n_head_kv; a.G = p.n_head / p.n_head_kv; a.n_tok = p.n_tok; a.n_past = p.n_past; a.T = p.n_past + p.n_tok;
    a.rows = a.G * p.n_tok; a.qkv_stride = p.qkv_stride; a.out_stride = out_stride;
    const int ctx_pad = p.kv.ctx_pad;
    // Both maps end at key T, not at n_ctx / ctx_pad: TMA zero-fills the rest of the last key tile.  Cache rows >= T are stale (an earlier
    // sequence, kv_write, load_kv) and may hold NaN or, for an fp32 value beyond 65504, Inf in the shadow; the masked probabilities are
    // exact zeros, but 0 x NaN and 0 x Inf in the P V product are NaN.
    CUtensorMap kmap, vmap;
    {   // k16 [n_ctx][n_head_kv][64]: box = 128 keys x 1 head x 64 dims -> 128 rows of 128 B
        const cuuint64_t gdim[3] = { 64, (cuuint64_t) p.n_head_kv, (cuuint64_t) a.T };
        const cuuint64_t gstr[2] = { 128, (cuuint64_t) p.n_head_kv * 128 };
        const cuuint32_t box[3] = { 64, 1, 128 }, estr[3] = { 1, 1, 1 };
        const CUresult rc = get_encode()(&kmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, (void *) p.kv.k16, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (rc != CUDA_SUCCESS) { fprintf(stderr, "b200: cuTensorMapEncodeTiled(k16) failed (%d)\n", (int) rc); exit(1); }
    }
    {   // vt16 [n_head_kv][64][ctx_pad]: box = 64 keys x 64 dims x 1 head -> 64 rows of 128 B (one half of a 128-key tile)
        const cuuint64_t gdim[3] = { (cuuint64_t) a.T, 64, (cuuint64_t) p.n_head_kv };
        const cuuint64_t gstr[2] = { (cuuint64_t) ctx_pad * 2, (cuuint64_t) ctx_pad * 128 };
        const cuuint32_t box[3] = { 64, 64, 1 }, estr[3] = { 1, 1, 1 };
        const CUresult rc = get_encode()(&vmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, (void *) p.kv.vt16, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (rc != CUDA_SUCCESS) { fprintf(stderr, "b200: cuTensorMapEncodeTiled(vt16) failed (%d)\n", (int) rc); exit(1); }
    }
    static bool set = false;
    if (!set) { B200_CUDA_CHECK(cudaFuncSetAttribute(attention_ws_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) SMEM_BYTES)); set = true; }
    dim3 grid((unsigned) ((a.rows + M - 1) / M), (unsigned) p.n_head_kv);
    attention_ws_kernel<<<grid, THREADS, SMEM_BYTES, stream>>>(kmap, vmap, a);
    B200_CUDA_CHECK(cudaGetLastError());
}
