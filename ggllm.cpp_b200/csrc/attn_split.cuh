// attn_split.cuh -- the frame of the split-KV decode attention (n_tok == 1, head_dim 64), shared by its two tiers: attention.cu's
// CUDA-core kernels up to attention_long_threshold() keys, attention_long.cu's tensor-core kernels above.  Numerics: attention.cu.
//
// Grid: (split, KV head, group of <= 16 of the KV head's G query heads).  A tier is two kernels:
//   scores: s = (q . k) * scale for the split's keys into the scratch row S[head][key], the split's maxima into pmax[head][split]
//   values: gmax = max over splits; e = LUT(s - gmax) for the split's keys and their sum in double; O_partial = sum_key V[key] e[key];
//           then split_combine: the LAST CTA of a (KV head, group) sums the partial sums and outputs in split order and scales by
//           (float) (1 / sum) -- ggml.c:12427-12449 multiplies each e by that factor before the product with V; scaling the product
//           instead is a reassociation-level difference (as the tensor-core prompt kernel does)
// Both kernels read n_past from a device scalar, so the captured decode graph serves every position.  The values kernel is launched
// programmatically behind the scores kernel (split_launch).  What differs between the tiers is only how keys are scored and how
// e . V is accumulated.
#pragma once
#include "kernels.h"
#include "actquant.cuh"

#define SPLIT_THREADS 128                // small CTAs: one fits beside ffn_up's two 256-thread CTAs on every SM
#define SPLIT_WARPS (SPLIT_THREADS / 32)
#define SPLIT_G 16                       // query heads per CTA (n_head / n_head_kv <= 16 per CTA, more in grid.z)
#define SPLIT_MAX 32                     // partials per head in the scratch: the most splits a tier may use
// keys per split: at least SPLIT_MIN_KEYS, so that a short context occupies few CTAs and the combine step reads few partials (at
// n_past < 64 one CTA per KV-head group does everything; the other CTAs of the fixed grid only check in at the counter)
#define SPLIT_MIN_KEYS 64

struct SplitArgs {
    const float * qkv; float * out;
    KvCache kv;                  // the layer's cache (kernels.h); its element type is the kernels' E
    float * S; float * pmax; double * psum; float * opart; unsigned * ctr;
    int n_head, n_head_kv, G, n_past; const int * n_past_dev; int n_ctx; int64_t qkv_stride;
    int n_splits;
    ActQ qA; int has_q;          // optional quantised copy of the output row (see AttnParams::qout)
    int fuse_rope; float theta_scale;     // see AttnParams::fuse_rope
};
// the fused append of this position's rows (elements e, e + 1 of K and V head kvh): every plane there is, through kernels.h's writer
__device__ __forceinline__ void split_append2(const SplitArgs & a, size_t o, int kvh, int e, int n_past, float2 k, float2 v) {
    kv_put_k(a.kv, o, k.x); kv_put_k(a.kv, o + 1, k.y);
    kv_put_v(a.kv, o, kvh, e, n_past, v.x); kv_put_v(a.kv, o + 1, kvh, e + 1, n_past, v.y);
}

__device__ __forceinline__ int split_keys(int T, int ns) { return max(SPLIT_MIN_KEYS, (T + ns - 1) / ns); }
__device__ __forceinline__ int splits_used(int T, int ns) { const int per = split_keys(T, ns); return (T + per - 1) / per; }
__device__ __forceinline__ void split_range(int T, int ns, int split, int & k_lo, int & k_hi) {
    const int per = split_keys(T, ns);
    k_lo = min(T, split * per); k_hi = min(T, k_lo + per);
}

// thread tid's 8 consecutive outputs (head hA of the CTA's group) -> the attention output row, plus wo's activation quantisation
__device__ __forceinline__ void split_store(const SplitArgs & a, const float (&y)[8], int h0, int hA, int G, int tid, int lane) {
    if (hA < G) {
        float4 * dst = reinterpret_cast<float4 *>(a.out + (size_t) h0 * 64) + 2 * tid;
        dst[0] = make_float4(y[0], y[1], y[2], y[3]); dst[1] = make_float4(y[4], y[5], y[6], y[7]);
    }
    if (a.has_q) {                                                      // here instead of in a kernel of its own
        const int k0 = h0 * 64 + 8 * tid;                               // a warp = 256 consecutive outputs = 4 heads
        if (a.qA.type == T_Q8_K) quantize_chunk8<T_Q8_K>(y, lane, a.qA, 0, k0, hA < G);
        else if (a.qA.type == T_Q8_1) quantize_chunk8<T_Q8_1>(y, lane, a.qA, 0, k0, hA < G);
        else quantize_chunk8<T_Q8_0>(y, lane, a.qA, 0, k0, hA < G);
    }
}

// The tail of both values kernels.  On entry, after a __syncthreads, a CTA whose split holds keys (nk > 0) has its per-warp partial
// outputs in shared memory, ow[warp][h * 32 + l] = dims 2 l, 2 l + 1 of head h, and its sums of e in dsum[r][h] (summed over r in
// order).  ns: the splits of the grid.  Sums run in a fixed order (warps, then splits): deterministic.
template <int WS, int R>
__device__ __forceinline__ void split_combine(const SplitArgs & a, const float2 (&ow)[SPLIT_WARPS][WS], const double (&dsum)[R][SPLIT_G],
                                              int ns, int n_used, int nk, int split, int h0, int G) {
    __shared__ float inv_s[SPLIT_G];
    __shared__ int s_last;
    const int tid = threadIdx.x, lane = tid & 31;
    auto cta_sum = [&](int h) {
        double s = 0.0;
#pragma unroll
        for (int r = 0; r < R; r++) s += dsum[r][h];
        return s;
    };
    if (n_used == 1) {
        // short context: split 0 holds every key; its CTA finishes from its own shared memory -- the same sums in the same order as the
        // general path below (warps, then the single split), no scratch round trip, no fence, no counter
        if (split != 0) return;
        if (tid < SPLIT_G) inv_s[tid] = (float) (1.0 / cta_sum(tid));
        __syncthreads();
        const int hA = tid / 8, l0 = 4 * (tid % 8);                          // thread = 8 consecutive outputs of head tid / 8 = lanes l0 .. l0 + 3
        float y[8];
        const float sc = hA < G ? inv_s[hA] : 0.f;
#pragma unroll
        for (int u = 0; u < 4; u++) {
            float2 r = ow[0][hA * 32 + l0 + u];
#pragma unroll
            for (int w = 1; w < SPLIT_WARPS; w++) { r.x += ow[w][hA * 32 + l0 + u].x; r.y += ow[w][hA * 32 + l0 + u].y; }
            y[2 * u] = __fmul_rn(r.x, sc); y[2 * u + 1] = __fmul_rn(r.y, sc);
        }
        split_store(a, y, h0, hA, G, tid, lane);
        return;
    }
    if (nk > 0) {                                                           // the split's partial sums and outputs (splits without keys write none)
        if (tid < G) a.psum[(size_t) (h0 + tid) * SPLIT_MAX + split] = cta_sum(tid);
        for (int i = tid; i < SPLIT_G * 32; i += SPLIT_THREADS) {
            const int h = i / 32, l = i % 32;
            float2 r = ow[0][h * 32 + l];
#pragma unroll
            for (int w = 1; w < SPLIT_WARPS; w++) { r.x += ow[w][h * 32 + l].x; r.y += ow[w][h * 32 + l].y; }
            if (h < G) *reinterpret_cast<float2 *>(a.opart + ((size_t) (split * a.n_head + h0 + h)) * 64 + 2 * l) = r;
        }
    }
    // the last CTA of this (KV head, group) combines the splits
    __threadfence();
    __syncthreads();
    unsigned * ctr = a.ctr + blockIdx.y * gridDim.z + blockIdx.z;
    if (tid == 0) { const unsigned old = atomicAdd(ctr, 1u); s_last = old == (unsigned) ns - 1; if (s_last) *ctr = 0; }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    if (tid < SPLIT_G) {
        double s = 0.0;
        if (tid < G) for (int sp = 0; sp < n_used; sp++) s += __ldcg(a.psum + (size_t) (h0 + tid) * SPLIT_MAX + sp);
        inv_s[tid] = (float) (1.0 / s);
    }
    __syncthreads();
    // 16 x 64 outputs as 256 float4 items, two per thread, every split's partial read once: batches of 8 splits x 2 items in
    // flight (this tail is the fixed cost of the kernel, keep it short)
    const int i0 = 2 * tid, i1 = 2 * tid + 1;                               // float4 items: thread = 8 consecutive outputs of head tid / 8
    float4 r0 = make_float4(0.f, 0.f, 0.f, 0.f), r1 = r0;
    const float * base = a.opart + (size_t) h0 * 64;
    const int hA = tid / 8;
#pragma unroll 1
    for (int sp = 0; sp < n_used; sp += 8) {
        float4 t0[8], t1[8];
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const float * ps = base + (size_t) (sp + u) * a.n_head * 64;
            const bool live = hA < G && sp + u < n_used;                  // partials of splits without keys were never written
            t0[u] = live ? __ldcg(reinterpret_cast<const float4 *>(ps) + i0) : make_float4(0.f, 0.f, 0.f, 0.f);
            t1[u] = live ? __ldcg(reinterpret_cast<const float4 *>(ps) + i1) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < 8; u++) {
            r0.x += t0[u].x; r0.y += t0[u].y; r0.z += t0[u].z; r0.w += t0[u].w;
            r1.x += t1[u].x; r1.y += t1[u].y; r1.z += t1[u].z; r1.w += t1[u].w;
        }
    }
    const float s = hA < G ? inv_s[hA] : 0.f;
    const float y[8] = { __fmul_rn(r0.x, s), __fmul_rn(r0.y, s), __fmul_rn(r0.z, s), __fmul_rn(r0.w, s),
                         __fmul_rn(r1.x, s), __fmul_rn(r1.y, s), __fmul_rn(r1.z, s), __fmul_rn(r1.w, s) };
    split_store(a, y, h0, hA, G, tid, lane);
}

// ---- host side
// Does the frame cover p?  (head groups x KV heads arrival counters must fit the counter block)
static inline bool split_fits(const AttnParams & p) {
    if (p.n_tok != 1 || p.head_dim != 64 || p.n_head % p.n_head_kv) return false;
    return (size_t) p.n_head_kv * ((p.n_head / p.n_head_kv + SPLIT_G - 1) / SPLIT_G) * sizeof(unsigned) <= ATTN_CTR_BYTES;
}
static inline size_t align256(size_t v) { return (v + 255) & ~(size_t) 255; }
// scratch: the counter block, S [n_head][n_ctx], pmax [n_head][SPLIT_MAX], psum [n_head][SPLIT_MAX], opart [SPLIT_MAX][n_head][64].
// Returns the bytes; with a buffer, also points a's arrays into it.
static inline size_t split_layout(const AttnParams & p, float * scratch, SplitArgs * a) {
    const size_t o_S = ATTN_CTR_BYTES, o_pmax = o_S + align256((size_t) p.n_head * p.n_ctx * 4);
    const size_t o_psum = o_pmax + align256((size_t) p.n_head * SPLIT_MAX * 4), o_opart = o_psum + align256((size_t) p.n_head * SPLIT_MAX * 8);
    if (scratch) {
        uint8_t * s = reinterpret_cast<uint8_t *>(scratch);
        a->ctr = reinterpret_cast<unsigned *>(s); a->S = reinterpret_cast<float *>(s + o_S); a->pmax = reinterpret_cast<float *>(s + o_pmax);
        a->psum = reinterpret_cast<double *>(s + o_psum); a->opart = reinterpret_cast<float *>(s + o_opart);
    }
    return o_opart + align256((size_t) SPLIT_MAX * p.n_head * 64 * 4);
}
// the kernels' arguments for p; n_splits and the quantised output are the caller's
static inline SplitArgs split_args(const float * qkv, float * out, const AttnParams & p, float * scratch) {
    SplitArgs a{};
    split_layout(p, scratch, &a);
    a.qkv = qkv; a.out = out; a.kv = p.kv;
    a.n_head = p.n_head; a.n_head_kv = p.n_head_kv; a.G = p.n_head / p.n_head_kv; a.n_past = p.n_past; a.n_past_dev = p.n_past_dev; a.n_ctx = p.n_ctx;
    a.qkv_stride = p.qkv_stride;
    a.fuse_rope = p.fuse_rope; a.theta_scale = p.rope_theta_scale;
    return a;
}
// scores, then values launched programmatically behind it (it may take the scores kernel's place on the SMs before that grid ends)
static inline void split_launch(void (*scores)(SplitArgs), void (*values)(SplitArgs), SplitArgs a, size_t values_smem, cudaStream_t stream) {
    const dim3 grid((unsigned) a.n_splits, (unsigned) a.n_head_kv, (unsigned) ((a.G + SPLIT_G - 1) / SPLIT_G));
    scores<<<grid, SPLIT_THREADS, 0, stream>>>(a);
    B200_CUDA_CHECK(cudaGetLastError());
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = dim3(SPLIT_THREADS); cfg.dynamicSmemBytes = values_smem; cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    B200_CUDA_CHECK(cudaLaunchKernelEx(&cfg, values, a));
}
