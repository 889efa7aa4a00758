// attention.cu -- multi-query / grouped-query attention over the f32 KV cache.
//
// Restates, as ONE kernel per layer, the seven graph nodes the reference pins to the CPU
// (libfalcon.cpp:2285-2366: K view/permute, mul_mat(K,Q) with cuda_op_directive=0, scale, diag_mask_inf, soft_max,
// mul_mat(V,P), permute+cpy) with the CPU numerics (SURVEY.md section 9.2):
//   s[p]  = (q . k_p) * (1/sqrt(head_dim))                           ggml.c:10911-11102, libfalcon.cpp:2313-2317
//   mask  : p > n_past + t  ->  -inf                                 ggml.c:12342-12348
//   e[p]  = f16->f32(LUT_exp[f32->f16(s[p] - max)]), sum in double, y = e * (float)(1/sum)     ggml.c:12427-12449
//   out   = sum_p V[p] * y[p]
// GQA head -> kv head map is the f32 mat-mul's  h / (n_head / n_head_kv)  (ggml.c:11074).
//
// KV cache layout on the device: K and V both [n_ctx][n_head_kv][head_dim] f32 per layer (the reference's K layout,
// libfalcon.cpp:2238-2242; its transposed, ping-ponged V copy with the O(n_past) re-copy per token,
// libfalcon.cpp:2256-2281, is replaced by a plain append -- values are identical).
//
// v1 kernel: one CTA per (query head, query token); scores live in shared memory (T floats).  Exact oracle
// semantics (global max before exp).  Fine for decode; prompts go through attention_ws.cu.
#include "kernels.h"
#include "actquant.cuh"

#define ATT_THREADS 128

__device__ __forceinline__ float exp_f16lut(float v) {      // table_exp_f16[f16(v)], ggml.c:4281-4290
    return __half2float(__float2half_rn(expf(__half2float(__float2half_rn(v)))));
}

__global__ void __launch_bounds__(ATT_THREADS) attention_kernel(const float * __restrict__ qkv, const float * __restrict__ kc, const float * __restrict__ vc,
                                                               float * __restrict__ out, int64_t out_stride, AttnParams p) {
    extern __shared__ __align__(16) float sm[];
    trace_begin(p.trace);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // wo's mat-vec may start prefetching its weights
    const int h = blockIdx.x, t = blockIdx.y, D = p.head_dim;
    const int n_past = p.n_past_dev ? *p.n_past_dev : p.n_past;
    const int T = n_past + t + 1;                            // keys visible to this query (causal)
    const int kvh = h / (p.n_head / p.n_head_kv);
    float * q = sm;                                          // [D]
    float * s = sm + D;                                      // [T]
    __shared__ float red_f[ATT_THREADS / 32];
    __shared__ double red_d[ATT_THREADS / 32];
    __shared__ float part[ATT_THREADS];

    for (int i = threadIdx.x; i < D; i += ATT_THREADS) q[i] = qkv[(size_t) t * p.qkv_stride + (size_t) h * D + i];
    __syncthreads();
    const float scale = 1.0f / sqrtf((float) D);
    const size_t kv_row = (size_t) p.n_head_kv * D;

    // scores: one thread per key, 16-byte loads along the head dimension
    float lmax = -INFINITY;
    for (int k = threadIdx.x; k < T; k += ATT_THREADS) {
        const float4 * kr = reinterpret_cast<const float4 *>(kc + (size_t) k * kv_row + (size_t) kvh * D);
        float acc = 0.f;
        for (int i = 0; i < D / 4; i++) {
            const float4 kv = kr[i];
            acc += kv.x * q[4 * i] + kv.y * q[4 * i + 1] + kv.z * q[4 * i + 2] + kv.w * q[4 * i + 3];
        }
        acc = __fmul_rn(acc, scale);
        s[k] = acc;
        lmax = fmaxf(lmax, acc);
    }
    lmax = warp_max(lmax);
    if ((threadIdx.x & 31) == 0) red_f[threadIdx.x >> 5] = lmax;
    __syncthreads();
    float gmax = red_f[0];
    for (int w = 1; w < ATT_THREADS / 32; w++) gmax = fmaxf(gmax, red_f[w]);

    double lsum = 0.0;
    for (int k = threadIdx.x; k < T; k += ATT_THREADS) { const float e = exp_f16lut(__fsub_rn(s[k], gmax)); s[k] = e; lsum += (double) e; }
    lsum = warp_sum_d(lsum);
    if ((threadIdx.x & 31) == 0) red_d[threadIdx.x >> 5] = lsum;
    __syncthreads();
    double gsum = 0.0;
    for (int w = 0; w < ATT_THREADS / 32; w++) gsum += red_d[w];
    const float inv = (float) (1.0 / gsum);

    // out[i] = sum_k V[k][i] * (e[k] * inv): thread = (key parity group, dim) so that a warp reads 128 contiguous bytes of V
    const int i = threadIdx.x % D, grp = threadIdx.x / D, ngrp = ATT_THREADS / D;     // D = 64 -> 2 groups
    float acc = 0.f;
    for (int k = grp; k < T; k += ngrp) acc += vc[(size_t) k * kv_row + (size_t) kvh * D + i] * __fmul_rn(s[k], inv);
    part[threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.x < D) {
        float r = part[threadIdx.x];
        for (int g = 1; g < ngrp; g++) r += part[g * D + threadIdx.x];
        out[(size_t) t * out_stride + (size_t) h * D + threadIdx.x] = r;
    }
    trace_end(p.trace);
}

// ------------------------------------------------------------------------------------------------------------------
// Split-KV decode attention (n_tok == 1, head_dim 64).  The kernel above walks a head's keys with one 128-thread CTA and
// re-reads the KV head's K / V once per query head: fine at 100 keys, far too slow at thousands
// (tools/ctx_decode.py shows the decode rate against the context position).  Here the G query heads of a KV head are processed TOGETHER (K / V are read
// once per KV head) and the keys are split over AT_SPLITS CTAs per KV head:
//   kernel 1 (scores): a warp takes one key per step, lane l holds dims 2l, 2l+1 of the key (one coalesced 256-byte row) and
//                      of the G <= 16 query vectors; G partial dots per lane are reduced with a transposing butterfly
//                      (16 shuffles); s = dot * scale goes to the scratch row S[head][key], per-(head, split) maxima on the side
//   kernel 2 (values) : gmax = max over splits; e = LUT(s - gmax) for the CTA's own keys (shared memory, [key][head]),
//                      their sum in double per (head, split); O_partial[head][d] += V[key][d] * e (lane = 2 dims, G heads
//                      in registers); the LAST CTA of a KV head sums the partial sums and outputs in split order and scales by
//                      (float)(1 / sum)  -- ggml.c:12427-12449 multiplies each e by that factor before the product with V;
//                      scaling the product instead is a reassociation-level difference (as the tensor-core prompt kernel does).
// Both kernels read n_past from a device scalar, so the captured decode graph serves every position.
#define AD_THREADS 128                   // small CTAs at <= 85 registers: one fits beside ffn_up's two 256-thread CTAs on every SM
#define AD_WARPS (AD_THREADS / 32)
#define AD_SPLITS 32
#define AD_B 4                           // key rows per warp step (plus the same number in flight for the next step)
#define AD_G 16                          // query heads per KV head handled together (n_head / n_head_kv <= 16)

struct AttnDecArgs {
    const float * qkv; const float * kc; const float * vc; float * out;
    float * S; float * pmax; double * psum; float * opart; unsigned * ctr;
    int n_head, n_head_kv, G, n_past; const int * n_past_dev; int n_ctx; int64_t qkv_stride;
    unsigned long long * trace;
    ActQ qA; int has_q;          // optional quantised copy of the output row (see AttnParams::qout)
    int fuse_rope; float theta_scale; float * kc_w; float * vc_w; __half * k16; __half * vt16; int ctx_pad;     // see AttnParams::fuse_rope
};

// 16 per-lane values -> lane l ends up with the warp total of value (l >> 1)
__device__ __forceinline__ float butterfly16(float (&v)[16], int lane) {
    float w8[8], w4[4], w2[2];
    const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4, b1 = lane & 2;
#pragma unroll
    for (int i = 0; i < 8; i++) { const float keep = b4 ? v[8 + i] : v[i], send = b4 ? v[i] : v[8 + i]; w8[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16); }
#pragma unroll
    for (int i = 0; i < 4; i++) { const float keep = b3 ? w8[4 + i] : w8[i], send = b3 ? w8[i] : w8[4 + i]; w4[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8); }
#pragma unroll
    for (int i = 0; i < 2; i++) { const float keep = b2 ? w4[2 + i] : w4[i], send = b2 ? w4[i] : w4[2 + i]; w2[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4); }
    const float keep = b1 ? w2[1] : w2[0], send = b1 ? w2[0] : w2[1];
    float r = keep + __shfl_xor_sync(0xffffffffu, send, 2);
    r += __shfl_xor_sync(0xffffffffu, r, 1);
    return r;
}
// keys per split: at least AD_MIN_KEYS, so that a short context occupies few CTAs and the combine step reads few partials (at
// n_past < 64 one CTA per KV-head group does everything; the other CTAs of the fixed grid only check in at the counter)
#define AD_MIN_KEYS 64
__device__ __forceinline__ int split_keys(int T) { return max(AD_MIN_KEYS, (T + AD_SPLITS - 1) / AD_SPLITS); }
__device__ __forceinline__ int splits_used(int T) { const int per = split_keys(T); return (T + per - 1) / per; }
__device__ __forceinline__ void split_range(int T, int split, int & k_lo, int & k_hi) {
    const int per = split_keys(T);
    k_lo = min(T, split * per); k_hi = min(T, k_lo + per);
}

__global__ void __launch_bounds__(AD_THREADS, 6) attn_dec_scores_kernel(const AttnDecArgs a) {
    __shared__ float wmax[AD_WARPS][AD_G];
    trace_begin(a.trace);
    const int split = blockIdx.x, kvh = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int h0 = kvh * a.G + blockIdx.z * AD_G, G = min(AD_G, a.G - (int) blockIdx.z * AD_G);      // this CTA's query heads: h0 .. h0 + G - 1
    const int n_past = a.n_past_dev ? *a.n_past_dev : a.n_past, T = n_past + 1;
    int k_lo, k_hi; split_range(T, split, k_lo, k_hi);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // the values kernel may take its place on the SMs now (it waits for this grid to finish)
    // the query rows do not depend on n_past: their loads are in flight while the device scalar arrives (every dependent round trip
    // counts here: beside ffn_up's streaming each one takes > 1 us, and at short contexts this kernel is nothing but such a chain)
    float2 q[AD_G];
#pragma unroll
    for (int h = 0; h < AD_G; h++)
        q[h] = h < G ? *reinterpret_cast<const float2 *>(a.qkv + (size_t) (h0 + h) * 64 + 2 * lane) : make_float2(0.f, 0.f);
    if (k_lo >= k_hi) { trace_end(a.trace); return; }            // a split without keys (short context): nothing to score, nobody reads its pmax
    const float scale = 1.0f / sqrtf(64.0f);
    const size_t kv_row = (size_t) a.n_head_kv * 64;
    // Fused RoPE + KV append (libfalcon.cpp:2229-2281).  A lane holds elements (2l, 2l+1) of a head; NeoX pairs element i < 32 with i + 32,
    // i.e. with the same component of lane l ^ 16.  Angles as rope_pair (ops.cu): theta = n_past * theta_scale^i by repeated fp32 products.
    float2 knew = make_float2(0.f, 0.f);
    if (a.fuse_rope) {
        const int i0 = (2 * lane) & 31;
        float th0 = (float) n_past;
        for (int k = 0; k < i0; k++) th0 = __fmul_rn(th0, a.theta_scale);
        const float th1 = __fmul_rn(th0, a.theta_scale);
        const float c0 = cosf(th0), s0 = sinf(th0), c1 = cosf(th1), s1 = sinf(th1);
        auto rot = [&](float2 v) {
            const float ox = __shfl_xor_sync(0xffffffffu, v.x, 16), oy = __shfl_xor_sync(0xffffffffu, v.y, 16);
            return lane < 16 ? make_float2(__fsub_rn(__fmul_rn(v.x, c0), __fmul_rn(ox, s0)), __fsub_rn(__fmul_rn(v.y, c1), __fmul_rn(oy, s1)))     // x0 c - x1 s
                             : make_float2(__fadd_rn(__fmul_rn(ox, s0), __fmul_rn(v.x, c0)), __fadd_rn(__fmul_rn(oy, s1), __fmul_rn(v.y, c1)));    // x0 s + x1 c
        };
#pragma unroll
        for (int h = 0; h < AD_G; h++) q[h] = rot(q[h]);
        knew = rot(*reinterpret_cast<const float2 *>(a.qkv + (size_t) (a.n_head + kvh) * 64 + 2 * lane));        // this position's key row, rotated
        if (blockIdx.z == 0 && warp == 0 && n_past >= k_lo && n_past < k_hi) {                                     // one warp appends K and V to the cache
            const size_t o = ((size_t) n_past * a.n_head_kv + kvh) * 64 + 2 * lane;
            const float2 vnew = *reinterpret_cast<const float2 *>(a.qkv + (size_t) (a.n_head + a.n_head_kv + kvh) * 64 + 2 * lane);
            *reinterpret_cast<float2 *>(a.kc_w + o) = knew;
            *reinterpret_cast<float2 *>(a.vc_w + o) = vnew;
            if (a.k16) {
                *reinterpret_cast<__half2 *>(a.k16 + o) = __floats2half2_rn(knew.x, knew.y);
                __half * vt = a.vt16 + ((size_t) kvh * 64 + 2 * lane) * a.ctx_pad + n_past;
                vt[0] = __float2half_rn(vnew.x); vt[a.ctx_pad] = __float2half_rn(vnew.y);
            }
        }
    }
    const int hh = lane >> 1;                                     // the head whose total this lane receives
    float lmax = -INFINITY;
    const float * kp = a.kc + (size_t) kvh * 64 + 2 * lane;
    // AD_B keys per warp and step, the next batch's rows already in flight (memory-level parallelism without more warps)
    float2 cur[AD_B], nxt[AD_B];
    const int k_new = a.fuse_rope ? n_past : -1;                 // this key is not in the cache yet (another CTA may be writing it right now): use the registers
    auto ld_key = [&](int kk) { return kk >= k_hi ? make_float2(0.f, 0.f) : kk == k_new ? knew : __ldg(reinterpret_cast<const float2 *>(kp + (size_t) kk * kv_row)); };
#pragma unroll
    for (int b = 0; b < AD_B; b++) cur[b] = ld_key(k_lo + warp + b * AD_WARPS);
    for (int k = k_lo + warp; k < k_hi; k += AD_B * AD_WARPS) {
#pragma unroll
        for (int b = 0; b < AD_B; b++) nxt[b] = ld_key(k + (AD_B + b) * AD_WARPS);
#pragma unroll
        for (int b = 0; b < AD_B; b++) {
            const int kk = k + b * AD_WARPS;
            float part[AD_G];
#pragma unroll
            for (int h = 0; h < AD_G; h++) part[h] = cur[b].x * q[h].x + cur[b].y * q[h].y;
            const float s = __fmul_rn(butterfly16(part, lane), scale);   // libfalcon.cpp:2313-2317
            if (hh < G && kk < k_hi) {
                if ((lane & 1) == 0) a.S[(size_t) (h0 + hh) * a.n_ctx + kk] = s;
                lmax = fmaxf(lmax, s);
            }
        }
#pragma unroll
        for (int b = 0; b < AD_B; b++) cur[b] = nxt[b];
    }
    if ((lane & 1) == 0 && hh < AD_G) wmax[warp][hh] = lmax;
    __syncthreads();
    if (threadIdx.x < G) {
        float mx = wmax[0][threadIdx.x];
#pragma unroll
        for (int w = 1; w < AD_WARPS; w++) mx = fmaxf(mx, wmax[w][threadIdx.x]);
        a.pmax[(size_t) (h0 + threadIdx.x) * AD_SPLITS + split] = mx;
    }
    trace_end(a.trace);
}

// thread tid's 8 consecutive outputs (head hA of the CTA's group) -> the attention output row, plus wo's activation quantisation
__device__ __forceinline__ void attn_dec_store(const AttnDecArgs & a, const float (&y)[8], int h0, int hA, int G, int tid, int lane) {
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

__global__ void __launch_bounds__(AD_THREADS, 6) attn_dec_values_kernel(const AttnDecArgs a, const int per_max) {
    extern __shared__ __align__(16) float sm_dyn[];                // es[per_max][AD_G]
    __shared__ float gmax[AD_G];
    __shared__ double dsum[AD_THREADS / AD_G][AD_G];
    __shared__ float2 oacc[AD_WARPS][AD_G][32];                    // per-warp partial outputs: [head][lane] = dims 2l, 2l+1
    __shared__ float inv_s[AD_G];
    __shared__ int s_last;
    float * es = sm_dyn;
    const int split = blockIdx.x, kvh = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int h0 = kvh * a.G + blockIdx.z * AD_G, G = min(AD_G, a.G - (int) blockIdx.z * AD_G);
    const int n_past = a.n_past_dev ? *a.n_past_dev : a.n_past, T = n_past + 1;
    int k_lo, k_hi; split_range(T, split, k_lo, k_hi);
    const int nk = k_hi - k_lo;
    const size_t kv_row = (size_t) a.n_head_kv * 64;
    trace_begin(a.trace);
    const int n_used = splits_used(T);                            // splits 0 .. n_used - 1 hold keys
    // V rows of EARLIER positions have been in the cache since their own decode steps: the first batch is fetched while the scores kernel
    // still runs (this position's row is appended by that kernel: loaded after the wait)
    const float * vp = a.vc + (size_t) kvh * 64 + 2 * lane;
    float2 cur[AD_B], nxt[AD_B];
#pragma unroll
    for (int b = 0; b < AD_B; b++) { const int jj = warp + b * AD_WARPS; cur[b] = jj < nk && k_lo + jj < n_past ? __ldg(reinterpret_cast<const float2 *>(vp + (size_t) (k_lo + jj) * kv_row)) : make_float2(0.f, 0.f); }
    asm volatile("griddepcontrol.wait;" ::: "memory");            // launched programmatically behind the scores kernel: its S / pmax / KV append are complete from here on
    if (nk > 0) {
    // the scores of the CTA's first AD_SPRE keys per thread are requested together with the split maxima (one round trip instead of two)
    constexpr int AD_SPRE = 8;
    const int eh = tid % AD_G, ej = tid / AD_G;
    const float * Sr = a.S + (size_t) (h0 + min(eh, G - 1)) * a.n_ctx + k_lo;
    float spre[AD_SPRE];
#pragma unroll
    for (int i = 0; i < AD_SPRE; i++) { const int j = ej + i * (AD_THREADS / AD_G); spre[i] = j < nk ? __ldcg(Sr + j) : 0.f; }
#pragma unroll
    for (int b = 0; b < AD_B; b++) { const int jj = warp + b * AD_WARPS; if (jj < nk && k_lo + jj >= n_past) cur[b] = *reinterpret_cast<const float2 *>(vp + (size_t) (k_lo + jj) * kv_row); }
    if (tid < AD_G) {
        float mx = -INFINITY;
        if (tid < G) for (int s = 0; s < n_used; s++) mx = fmaxf(mx, a.pmax[(size_t) (h0 + tid) * AD_SPLITS + s]);
        gmax[tid] = mx;
    }
    __syncthreads();
    // e = table_exp_f16[f16(s - max)] (ggml.c:12427-12440) for the CTA's keys, sums in double
    {
        double s = 0.0;
        if (eh < G) {
            const float gm = gmax[eh];
#pragma unroll
            for (int i = 0; i < AD_SPRE; i++) {
                const int j = ej + i * (AD_THREADS / AD_G);
                if (j < nk) { const float e = exp_f16lut(__fsub_rn(spre[i], gm)); es[j * AD_G + eh] = e; s += (double) e; }
            }
            for (int j = ej + AD_SPRE * (AD_THREADS / AD_G); j < nk; j += AD_THREADS / AD_G) {
                const float e = exp_f16lut(__fsub_rn(__ldcg(Sr + j), gm));
                es[j * AD_G + eh] = e; s += (double) e;
            }
        } else for (int j = ej; j < nk; j += AD_THREADS / AD_G) es[j * AD_G + eh] = 0.f;
        dsum[ej][eh] = s;
    }
    __syncthreads();
    if (tid < G && n_used > 1) {
        double s = 0.0;
#pragma unroll
        for (int r = 0; r < AD_THREADS / AD_G; r++) s += dsum[r][tid];
        a.psum[(size_t) (h0 + tid) * AD_SPLITS + split] = s;
    }
    // O_partial[h][2l..2l+1] = sum over the warp's keys of V[key][2l..2l+1] * e[key][h]
    float2 acc[AD_G];
#pragma unroll
    for (int h = 0; h < AD_G; h++) acc[h] = make_float2(0.f, 0.f);
    for (int j = warp; j < nk; j += AD_B * AD_WARPS) {
#pragma unroll
        for (int b = 0; b < AD_B; b++) { const int jj = j + (AD_B + b) * AD_WARPS; nxt[b] = jj < nk ? __ldg(reinterpret_cast<const float2 *>(vp + (size_t) (k_lo + jj) * kv_row)) : make_float2(0.f, 0.f); }
#pragma unroll
        for (int b = 0; b < AD_B; b++) {
            const int jj = j + b * AD_WARPS;
            if (jj < nk) {                                                    // warp-uniform
                const float4 * er = reinterpret_cast<const float4 *>(es + jj * AD_G);
                const float2 vv = cur[b];
#pragma unroll
                for (int c = 0; c < AD_G / 4; c++) {
                    const float4 e = er[c];
                    acc[4 * c].x += vv.x * e.x;     acc[4 * c].y += vv.y * e.x;
                    acc[4 * c + 1].x += vv.x * e.y; acc[4 * c + 1].y += vv.y * e.y;
                    acc[4 * c + 2].x += vv.x * e.z; acc[4 * c + 2].y += vv.y * e.z;
                    acc[4 * c + 3].x += vv.x * e.w; acc[4 * c + 3].y += vv.y * e.w;
                }
            }
        }
#pragma unroll
        for (int b = 0; b < AD_B; b++) cur[b] = nxt[b];
    }
#pragma unroll
    for (int h = 0; h < AD_G; h++) oacc[warp][h][lane] = acc[h];
    __syncthreads();
    if (n_used > 1)
    for (int i = tid; i < AD_G * 32; i += AD_THREADS) {             // fixed warp order: deterministic
        const int h = i / 32, l = i % 32;
        float2 r = oacc[0][h][l];
#pragma unroll
        for (int w = 1; w < AD_WARPS; w++) { r.x += oacc[w][h][l].x; r.y += oacc[w][h][l].y; }
        if (h < G) *reinterpret_cast<float2 *>(a.opart + ((size_t) (split * a.n_head + h0 + h)) * 64 + 2 * l) = r;
    }
    }   // nk > 0
    if (n_used == 1) {
        // short context: split 0 holds every key; its CTA finishes from its own shared memory -- the same sums in the same order as the
        // general path below (warps, then the single split), no scratch round trip, no fence, no counter
        if (split != 0) { trace_end(a.trace); return; }
        if (tid < AD_G) {
            double s = 0.0;
#pragma unroll
            for (int r = 0; r < AD_THREADS / AD_G; r++) s += dsum[r][tid];
            inv_s[tid] = (float) (1.0 / s);
        }
        __syncthreads();
        const int hA = tid / 8, l0 = 4 * (tid % 8);                          // thread = 8 consecutive outputs of head tid / 8 = lanes l0 .. l0 + 3 of oacc
        float y[8];
        const float sc = hA < G ? inv_s[hA] : 0.f;
#pragma unroll
        for (int u = 0; u < 4; u++) {
            float2 r = oacc[0][hA][l0 + u];
#pragma unroll
            for (int w = 1; w < AD_WARPS; w++) { r.x += oacc[w][hA][l0 + u].x; r.y += oacc[w][hA][l0 + u].y; }
            y[2 * u] = __fmul_rn(r.x, sc); y[2 * u + 1] = __fmul_rn(r.y, sc);
        }
        attn_dec_store(a, y, h0, hA, G, tid, lane);
        trace_end(a.trace);
        return;
    } else {
    // the last CTA of this KV head combines the splits
    __threadfence();
    __syncthreads();
    unsigned * ctr = a.ctr + kvh * gridDim.z + blockIdx.z;
    if (tid == 0) { const unsigned old = atomicAdd(ctr, 1u); s_last = old == AD_SPLITS - 1; if (s_last) *ctr = 0; }
    __syncthreads();
    if (!s_last) { trace_end(a.trace); return; }
    __threadfence();
    }
    if (tid < AD_G) {
        double s = 0.0;
        if (tid < G) for (int sp = 0; sp < n_used; sp++) s += __ldcg(a.psum + (size_t) (h0 + tid) * AD_SPLITS + sp);
        inv_s[tid] = (float) (1.0 / s);
    }
    __syncthreads();
    // 16 x 64 outputs as 256 float4 items, two per thread, every split's partial read once: batches of 8 splits x 2 items in
    // flight (this tail is the fixed cost of the kernel, keep it short)
    {
        const int i0 = 2 * tid, i1 = 2 * tid + 1;                           // float4 items: thread = 8 consecutive outputs of head tid / 8
        float4 r0 = make_float4(0.f, 0.f, 0.f, 0.f), r1 = r0;
        const float * base = a.opart + (size_t) h0 * 64;
        const int hA = tid / 8;
#pragma unroll 1
        for (int sp = 0; sp < n_used; sp += 8) {
            float4 t0[8], t1[8];
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const float * ps = base + (size_t) (sp + u) * a.n_head * 64;
                const bool live = hA < G && sp + u < n_used;              // partials of splits without keys were never written
                t0[u] = live ? __ldcg(reinterpret_cast<const float4 *>(ps) + i0) : make_float4(0.f, 0.f, 0.f, 0.f);
                t1[u] = live ? __ldcg(reinterpret_cast<const float4 *>(ps) + i1) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int u = 0; u < 8; u++) {                                   // fixed split order: deterministic
                r0.x += t0[u].x; r0.y += t0[u].y; r0.z += t0[u].z; r0.w += t0[u].w;
                r1.x += t1[u].x; r1.y += t1[u].y; r1.z += t1[u].z; r1.w += t1[u].w;
            }
        }
        const float s = hA < G ? inv_s[hA] : 0.f;
        const float y[8] = { __fmul_rn(r0.x, s), __fmul_rn(r0.y, s), __fmul_rn(r0.z, s), __fmul_rn(r0.w, s),
                             __fmul_rn(r1.x, s), __fmul_rn(r1.y, s), __fmul_rn(r1.z, s), __fmul_rn(r1.w, s) };
        attn_dec_store(a, y, h0, hA, G, tid, lane);
    }
    trace_end(a.trace);
}

static size_t align256(size_t v) { return (v + 255) & ~(size_t) 255; }
#define AD_CTR_BYTES 4096                 // arrival counters at the START of the scratch block (n_head_kv * head groups <= 1024)
size_t attention_scratch_bytes(const AttnParams & p) {
    if (p.n_tok != 1 || p.head_dim != 64) return 0;
    return AD_CTR_BYTES + align256((size_t) p.n_head * p.n_ctx * 4) + align256((size_t) p.n_head * AD_SPLITS * 4) + align256((size_t) p.n_head * AD_SPLITS * 8) +
           align256((size_t) AD_SPLITS * p.n_head * 64 * 4);
}
// scratch: attention_scratch_bytes(p) bytes whose first AD_CTR_BYTES were zeroed once by the owner (the counters re-arm themselves)
static bool launch_attention_split(const float * qkv, const float * k_cache, const float * v_cache, float * out, const AttnParams & p, float * scratch, cudaStream_t stream) {
    if (!scratch || p.n_tok != 1 || p.head_dim != 64 || p.n_head % p.n_head_kv || getenv("B200_ATTN_NOSPLIT")) return false;
    const int G = p.n_head / p.n_head_kv, groups = (G + AD_G - 1) / AD_G;
    if ((size_t) p.n_head_kv * groups * 4 > AD_CTR_BYTES) return false;
    const int per_max = max(AD_MIN_KEYS, (p.n_ctx + AD_SPLITS - 1) / AD_SPLITS);
    const size_t smem = (size_t) per_max * AD_G * 4;
    if (smem > 160 * 1024) return false;
    AttnDecArgs a;
    uint8_t * s = reinterpret_cast<uint8_t *>(scratch);
    a.ctr = reinterpret_cast<unsigned *>(s); s += AD_CTR_BYTES;
    a.S = reinterpret_cast<float *>(s); s += align256((size_t) p.n_head * p.n_ctx * 4);
    a.pmax = reinterpret_cast<float *>(s); s += align256((size_t) p.n_head * AD_SPLITS * 4);
    a.psum = reinterpret_cast<double *>(s); s += align256((size_t) p.n_head * AD_SPLITS * 8);
    a.opart = reinterpret_cast<float *>(s);
    a.qkv = qkv; a.kc = k_cache; a.vc = v_cache; a.out = out;
    a.n_head = p.n_head; a.n_head_kv = p.n_head_kv; a.G = p.n_head / p.n_head_kv; a.n_past = p.n_past; a.n_past_dev = p.n_past_dev; a.n_ctx = p.n_ctx;
    a.qkv_stride = p.qkv_stride;
    a.fuse_rope = p.fuse_rope; a.theta_scale = p.rope_theta_scale; a.kc_w = const_cast<float *>(k_cache); a.vc_w = const_cast<float *>(v_cache);
    a.k16 = p.k16; a.vt16 = p.vt16; a.ctx_pad = attention_ctx_pad(p.n_ctx);
    // Q8_K blocks are 256 outputs = 4 heads: they must not straddle the 16-head groups the CTAs combine
    a.has_q = p.qout != nullptr && (p.qout->type != T_Q8_K || G % 4 == 0);
    if (a.has_q) a.qA = *p.qout;
    B200_ASSERT(p.qout == nullptr || a.has_q);
    static bool set = false;
    if (!set) {
        B200_CUDA_CHECK(cudaFuncSetAttribute(attn_dec_values_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
        B200_CUDA_CHECK(cudaFuncSetAttribute(attn_dec_scores_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, B200_CARVEOUT));
        B200_CUDA_CHECK(cudaFuncSetAttribute(attn_dec_values_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, B200_CARVEOUT));
        set = true;
    }
    dim3 grid(AD_SPLITS, (unsigned) p.n_head_kv, (unsigned) groups);
    a.trace = b200_trace_slot("attn_scores");
    attn_dec_scores_kernel<<<grid, AD_THREADS, 0, stream>>>(a);
    B200_CUDA_CHECK(cudaGetLastError());
    a.trace = b200_trace_slot("attn_values");
    {
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = grid; cfg.blockDim = dim3(AD_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr; cfg.numAttrs = getenv("B200_NO_PDL") ? 0 : 1;
        B200_CUDA_CHECK(cudaLaunchKernelEx(&cfg, attn_dec_values_kernel, a, per_max));
    }
    return true;
}

bool launch_attention_long(const float * qkv, const float * k_cache, const float * v_cache, float * out, const AttnParams & p, float * scratch, cudaStream_t stream);   // attention_long.cu
int attention_long_threshold() {             // read on every call (graph builds and eager launches only): tests move it
    const char * e = getenv("B200_ATTN_LONG_FROM");
    return e ? atoi(e) : 1024;
}

// returns the number of kernels launched
int launch_attention(const float * qkv, const float * k_cache, const float * v_cache, float * out, int64_t out_stride,
                      const AttnParams & p, float * scratch, cudaStream_t stream) {
    if (p.n_tok <= 0) return 0;
    // long contexts: one-wave tensor-core kernels with cp.async rings (measured crossover, see attention_long.cu)
    const bool long_ctx = p.n_past_dev ? p.long_ctx != 0 : p.n_past + 1 > attention_long_threshold();
    if (long_ctx && launch_attention_long(qkv, k_cache, v_cache, out, p, scratch, stream)) return 2;
    if (launch_attention_split(qkv, k_cache, v_cache, out, p, scratch, stream)) return 2;
    if (p.fuse_rope) {                                         // fallback kernel: RoPE + append in their own kernel, in place, as before
        AttnParams pr = p; pr.fuse_rope = 0;
        launch_rope_kv_append(const_cast<float *>(qkv), const_cast<float *>(k_cache), const_cast<float *>(v_cache), pr, p.rope_theta_scale, stream);
    }
    B200_ASSERT(p.qout == nullptr && "attention: a quantised output copy needs the split-KV kernels");
    B200_ASSERT(p.head_dim % 4 == 0 && ATT_THREADS % p.head_dim == 0);
    // shared memory is sized for the worst case so that a captured graph stays valid while n_past grows
    const int t_max = p.n_past_dev ? p.n_ctx : p.n_past + p.n_tok;
    const size_t smem = (size_t) (p.head_dim + t_max) * sizeof(float);
    static bool set = false;
    if (!set) { B200_CUDA_CHECK(cudaFuncSetAttribute(attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        B200_CUDA_CHECK(cudaFuncSetAttribute(attention_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, B200_CARVEOUT)); set = true; }
    B200_ASSERT(smem <= 200 * 1024);
    dim3 grid((unsigned) p.n_head, (unsigned) p.n_tok);
    AttnParams pt = p; pt.trace = b200_trace_slot("attention");
    attention_kernel<<<grid, ATT_THREADS, smem, stream>>>(qkv, k_cache, v_cache, out, out_stride, pt);
    B200_CUDA_CHECK(cudaGetLastError());
    return p.fuse_rope ? 2 : 1;
}
