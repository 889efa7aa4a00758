// attention.cu -- multi-query / grouped-query attention over the f32 KV cache, and launch_attention, which picks the kernel for every
// call.
//
// Restates the seven graph nodes the reference pins to the CPU (libfalcon.cpp:2285-2366: K view/permute, mul_mat(K,Q) with
// cuda_op_directive=0, scale, diag_mask_inf, soft_max, mul_mat(V,P), permute+cpy) with the CPU numerics (SURVEY.md section 9.2):
//   s[p]  = (q . k_p) * (1/sqrt(head_dim))                           ggml.c:10911-11102, libfalcon.cpp:2313-2317
//   mask  : p > n_past + t  ->  -inf                                 ggml.c:12342-12348
//   e[p]  = f16->f32(LUT_exp[f32->f16(s[p] - max)]), sum in double, y = e * (float)(1/sum)     ggml.c:12427-12449
//   out   = sum_p V[p] * y[p]
// GQA head -> kv head map is the f32 mat-mul's  h / (n_head / n_head_kv)  (ggml.c:11074).
//
// KV cache layout on the device: K and V both [n_ctx][n_head_kv][head_dim] f32 per layer (the reference's K layout,
// libfalcon.cpp:2238-2242; its transposed, ping-ponged V copy with the O(n_past) re-copy per token,
// libfalcon.cpp:2256-2281, is replaced by a plain append -- values are identical), or fp16 in the same layout: every kernel reads the
// layer's KvCache (kernels.h) as a template on its element type E, widens what it loads and otherwise runs the same arithmetic.
//
// Kernels: decode (one token) on the split-KV frame of attn_split.cuh, this file's CUDA-core tier up to attention_long_threshold()
// keys and attention_long.cu's tensor-core tier above; attention_kernel below where that frame does not apply (head_dim != 64) or
// B200_ATTN_NOSPLIT turns the short tier off.  Prompts: attention_ws.cu (wgmma over the fp16 KV shadow), else attention_prefill.cu.
#include "attn_split.cuh"

#define ATT_THREADS 128

// one CTA per query head of the one new token; scores live in shared memory (T floats).  Exact oracle semantics (global max before exp).
template <typename E>
__global__ void __launch_bounds__(ATT_THREADS) attention_kernel(const float * __restrict__ qkv, float * __restrict__ out, AttnParams p) {
    extern __shared__ __align__(16) float sm[];
    const E * __restrict__ kc = kv_k<E>(p.kv), * __restrict__ vc = kv_v<E>(p.kv);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // wo's mat-vec may start prefetching its weights
    const int h = blockIdx.x, D = p.head_dim;
    const int n_past = p.n_past_dev ? *p.n_past_dev : p.n_past;
    const int T = n_past + 1;                                // keys visible to the query (causal)
    const int kvh = h / (p.n_head / p.n_head_kv);
    float * q = sm;                                          // [D]
    float * s = sm + D;                                      // [T]
    __shared__ float red_f[ATT_THREADS / 32];
    __shared__ double red_d[ATT_THREADS / 32];
    __shared__ float part[ATT_THREADS];

    for (int i = threadIdx.x; i < D; i += ATT_THREADS) q[i] = qkv[(size_t) h * D + i];
    __syncthreads();
    const float scale = 1.0f / sqrtf((float) D);
    const size_t kv_row = (size_t) p.n_head_kv * D;

    // scores: one thread per key, 16-byte loads along the head dimension
    float lmax = -INFINITY;
    for (int k = threadIdx.x; k < T; k += ATT_THREADS) {
        const E * kr = kc + (size_t) k * kv_row + (size_t) kvh * D;
        float acc = 0.f;
        for (int i = 0; i < D / 4; i++) {
            const float4 kv = kv_ld4(kr, i);
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
    for (int k = grp; k < T; k += ngrp) acc += kv_ld(vc + (size_t) k * kv_row + (size_t) kvh * D + i) * __fmul_rn(s[k], inv);
    part[threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.x < D) {
        float r = part[threadIdx.x];
        for (int g = 1; g < ngrp; g++) r += part[g * D + threadIdx.x];
        out[(size_t) h * D + threadIdx.x] = r;
    }
}

// ---- the CUDA-core tier of the split-KV frame (attn_split.cuh), up to attention_long_threshold() keys.  attention_kernel walks a head's
// keys with one CTA and re-reads the KV head's K / V once per query head: fine at 100 keys, far too slow at thousands
// (tools/ctx_decode.py shows the decode rate against the context position).  Here K / V are read once per KV head, over SPLIT_MAX splits:
//   scores: a warp takes one key per step, lane l holds dims 2l, 2l+1 of the key (one coalesced 256-byte row) and of the G <= 16 query
//           vectors; G partial dots per lane are reduced with a transposing butterfly (16 shuffles)
//   values: e for the CTA's own keys in shared memory ([key][head]); O_partial[head][d] += V[key][d] * e (lane = 2 dims, G heads in registers)
#define AD_B 4                           // key rows per warp step (plus the same number in flight for the next step)

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

template <typename E>
__global__ void __launch_bounds__(SPLIT_THREADS, 6) attn_dec_scores_kernel(const SplitArgs a) {
    __shared__ float wmax[SPLIT_WARPS][SPLIT_G];
    const int split = blockIdx.x, kvh = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int h0 = kvh * a.G + blockIdx.z * SPLIT_G, G = min(SPLIT_G, a.G - (int) blockIdx.z * SPLIT_G);      // this CTA's query heads: h0 .. h0 + G - 1
    const int n_past = a.n_past_dev ? *a.n_past_dev : a.n_past, T = n_past + 1;
    int k_lo, k_hi; split_range(T, SPLIT_MAX, split, k_lo, k_hi);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // the values kernel may take its place on the SMs now (it waits for this grid to finish)
    // the query rows do not depend on n_past: their loads are in flight while the device scalar arrives (every dependent round trip
    // counts here: beside ffn_up's streaming each one takes > 1 us, and at short contexts this kernel is nothing but such a chain)
    float2 q[SPLIT_G];
#pragma unroll
    for (int h = 0; h < SPLIT_G; h++)
        q[h] = h < G ? *reinterpret_cast<const float2 *>(a.qkv + (size_t) (h0 + h) * 64 + 2 * lane) : make_float2(0.f, 0.f);
    if (k_lo >= k_hi) return;                                   // a split without keys (short context): nothing to score, nobody reads its pmax
    const float scale = 1.0f / sqrtf(64.0f);
    const size_t kv_row = (size_t) a.n_head_kv * 64;
    // Fused RoPE + KV append (libfalcon.cpp:2229-2281).  A lane holds elements (2l, 2l+1) of a head; NeoX pairs element i < 32 with i + 32,
    // i.e. with the same component of lane l ^ 16.
    float2 knew = make_float2(0.f, 0.f);
    if (a.fuse_rope) {
        const float th0 = rope_theta(n_past, (2 * lane) & 31, a.theta_scale);
        const float th1 = __fmul_rn(th0, a.theta_scale);
        const float c0 = cosf(th0), s0 = sinf(th0), c1 = cosf(th1), s1 = sinf(th1);
        auto rot = [&](float2 v) {
            const float ox = __shfl_xor_sync(0xffffffffu, v.x, 16), oy = __shfl_xor_sync(0xffffffffu, v.y, 16);
            return lane < 16 ? make_float2(rope_rotate(v.x, ox, c0, s0).x, rope_rotate(v.y, oy, c1, s1).x)
                             : make_float2(rope_rotate(ox, v.x, c0, s0).y, rope_rotate(oy, v.y, c1, s1).y);
        };
#pragma unroll
        for (int h = 0; h < SPLIT_G; h++) q[h] = rot(q[h]);
        knew = rot(*reinterpret_cast<const float2 *>(a.qkv + (size_t) (a.n_head + kvh) * 64 + 2 * lane));        // this position's key row, rotated
        if (blockIdx.z == 0 && warp == 0 && n_past >= k_lo && n_past < k_hi) {                                     // one warp appends K and V to the cache
            const size_t o = ((size_t) n_past * a.n_head_kv + kvh) * 64 + 2 * lane;
            split_append2(a, o, kvh, 2 * lane, n_past, knew, *reinterpret_cast<const float2 *>(a.qkv + (size_t) (a.n_head + a.n_head_kv + kvh) * 64 + 2 * lane));
        }
        knew = make_float2(kv_seen(knew.x, (const E *) nullptr), kv_seen(knew.y, (const E *) nullptr));           // scored as the cache holds it
    }
    const int hh = lane >> 1;                                     // the head whose total this lane receives
    float lmax = -INFINITY;
    const E * kp = kv_k<E>(a.kv) + (size_t) kvh * 64 + 2 * lane;
    // AD_B keys per warp and step, the next batch's rows already in flight (memory-level parallelism without more warps)
    float2 cur[AD_B], nxt[AD_B];
    const int k_new = a.fuse_rope ? n_past : -1;                 // this key is not in the cache yet (another CTA may be writing it right now): use the registers
    auto ld_key = [&](int kk) { return kk >= k_hi ? make_float2(0.f, 0.f) : kk == k_new ? knew : kv_ld2(kp + (size_t) kk * kv_row); };
#pragma unroll
    for (int b = 0; b < AD_B; b++) cur[b] = ld_key(k_lo + warp + b * SPLIT_WARPS);
    for (int k = k_lo + warp; k < k_hi; k += AD_B * SPLIT_WARPS) {
#pragma unroll
        for (int b = 0; b < AD_B; b++) nxt[b] = ld_key(k + (AD_B + b) * SPLIT_WARPS);
#pragma unroll
        for (int b = 0; b < AD_B; b++) {
            const int kk = k + b * SPLIT_WARPS;
            float part[SPLIT_G];
#pragma unroll
            for (int h = 0; h < SPLIT_G; h++) part[h] = cur[b].x * q[h].x + cur[b].y * q[h].y;
            const float s = __fmul_rn(butterfly16(part, lane), scale);   // libfalcon.cpp:2313-2317
            if (hh < G && kk < k_hi) {
                if ((lane & 1) == 0) a.S[(size_t) (h0 + hh) * a.n_ctx + kk] = s;
                lmax = fmaxf(lmax, s);
            }
        }
#pragma unroll
        for (int b = 0; b < AD_B; b++) cur[b] = nxt[b];
    }
    if ((lane & 1) == 0 && hh < SPLIT_G) wmax[warp][hh] = lmax;
    __syncthreads();
    if (threadIdx.x < G) {
        float mx = wmax[0][threadIdx.x];
#pragma unroll
        for (int w = 1; w < SPLIT_WARPS; w++) mx = fmaxf(mx, wmax[w][threadIdx.x]);
        a.pmax[(size_t) (h0 + threadIdx.x) * SPLIT_MAX + split] = mx;
    }
}

template <typename E>
__global__ void __launch_bounds__(SPLIT_THREADS, 6) attn_dec_values_kernel(const SplitArgs a) {
    extern __shared__ __align__(16) float sm_dyn[];                // es[keys per split][SPLIT_G]
    __shared__ float gmax[SPLIT_G];
    __shared__ double dsum[SPLIT_THREADS / SPLIT_G][SPLIT_G];
    __shared__ float2 oacc[SPLIT_WARPS][SPLIT_G * 32];             // per-warp partial outputs: [head * 32 + lane] = dims 2l, 2l+1
    float * es = sm_dyn;
    const int split = blockIdx.x, kvh = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int h0 = kvh * a.G + blockIdx.z * SPLIT_G, G = min(SPLIT_G, a.G - (int) blockIdx.z * SPLIT_G);
    const int n_past = a.n_past_dev ? *a.n_past_dev : a.n_past, T = n_past + 1;
    int k_lo, k_hi; split_range(T, SPLIT_MAX, split, k_lo, k_hi);
    const int nk = k_hi - k_lo;
    const size_t kv_row = (size_t) a.n_head_kv * 64;
    const int n_used = splits_used(T, SPLIT_MAX);                 // splits 0 .. n_used - 1 hold keys
    // V rows of EARLIER positions have been in the cache since their own decode steps: the first batch is fetched while the scores kernel
    // still runs (this position's row is appended by that kernel: loaded after the wait)
    const E * vp = kv_v<E>(a.kv) + (size_t) kvh * 64 + 2 * lane;
    float2 cur[AD_B], nxt[AD_B];
#pragma unroll
    for (int b = 0; b < AD_B; b++) { const int jj = warp + b * SPLIT_WARPS; cur[b] = jj < nk && k_lo + jj < n_past ? kv_ld2(vp + (size_t) (k_lo + jj) * kv_row) : make_float2(0.f, 0.f); }
    asm volatile("griddepcontrol.wait;" ::: "memory");            // launched programmatically behind the scores kernel: its S / pmax / KV append are complete from here on
    if (nk > 0) {
    // the scores of the CTA's first AD_SPRE keys per thread are requested together with the split maxima (one round trip instead of two)
    constexpr int AD_SPRE = 8;
    const int eh = tid % SPLIT_G, ej = tid / SPLIT_G;
    const float * Sr = a.S + (size_t) (h0 + min(eh, G - 1)) * a.n_ctx + k_lo;
    float spre[AD_SPRE];
#pragma unroll
    for (int i = 0; i < AD_SPRE; i++) { const int j = ej + i * (SPLIT_THREADS / SPLIT_G); spre[i] = j < nk ? __ldcg(Sr + j) : 0.f; }
#pragma unroll
    for (int b = 0; b < AD_B; b++) { const int jj = warp + b * SPLIT_WARPS; if (jj < nk && k_lo + jj >= n_past) cur[b] = kv_ld2_new(vp + (size_t) (k_lo + jj) * kv_row); }
    if (tid < SPLIT_G) {
        float mx = -INFINITY;
        if (tid < G) for (int s = 0; s < n_used; s++) mx = fmaxf(mx, a.pmax[(size_t) (h0 + tid) * SPLIT_MAX + s]);
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
                const int j = ej + i * (SPLIT_THREADS / SPLIT_G);
                if (j < nk) { const float e = exp_f16lut(__fsub_rn(spre[i], gm)); es[j * SPLIT_G + eh] = e; s += (double) e; }
            }
            for (int j = ej + AD_SPRE * (SPLIT_THREADS / SPLIT_G); j < nk; j += SPLIT_THREADS / SPLIT_G) {
                const float e = exp_f16lut(__fsub_rn(__ldcg(Sr + j), gm));
                es[j * SPLIT_G + eh] = e; s += (double) e;
            }
        } else for (int j = ej; j < nk; j += SPLIT_THREADS / SPLIT_G) es[j * SPLIT_G + eh] = 0.f;
        dsum[ej][eh] = s;
    }
    __syncthreads();
    // O_partial[h][2l..2l+1] = sum over the warp's keys of V[key][2l..2l+1] * e[key][h]
    float2 acc[SPLIT_G];
#pragma unroll
    for (int h = 0; h < SPLIT_G; h++) acc[h] = make_float2(0.f, 0.f);
    for (int j = warp; j < nk; j += AD_B * SPLIT_WARPS) {
#pragma unroll
        for (int b = 0; b < AD_B; b++) { const int jj = j + (AD_B + b) * SPLIT_WARPS; nxt[b] = jj < nk ? kv_ld2(vp + (size_t) (k_lo + jj) * kv_row) : make_float2(0.f, 0.f); }
#pragma unroll
        for (int b = 0; b < AD_B; b++) {
            const int jj = j + b * SPLIT_WARPS;
            if (jj < nk) {                                                    // warp-uniform
                const float4 * er = reinterpret_cast<const float4 *>(es + jj * SPLIT_G);
                const float2 vv = cur[b];
#pragma unroll
                for (int c = 0; c < SPLIT_G / 4; c++) {
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
    for (int h = 0; h < SPLIT_G; h++) oacc[warp][h * 32 + lane] = acc[h];
    __syncthreads();
    }   // nk > 0
    split_combine(a, oacc, dsum, SPLIT_MAX, n_used, nk, split, h0, G);
}

// the values kernel's e array, es[keys per split][SPLIT_G], sized for n_ctx keys
static size_t dec_values_smem(int n_ctx) { return (size_t) max(SPLIT_MIN_KEYS, (n_ctx + SPLIT_MAX - 1) / SPLIT_MAX) * SPLIT_G * 4; }
template <typename E> static void launch_attention_split(SplitArgs a, cudaStream_t stream) {
    static bool set = false;
    if (!set) {
        B200_CUDA_CHECK(cudaFuncSetAttribute(attn_dec_values_kernel<E>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
        B200_CUDA_CHECK(cudaFuncSetAttribute(attn_dec_scores_kernel<E>, cudaFuncAttributePreferredSharedMemoryCarveout, B200_CARVEOUT));
        B200_CUDA_CHECK(cudaFuncSetAttribute(attn_dec_values_kernel<E>, cudaFuncAttributePreferredSharedMemoryCarveout, B200_CARVEOUT));
        set = true;
    }
    a.n_splits = SPLIT_MAX;
    split_launch(attn_dec_scores_kernel<E>, attn_dec_values_kernel<E>, a, dec_values_smem(a.n_ctx), stream);
}
void launch_attention_long(SplitArgs a, cudaStream_t stream);                                                      // attention_long.cu
bool attention_ws_covers(const AttnParams & p);                                                                     // attention_ws.cu
void launch_attention_ws(const float * qkv, float * out, int64_t out_stride, const AttnParams & p, cudaStream_t stream);
size_t attention_prefill_scratch_bytes(int n_head, int n_tok, int T);                                               // attention_prefill.cu
void launch_attention_prefill(const float * qkv, float * out, int64_t out_stride, const AttnParams & p, float * scratch, cudaStream_t stream);

int attention_long_threshold() {             // read on every call (graph builds and eager launches only): tests move it
    const char * e = getenv("B200_ATTN_LONG_FROM");
    return e ? atoi(e) : 1024;
}
// the split-KV tier a decode call takes: 2 = attention_long.cu (one-wave tensor-core kernels, measured crossover), 1 = this file's,
// 0 = none (attention_kernel)
static int split_tier(const AttnParams & p) {
    if (!split_fits(p)) return 0;
    const bool long_ctx = p.n_past_dev ? p.long_ctx != 0 : p.n_past + 1 > attention_long_threshold();
    if (long_ctx) return 2;
    return !getenv("B200_ATTN_NOSPLIT") && dec_values_smem(p.n_ctx) <= 160 * 1024 ? 1 : 0;
}

size_t attention_scratch_bytes(const AttnParams & p) {
    if (p.n_tok == 1) return split_fits(p) ? split_layout(p, nullptr, nullptr) : 0;
    if (p.n_tok <= 0 || attention_ws_covers(p)) return 0;
    return ATTN_CTR_BYTES + attention_prefill_scratch_bytes(p.n_head, p.n_tok, p.n_past + p.n_tok);
}

int launch_attention(float * qkv, float * out, int64_t out_stride, const AttnParams & p, float * scratch, cudaStream_t stream, bool * folded,
                     bool * rope_in_place) {
    if (folded) *folded = false;
    if (rope_in_place) *rope_in_place = false;
    if (p.n_tok <= 0) return 0;
    const int tier = p.n_tok == 1 ? split_tier(p) : 0;
    int n = 0;
    if (rope_in_place) *rope_in_place = !tier || !p.fuse_rope;
    if (!tier || !p.fuse_rope) { launch_rope_kv_append(qkv, p, stream); n++; }       // in place
    bool fold = false;
    if (tier) {
        B200_ASSERT(scratch != nullptr);
        SplitArgs a = split_args(qkv, out, p, scratch);
        // wo's activation quantisation in the combine step.  Q8_K blocks are 256 outputs = 4 heads: they must not straddle the 16-head
        // groups the CTAs combine
        fold = p.qout && !getenv("B200_ATTN_NOFOLD") && (p.qout->type != T_Q8_K || a.G % 4 == 0);
        if (fold) { a.has_q = 1; a.qA = *p.qout; }
        if (tier == 2) launch_attention_long(a, stream);
        else if (kv_f16(a.kv)) launch_attention_split<__half>(a, stream);
        else launch_attention_split<float>(a, stream);
        n += 2;
    } else if (p.n_tok == 1) {
        B200_ASSERT(p.head_dim % 4 == 0 && ATT_THREADS % p.head_dim == 0);
        // shared memory is sized for the worst case so that a captured graph stays valid while n_past grows
        const size_t smem = (size_t) (p.head_dim + (p.n_past_dev ? p.n_ctx : p.n_past + 1)) * sizeof(float);
        static bool set = false;
        if (!set) {
            for (const void * k : { (const void *) attention_kernel<float>, (const void *) attention_kernel<__half> }) {
                B200_CUDA_CHECK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
                B200_CUDA_CHECK(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, B200_CARVEOUT));
            }
            set = true;
        }
        B200_ASSERT(smem <= 200 * 1024);
        if (kv_f16(p.kv)) attention_kernel<__half><<<p.n_head, ATT_THREADS, smem, stream>>>(qkv, out, p);
        else attention_kernel<float><<<p.n_head, ATT_THREADS, smem, stream>>>(qkv, out, p);
        B200_CUDA_CHECK(cudaGetLastError());
        n++;
    } else if (attention_ws_covers(p)) {
        launch_attention_ws(qkv, out, out_stride, p, stream);
        n++;
    } else {
        B200_ASSERT(scratch != nullptr);
        launch_attention_prefill(qkv, out, out_stride, p, scratch + ATTN_CTR_BYTES / sizeof(float), stream);
        n += 2;
    }
    if (p.qout && !fold) { launch_quantize_act(out, out_stride, *p.qout, stream); n++; }
    if (folded) *folded = fold;
    return n;
}
