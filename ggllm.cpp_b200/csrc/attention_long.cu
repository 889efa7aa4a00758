// attention_long.cu -- split-KV decode attention (n_tok == 1, head_dim 64) for LONG contexts.
//
// Same contract and scratch layout as the split-KV kernels of attention.cu (see there for the numerics, libfalcon.cpp:2285-2366); what
// differs is how the work is laid out, because at thousands of keys these kernels stop being hidden beside ffn_up / ffn_down:
//   * ONE WAVE: n_splits x n_head_kv x head groups ~ the SM count.  Beside the mat-vec CTAs an SM has registers for exactly one of these
//     128-thread CTAs, so the 256-CTA grid of attention.cu runs as two waves of latency-bound CTAs
//   * rows stream through a warp-private cp.async ring (AL_KR stages of AL_KB = 8 rows, padded against bank conflicts): only __syncwarp
//     is involved and the next stage is in flight while one is consumed, without holding registers
//   * both products run on the TENSOR CORES: the G <= 16 query heads of a KV head are exactly the M = 16 of a warp-level mma.  At 8k keys
//     attention.cu's kernels are latency-bound instruction streams (one warp per scheduler, ~270 instructions per key) that also take
//     issue slots from the mat-vec CTAs beside them; mma.sync m16n8k16 (scores) / m16n8k8 (values) with the fp32 operands split into
//     fp16 hi + lo terms needs ~60 instructions per key
//   * values: the exponentials come out directly in A-fragment layout (lane = heads gid, gid + 8 x keys 2 tig, 2 tig + 1), no separate pass,
//     no [key][head] array, no shuffles; the scores travel through the same ring as the V rows
// Against the oracle the tiny-model evals stay at the 1e-8 * S level.  Short contexts gain nothing:
// launch_attention picks this path above attention_long_threshold() keys; the decode graphs of engine.cu are captured per tier.
#include "kernels.h"
#include "actquant.cuh"

__device__ __forceinline__ float exp_f16lut_l(float v) {      // table_exp_f16[f16(v)], ggml.c:4281-4290
    return __half2float(__float2half_rn(expf(__half2float(__float2half_rn(v)))));
}

#define AL_THREADS 128                   // small CTAs (<= 104 registers): one fits beside ffn_up's two 256-thread CTAs on every SM
#define AL_WARPS (AL_THREADS / 32)
#define AL_MAX_SPLITS 32                 // the scratch holds this many partials per head (attention.cu's layout); the launcher picks n_splits <= it
#define AL_G 16                          // query heads per KV head handled together (n_head / n_head_kv <= 16 per CTA, more in grid.z)

struct AttnLongArgs {
    const float * qkv; const float * kc; const float * vc; float * out;
    float * S; float * pmax; double * psum; float * opart; unsigned * ctr;
    int n_head, n_head_kv, G, n_past; const int * n_past_dev; int n_ctx; int64_t qkv_stride;
    int n_splits;
    unsigned long long * trace;
    ActQ qA; int has_q;          // optional quantised copy of the output row (see AttnParams::qout)
    int fuse_rope; float theta_scale; float * kc_w; float * vc_w; __half * k16; __half * vt16; int ctx_pad;     // see AttnParams::fuse_rope
};

__device__ __forceinline__ void cp_async16(void * smem, const void * g) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(smem_u32(smem)), "l"(g) : "memory"); }
__device__ __forceinline__ void cp_async4(void * smem, const void * g) { asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" :: "r"(smem_u32(smem)), "l"(g) : "memory"); }
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N) : "memory"); }

// keys per split: at least AL_MIN_KEYS, so that a short context occupies few CTAs and the combine step reads few partials (at
// n_past < 64 one CTA per KV-head group does everything; the other CTAs of the fixed grid only check in at the counter)
#define AL_MIN_KEYS 64
__device__ __forceinline__ int split_keys(int T, int ns) { return max(AL_MIN_KEYS, (T + ns - 1) / ns); }
__device__ __forceinline__ int splits_used(int T, int ns) { const int per = split_keys(T, ns); return (T + per - 1) / per; }
__device__ __forceinline__ void split_range(int T, int ns, int split, int & k_lo, int & k_hi) {
    const int per = split_keys(T, ns);
    k_lo = min(T, split * per); k_hi = min(T, k_lo + per);
}

// ---- tensor-core helpers.  The G <= 16 query heads of a KV head are exactly the M = 16 of a warp-level mma: scores = Q[16 x 64] K^T and
// O += E[16 x keys] V run on the tensor cores (legacy mma.sync, the right size for a 16-row problem), which takes the instruction count
// per key from 79 + 97 (the CUDA-core version of this file) to 24 + 39.  fp32 operands are split into two fp16 terms (hi = fp16(x), lo = fp16(x - hi):
// 22 significant bits); products of fp16 pairs are exact in the fp32 accumulator, the dropped lo x lo term is 2^-22 of the product -- the
// fp32 dot product's own rounding level (below |x| = 0.125 the lo term is an fp16 subnormal: the error is then absolute, <= 2^-25 per
// element; tests/test_host.py emulates both regimes; an operand beyond fp16's 65504 would overflow the hi term -- Falcon's rotated q / k
// rows and v rows are O(1) .. O(100)).  e = table_exp_f16[...] IS an fp16 value: the A operand of the second product is exact.
__device__ __forceinline__ void split_h2(float x0, float x1, uint32_t & hi, uint32_t & lo) {
    const __half2 h = __floats2half2_rn(x0, x1);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn(__fsub_rn(x0, hf.x), __fsub_rn(x1, hf.y));
    hi = *reinterpret_cast<const uint32_t *>(&h); lo = *reinterpret_cast<const uint32_t *>(&l);
}
// D[16 x 8] += A[16 x 16] B[16 x 8]   (fp16 operands, fp32 accumulate); fragment layouts: PTX ISA "mma.m16n8k16", gid = lane / 4, tig = lane % 4
__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// D[16 x 8] += A[16 x 8] B[8 x 8]
__device__ __forceinline__ void mma_1688(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t b0) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5}, {%6}, {%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a0), "r"(a1), "r"(b0));
}
#define AL_KB 8                          // keys per warp and ring stage = the N of one mma
#define AL_KR 2                          // ring stages per warp (double buffer)
#define AL_KS 72                         // floats per K row in the ring: 64 + 8 keeps the B-fragment LDS.64s of a half-warp on distinct banks
#define AL_VS 68                         // floats per V row in the ring: 64 + 4 does the same for the LDS.32s of the second product
// 8-key blocks of a split go round-robin to the warps: block b = stage * AL_WARPS + warp
__device__ __forceinline__ int warp_blocks(int nk, int warp) { const int nb = (nk + AL_KB - 1) / AL_KB; return nb > warp ? (nb - warp + AL_WARPS - 1) / AL_WARPS : 0; }

__global__ void __launch_bounds__(AL_THREADS, 4) attn_long_scores_kernel(const AttnLongArgs a) {
    __shared__ float wmax[AL_WARPS][AL_G];
    __shared__ __align__(16) float ring[AL_WARPS][AL_KR][AL_KB][AL_KS];    // 18 KB: K rows in flight
    __shared__ __align__(16) float qs[AL_G][64];                           // this position's query rows, rotated
    __shared__ __align__(16) float knew_s[AL_KS];                          // this position's key row, rotated (not in the cache yet)
    trace_begin(a.trace);
    const int split = blockIdx.x, kvh = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int h0 = kvh * a.G + blockIdx.z * AL_G, G = min(AL_G, a.G - (int) blockIdx.z * AL_G);      // this CTA's query heads: h0 .. h0 + G - 1
    const int n_past = a.n_past_dev ? *a.n_past_dev : a.n_past, T = n_past + 1;
    int k_lo, k_hi; split_range(T, a.n_splits, split, k_lo, k_hi);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // the values kernel may take its place on the SMs now (it waits for this grid to finish)
    // RoPE work of thread t: pair i = t % 32 (elements i, i + 32) of heads t / 32 + 4 r and, for t < 32, of the key row.  The rows do not
    // depend on n_past: their loads are in flight while the device scalar arrives.
    const int ri = tid & 31, rh = tid >> 5;
    float qa[AL_G / AL_WARPS], qb[AL_G / AL_WARPS];
#pragma unroll
    for (int r = 0; r < AL_G / AL_WARPS; r++) {
        const int h = rh + AL_WARPS * r;
        const float * src = a.qkv + (size_t) (h0 + min(h, G - 1)) * 64;
        qa[r] = src[ri]; qb[r] = src[ri + 32];
    }
    const float * ksrc = a.qkv + (size_t) (a.n_head + kvh) * 64;
    const float ka = ksrc[ri], kb_ = ksrc[ri + 32];
    if (k_lo >= k_hi) { trace_end(a.trace); return; }            // a split without keys (short context): nothing to score, nobody reads its pmax
    const int nk = k_hi - k_lo, nst = warp_blocks(nk, warp);
    const int j_new = a.fuse_rope ? n_past - k_lo : -1;           // this position's key is not in the cache yet (another CTA may be writing it right now)
    const size_t kv_row = (size_t) a.n_head_kv * 64;
    const int gid = lane >> 2, tig = lane & 3;
    const float * kp = a.kc + (size_t) kvh * 64 + 16 * tig + (size_t) k_lo * kv_row;
    auto issue = [&](int i) {                                     // lane copies 64 bytes: dims 16 tig .. 16 tig + 15 of key gid of the block
        if (i < nst) {
            const int jj = (i * AL_WARPS + warp) * AL_KB + gid;
            if (jj < nk && jj != j_new) {
                float * dst = &ring[warp][i % AL_KR][gid][16 * tig];
                const float * src = kp + (size_t) jj * kv_row;
#pragma unroll
                for (int c = 0; c < 4; c++) cp_async16(dst + 4 * c, src + 4 * c);
            }
        }
        cp_async_commit();
    };
#pragma unroll
    for (int i = 0; i < AL_KR - 1; i++) issue(i);                // the first rows travel while RoPE runs
    // Fused RoPE + KV append (libfalcon.cpp:2229-2281), arithmetic of rope_pair (ops.cu): theta = n_past * theta_scale^i by repeated fp32 products
    {
        float c = 1.f, sn = 0.f;
        if (a.fuse_rope) {
            float th = (float) n_past;
            for (int k = 0; k < ri; k++) th = __fmul_rn(th, a.theta_scale);
            c = cosf(th); sn = sinf(th);
        }
        auto rot = [&](float x0, float x1, float & y0, float & y1) {
            if (a.fuse_rope) { y0 = __fsub_rn(__fmul_rn(x0, c), __fmul_rn(x1, sn)); y1 = __fadd_rn(__fmul_rn(x0, sn), __fmul_rn(x1, c)); }
            else { y0 = x0; y1 = x1; }
        };
#pragma unroll
        for (int r = 0; r < AL_G / AL_WARPS; r++) {
            const int h = rh + AL_WARPS * r;
            float y0, y1; rot(qa[r], qb[r], y0, y1);
            qs[h][ri] = h < G ? y0 : 0.f; qs[h][ri + 32] = h < G ? y1 : 0.f;
        }
        if (a.fuse_rope && warp == 0) {
            float y0, y1; rot(ka, kb_, y0, y1);
            knew_s[ri] = y0; knew_s[ri + 32] = y1;
            if (blockIdx.z == 0 && n_past >= k_lo && n_past < k_hi) {                                                  // one warp appends K and V to the cache
                const size_t o = ((size_t) n_past * a.n_head_kv + kvh) * 64;
                const float * vsrc = a.qkv + (size_t) (a.n_head + a.n_head_kv + kvh) * 64;
                const float v0 = vsrc[ri], v1 = vsrc[ri + 32];
                a.kc_w[o + ri] = y0; a.kc_w[o + ri + 32] = y1;
                a.vc_w[o + ri] = v0; a.vc_w[o + ri + 32] = v1;
                if (a.k16) {
                    a.k16[o + ri] = __float2half_rn(y0); a.k16[o + ri + 32] = __float2half_rn(y1);
                    __half * vt = a.vt16 + (size_t) kvh * 64 * a.ctx_pad + n_past;
                    vt[(size_t) ri * a.ctx_pad] = __float2half_rn(v0); vt[(size_t) (ri + 32) * a.ctx_pad] = __float2half_rn(v1);
                }
            }
        }
    }
    __syncthreads();
    // A fragments of Q (16 heads x 64 dims = 4 k-steps), hi and lo terms: rows gid / gid + 8, columns 16 t + 2 tig (+1) and + 8 (+9)
    uint32_t ah[4][4], al[4][4];
#pragma unroll
    for (int t = 0; t < 4; t++)
#pragma unroll
        for (int r = 0; r < 4; r++) {
            const float2 q2 = *reinterpret_cast<const float2 *>(&qs[gid + 8 * (r & 1)][16 * t + 2 * tig + 8 * (r >> 1)]);
            split_h2(q2.x, q2.y, ah[t][r], al[t][r]);
        }
    const float scale = 1.0f / sqrtf(64.0f);
    float lmax0 = -INFINITY, lmax1 = -INFINITY;                   // heads gid, gid + 8 over this lane's keys
    for (int i = 0; i < nst; i++) {
        issue(i + AL_KR - 1);                                     // refills the stage consumed in the previous iteration
        cp_async_wait<AL_KR - 1>();
        __syncwarp();                                             // the four lanes of a key copied a quarter of its row each
        const int jj0 = (i * AL_WARPS + warp) * AL_KB;
        const float * krow = jj0 + gid == j_new ? knew_s : &ring[warp][i % AL_KR][gid][0];     // B column gid = key jj0 + gid
        float c[4] = { 0.f, 0.f, 0.f, 0.f };
#pragma unroll
        for (int t = 0; t < 4; t++) {
            const float2 p0 = *reinterpret_cast<const float2 *>(krow + 16 * t + 2 * tig), p1 = *reinterpret_cast<const float2 *>(krow + 16 * t + 2 * tig + 8);
            uint32_t bh0, bl0, bh1, bl1;
            split_h2(p0.x, p0.y, bh0, bl0); split_h2(p1.x, p1.y, bh1, bl1);
            mma_16816(c, ah[t], bh0, bh1); mma_16816(c, ah[t], bl0, bl1); mma_16816(c, al[t], bh0, bh1);
        }
        // c0, c1: head gid, keys jj0 + 2 tig, + 1;  c2, c3: head gid + 8.  A key past the split's end had an unwritten ring row: its column is not stored
#pragma unroll
        for (int u = 0; u < 2; u++) {
            const int jj = jj0 + 2 * tig + u;
            if (jj < nk) {
                const float s0 = __fmul_rn(c[u], scale), s1 = __fmul_rn(c[2 + u], scale);   // libfalcon.cpp:2313-2317
                if (gid < G)     { a.S[(size_t) (h0 + gid) * a.n_ctx + k_lo + jj] = s0; lmax0 = fmaxf(lmax0, s0); }
                if (gid + 8 < G) { a.S[(size_t) (h0 + gid + 8) * a.n_ctx + k_lo + jj] = s1; lmax1 = fmaxf(lmax1, s1); }
            }
        }
        __syncwarp();                                             // all reads of this stage are done before the next iteration refills it
    }
    cp_async_wait<0>();
    lmax0 = fmaxf(lmax0, __shfl_xor_sync(0xffffffffu, lmax0, 1)); lmax0 = fmaxf(lmax0, __shfl_xor_sync(0xffffffffu, lmax0, 2));
    lmax1 = fmaxf(lmax1, __shfl_xor_sync(0xffffffffu, lmax1, 1)); lmax1 = fmaxf(lmax1, __shfl_xor_sync(0xffffffffu, lmax1, 2));
    if (tig == 0) { wmax[warp][gid] = lmax0; wmax[warp][gid + 8] = lmax1; }
    __syncthreads();
    if (tid < G) {
        float mx = wmax[0][tid];
#pragma unroll
        for (int w = 1; w < AL_WARPS; w++) mx = fmaxf(mx, wmax[w][tid]);
        a.pmax[(size_t) (h0 + tid) * AL_MAX_SPLITS + split] = mx;
    }
    trace_end(a.trace);
}

// thread tid's 8 consecutive outputs (head hA of the CTA's group) -> the attention output row, plus wo's activation quantisation
__device__ __forceinline__ void attn_long_store(const AttnLongArgs & a, const float (&y)[8], int h0, int hA, int G, int tid, int lane) {
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

// fixed order: deterministic
__device__ __forceinline__ double dsum_total(const double (&d)[AL_WARPS][2][AL_G], int h) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < AL_WARPS; w++) s += d[w][0][h] + d[w][1][h];
    return s;
}

__global__ void __launch_bounds__(AL_THREADS, 4) attn_long_values_kernel(const AttnLongArgs a) {
    // V rows in flight; once a warp has consumed its rows the same memory holds its partial outputs [head][64]
    __shared__ __align__(16) float2 vring[AL_WARPS][AL_KR * AL_KB * AL_VS / 2];
    __shared__ float sring[AL_WARPS][AL_KR][32][4];                // the scores of those rows, lane-private: (gid, 2 tig), (gid, 2 tig + 1), (gid + 8, ..)
    __shared__ float gmax[AL_G];
    __shared__ double dsum[AL_WARPS][2][AL_G];
    __shared__ float inv_s[AL_G];
    __shared__ int s_last;
    static_assert(AL_KR * AL_KB * AL_VS / 2 >= AL_G * 32, "a warp's ring doubles as its [AL_G][64] partial-output block");
    const int split = blockIdx.x, kvh = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int h0 = kvh * a.G + blockIdx.z * AL_G, G = min(AL_G, a.G - (int) blockIdx.z * AL_G);
    const int n_past = a.n_past_dev ? *a.n_past_dev : a.n_past, T = n_past + 1;
    int k_lo, k_hi; split_range(T, a.n_splits, split, k_lo, k_hi);
    const int nk = k_hi - k_lo, nst = warp_blocks(nk, warp);
    const size_t kv_row = (size_t) a.n_head_kv * 64;
    trace_begin(a.trace);
    const int n_used = splits_used(T, a.n_splits);                // splits 0 .. n_used - 1 hold keys
    const int j_new = n_past - k_lo;                              // this position's V row is appended by the scores kernel: read after the wait
    const int gid = lane >> 2, tig = lane & 3;
    const float * vp = a.vc + (size_t) kvh * 64 + 16 * tig + (size_t) k_lo * kv_row;
    const float * S0 = a.S + (size_t) (h0 + min(gid, G - 1)) * a.n_ctx + k_lo, * S1 = a.S + (size_t) (h0 + min(gid + 8, G - 1)) * a.n_ctx + k_lo;
    float (*vr)[AL_KB][AL_VS] = reinterpret_cast<float (*)[AL_KB][AL_VS]>(vring[warp]);
    auto issue = [&](int i, bool v, bool s) {
        if (i < nst) {
            const int jj0 = (i * AL_WARPS + warp) * AL_KB;
            if (v) {                                              // lane copies 64 bytes: dims 16 tig .. + 15 of key gid; rows past the end are zeroed (0 x garbage could be NaN)
                const int jj = jj0 + gid;
                float * dst = &vr[i % AL_KR][gid][16 * tig];
                if (jj < nk && jj != j_new) {
                    const float * src = vp + (size_t) jj * kv_row;
#pragma unroll
                    for (int c = 0; c < 4; c++) cp_async16(dst + 4 * c, src + 4 * c);
                } else if (jj >= nk) {
#pragma unroll
                    for (int c = 0; c < 4; c++) *reinterpret_cast<float4 *>(dst + 4 * c) = make_float4(0.f, 0.f, 0.f, 0.f);
                }
            }
            if (s) {
#pragma unroll
                for (int u = 0; u < 2; u++) {
                    const int jj = jj0 + 2 * tig + u;
                    if (jj < nk) { cp_async4(&sring[warp][i % AL_KR][lane][u], S0 + jj); cp_async4(&sring[warp][i % AL_KR][lane][2 + u], S1 + jj); }
                }
            }
        }
        cp_async_commit();
    };
    // V rows of EARLIER positions have been in the cache since their own decode steps: the first stage travels while the scores kernel still runs
#pragma unroll
    for (int i = 0; i < AL_KR - 1; i++) issue(i, true, false);
    asm volatile("griddepcontrol.wait;" ::: "memory");            // launched programmatically behind the scores kernel: its S / pmax / KV append are complete from here on
    if (nk > 0) {
#pragma unroll
    for (int i = 0; i < AL_KR - 1; i++) issue(i, false, true);    // their scores, together with the split maxima: one round trip
    const bool has_new = j_new >= 0 && j_new < nk;
    const float2 vnew = has_new ? *reinterpret_cast<const float2 *>(a.vc + (size_t) kvh * 64 + 2 * lane + (size_t) (k_lo + j_new) * kv_row) : make_float2(0.f, 0.f);
    if (tid < AL_G) {
        float mx = -INFINITY;
        if (tid < G) for (int s = 0; s < n_used; s++) mx = fmaxf(mx, a.pmax[(size_t) (h0 + tid) * AL_MAX_SPLITS + s]);
        gmax[tid] = mx;
    }
    __syncthreads();
    const float gm0 = gmax[gid], gm1 = gmax[gid + 8];
    double lsum0 = 0.0, lsum1 = 0.0;                               // heads gid, gid + 8: sum of e over this lane's keys
    // O[16 heads x 64 dims] += E[16 x 8 keys] V[8 x 64] per stage: 8 n-tiles of 8 dims, accumulators c0, c1 = (gid, 8 nt + 2 tig, + 1), c2, c3 = (gid + 8, ..)
    float acc[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; nt++) { acc[nt][0] = 0.f; acc[nt][1] = 0.f; acc[nt][2] = 0.f; acc[nt][3] = 0.f; }
    for (int i = 0; i < nst; i++) {
        issue(i + AL_KR - 1, true, true);
        cp_async_wait<AL_KR - 1>();
        __syncwarp();
        const int jj0 = (i * AL_WARPS + warp) * AL_KB, st = i % AL_KR;
        if (has_new && j_new >= jj0 && j_new < jj0 + AL_KB) {     // this position's V row goes into its ring row now
            *reinterpret_cast<float2 *>(&vr[st][j_new - jj0][2 * lane]) = vnew;
            __syncwarp();
        }
        // e = table_exp_f16[f16(s - max)] (ggml.c:12427-12440), produced directly in A-fragment layout: a0 = (gid; keys 2 tig, + 1), a1 = (gid + 8; ..)
        float e[4];
#pragma unroll
        for (int u = 0; u < 2; u++) {
            const bool live = jj0 + 2 * tig + u < nk;
            e[u]     = live && gid < G     ? exp_f16lut_l(__fsub_rn(sring[warp][st][lane][u], gm0)) : 0.f;
            e[2 + u] = live && gid + 8 < G ? exp_f16lut_l(__fsub_rn(sring[warp][st][lane][2 + u], gm1)) : 0.f;
        }
        lsum0 += (double) e[0] + (double) e[1]; lsum1 += (double) e[2] + (double) e[3];
        const __half2 e0h = __floats2half2_rn(e[0], e[1]), e1h = __floats2half2_rn(e[2], e[3]);       // exact: e is an fp16 value
        const uint32_t a0 = *reinterpret_cast<const uint32_t *>(&e0h), a1 = *reinterpret_cast<const uint32_t *>(&e1h);
#pragma unroll
        for (int nt = 0; nt < 8; nt++) {                                         // B column gid = dim 8 nt + gid, rows = keys 2 tig, 2 tig + 1
            uint32_t bh, bl;
            split_h2(vr[st][2 * tig][8 * nt + gid], vr[st][2 * tig + 1][8 * nt + gid], bh, bl);
            mma_1688(acc[nt], a0, a1, bh); mma_1688(acc[nt], a0, a1, bl);
        }
        __syncwarp();                                             // all reads of this stage are done before the next iteration refills it
    }
    cp_async_wait<0>();
    lsum0 += __shfl_xor_sync(0xffffffffu, lsum0, 1); lsum0 += __shfl_xor_sync(0xffffffffu, lsum0, 2);
    lsum1 += __shfl_xor_sync(0xffffffffu, lsum1, 1); lsum1 += __shfl_xor_sync(0xffffffffu, lsum1, 2);
    if (tig == 0) { dsum[warp][0][gid] = lsum0; dsum[warp][0][gid + 8] = lsum1; dsum[warp][1][gid] = 0.0; dsum[warp][1][gid + 8] = 0.0; }
    __syncwarp();                                                              // every lane is done with the ring: it becomes the warp's partial-output block [head][64]
#pragma unroll
    for (int nt = 0; nt < 8; nt++) {
        vring[warp][gid * 32 + 4 * nt + tig] = make_float2(acc[nt][0], acc[nt][1]);
        vring[warp][(gid + 8) * 32 + 4 * nt + tig] = make_float2(acc[nt][2], acc[nt][3]);
    }
    __syncthreads();
    if (n_used > 1) {
        if (tid < G) a.psum[(size_t) (h0 + tid) * AL_MAX_SPLITS + split] = dsum_total(dsum, tid);
        for (int i = tid; i < AL_G * 32; i += AL_THREADS) {             // fixed warp order: deterministic
            const int h = i / 32, l = i % 32;
            float2 r = vring[0][h * 32 + l];
#pragma unroll
            for (int w = 1; w < AL_WARPS; w++) { r.x += vring[w][h * 32 + l].x; r.y += vring[w][h * 32 + l].y; }
            if (h < G) *reinterpret_cast<float2 *>(a.opart + ((size_t) (split * a.n_head + h0 + h)) * 64 + 2 * l) = r;
        }
    }
    }   // nk > 0
    if (n_used == 1) {
        // short context: split 0 holds every key; its CTA finishes from its own shared memory -- the same sums in the same order as the
        // general path below (warps, then the single split), no scratch round trip, no fence, no counter
        if (split != 0) { trace_end(a.trace); return; }
        if (tid < AL_G) inv_s[tid] = (float) (1.0 / dsum_total(dsum, tid));
        __syncthreads();
        const int hA = tid / 8, l0 = 4 * (tid % 8);                          // thread = 8 consecutive outputs of head tid / 8 = lanes l0 .. l0 + 3 of the partial blocks
        float y[8];
        const float sc = hA < G ? inv_s[hA] : 0.f;
#pragma unroll
        for (int u = 0; u < 4; u++) {
            float2 r = vring[0][hA * 32 + l0 + u];
#pragma unroll
            for (int w = 1; w < AL_WARPS; w++) { r.x += vring[w][hA * 32 + l0 + u].x; r.y += vring[w][hA * 32 + l0 + u].y; }
            y[2 * u] = __fmul_rn(r.x, sc); y[2 * u + 1] = __fmul_rn(r.y, sc);
        }
        attn_long_store(a, y, h0, hA, G, tid, lane);
        trace_end(a.trace);
        return;
    }
    // the last CTA of this KV head group combines the splits
    __threadfence();
    __syncthreads();
    unsigned * ctr = a.ctr + kvh * gridDim.z + blockIdx.z;
    if (tid == 0) { const unsigned old = atomicAdd(ctr, 1u); s_last = old == (unsigned) a.n_splits - 1; if (s_last) *ctr = 0; }
    __syncthreads();
    if (!s_last) { trace_end(a.trace); return; }
    __threadfence();
    if (tid < AL_G) {
        double s = 0.0;
        if (tid < G) for (int sp = 0; sp < n_used; sp++) s += __ldcg(a.psum + (size_t) (h0 + tid) * AL_MAX_SPLITS + sp);
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
        attn_long_store(a, y, h0, hA, G, tid, lane);
    }
    trace_end(a.trace);
}

static size_t align256(size_t v) { return (v + 255) & ~(size_t) 255; }
#define AL_CTR_BYTES 4096                 // as AD_CTR_BYTES in attention.cu: the two variants share one scratch block
// scratch: attention_scratch_bytes(p) bytes whose first AL_CTR_BYTES were zeroed once by the owner (the counters re-arm themselves)
static int g_long_launches = 0;
extern "C" int b200_attention_long_launches(void) { return g_long_launches; }       // diagnostics / tests: launches (eager or captured) of this path

bool launch_attention_long(const float * qkv, const float * k_cache, const float * v_cache, float * out, const AttnParams & p, float * scratch, cudaStream_t stream) {
    if (!scratch || p.n_tok != 1 || p.head_dim != 64 || p.n_head % p.n_head_kv || getenv("B200_ATTN_NOLONG")) return false;
    const int G = p.n_head / p.n_head_kv, groups = (G + AL_G - 1) / AL_G;
    if ((size_t) p.n_head_kv * groups * 4 > AL_CTR_BYTES) return false;
    AttnLongArgs a;
    uint8_t * s = reinterpret_cast<uint8_t *>(scratch);
    a.ctr = reinterpret_cast<unsigned *>(s); s += AL_CTR_BYTES;
    a.S = reinterpret_cast<float *>(s); s += align256((size_t) p.n_head * p.n_ctx * 4);
    a.pmax = reinterpret_cast<float *>(s); s += align256((size_t) p.n_head * AL_MAX_SPLITS * 4);
    a.psum = reinterpret_cast<double *>(s); s += align256((size_t) p.n_head * AL_MAX_SPLITS * 8);
    a.opart = reinterpret_cast<float *>(s);
    a.qkv = qkv; a.kc = k_cache; a.vc = v_cache; a.out = out;
    a.n_head = p.n_head; a.n_head_kv = p.n_head_kv; a.G = p.n_head / p.n_head_kv; a.n_past = p.n_past; a.n_past_dev = p.n_past_dev; a.n_ctx = p.n_ctx;
    a.qkv_stride = p.qkv_stride;
    a.fuse_rope = p.fuse_rope; a.theta_scale = p.rope_theta_scale; a.kc_w = const_cast<float *>(k_cache); a.vc_w = const_cast<float *>(v_cache);
    a.k16 = p.k16; a.vt16 = p.vt16; a.ctx_pad = attention_ctx_pad(p.n_ctx);
    // one wave: as many key splits as SMs divided by the (KV head, head group) pairs -- Falcon-40B 18, 180B 9, 7B 29
    static int force = -1;
    if (force < 0) { const char * e = getenv("B200_ATTN_SPLITS"); force = e ? atoi(e) : 0; }
    a.n_splits = force > 0 ? force : num_sms() / (p.n_head_kv * groups);
    a.n_splits = a.n_splits < 4 ? 4 : a.n_splits > AL_MAX_SPLITS ? AL_MAX_SPLITS : a.n_splits;
    // Q8_K blocks are 256 outputs = 4 heads: they must not straddle the 16-head groups the CTAs combine
    a.has_q = p.qout != nullptr && (p.qout->type != T_Q8_K || G % 4 == 0);
    if (a.has_q) a.qA = *p.qout;
    B200_ASSERT(p.qout == nullptr || a.has_q);
    static bool set = false;
    if (!set) {
        B200_CUDA_CHECK(cudaFuncSetAttribute(attn_long_scores_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, B200_CARVEOUT));
        B200_CUDA_CHECK(cudaFuncSetAttribute(attn_long_values_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, B200_CARVEOUT));
        set = true;
    }
    dim3 grid((unsigned) a.n_splits, (unsigned) p.n_head_kv, (unsigned) groups);
    g_long_launches++;
    a.trace = b200_trace_slot("attn_scores");
    attn_long_scores_kernel<<<grid, AL_THREADS, 0, stream>>>(a);
    B200_CUDA_CHECK(cudaGetLastError());
    a.trace = b200_trace_slot("attn_values");
    {
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = grid; cfg.blockDim = dim3(AL_THREADS); cfg.dynamicSmemBytes = 0; cfg.stream = stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr; cfg.numAttrs = getenv("B200_NO_PDL") ? 0 : 1;
        B200_CUDA_CHECK(cudaLaunchKernelEx(&cfg, attn_long_values_kernel, a));
    }
    return true;
}

