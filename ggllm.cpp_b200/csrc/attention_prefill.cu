// attention_prefill.cu -- causal grouped-query attention for a batch of N > 1 new tokens (prompt processing) where attention_ws.cu
// does not apply (N <= 8, no fp16 shadow, head_dim != 64), over the layer's KvCache, f32 or fp16 (template on the element type E).
//
// Same arithmetic contract as attention.cu (libfalcon.cpp:2285-2366, ggml.c:12389-12458): fp32 scores, softmax with the
// row's GLOBAL maximum subtracted before an fp16-LUT exp, the sum accumulated in double, probabilities scaled by
// (float)(1/sum) BEFORE the product with V.  The global maximum is why this is not an online-softmax kernel:
//   kernel 1 (scores): per (kv head, tile of 64 query rows) S = scale * Q K^T over the visible keys, written to a
//                      scratch matrix while tracking the row maxima; then a second sweep over its own (L2-resident)
//                      rows turns S into e = LUT(S - max), accumulates the row sums in double, stores inv = 1/sum
//   kernel 2 (PV)    : O = (e * inv) V, a [64 rows x T] x [T x 64] product per tile
// The 16 (40B) / 29 (180B) / 71 (7B) query heads that share one KV head are stacked into the row dimension
// (row = token * G + head_in_group), so every K / V tile read from HBM/L2 serves all of them.
// CUDA-core fp32 tiles (4x4 outputs per thread); the tensor-core version is future work (DESIGN.md).
#include "kernels.h"

#define PT 64          // tile: 64 rows x 64 keys (scores) / 64 rows x 64 dims (PV)
#define PTHREADS 256

struct PrefillArgs {
    const float * qkv; KvCache kv; float * out; float * S; float * inv;     // kv: read as the kernels' E
    int n_head, n_head_kv, G, D, n_tok, n_past, T;      // T = n_past + n_tok
    int64_t qkv_stride, out_stride, s_stride;           // s_stride = T rounded up to 64
    int rows;                                           // G * n_tok rows per kv head
};

// row -> (token, head)
__device__ __forceinline__ void row_to(const PrefillArgs & a, int g, int row, int & t, int & h) { t = row / a.G; h = g * a.G + row % a.G; }

// 4 CTAs per SM (64 registers): left to itself, ptxas takes 74-78 registers for this kernel, depending on the size of its parameters
template <typename E>
__global__ void __launch_bounds__(PTHREADS, 4) prefill_scores_kernel(const PrefillArgs a) {
    __shared__ float sq[PT][PT + 1];      // [row][d]
    __shared__ float sk[PT][PT + 1];      // [key][d]
    __shared__ float smax[PT];
    const int g = blockIdx.y, r0 = blockIdx.x * PT;
    const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;          // thread -> keys tx*4.., rows ty*4..
    const float scale = 1.0f / sqrtf((float) a.D);
    // query tile
    for (int i = threadIdx.x; i < PT * PT; i += PTHREADS) {
        const int r = i / PT, d = i % PT, row = r0 + r;
        float v = 0.f;
        if (row < a.rows && d < a.D) { int t, h; row_to(a, g, row, t, h); v = a.qkv[(size_t) t * a.qkv_stride + (size_t) h * a.D + d]; }
        sq[r][d] = v;
    }
    if (threadIdx.x < PT) smax[threadIdx.x] = -INFINITY;
    const int last_row = min(r0 + PT, a.rows) - 1;
    const int t_last = last_row / a.G;
    const int kmax = a.n_past + t_last + 1;                          // keys visible to the last row of the tile
    float * Sg = a.S + (size_t) g * a.rows * a.s_stride;
    for (int k0 = 0; k0 < kmax; k0 += PT) {
        __syncthreads();
        for (int i = threadIdx.x; i < PT * PT; i += PTHREADS) {
            const int kk = i / PT, d = i % PT, key = k0 + kk;
            sk[kk][d] = (key < a.T && d < a.D) ? kv_ld(kv_k<E>(a.kv) + ((size_t) key * a.n_head_kv + g) * a.D + d) : 0.f;
        }
        __syncthreads();
        float acc[4][4] = {};
#pragma unroll 8
        for (int d = 0; d < PT; d++) {
            float qv[4], kv[4];
#pragma unroll
            for (int i = 0; i < 4; i++) { qv[i] = sq[ty * 4 + i][d]; kv[i] = sk[tx * 4 + i][d]; }
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[i][j] += qv[i] * kv[j];
        }
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int row = r0 + ty * 4 + i;
            const int t = row / a.G, vis = row < a.rows ? a.n_past + t + 1 : 0;   // causal: keys < vis (no keys for rows past the end)
            float m = -INFINITY;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int key = k0 + tx * 4 + j;
                if (key < vis) { const float s = __fmul_rn(acc[i][j], scale); Sg[(size_t) row * a.s_stride + key] = s; m = fmaxf(m, s); }
            }
            // max over the 16 threads (same ty) that share this row: lanes tx = 0..15 of a half-warp
#pragma unroll
            for (int o = 8; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o, 16));
            if (tx == 0) smax[ty * 4 + i] = fmaxf(smax[ty * 4 + i], m);
        }
    }
    __syncthreads();
    // second sweep: e = LUT(s - max), sum in double (4 threads per row), inv = (float)(1/sum)
    {
        const int r = threadIdx.x / 4, part = threadIdx.x % 4, row = r0 + r;
        double sum = 0.0;
        if (row < a.rows) {
            const int t = row / a.G, vis = a.n_past + t + 1;
            const float mx = smax[r];
            float * Sr = Sg + (size_t) row * a.s_stride;
            for (int k = part; k < vis; k += 4) { const float e = exp_f16lut(__fsub_rn(Sr[k], mx)); Sr[k] = e; sum += (double) e; }
        }
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        sum += __shfl_xor_sync(0xffffffffu, sum, 2);
        if (part == 0 && row < a.rows) { int t, h; row_to(a, g, row, t, h); a.inv[(size_t) h * a.n_tok + t] = (float) (1.0 / sum); }
    }
}

template <typename E>
__global__ void __launch_bounds__(PTHREADS) prefill_pv_kernel(const PrefillArgs a) {
    __shared__ float sp[PT][PT + 1];      // [row][key]
    __shared__ float sv[PT][PT + 1];      // [key][d]
    const int g = blockIdx.y, r0 = blockIdx.x * PT;
    const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;          // thread -> dims tx*4.., rows ty*4..
    const int last_row = min(r0 + PT, a.rows) - 1;
    const int kmax = a.n_past + last_row / a.G + 1;
    const float * Sg = a.S + (size_t) g * a.rows * a.s_stride;
    float acc[4][4] = {};
    for (int k0 = 0; k0 < kmax; k0 += PT) {
        __syncthreads();
        for (int i = threadIdx.x; i < PT * PT; i += PTHREADS) {
            const int r = i / PT, kk = i % PT, row = r0 + r, key = k0 + kk;
            float p = 0.f;
            if (row < a.rows) {
                const int t = row / a.G, h = g * a.G + row % a.G;
                if (key < a.n_past + t + 1) p = __fmul_rn(Sg[(size_t) row * a.s_stride + key], a.inv[(size_t) h * a.n_tok + t]);
            }
            sp[r][kk] = p;
            const int kv = i / PT, d = i % PT, key2 = k0 + kv;
            sv[kv][d] = (key2 < a.T && d < a.D) ? kv_ld(kv_v<E>(a.kv) + ((size_t) key2 * a.n_head_kv + g) * a.D + d) : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int kk = 0; kk < PT; kk++) {
            float pv[4], vv[4];
#pragma unroll
            for (int i = 0; i < 4; i++) { pv[i] = sp[ty * 4 + i][kk]; vv[i] = sv[kk][tx * 4 + i]; }
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[i][j] += pv[i] * vv[j];
        }
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int row = r0 + ty * 4 + i;
        if (row >= a.rows) continue;
        int t, h; row_to(a, g, row, t, h);
#pragma unroll
        for (int j = 0; j < 4; j++) { const int d = tx * 4 + j; if (d < a.D) a.out[(size_t) t * a.out_stride + (size_t) h * a.D + d] = acc[i][j]; }
    }
}

size_t attention_prefill_scratch_bytes(int n_head, int n_tok, int T) {
    const size_t s_stride = (size_t) (T + 63) / 64 * 64;
    return (size_t) n_head * n_tok * s_stride * 4 + (size_t) n_head * n_tok * 4 + 256;
}

void launch_attention_prefill(const float * qkv, float * out, int64_t out_stride, const AttnParams & p, float * scratch, cudaStream_t stream) {
    B200_ASSERT(p.head_dim <= PT && p.n_past_dev == nullptr);
    PrefillArgs a;
    const bool kv16 = kv_f16(p.kv);
    a.qkv = qkv; a.kv = p.kv; a.out = out;
    a.n_head = p.n_head; a.n_head_kv = p.n_head_kv; a.G = p.n_head / p.n_head_kv; a.D = p.head_dim; a.n_tok = p.n_tok; a.n_past = p.n_past;
    a.T = p.n_past + p.n_tok; a.qkv_stride = p.qkv_stride; a.out_stride = out_stride; a.s_stride = (a.T + 63) / 64 * 64;
    a.rows = a.G * p.n_tok;
    a.S = scratch; a.inv = scratch + (size_t) p.n_head * p.n_tok * a.s_stride;
    dim3 grid((unsigned) ((a.rows + PT - 1) / PT), (unsigned) p.n_head_kv);
    if (kv16) prefill_scores_kernel<__half><<<grid, PTHREADS, 0, stream>>>(a);
    else prefill_scores_kernel<float><<<grid, PTHREADS, 0, stream>>>(a);
    B200_CUDA_CHECK(cudaGetLastError());
    if (kv16) prefill_pv_kernel<__half><<<grid, PTHREADS, 0, stream>>>(a);
    else prefill_pv_kernel<float><<<grid, PTHREADS, 0, stream>>>(a);
    B200_CUDA_CHECK(cudaGetLastError());
}
