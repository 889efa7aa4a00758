// ops.cu -- the non-matmul operators of the Falcon graph, with the CPU oracle's numerics (SURVEY.md section 9.2):
//   LayerNorm  ggml_compute_forward_norm_f32 (ggml.c:10540-10599) + gamma/beta mul/add (libfalcon.cpp:2166-2185)
//   GELU       fp16-LUT semantics (ggml.c:3461-3484)
//   RoPE       NeoX mode with dynamic NTK alpha (ggml.c:12875-12898, 12957-12979)
//   add / mul / scale glue (libfalcon.cpp:2399-2400; ggml-cuda.cu:181-206 add_f32/mul_f32/scale_f32)
// None of these has a usable kernel in the reference backend (no LayerNorm, no GELU, RoPE mode 0 only).
#include "kernels.h"
#include "actquant.cuh"
#include <cmath>

// ---------------------------------------------------------------------------------------------- block reductions
template <int NT> __device__ __forceinline__ double block_sum_d(double v, double * sh) {
    v = warp_sum_d(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();                       // protect sh reuse
    if (l == 0) sh[w] = v;
    __syncthreads();
    double t = (l < NT / 32) ? sh[l] : 0.0;
    t = warp_sum_d(t);
    return t;                              // every thread gets the total
}

// ---------------------------------------------------------------------------------------------- LayerNorm
// One CTA per row.  Sums in double like the CPU (ggml_float), everything else fp32 with separately rounded
// multiply and add (no FMA) so the result is bit-identical to the oracle up to double-summation order.
#define LN_THREADS 512
__global__ void __launch_bounds__(LN_THREADS) layernorm_kernel(const float * __restrict__ x, int64_t x_stride, const float * __restrict__ g,
                                                             const float * __restrict__ b, float * __restrict__ y, int64_t y_stride, int n) {
    __shared__ double sh[LN_THREADS / 32];
    const float * xr = x + (size_t) blockIdx.x * x_stride;
    float * yr = y + (size_t) blockIdx.x * y_stride;
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += LN_THREADS) s += (double) xr[i];
    const float mean = (float) (block_sum_d<LN_THREADS>(s, sh) / n);
    double s2 = 0.0;
    for (int i = threadIdx.x; i < n; i += LN_THREADS) { const float v = __fsub_rn(xr[i], mean); s2 += (double) __fmul_rn(v, v); }
    const float var = (float) (block_sum_d<LN_THREADS>(s2, sh) / n);
    const float scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(var, 1e-5f)));
    for (int i = threadIdx.x; i < n; i += LN_THREADS) {
        float v = __fmul_rn(__fsub_rn(xr[i], mean), scale);
        if (g) v = __fmul_rn(v, g[i]);
        if (b) v = __fadd_rn(v, b[i]);
        yr[i] = v;
    }
}
void launch_layernorm(const float * x, int64_t x_stride, const float * g, const float * b, float * y, int64_t y_stride, int n, int rows, cudaStream_t stream) {
    if (rows <= 0) return;
    layernorm_kernel<<<rows, LN_THREADS, 0, stream>>>(x, x_stride, g, b, y, y_stride, n);
    B200_CUDA_CHECK(cudaGetLastError());
}

__device__ __forceinline__ void store_f32x8(float * p, const float (&v)[8]) {
    *reinterpret_cast<float4 *>(p) = make_float4(v[0], v[1], v[2], v[3]); *reinterpret_cast<float4 *>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
}
// Fused: [residual add] + normalise once + apply up to two (gamma, beta) pairs (Falcon-40B's ln_attn and ln_mlp read
// the same input, libfalcon.cpp:2166-2188) + write each result directly as quantised activations for the following
// mat-mul.  With ra/rb given the row is first updated to x = (ra + rb) + x and written back: the two residual adds
// that close the previous layer (libfalcon.cpp:2399-2400), in that order.  YO: rows from y_row0 on also store the first pair's fp32
// result, the values it quantises, at y + (row - y_row0) * y_stride (the final LayerNorm's "result_norm" row, libfalcon.cpp:2422-2431).
template <int ATYPE, bool YO>
__global__ void __launch_bounds__(LN_THREADS) layernorm_q_kernel(float * __restrict__ x, int64_t x_stride,
        const float * __restrict__ ra, const float * __restrict__ rb, int64_t r_stride,
        const float * __restrict__ g1, const float * __restrict__ b1, ActQ A1,
        const float * __restrict__ g2, const float * __restrict__ b2, ActQ A2, int has2, int n,
        float * __restrict__ y, int64_t y_stride, int y_row0) {
    __shared__ double sh[LN_THREADS / 32];
    extern __shared__ float vn[];                                     // the row: raw, then normalised
    const int row = blockIdx.x;
    float * xr = x + (size_t) row * x_stride;
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += LN_THREADS) {
        float v = xr[i];
        if (ra) { v = __fadd_rn(__fadd_rn(ra[(size_t) row * r_stride + i], rb[(size_t) row * r_stride + i]), v); xr[i] = v; }
        vn[i] = v;
        s += (double) v;
    }
    const float mean = (float) (block_sum_d<LN_THREADS>(s, sh) / n);
    double s2 = 0.0;
    for (int i = threadIdx.x; i < n; i += LN_THREADS) { const float v = __fsub_rn(vn[i], mean); s2 += (double) __fmul_rn(v, v); }
    const float var = (float) (block_sum_d<LN_THREADS>(s2, sh) / n);
    const float scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(var, 1e-5f)));
    for (int i = threadIdx.x; i < n; i += LN_THREADS) vn[i] = __fmul_rn(__fsub_rn(vn[i], mean), scale);   // each thread rewrites only its own entries
    __syncthreads();
    const int lane = threadIdx.x & 31;
    // chunks of 8 values; a warp always works on 32 consecutive chunks = one 256-block (or eight 32-blocks)
    for (int c0 = (threadIdx.x >> 5) * 32; c0 < n / 8; c0 += LN_THREADS) {
        const int c = c0 + lane;
        if (c < n / 8) {         // n % 256 == 0 for Q8_K, n % 32 == 0 otherwise: blocks never straddle the guard
            float v[8];
#pragma unroll
            for (int j = 0; j < 8; j++) v[j] = __fadd_rn(__fmul_rn(vn[c * 8 + j], g1[c * 8 + j]), b1[c * 8 + j]);
            if (YO && row >= y_row0) store_f32x8(y + (size_t) (row - y_row0) * y_stride + c * 8, v);
            quantize_chunk8<ATYPE>(v, lane, A1, row, c * 8);
            if (has2) {
#pragma unroll
                for (int j = 0; j < 8; j++) v[j] = __fadd_rn(__fmul_rn(vn[c * 8 + j], g2[c * 8 + j]), b2[c * 8 + j]);
                quantize_chunk8<ATYPE>(v, lane, A2, row, c * 8);
            }
        }
    }
}
// Register-resident variant for rows of up to 16384 values (every Falcon n_embd): 1024 threads, each owns one or two
// chunks of 8 consecutive values, so the row is read from global memory exactly once, a warp's 32 chunks are one Q8_K
// block (or eight 32-blocks) and the quantisation needs no shared memory.  On the decode critical path this kernel
// runs alone on one SM, so what matters is its dependent-latency chain: 1 load round, 2 block reductions, 1 store round.
#define LNR_THREADS 1024
template <int ATYPE, int CH, bool YO>
__global__ void __launch_bounds__(LNR_THREADS) layernorm_q_reg_kernel(float * __restrict__ x, int64_t x_stride,
        const float * __restrict__ ra, const float * __restrict__ rb, int64_t r_stride,
        const float * __restrict__ g1, const float * __restrict__ b1, ActQ A1,
        const float * __restrict__ g2, const float * __restrict__ b2, ActQ A2, int has2, int n,
        float * __restrict__ y, int64_t y_stride, int y_row0) {
    __shared__ double sh[LNR_THREADS / 32];
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // the mat-vecs that follow may start prefetching their weights now
    const int row = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // launched with programmatic stream serialisation: gamma / beta do not depend on the previous kernel, so they are
    // pulled into L2 while it drains; everything below the wait reads what it wrote
#pragma unroll
    for (int c = 0; c < CH; c++) {
        const int e = (c * LNR_THREADS + threadIdx.x) * 8;
        if (e < n) {
            asm volatile("prefetch.global.L2 [%0];" :: "l"(g1 + e)); asm volatile("prefetch.global.L2 [%0];" :: "l"(b1 + e));
            if (has2) { asm volatile("prefetch.global.L2 [%0];" :: "l"(g2 + e)); asm volatile("prefetch.global.L2 [%0];" :: "l"(b2 + e)); }
        }
    }
    asm volatile("griddepcontrol.wait;" ::: "memory");
    float * xr = x + (size_t) row * x_stride;
    float v[CH][8];
    bool ok[CH];
    double s = 0.0;
#pragma unroll
    for (int c = 0; c < CH; c++) {
        const int e = (c * LNR_THREADS + threadIdx.x) * 8;
        ok[c] = e < n;
        if (ok[c]) {
            float4 p = *reinterpret_cast<const float4 *>(xr + e), q = *reinterpret_cast<const float4 *>(xr + e + 4);
            if (ra) {
                const float4 a0 = *reinterpret_cast<const float4 *>(ra + (size_t) row * r_stride + e), a1 = *reinterpret_cast<const float4 *>(ra + (size_t) row * r_stride + e + 4);
                const float4 c0 = *reinterpret_cast<const float4 *>(rb + (size_t) row * r_stride + e), c1 = *reinterpret_cast<const float4 *>(rb + (size_t) row * r_stride + e + 4);
                p.x = __fadd_rn(__fadd_rn(a0.x, c0.x), p.x); p.y = __fadd_rn(__fadd_rn(a0.y, c0.y), p.y); p.z = __fadd_rn(__fadd_rn(a0.z, c0.z), p.z); p.w = __fadd_rn(__fadd_rn(a0.w, c0.w), p.w);
                q.x = __fadd_rn(__fadd_rn(a1.x, c1.x), q.x); q.y = __fadd_rn(__fadd_rn(a1.y, c1.y), q.y); q.z = __fadd_rn(__fadd_rn(a1.z, c1.z), q.z); q.w = __fadd_rn(__fadd_rn(a1.w, c1.w), q.w);
                *reinterpret_cast<float4 *>(xr + e) = p; *reinterpret_cast<float4 *>(xr + e + 4) = q;
            }
            v[c][0] = p.x; v[c][1] = p.y; v[c][2] = p.z; v[c][3] = p.w; v[c][4] = q.x; v[c][5] = q.y; v[c][6] = q.z; v[c][7] = q.w;
#pragma unroll
            for (int i = 0; i < 8; i++) s += (double) v[c][i];
        } else {
#pragma unroll
            for (int i = 0; i < 8; i++) v[c][i] = 0.f;
        }
    }
    auto block_total = [&](double t) -> double {
        t = warp_sum_d(t);
        __syncthreads();
        if (lane == 0) sh[warp] = t;
        __syncthreads();
        double r = sh[lane];                           // 32 warps -> one value per lane
        return warp_sum_d(r);
    };
    const float mean = (float) (block_total(s) / n);
    double s2 = 0.0;
#pragma unroll
    for (int c = 0; c < CH; c++) if (ok[c]) {
#pragma unroll
        for (int i = 0; i < 8; i++) { v[c][i] = __fsub_rn(v[c][i], mean); s2 += (double) __fmul_rn(v[c][i], v[c][i]); }
    }
    const float var = (float) (block_total(s2) / n);
    const float scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(var, 1e-5f)));
#pragma unroll
    for (int c = 0; c < CH; c++) {
        const int e = (c * LNR_THREADS + threadIdx.x) * 8;
        if (!ok[c]) continue;                          // whole warps drop out together (n is a multiple of 256 for Q8_K, of 32 otherwise)
        float yv[8];
        const float4 ga = *reinterpret_cast<const float4 *>(g1 + e), gb = *reinterpret_cast<const float4 *>(g1 + e + 4);
        const float4 ba = *reinterpret_cast<const float4 *>(b1 + e), bb = *reinterpret_cast<const float4 *>(b1 + e + 4);
        const float gg[8] = { ga.x, ga.y, ga.z, ga.w, gb.x, gb.y, gb.z, gb.w }, bv[8] = { ba.x, ba.y, ba.z, ba.w, bb.x, bb.y, bb.z, bb.w };
#pragma unroll
        for (int i = 0; i < 8; i++) yv[i] = __fadd_rn(__fmul_rn(__fmul_rn(v[c][i], scale), gg[i]), bv[i]);
        if (YO && row >= y_row0) store_f32x8(y + (size_t) (row - y_row0) * y_stride + e, yv);
        quantize_chunk8<ATYPE>(yv, lane, A1, row, e);
        if (has2) {
            const float4 ha = *reinterpret_cast<const float4 *>(g2 + e), hb = *reinterpret_cast<const float4 *>(g2 + e + 4);
            const float4 ca = *reinterpret_cast<const float4 *>(b2 + e), cb = *reinterpret_cast<const float4 *>(b2 + e + 4);
            const float g2v[8] = { ha.x, ha.y, ha.z, ha.w, hb.x, hb.y, hb.z, hb.w }, b2v[8] = { ca.x, ca.y, ca.z, ca.w, cb.x, cb.y, cb.z, cb.w };
#pragma unroll
            for (int i = 0; i < 8; i++) yv[i] = __fadd_rn(__fmul_rn(__fmul_rn(v[c][i], scale), g2v[i]), b2v[i]);
            quantize_chunk8<ATYPE>(yv, lane, A2, row, e);
        }
    }
}

// Decode (one row): the same LayerNorm + quantisation spread over a thread-block CLUSTER of ceil(n / 1024) <= 8 CTAs x 128 threads,
// 8 values per thread.  The 1024-thread single-CTA kernel above needs a whole SM's registers, so it cannot become resident
// before the previous mat-vec has drained, and its ~64 registers per thread leave no room to have gamma / beta in flight
// early: a gap between the end of wo and the first qkv row.  Here every CTA is small enough
// to sit beside the mat-vec's CTAs, loads its gamma / beta BEFORE griddepcontrol.wait, and after the wait pays one L2 round
// trip plus two cluster reductions through distributed shared memory (fixed summation order: deterministic).
#define LNC_THREADS 128
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ double ld_dsmem_f64(const double * local, int rank) {
    uint32_t raddr; double v;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(raddr) : "r"(smem_u32(local)), "r"(rank));
    asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(raddr) : "memory");
    return v;
}
template <int ATYPE, bool YO>
__global__ void __launch_bounds__(LNC_THREADS) layernorm_q_cluster_kernel(float * __restrict__ x, const float * __restrict__ ra, const float * __restrict__ rb,
        const float * __restrict__ g1, const float * __restrict__ b1, ActQ A1,
        const float * __restrict__ g2, const float * __restrict__ b2, ActQ A2, int has2, int n, float * __restrict__ yout) {
    __shared__ double wsum[LNC_THREADS / 32];
    __shared__ double part[2];                                        // this CTA's partial sum / sum of squares, read by the whole cluster
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, C = gridDim.x;
    const int e = ((int) blockIdx.x * LNC_THREADS + threadIdx.x) * 8;
    const bool ok = e < n;                                            // the last CTA of a row that is not a multiple of 1024 has idle lanes
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    // weights first: they do not depend on the previous kernel
    float4 ga = z4, gb = z4, ba = z4, bb = z4;
    if (ok) { ga = __ldg(reinterpret_cast<const float4 *>(g1 + e)); gb = __ldg(reinterpret_cast<const float4 *>(g1 + e + 4));
              ba = __ldg(reinterpret_cast<const float4 *>(b1 + e)); bb = __ldg(reinterpret_cast<const float4 *>(b1 + e + 4)); }
    float4 ha = ga, hb = gb, ca = ba, cb = bb;
    if (has2 && ok) { ha = __ldg(reinterpret_cast<const float4 *>(g2 + e)); hb = __ldg(reinterpret_cast<const float4 *>(g2 + e + 4));
                      ca = __ldg(reinterpret_cast<const float4 *>(b2 + e)); cb = __ldg(reinterpret_cast<const float4 *>(b2 + e + 4)); }
    asm volatile("griddepcontrol.wait;" ::: "memory");
    float4 p = z4, q = z4;
    if (ok) {
        p = *reinterpret_cast<const float4 *>(x + e); q = *reinterpret_cast<const float4 *>(x + e + 4);
        if (ra) {
            const float4 a0 = *reinterpret_cast<const float4 *>(ra + e), a1 = *reinterpret_cast<const float4 *>(ra + e + 4);
            const float4 c0 = *reinterpret_cast<const float4 *>(rb + e), c1 = *reinterpret_cast<const float4 *>(rb + e + 4);
            p.x = __fadd_rn(__fadd_rn(a0.x, c0.x), p.x); p.y = __fadd_rn(__fadd_rn(a0.y, c0.y), p.y); p.z = __fadd_rn(__fadd_rn(a0.z, c0.z), p.z); p.w = __fadd_rn(__fadd_rn(a0.w, c0.w), p.w);
            q.x = __fadd_rn(__fadd_rn(a1.x, c1.x), q.x); q.y = __fadd_rn(__fadd_rn(a1.y, c1.y), q.y); q.z = __fadd_rn(__fadd_rn(a1.z, c1.z), q.z); q.w = __fadd_rn(__fadd_rn(a1.w, c1.w), q.w);
            *reinterpret_cast<float4 *>(x + e) = p; *reinterpret_cast<float4 *>(x + e + 4) = q;
        }
    }
    float v[8] = { p.x, p.y, p.z, p.w, q.x, q.y, q.z, q.w };
    auto cluster_total = [&](double t, int slot) -> double {
        t = warp_sum_d(t);
        if (lane == 0) wsum[warp] = t;
        __syncthreads();
        if (threadIdx.x == 0) { double r = 0.0; for (int w = 0; w < LNC_THREADS / 32; w++) r += wsum[w]; part[slot] = r; }
        cluster_sync_all();                                           // every CTA's partial is published
        double r = 0.0;
        for (int k = 0; k < C; k++) r += ld_dsmem_f64(part + slot, k);
        return r;
    };
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < 8; i++) s += (double) v[i];                   // idle lanes hold zeros
    const float mean = (float) (cluster_total(s, 0) / n);
    double s2 = 0.0;
#pragma unroll
    for (int i = 0; i < 8; i++) { v[i] = __fsub_rn(v[i], mean); if (ok) s2 += (double) __fmul_rn(v[i], v[i]); }
    const float scale = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn((float) (cluster_total(s2, 1) / n), 1e-5f)));
    float y[8];
    const float gg[8] = { ga.x, ga.y, ga.z, ga.w, gb.x, gb.y, gb.z, gb.w }, bv[8] = { ba.x, ba.y, ba.z, ba.w, bb.x, bb.y, bb.z, bb.w };
#pragma unroll
    for (int i = 0; i < 8; i++) y[i] = ok ? __fadd_rn(__fmul_rn(__fmul_rn(v[i], scale), gg[i]), bv[i]) : 0.f;
    if (YO && ok) store_f32x8(yout + e, y);
    quantize_chunk8<ATYPE>(y, lane, A1, 0, e, ok);
    if (has2) {
        const float g2v[8] = { ha.x, ha.y, ha.z, ha.w, hb.x, hb.y, hb.z, hb.w }, b2v[8] = { ca.x, ca.y, ca.z, ca.w, cb.x, cb.y, cb.z, cb.w };
#pragma unroll
        for (int i = 0; i < 8; i++) y[i] = ok ? __fadd_rn(__fmul_rn(__fmul_rn(v[i], scale), g2v[i]), b2v[i]) : 0.f;
        quantize_chunk8<ATYPE>(y, lane, A2, 0, e, ok);
    }
    cluster_sync_all();                                               // nobody leaves while a peer may still read its `part`
}

void launch_layernorm_q(float * x, int64_t x_stride, const float * ra, const float * rb, int64_t r_stride,
                        const float * g1, const float * b1, const ActQ * A1,
                        const float * g2, const float * b2, const ActQ * A2, int n, int rows, cudaStream_t stream,
                        float * y, int64_t y_stride, int y_row0) {
    if (rows <= 0) return;
    const ActQ a2 = A2 ? *A2 : *A1;
    B200_ASSERT(!A2 || A2->type == A1->type);
    const bool yo = y && y_row0 < rows;                              // the fp32 rows go out with vector stores
    B200_ASSERT(!yo || (y_row0 >= 0 && n % 8 == 0 && y_stride % 4 == 0 && ((uintptr_t) y & 15) == 0));
    const int qblk = A1->type == T_Q8_K ? 256 : 32;                  // whole quantisation blocks per row: idle lanes come in whole blocks
    if (rows == 1 && n % qblk == 0 && (n + LNC_THREADS * 8 - 1) / (LNC_THREADS * 8) <= 8 && !getenv("B200_LN_NOCLUSTER")) {
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3((unsigned) ((n + LNC_THREADS * 8 - 1) / (LNC_THREADS * 8))); cfg.blockDim = dim3(LNC_THREADS); cfg.stream = stream;
        cudaLaunchAttribute attr[2];
        attr[0].id = cudaLaunchAttributeClusterDimension; attr[0].val.clusterDim.x = cfg.gridDim.x; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
        attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[1].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr; cfg.numAttrs = 2;
        const int has2 = A2 != nullptr;
#define LNCQ1(T, YO) do { static bool set = false; if (!set) { B200_CUDA_CHECK(cudaFuncSetAttribute(layernorm_q_cluster_kernel<T, YO>, cudaFuncAttributePreferredSharedMemoryCarveout, B200_CARVEOUT)); set = true; } \
        B200_CUDA_CHECK(cudaLaunchKernelEx(&cfg, layernorm_q_cluster_kernel<T, YO>, x, ra, rb, g1, b1, *A1, g2, b2, a2, has2, n, y)); } while (0)
#define LNCQ(T) do { if (yo) LNCQ1(T, true); else LNCQ1(T, false); } while (0)
        switch (A1->type) {
            case T_Q8_0: LNCQ(T_Q8_0); break;
            case T_Q8_1: LNCQ(T_Q8_1); break;
            case T_Q8_K: LNCQ(T_Q8_K); break;
            default: B200_ASSERT(!"layernorm_q: bad activation type");
        }
#undef LNCQ
#undef LNCQ1
        return;
    }
    if (n <= 16384 && n % 8 == 0 && !getenv("B200_LN_SMEM")) {
        const bool two = n > 8192;
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3((unsigned) rows); cfg.blockDim = dim3(LNR_THREADS); cfg.stream = stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr; cfg.numAttrs = 1;
        const int has2 = A2 != nullptr;
#define LNRQ1(T, CH, YO) B200_CUDA_CHECK(cudaLaunchKernelEx(&cfg, layernorm_q_reg_kernel<T, CH, YO>, x, x_stride, ra, rb, r_stride, g1, b1, *A1, g2, b2, a2, has2, n, y, y_stride, y_row0))
#define LNRQ(T) do { if (two) { if (yo) LNRQ1(T, 2, true); else LNRQ1(T, 2, false); } \
                     else     { if (yo) LNRQ1(T, 1, true); else LNRQ1(T, 1, false); } } while (0)
        switch (A1->type) {
            case T_Q8_0: LNRQ(T_Q8_0); break;
            case T_Q8_1: LNRQ(T_Q8_1); break;
            case T_Q8_K: LNRQ(T_Q8_K); break;
            default: B200_ASSERT(!"layernorm_q: bad activation type");
        }
#undef LNRQ
#undef LNRQ1
        B200_CUDA_CHECK(cudaGetLastError());
        return;
    }
    const size_t smem = (size_t) n * 4;
#define LNQ1(T, YO) do { static bool set = false; if (!set) { B200_CUDA_CHECK(cudaFuncSetAttribute(layernorm_q_kernel<T, YO>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024)); set = true; } \
        layernorm_q_kernel<T, YO><<<rows, LN_THREADS, smem, stream>>>(x, x_stride, ra, rb, r_stride, g1, b1, *A1, g2, b2, a2, A2 != nullptr, n, y, y_stride, y_row0); } while (0)
#define LNQ(T) do { if (yo) LNQ1(T, true); else LNQ1(T, false); } while (0)
    switch (A1->type) {
        case T_Q8_0: LNQ(T_Q8_0); break;
        case T_Q8_1: LNQ(T_Q8_1); break;
        case T_Q8_K: LNQ(T_Q8_K); break;
        default: B200_ASSERT(!"layernorm_q: bad activation type");
    }
#undef LNQ
#undef LNQ1
    B200_CUDA_CHECK(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------- elementwise
__global__ void gelu_kernel(const float * __restrict__ x, float * __restrict__ y, int64_t n) {
    for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) y[i] = gelu_f16lut(x[i]);
}
__global__ void add_kernel(const float * __restrict__ a, const float * __restrict__ b, float * __restrict__ y, int64_t n) {
    for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) y[i] = __fadd_rn(a[i], b[i]);
}
__global__ void add3_kernel(const float * __restrict__ a, const float * __restrict__ b, const float * __restrict__ c, float * __restrict__ y, int64_t n) {
    for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) y[i] = __fadd_rn(__fadd_rn(a[i], b[i]), c[i]);
}
__global__ void mul_bcast_kernel(const float * __restrict__ a, const float * __restrict__ b, float * __restrict__ y, int64_t n, int64_t nb) {
    for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) y[i] = __fmul_rn(a[i], b[i % nb]);
}
__global__ void add_bcast_kernel(const float * __restrict__ a, const float * __restrict__ b, float * __restrict__ y, int64_t n, int64_t nb) {
    for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) y[i] = __fadd_rn(a[i], b[i % nb]);
}
__global__ void scale_kernel(const float * __restrict__ a, float s, float * __restrict__ y, int64_t n) {
    for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) y[i] = __fmul_rn(a[i], s);
}
__global__ void f32_to_f16_kernel(const float * __restrict__ x, __half * __restrict__ y, int64_t n) {       // ggml_fp32_to_fp16_row
    for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) y[i] = __float2half_rn(x[i]);
}
unsigned ew_grid(int64_t n) { int64_t g = (n + 255) / 256; return (unsigned) (g < 1 ? 1 : (g > 132 * 16 ? 132 * 16 : g)); }
void launch_f32_to_f16(const float * x, __half * y, int64_t n, cudaStream_t s) { f32_to_f16_kernel<<<ew_grid(n), 256, 0, s>>>(x, y, n); B200_CUDA_CHECK(cudaGetLastError()); }
void launch_gelu(const float * x, float * y, int64_t n, cudaStream_t s) { gelu_kernel<<<ew_grid(n), 256, 0, s>>>(x, y, n); B200_CUDA_CHECK(cudaGetLastError()); }
void launch_add(const float * a, const float * b, float * y, int64_t n, cudaStream_t s) { add_kernel<<<ew_grid(n), 256, 0, s>>>(a, b, y, n); B200_CUDA_CHECK(cudaGetLastError()); }
void launch_add3(const float * a, const float * b, const float * c, float * y, int64_t n, cudaStream_t s) { add3_kernel<<<ew_grid(n), 256, 0, s>>>(a, b, c, y, n); B200_CUDA_CHECK(cudaGetLastError()); }
void launch_mul_bcast(const float * a, const float * b, float * y, int64_t n, int64_t nb, cudaStream_t s) { mul_bcast_kernel<<<ew_grid(n), 256, 0, s>>>(a, b, y, n, nb); B200_CUDA_CHECK(cudaGetLastError()); }
void launch_add_bcast(const float * a, const float * b, float * y, int64_t n, int64_t nb, cudaStream_t s) { add_bcast_kernel<<<ew_grid(n), 256, 0, s>>>(a, b, y, n, nb); B200_CUDA_CHECK(cudaGetLastError()); }
void launch_scale(const float * a, float sc, float * y, int64_t n, cudaStream_t s) { scale_kernel<<<ew_grid(n), 256, 0, s>>>(a, sc, y, n); B200_CUDA_CHECK(cudaGetLastError()); }

// ---------------------------------------------------------------------------------------------- transpose
// One CTA moves a 32 x 32 tile through shared memory: warp-wide reads along a source row, warp-wide writes along a destination row.
// The padding column keeps the column-wise accesses to the tile free of bank conflicts.
__global__ void __launch_bounds__(256) transpose_f32_kernel(const float * __restrict__ src, int64_t ld_src, int rows, int cols,
                                                            float * __restrict__ dst, int64_t ld_dst) {
    __shared__ float tile[32][33];
    const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32, tx = threadIdx.x;
    for (int i = threadIdx.y; i < 32; i += 8)
        if (r0 + i < rows && c0 + tx < cols) tile[i][tx] = src[(int64_t) (r0 + i) * ld_src + c0 + tx];
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += 8)
        if (c0 + i < cols && r0 + tx < rows) dst[(int64_t) (c0 + i) * ld_dst + r0 + tx] = tile[tx][i];
}
void launch_transpose_f32(const float * src, int64_t ld_src, int rows, int cols, float * dst, int64_t ld_dst, cudaStream_t s) {
    if (rows <= 0 || cols <= 0) return;
    B200_ASSERT((rows + 31) / 32 <= 65535);
    transpose_f32_kernel<<<dim3((unsigned) ((cols + 31) / 32), (unsigned) ((rows + 31) / 32)), dim3(32, 8), 0, s>>>(src, ld_src, rows, cols, dst, ld_dst);
    B200_CUDA_CHECK(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------- RoPE
// theta_scale is computed on the host exactly as the CPU does (powf in fp32, ggml.c:12875-12898) and passed in.
float rope_theta_scale_host(int head_dim, int n_ctx_rope, int dynamic_mode, float ntk_alpha, int freq_base) {
    const float fb = (float) (freq_base ? freq_base : 10000);
    float alpha = 1.0f;
    if (dynamic_mode) {
        if (n_ctx_rope >= 2048) alpha = powf(((n_ctx_rope / 2048) - 1) * ntk_alpha + 1, head_dim / (head_dim - 2.0));
    } else if (ntk_alpha != 0.0f) alpha = powf(ntk_alpha, head_dim / (head_dim - 2.0));
    return powf(alpha * fb, -2.0f / head_dim);
}
float falcon_rope_theta_scale(int head_dim, int n_ctx_rope, int n_ctx) { return rope_theta_scale_host(head_dim, n_ctx_rope ? n_ctx_rope : n_ctx, 1, 2.0f, 0); }
// pair i of a head at position p, in place
__device__ __forceinline__ void rope_pair(float * v, int half, int i, int p, float theta_scale) {
    const float theta = rope_theta(p, i, theta_scale);
    const float c = cosf(theta), s = sinf(theta);
    const float2 r = rope_rotate(v[i], v[i + half], c, s);
    v[i] = r.x; v[i + half] = r.y;
}
__global__ void rope_neox_kernel(float * __restrict__ x, int n_head, int head_dim, int64_t tok_stride, int n_past, const int * __restrict__ n_past_dev, float theta_scale) {
    const int t = blockIdx.y, h = blockIdx.x, i = threadIdx.x;
    if (h >= n_head || i >= head_dim / 2) return;
    const int p = (n_past_dev ? *n_past_dev : n_past) + t;
    rope_pair(x + (size_t) t * tok_stride + (size_t) h * head_dim, head_dim / 2, i, p, theta_scale);
}
void launch_rope_neox(float * x, int n_tok, int n_head, int head_dim, int64_t tok_stride, int n_past, const int * n_past_dev, float theta_scale, cudaStream_t stream) {
    if (n_tok <= 0) return;
    dim3 grid((unsigned) n_head, (unsigned) n_tok);
    rope_neox_kernel<<<grid, head_dim / 2, 0, stream>>>(x, n_head, head_dim, tok_stride, n_past, n_past_dev, theta_scale);
    B200_CUDA_CHECK(cudaGetLastError());
}

// fused RoPE(Q) + RoPE(K) + K append + V append (libfalcon.cpp:2229-2281): one CTA per (token, head slot)
__global__ void rope_kv_append_kernel(float * __restrict__ qkv, AttnParams p) {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const int t = blockIdx.y, slot = blockIdx.x, i = threadIdx.x, D = p.head_dim, half = D / 2;
    const int n_past = p.n_past_dev ? *p.n_past_dev : p.n_past;
    const int pos = n_past + t;
    float * v = qkv + (size_t) t * p.qkv_stride + (size_t) slot * D;             // slots: Q heads | K heads | V heads
    if (slot < p.n_head + p.n_head_kv) rope_pair(v, half, i, pos, p.rope_theta_scale);
    if (slot >= p.n_head) {
        const bool is_k = slot < p.n_head + p.n_head_kv;
        const int kvh = slot - p.n_head - (is_k ? 0 : p.n_head_kv);
        const size_t o = ((size_t) pos * p.n_head_kv + kvh) * D;
        if (is_k) { kv_put_k(p.kv, o + i, v[i]); kv_put_k(p.kv, o + i + half, v[i + half]); }
        else { kv_put_v(p.kv, o + i, kvh, i, pos, v[i]); kv_put_v(p.kv, o + i + half, kvh, i + half, pos, v[i + half]); }
    }
}
// The same work for a batch of tokens (prompt).  The single-token kernel above recomputes the 32 rotation angles of a position in every
// one of its (n_head + 2 n_head_kv) x n_tok tiny CTAs and scatters V^T two bytes at a time (at 512 tokens
// about as long as the attention itself).  Here one CTA per token computes its cos / sin once and walks the row coalesced, and the V^T shadow
// is written by extra CTAs that transpose 64 tokens x 64 dims through shared memory (128-byte rows).  Same arithmetic, same bits.
__global__ void __launch_bounds__(256) rope_kv_append_batch_kernel(float * __restrict__ qkv, AttnParams p) {
    const int D = p.head_dim, half = D / 2, H = p.n_head, HKV = p.n_head_kv, N = p.n_tok;
    const int n_past = p.n_past_dev ? *p.n_past_dev : p.n_past;
    if ((int) blockIdx.x < N) {
        __shared__ float cs[64], sn[64];
        const int t = blockIdx.x, pos = n_past + t;
        if ((int) threadIdx.x < half) {
            const float theta = rope_theta(pos, threadIdx.x, p.rope_theta_scale);
            cs[threadIdx.x] = cosf(theta); sn[threadIdx.x] = sinf(theta);
        }
        __syncthreads();
        float * row = qkv + (size_t) t * p.qkv_stride;
        for (int idx = threadIdx.x; idx < (H + HKV) * half; idx += 256) {
            const int slot = idx / half, i = idx % half;
            float * v = row + (size_t) slot * D;
            const float2 r = rope_rotate(v[i], v[i + half], cs[i], sn[i]);
            const float r0 = r.x, r1 = r.y;
            v[i] = r0; v[i + half] = r1;
            if (slot >= H) {
                const size_t o = ((size_t) pos * HKV + (slot - H)) * D;
                kv_put_k(p.kv, o + i, r0); kv_put_k(p.kv, o + i + half, r1);
            }
        }
        for (int idx = threadIdx.x; idx < HKV * D; idx += 256)         // V^T: the CTAs below
            kv_put_v_rows(p.kv, (size_t) pos * HKV * D + idx, row[(size_t) (H + HKV) * D + idx]);
    } else if (p.kv.vt16) {
        __shared__ __half sm[64][66];
        const int tile = (int) blockIdx.x - N, tt = tile / HKV, kvh = tile % HKV;
        for (int idx = threadIdx.x; idx < 64 * 64; idx += 256) {
            const int tl = idx >> 6, d = idx & 63, t = tt * 64 + tl;
            sm[tl][d] = t < N ? __float2half_rn(qkv[(size_t) t * p.qkv_stride + (size_t) (H + HKV + kvh) * 64 + d]) : __float2half_rn(0.f);
        }
        __syncthreads();
        for (int idx = threadIdx.x; idx < 64 * 64; idx += 256) {
            const int d = idx >> 6, tl = idx & 63, t = tt * 64 + tl;
            if (t < N) p.kv.vt16[((size_t) kvh * 64 + d) * p.kv.ctx_pad + n_past + t] = sm[tl][d];
        }
    }
}

void launch_rope_kv_append(float * qkv, const AttnParams & p, cudaStream_t stream) {
    if (p.n_tok <= 0) return;
    if (p.n_tok > 1 && p.head_dim <= 128 && (!p.kv.vt16 || p.head_dim == 64)) {
        const unsigned grid = (unsigned) (p.n_tok + (p.kv.vt16 ? (p.n_tok + 63) / 64 * p.n_head_kv : 0));
        rope_kv_append_batch_kernel<<<grid, 256, 0, stream>>>(qkv, p);
        B200_CUDA_CHECK(cudaGetLastError());
        return;
    }
    dim3 grid((unsigned) (p.n_head + 2 * p.n_head_kv), (unsigned) p.n_tok);
    static bool set = false;
    if (!set) { B200_CUDA_CHECK(cudaFuncSetAttribute(rope_kv_append_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, B200_CARVEOUT)); set = true; }
    rope_kv_append_kernel<<<grid, p.head_dim / 2, 0, stream>>>(qkv, p);
    B200_CUDA_CHECK(cudaGetLastError());
}

// ---------------------------------------------------------------------------------------------- greedy sampling
// arg-max of one logits row; ties -> lowest index (what a sequential `if (x > best)` scan returns).  Graph-replayable: the id also goes
// to hist[*step], and the step counter advances
__global__ void __launch_bounds__(1024) argmax_hist_kernel(const float * __restrict__ x, int n, int32_t * __restrict__ out, int32_t * __restrict__ hist, int * __restrict__ step) {
    __shared__ float sv[32]; __shared__ int si[32];
    float best = -INFINITY; int bi = 0x7fffffff;
    for (int i = threadIdx.x; i < n; i += blockDim.x) { const float v = x[i]; if (v > best || (v == best && i < bi)) { best = v; bi = i; } }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = best; si[threadIdx.x >> 5] = bi; }
    __syncthreads();
    if (threadIdx.x < 32) {
        best = sv[threadIdx.x]; bi = si[threadIdx.x];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, best, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
        }
        if (threadIdx.x == 0) { *out = bi; const int k = *step; hist[k] = bi; *step = k + 1; }
    }
}
void launch_argmax_hist(const float * x, int n, int32_t * out, int32_t * hist, int * step, cudaStream_t stream) {
    argmax_hist_kernel<<<1, 1024, 0, stream>>>(x, n, out, hist, step);
    B200_CUDA_CHECK(cudaGetLastError());
}
