// actquant.cu -- activation quantisation to the weight type's "vec_dot_type" (Q8_0 / Q8_1 / Q8_K).
//
// This is the INIT pass of the CPU mat-mul (ggml_compute_forward_mul_mat_q_f32, ggml.c:11462-11476), which the
// reference CUDA kernels skip (they multiply fp32 activations).  Reproducing it makes the GPU mat-vec compute the
// same integer block dots as the CPU oracle, and shrinks the activation tile staged in shared memory 4x.
// Codes and scales are bit-exact with the CPU (tests/test_actq_edges_gpu.py, on ties, half-way products and clamps):
//   Q8_K : quantize_row_q8_K_reference, k_quants.c:899-934 (iscale = -128/max, round-half-even, min(127,.))
//   Q8_0 : the AVX/AVX2 body an x86 host runs, ggml.c:1201-1237 (id = 127/amax, round-half-even, d -> fp16)
//   Q8_1 : ggml.c:1421-1470 (same, d kept in fp32, s = d * sum(q))
#include "kernels.h"
#include "actquant.cuh"

size_t actq_bytes(int t, int K, int N) {
    const int blk = act_block(t);
    size_t b = round_up((size_t) N * K, 256);                       // q
    b += round_up((size_t) N * (K / blk) * 4, 256);                 // d
    if (t == T_Q8_1) b += round_up((size_t) N * (K / 32) * 4, 256); // s
    b += round_up((size_t) N * (K / (t == T_Q8_K ? 16 : 32)) * 2, 256); // bsums (Q8_K: per 16 codes; Q8_0/1: per block)
    return b;
}
void actq_bind(ActQ & A, int t, int K, int N, void * base) {
    const int blk = act_block(t);
    uint8_t * p = (uint8_t *) base;
    A.type = t; A.K = K; A.N = N;
    A.q = (int8_t *) p; p += round_up((size_t) N * K, 256);
    A.d = (float *) p;  p += round_up((size_t) N * (K / blk) * 4, 256);
    A.s = nullptr; A.bs = nullptr; A.h = nullptr;
    if (t == T_Q8_1) { A.s = (float *) p; p += round_up((size_t) N * (K / 32) * 4, 256); }
    A.bs = (int16_t *) p;
}

template <int TYPE>
__global__ void __launch_bounds__(256) quantize_act_kernel(const float * __restrict__ x, int64_t x_stride, ActQ A) {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const int lane = threadIdx.x & 31;
    const int64_t chunk = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x);     // index of this lane's 8-value chunk
    const int64_t chunks_per_row = A.K / 8;
    if (chunk >= chunks_per_row * A.N) return;                       // K % 32 == 0, so whole blocks drop out together
    const int n = (int) (chunk / chunks_per_row);
    const int k0 = (int) (chunk % chunks_per_row) * 8;
    const float4 a = *reinterpret_cast<const float4 *>(x + n * x_stride + k0);
    const float4 b = *reinterpret_cast<const float4 *>(x + n * x_stride + k0 + 4);
    const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    quantize_chunk8<TYPE>(v, lane, A, n, k0);
}

void launch_quantize_act(const float * x, int64_t x_stride, const ActQ & A, cudaStream_t stream) {
    B200_ASSERT(A.K % act_block(A.type) == 0);
    const int64_t chunks = (int64_t) A.N * A.K / 8;
    const unsigned grid = (unsigned) ((chunks + 255) / 256);
    if (grid == 0) return;
    switch (A.type) {
        case T_Q8_0: quantize_act_kernel<T_Q8_0><<<grid, 256, 0, stream>>>(x, x_stride, A); break;
        case T_Q8_1: quantize_act_kernel<T_Q8_1><<<grid, 256, 0, stream>>>(x, x_stride, A); break;
        case T_Q8_K: quantize_act_kernel<T_Q8_K><<<grid, 256, 0, stream>>>(x, x_stride, A); break;
        default: B200_ASSERT(!"bad activation type");
    }
    B200_CUDA_CHECK(cudaGetLastError());
}

// GEMM B-operand: the dequantised activation d*q rounded to fp16 (exact for the int8 code, one rounding for the product)
__global__ void actq_to_f16_kernel(ActQ A, __half * __restrict__ dst, int64_t dst_stride, int blk) {
    const int64_t i = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) * 8;
    if (i >= (int64_t) A.N * A.K) return;
    const int n = (int) (i / A.K), k0 = (int) (i % A.K);
    const uint2 c = *reinterpret_cast<const uint2 *>(A.q + (size_t) n * A.K + k0);
    const float d = A.d[(size_t) n * (A.K / blk) + k0 / blk];
    __half h[8];
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const int8_t qv = (int8_t) ((j < 4 ? c.x >> (8 * j) : c.y >> (8 * (j - 4))) & 0xff);
        h[j] = __float2half_rn(__fmul_rn(d, (float) qv));
    }
    *reinterpret_cast<uint4 *>(dst + (size_t) n * dst_stride + k0) = *reinterpret_cast<const uint4 *>(h);
}
void launch_actq_to_f16(const ActQ & A, __half * dst, int64_t dst_stride, cudaStream_t stream) {
    const int64_t chunks = (int64_t) A.N * A.K / 8;
    if (chunks == 0) return;
    actq_to_f16_kernel<<<(unsigned) ((chunks + 255) / 256), 256, 0, stream>>>(A, dst, dst_stride, act_block(A.type));
    B200_CUDA_CHECK(cudaGetLastError());
}
