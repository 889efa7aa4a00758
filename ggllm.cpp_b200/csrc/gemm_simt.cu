// gemm_simt.cu -- plain CUDA-core tiled GEMM with on-the-fly dequantisation.
//
// NOT the product path for the prompt mat-mat: it exists (a) as the first correct implementation of
// Y[n][m] = sum_k fp16(W[m][k]) * X_f16[n][k] against which the wgmma kernel (gemm_tc.cu) is bit-compared in the
// tests, and (b) as the N-tail handler for shapes the tensor-core tiling does not cover.  Same operand rounding
// as the tensor-core kernel: weights dequantised bit-exactly to fp32 then rounded once to fp16, activations fp16,
// fp32 accumulation.
#include "kernels.h"

#define TS 64      // tile of 64 (m) x 64 (n)
#define KS 32

__global__ void __launch_bounds__(256) gemm_simt_kernel(const WPlanes W, const __half * __restrict__ X, int64_t x_stride, int N,
                                                       float * __restrict__ Y, int64_t y_stride, int epi_gelu) {
    __shared__ float ws[KS][TS + 1];
    __shared__ float xs[KS][TS + 1];
    const int m0 = blockIdx.x * TS, n0 = blockIdx.y * TS;
    const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;       // thread computes m = m0 + tx*4.., n = n0 + ty*4..
    float acc[4][4] = {};
    for (int k0 = 0; k0 < W.K; k0 += KS) {
        for (int i = threadIdx.x; i < TS * KS; i += 256) {
            const int r = i / KS, k = i % KS;
            const int m = m0 + r, n = n0 + r;
            ws[k][r] = m < W.M ? __half2float(__float2half_rn(dequant_elem(W, (size_t) m, k0 + k))) : 0.f;
            xs[k][r] = n < N ? __half2float(X[(size_t) n * x_stride + k0 + k]) : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int k = 0; k < KS; k++) {
            float a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; i++) { a[i] = ws[k][tx * 4 + i]; b[i] = xs[k][ty * 4 + i]; }
#pragma unroll
            for (int j = 0; j < 4; j++)
#pragma unroll
                for (int i = 0; i < 4; i++) acc[j][i] += a[i] * b[j];
        }
        __syncthreads();
    }
    for (int j = 0; j < 4; j++) {
        const int n = n0 + ty * 4 + j;
        if (n >= N) continue;
        for (int i = 0; i < 4; i++) {
            const int m = m0 + tx * 4 + i;
            if (m < W.M) {
                float v = acc[j][i];
                if (epi_gelu) v = gelu_f16lut(v);
                Y[(size_t) n * y_stride + m] = v;
            }
        }
    }
}

void launch_gemm_simt(const WPlanes & W, const __half * X, int64_t x_stride, int N, float * Y, int64_t y_stride, int epi_gelu, cudaStream_t stream) {
    if (N <= 0) return;
    dim3 grid((unsigned) ((W.M + TS - 1) / TS), (unsigned) ((N + TS - 1) / TS));
    gemm_simt_kernel<<<grid, 256, 0, stream>>>(W, X, x_stride, N, Y, y_stride, epi_gelu);
    B200_CUDA_CHECK(cudaGetLastError());
}
