// gemm.cu -- prompt mat-mat dispatch: Y[n][m] = sum_k W[m][k] * X[n][k] for N > b200_mmv_max_n().
#include "kernels.h"

void launch_gemm_simt(const WPlanes & W, const __half * X, int64_t x_stride, int N, float * Y, int64_t y_stride, int epi_gelu, cudaStream_t stream);
bool launch_gemm_tc(const WPlanes & W, const __half * X, int64_t x_stride, int N, float * Y, int64_t y_stride, int epi_gelu, cudaStream_t stream);

// wgmma kernel in chunks of <= 512 tokens (it tiles the tokens by up to 256 per CTA); shapes it does not cover
// (K not a multiple of 64) go to the CUDA-core kernel
void launch_mmq_gemm(const WPlanes & W, const __half * X, int64_t x_stride, int N, float * Y, int64_t y_stride, int epi_gelu, cudaStream_t stream) {
    const bool force_simt = getenv("B200_GEMM_SIMT") != nullptr;
    for (int n0 = 0; n0 < N; n0 += 512) {
        const int n = N - n0 < 512 ? N - n0 : 512;
        if (force_simt || !launch_gemm_tc(W, X + (size_t) n0 * x_stride, x_stride, n, Y + (size_t) n0 * y_stride, y_stride, epi_gelu, stream))
            launch_gemm_simt(W, X + (size_t) n0 * x_stride, x_stride, n, Y + (size_t) n0 * y_stride, y_stride, epi_gelu, stream);
    }
}
