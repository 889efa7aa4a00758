// gemm.cu -- mat-mul dispatch: Y[n][m] = sum_k W[m][k] * X[n][k], the mat-vec for N <= MMV_MAX_N, the prompt GEMM above.
#include "kernels.h"

// wgmma kernel in chunks of <= 512 tokens (it tiles the tokens by up to 256 per CTA); shapes it does not cover
// (K not a multiple of 64) go to the CUDA-core kernel
void launch_mmq_gemm(const WPlanes & W, const __half * X, int64_t x_stride, int N, float * Y, int64_t y_stride, int epi_gelu, cudaStream_t stream) {
    for (int n0 = 0; n0 < N; n0 += 512) {
        const int n = N - n0 < 512 ? N - n0 : 512;
        if (!launch_gemm_tc(W, X + (size_t) n0 * x_stride, x_stride, n, Y + (size_t) n0 * y_stride, y_stride, epi_gelu, stream))
            launch_gemm_simt(W, X + (size_t) n0 * x_stride, x_stride, n, Y + (size_t) n0 * y_stride, y_stride, epi_gelu, stream);
    }
}

int launch_mul_mat_q(const WPlanes & W, const ActQ & A, int N, float * y, int64_t y_stride, int epi, cudaStream_t stream) {
    ActQ a = A; a.N = N;
    if (N <= MMV_MAX_N) launch_mmv(W, a, y, y_stride, { epi, nullptr, nullptr }, stream);
    else {
        B200_ASSERT(epi != EPI_ADD2 && a.h);                   // the producer of the codes wrote the fp16 operand beside them
        launch_mmq_gemm(W, a.h, W.K, N, y, y_stride, epi == EPI_GELU, stream);
    }
    return 1;
}

size_t mul_mat_scratch_bytes(const WPlanes & W, int N) {
    const int at = act_type_for(W.type);
    if (at < 0) return 0;
    return actq_bytes(at, W.K, N) + (N > MMV_MAX_N ? (size_t) N * W.K * sizeof(__half) : 0);
}

// The activation format is made on the spot for this matrix: Q8_0 / Q8_1 / Q8_K codes for a quantised one (the INIT pass of ggml's
// MUL_MAT, ggml.c:11462-11476), the rows themselves for F16 / F32 weights.
int launch_mul_mat(const WPlanes & W, const float * x, int64_t x_stride, int N, float * y, int64_t y_stride, int epi, void * scratch,
                   cudaStream_t stream) {
    if (W.type == T_F32 || W.type == T_F16) {
        launch_mmv_f(W, x, x_stride, N, y, y_stride, stream);
        if (epi != EPI_GELU) return 1;
        B200_ASSERT(y_stride == W.M);
        launch_gelu(y, y, (int64_t) N * W.M, stream);                                    // ggml.c:10298-10337
        return 2;
    }
    const int at = act_type_for(W.type);
    ActQ A; actq_bind(A, at, W.K, N, scratch);
    if (N > MMV_MAX_N) A.h = (__half *) ((uint8_t *) scratch + actq_bytes(at, W.K, N));
    launch_quantize_act(x, x_stride, A, stream);
    return 1 + launch_mul_mat_q(W, A, N, y, y_stride, epi, stream);
}
