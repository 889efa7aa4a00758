// weights.cu -- device residency of quantised weight matrices: upload + AoS->planar repack, row dequantisation.
//
// Replaces ggml_cuda_transform_tensor's blocking per-tensor cudaMemcpy of raw blocks (ggml-cuda.cu:3030-3073)
// and the dequantize_block_* family (ggml-cuda.cu:318-473, 1084-1100) -- the latter only as a standalone
// checker / get_rows producer; in the hot path dequantisation is fused into the mat-vec and GEMM kernels.
#include "formats.cuh"
#include "kernels.h"

size_t wplanes_layout(WPlanes & W, int type, int K, int M) {
    const TypeSpec ts = type_spec(type);
    B200_ASSERT(ts.blk_elems > 0 && K % ts.blk_elems == 0);
    W.type = type; W.K = K; W.M = M; W.nb = K / ts.blk_elems;
    size_t off = 0;
    for (int i = 0; i < B200_MAX_PLANES; i++) {
        if (i < ts.n_planes) {
            W.stride[i] = (uint32_t) round_up((size_t) W.nb * ts.plane[i].bytes, 16);
            W.p[i] = reinterpret_cast<uint8_t *>(off);      // offsets for now; rebased by the caller
            off += round_up((size_t) W.stride[i] * M, 256);
        } else { W.stride[i] = 0; W.p[i] = nullptr; }
    }
    W.bytes = off;
    return off;
}

// one thread per (row, block): scatter the block's fields into their planes
__global__ void repack_kernel(const uint8_t * __restrict__ src, WPlanes W, TypeSpec ts, int64_t row0, int64_t nrows) {
    const int64_t idx = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= nrows * W.nb) return;
    const int64_t r = idx / W.nb; const int b = (int) (idx % W.nb);
    const uint8_t * s = src + (size_t) idx * ts.blk_bytes;
    for (int p = 0; p < ts.n_planes; p++) {
        uint8_t * d = W.p[p] + (size_t) (row0 + r) * W.stride[p] + (size_t) b * ts.plane[p].bytes;
        const uint8_t * f = s + ts.plane[p].src_off;
        if (ts.plane[p].kind == 1) {                      // expand the 6-bit (scale, min) pairs, see PlaneSpec
            for (int pr = 0; pr < 4; pr++) {
                int s0, m0, s1, m1; unpack_sm6(2 * pr, f, s0, m0); unpack_sm6(2 * pr + 1, f, s1, m1);
                d[4 * pr] = (uint8_t) s0; d[4 * pr + 1] = (uint8_t) s1; d[4 * pr + 2] = (uint8_t) m0; d[4 * pr + 3] = (uint8_t) m1;
            }
        } else if (ts.plane[p].kind == 2) {               // Q3_K scales, see PlaneSpec
            for (int j = 0; j < 16; j++) d[4 * (2 * (j >> 3) + (j & 1)) + ((j >> 1) & 3)] = (uint8_t) (int8_t) (q3_scale(f, j) - 32);
        } else for (int i = 0; i < ts.plane[p].bytes; i++) d[i] = f[i];
    }
}

// Points the planes of a laid-out (or already placed) matrix at `base`, one allocation of W.bytes, keeping their offsets.
void wplanes_place(WPlanes & W, uint8_t * base) {
    const int n = type_spec(W.type).n_planes;
    const uint8_t * p0 = W.p[0];
    for (int i = n - 1; i >= 0; i--) W.p[i] = base + (size_t) (W.p[i] - p0);
}

static void wplanes_alloc(WPlanes & W, int type, int K, int M) {
    wplanes_layout(W, type, K, M);
    uint8_t * base = nullptr;
    B200_CUDA_CHECK(cudaMalloc(&base, W.bytes));
    wplanes_place(W, base);
}

// Fill a placed matrix from `M` rows of raw ggml blocks (host pointer, row-major, rows of K/blk blocks), in planar form.  Staged
// through a bounded device scratch so a 100 GB model never needs 2x its size.
void wplanes_fill(const WPlanes & W, const void * host_raw, cudaStream_t stream) {
    const TypeSpec ts = type_spec(W.type);
    const size_t M = (size_t) W.M;
    const size_t row_bytes = (size_t) W.nb * ts.blk_bytes;
    if (ts.n_planes == 1) {   // f32 / f16: rows are already planar; strided copy handles the 16 B row padding
        B200_CUDA_CHECK(cudaMemcpy2DAsync(W.p[0], W.stride[0], host_raw, row_bytes, row_bytes, M, cudaMemcpyHostToDevice, stream));
        B200_CUDA_CHECK(cudaStreamSynchronize(stream));
        return;
    }
    const size_t chunk_rows = (256u << 20) / row_bytes > 0 ? (256u << 20) / row_bytes : 1;
    uint8_t * stage = nullptr;
    const size_t stage_rows = chunk_rows < M ? chunk_rows : M;
    B200_CUDA_CHECK(cudaMalloc(&stage, stage_rows * row_bytes));
    for (size_t r0 = 0; r0 < M; r0 += stage_rows) {
        const size_t nr = r0 + stage_rows <= M ? stage_rows : M - r0;
        B200_CUDA_CHECK(cudaMemcpyAsync(stage, (const uint8_t *) host_raw + r0 * row_bytes, nr * row_bytes, cudaMemcpyHostToDevice, stream));
        launch_repack_rows(W, stage, (int64_t) r0, (int64_t) nr, stream);
    }
    B200_CUDA_CHECK(cudaStreamSynchronize(stream));
    B200_CUDA_CHECK(cudaFree(stage));
}

void wplanes_upload(WPlanes & W, int type, int K, int M, const void * host_raw, cudaStream_t stream) {
    wplanes_alloc(W, type, K, M);
    if (host_raw) wplanes_fill(W, host_raw, stream);
}

// rows [row0, row0 + nrows) of an allocated matrix from their raw blocks staged on the device (the streaming loader, engine.cu)
void launch_repack_rows(const WPlanes & W, const void * stage_dev, int64_t row0, int64_t nrows, cudaStream_t stream) {
    const int64_t n = nrows * W.nb;
    if (n <= 0) return;
    repack_kernel<<<(unsigned) ((n + 255) / 256), 256, 0, stream>>>((const uint8_t *) stage_dev, W, type_spec(W.type), row0, nrows);
    B200_CUDA_CHECK(cudaGetLastError());
}

void wplanes_free(WPlanes & W) {
    if (W.p[0]) B200_CUDA_CHECK(cudaFree(W.p[0]));
    for (int i = 0; i < B200_MAX_PLANES; i++) W.p[i] = nullptr;
    W.bytes = 0;
}

// Fill the planes with pseudo-random but well-formed blocks (hash of the byte address): quant bytes uniform,
// fp16 scales in a sane range, 6-bit fields as they come.  For throughput runs on 40B/180B-sized synthetic
// models (SURVEY.md section 8d: "random blocks with sane fp16 scales ... the reference loader accepts any
// bytes"); parity runs use real quantised weights instead.
__device__ __forceinline__ uint32_t mix32(uint64_t x) {
    x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33;
    return (uint32_t) x;
}
__global__ void fill_random_kernel(WPlanes W, TypeSpec ts, uint64_t seed) {
    const int64_t total = (int64_t) W.M * W.nb;
    for (int64_t idx = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t) gridDim.x * blockDim.x) {
        const int64_t r = idx / W.nb; const int b = (int) (idx % W.nb);
        for (int p = 0; p < ts.n_planes; p++) {
            uint8_t * d = W.p[p] + (size_t) r * W.stride[p] + (size_t) b * ts.plane[p].bytes;
            const int nbytes = ts.plane[p].bytes;
            for (int i = 0; i < nbytes; i += 4) {
                uint32_t v = mix32(seed ^ (((uint64_t) idx * 8 + p) << 20) ^ (uint64_t) i);
                if (ts.plane[p].kind == 1) v &= 0x3f3f3f3fu;         // expanded 6-bit scales / mins
                if (ts.plane[p].kind == 2) v = (((v & 0x3f3f3f3fu) | 0x80808080u) - 0x20202020u) ^ 0x80808080u;   // per byte: 6-bit value - 32 as int8 (borrow-free SWAR)
                for (int k = 0; k < 4 && i + k < nbytes; k++) d[i + k] = (uint8_t) (v >> (8 * k));
            }
        }
        // overwrite the fp16 scale fields with sane magnitudes (weights end up O(1e-2))
        const uint32_t h = mix32(seed ^ 0x9e3779b97f4a7c15ULL ^ (uint64_t) idx);
        const float unit = ts.blk_elems == 256 ? 1e-4f : 2e-3f;      // K-quants multiply d by a 4..8-bit sub-scale
        const float dsm = unit * (1.f + 2.f * (float) (h & 0xffff) / 65536.f);
        const uint16_t d16 = __half_as_ushort(__float2half_rn(dsm)), m16 = __half_as_ushort(__float2half_rn(dsm * 4.f));
        auto put16 = [&](int plane, int off, uint16_t v) {
            *reinterpret_cast<uint16_t *>(W.p[plane] + (size_t) r * W.stride[plane] + (size_t) b * ts.plane[plane].bytes + off) = v;
        };
        switch (W.type) {
            case T_Q4_0: case T_Q8_0: put16(1, 0, d16); break;
            case T_Q4_1: put16(1, 0, d16); put16(1, 2, m16); break;
            case T_Q5_0: put16(2, 0, d16); break;
            case T_Q5_1: put16(2, 0, d16); put16(2, 2, m16); break;
            case T_Q2_K: put16(2, 0, d16); put16(2, 2, d16); break;
            case T_Q3_K: put16(3, 0, d16); break;
            case T_Q4_K: put16(2, 0, d16); put16(2, 2, d16); break;
            case T_Q5_K: put16(3, 0, d16); put16(3, 2, d16); break;
            case T_Q6_K: put16(3, 0, d16); break;
            case T_F16: put16(0, 0, __half_as_ushort(__float2half_rn(dsm * 10.f - 0.02f))); break;
            case T_F32: *reinterpret_cast<float *>(W.p[0] + (size_t) r * W.stride[0] + (size_t) b * 4) = dsm * 10.f - 0.02f; break;
        }
    }
}
void wplanes_fill_random(const WPlanes & W, uint64_t seed, cudaStream_t stream) {
    fill_random_kernel<<<132 * 8, 256, 0, stream>>>(W, type_spec(W.type), seed);
    B200_CUDA_CHECK(cudaGetLastError());
}
void wplanes_alloc_random(WPlanes & W, int type, int K, int M, uint64_t seed, cudaStream_t stream) {
    wplanes_alloc(W, type, K, M);
    wplanes_fill_random(W, seed, stream);
}

// dst[r][e] = dequant(W[rows[r]][e]) -- ggml_get_rows on a quantised matrix (ggml.c:11975-12002), also the
// standalone bit-exactness checker.  rows == nullptr means rows 0..nrows-1.
__global__ void dequant_rows_kernel(WPlanes W, const int32_t * __restrict__ rows, int nrows, float * __restrict__ dst, int64_t dst_stride) {
    const int r = blockIdx.y;
    // device-side row ids (token ids fed back by the on-device samplers) cannot be checked by the host: clamp into the matrix
    const size_t row = rows ? (size_t) min(max(rows[r], 0), W.M - 1) : (size_t) r;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < W.K; e += gridDim.x * blockDim.x)
        dst[(size_t) r * dst_stride + e] = dequant_elem(W, row, e);
}
void launch_dequant_rows(const WPlanes & W, const int32_t * rows_dev, int nrows, float * dst, int64_t dst_stride, cudaStream_t stream) {
    if (nrows <= 0) return;
    dim3 grid((unsigned) ((W.K + 255) / 256 < 64 ? (W.K + 255) / 256 : 64), (unsigned) nrows);
    dequant_rows_kernel<<<grid, 256, 0, stream>>>(W, rows_dev, nrows, dst, dst_stride);
    B200_CUDA_CHECK(cudaGetLastError());
}
