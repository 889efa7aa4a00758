// mmv_fast.cu -- the decode mat-vec for the types the BASELINE configs use (Q4_K, Q4_0), tuned for issue slots.
//
// Profiling the generic ring kernel showed the mat-vec is NOT limited by HBM latency but
// by instruction issue and the L1/shared-memory data path: 101 warp-instructions per 512 B of weights, most of them
// address arithmetic, nibble shifts, 6-bit scale unpacking and shared-memory reads of the activation.  This kernel
// removes them instead of hiding them:
//   * the activation lives in REGISTERS.  Thread t of a CTA always handles the same 16-byte "piece" position of a
//     row (piece g = j*NT + t), so the 32 activation codes, their block sums and scale that piece needs are loaded
//     once (TMA bulk copy global->shared, then one read into registers) and reused for every row the CTA owns
//   * weights go HBM -> registers with one coalesced 16-byte ld.global.nc per piece (a warp reads 512 contiguous
//     bytes of the row), double-buffered: the next group of rows is in flight while the current one is computed
//   * high nibbles are dotted in place (x16, exact) instead of shifted; the four 6-bit scale/min values of a
//     sub-block pair come pre-expanded in one 32-bit word and are applied with two dp2a
//   * the K dimension is split across the warps of the CTA; G rows are reduced together with a transposing
//     butterfly (6 shuffles per 4 rows) and a fixed-order sum over warps through shared memory -> deterministic
// Arithmetic is identical to mmv.cu / the CPU's integer block dots (ggml.c:2591-2609, k_quants.c:1999-2055).
#include "kernels.h"

#include "mmv_fast.cuh"

// D = rows in flight per thread (register ring), reduced G = min(D, 4) rows at a time.  D * J = 8 pieces = 192 B in
// flight per thread at all times (>= 96 KB per SM): the ring is refilled one row at a time, right after that row's
// slot has been consumed, so the depth never drops while a group is being computed.
// Shared memory: the activation's mbarrier, partial[2][NT / 32][4] (ring_pass), then the activation codes (TMA destination).
constexpr int xq_offset(int nt) { return 16 + 2 * (nt / 32) * 4 * 4; }

template <int TYPE, int NT, int J, int D>
// 96 registers for the 256-thread shapes: two CTAs per SM leave a quarter of the register file to the small attention
// kernels of the other stream, which then run beside ffn_up instead of after it
__global__ void __launch_bounds__(NT) __maxnreg__(NT <= 256 ? 96 : 128) mmv_fast_kernel(const WPlanes W, const ActQ A, float * __restrict__ y, int64_t y_stride, const Epi epi) {
    using T = FX<TYPE>;
    extern __shared__ __align__(16) uint8_t smem[];
    uint64_t * bar = reinterpret_cast<uint64_t *>(smem);
    float * partial = reinterpret_cast<float *>(smem + 16);
    int8_t * xq = reinterpret_cast<int8_t *>(smem + xq_offset(NT));
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cta = blockIdx.x, nctas = gridDim.x, n = blockIdx.y;
    const int P = W.nb * T::PPB;

    if (tid == 0) { mbar_init(bar, 1); mbar_fence_init(); }
    // rows [row0, row1) of this CTA, balanced to +-1
    const int per = W.M / nctas, rem = W.M % nctas;
    const int row0 = cta * per + min(cta, rem), row1 = row0 + per + (cta < rem ? 1 : 0);
    const int nrows = row1 - row0;

    int gidx[J]; bool valid[J];
    WP wp[J];
    int aux[J];
#pragma unroll
    for (int j = 0; j < J; j++) { const int g = j * NT + tid; valid[j] = g < P; gidx[j] = valid[j] ? g : P - 1; wp[j] = T::wp(W, gidx[j]); aux[j] = piece_aux<TYPE>(gidx[j]); }

    typename T::WR w[D][J];
    ring_fill<TYPE, J, D>(w, wp, row0, row1);                                // weights are in flight before the activation arrives

    // everything above touched only weights; the activation row is produced by the previous kernel(s) of the stream
    if (!epi.late_wait) asm volatile("griddepcontrol.wait;" ::: "memory");
    if (tid == 0) {
        mbar_expect_tx(bar, (uint32_t) W.K);
        tma_load_1d(xq, A.q + (size_t) n * W.K, (uint32_t) W.K, bar);       // activation codes: global -> shared by TMA
    }
    __syncthreads();                                                          // barrier initialised (thread 0 did it before issuing)
    mbar_wait(bar, 0);
    typename T::XR xr[J];
#pragma unroll
    for (int j = 0; j < J; j++) xr[j] = valid[j] ? T::load_x(xq, A, n, gidx[j]) : zero_xr<TYPE>();

    // Programmatic dependent launch: the next kernel of the stream is released once this CTA is about to issue its last
    // weight loads.  Triggering earlier would park the dependent grid's CTAs at the head of the hardware queue for the
    // whole duration of this kernel and keep the small attention kernels of the other stream from being scheduled.
    const int ekind = epi.kind; const float * r1p = epi.r1, * r2p = epi.r2;
    ring_run<TYPE, NT, J, D>(w, wp, row0, row1, xr, aux, partial, tid,
        [&](int row, float v) {
            if (ekind == EPI_GELU) v = gelu_f16lut(v);
            else if (ekind == EPI_ADD2) v = (v + r1p[(size_t) n * y_stride + row]) + r2p[(size_t) n * y_stride + row];
            y[(size_t) n * y_stride + row] = v;
        },
        [&]() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); });
    if (epi.late_wait) asm volatile("griddepcontrol.wait;" ::: "memory");      // see MmvEpilogue::late_wait
    if (epi.qctr) {
        // Quantise the finished output row for the next mat-mul, 256 values at a time.  A chunk's rows belong to up to
        // three CTAs; each adds its row count to the chunk's counter once its own rows are stored and fenced, and the CTA
        // that completes the count quantises the chunk (one warp) and re-arms the counter for the next launch.
        __shared__ int s_do;
        __threadfence();
        __syncthreads();
        if (nrows > 0) {
            for (int b = row0 >> 8; b <= (row1 - 1) >> 8; b++) {
                if (tid == 0) {
                    const unsigned cnt = (unsigned) (min(row1, (b + 1) << 8) - max(row0, b << 8));
                    const unsigned old = atomicAdd(epi.qctr + b, cnt);
                    s_do = old + cnt == 256u;
                    if (s_do) epi.qctr[b] = 0;
                }
                __syncthreads();
                if (s_do && warp == 0) {
                    __threadfence();
                    const float * src = y + (size_t) n * y_stride + (b << 8) + lane * 8;
                    const float4 p = __ldcg(reinterpret_cast<const float4 *>(src)), q = __ldcg(reinterpret_cast<const float4 *>(src) + 1);
                    const float v[8] = { p.x, p.y, p.z, p.w, q.x, q.y, q.z, q.w };
                    if (epi.qA.type == T_Q8_K) quantize_chunk8<T_Q8_K>(v, lane, epi.qA, n, (b << 8) + lane * 8);
                    else quantize_chunk8<T_Q8_0>(v, lane, epi.qA, n, (b << 8) + lane * 8);
                }
                __syncthreads();
            }
        }
    }
}

template <int TYPE, int NT, int J, int D>
static void launch_cfg(const WPlanes & W, const ActQ & A, float * y, int64_t y_stride, Epi epi, cudaStream_t stream) {
    const size_t smem = xq_offset(NT) + (size_t) ((W.K + 15) & ~15);
    static bool set = false;
    if (!set) { B200_CUDA_CHECK(cudaFuncSetAttribute(mmv_fast_kernel<TYPE, NT, J, D>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
        // same L1/shared split as the small kernels of the other stream: an SM cannot host kernels with different carve-outs at once
        B200_CUDA_CHECK(cudaFuncSetAttribute(mmv_fast_kernel<TYPE, NT, J, D>, cudaFuncAttributePreferredSharedMemoryCarveout, B200_CARVEOUT)); set = true; }
    int ctas = num_sms() * (NT == 128 ? 4 : NT == 160 || NT == 192 ? 3 : NT == 256 ? 2 : 1);
    if (ctas > (W.M + 3) / 4) ctas = (W.M + 3) / 4;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned) ctas, (unsigned) A.N); cfg.blockDim = dim3(NT); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;          // PDL: may start while the previous kernel of the stream drains
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    B200_CUDA_CHECK(cudaLaunchKernelEx(&cfg, mmv_fast_kernel<TYPE, NT, J, D>, W, A, y, y_stride, epi));
}

// The launch shape (NT threads, J pieces per thread, ring depth D) for a row of K weights;
// nt == 0: not covered, the caller uses the generic ring kernel of mmv.cu
template <int TYPE>
static MmvShape pick_shape_t(int K) {
    const int P = K / (TYPE == T_Q4_0 ? 32 : 256) * FX<TYPE>::PPB;
    if (K > 64 * 1024) return {};
    constexpr int D1 = FX<TYPE>::D256;                        // ring depth for one piece per thread; D * J stays constant
    if (P <= 128 && D1 == 4) return { 128, 1, D1 };                                        // 64-weight pieces (Q3_K): K = 8192 is 128 pieces
    if (P > 128 && P <= 160 && D1 == 8) return { 160, 1, D1 };                             // Falcon-7B: K = 4544 is 142 pieces
    if (P <= 256) return { 256, 1, D1 };
    // Falcon-180B (K = 14848: 464 pieces): two 256-thread CTAs at 96 registers instead of one 512-thread CTA at 128 leave a quarter of the
    // register file to the attention kernels of the other stream, as the K = 8192 shape does
    if (P > 256 && P <= 512 && D1 == 8) return { 256, 2, D1 / 2 };
    if (P <= 512) return { 512, 1, D1 };
    // Falcon-7B's ffn_down (K = 18176: 568 pieces): 3 pieces per thread of a 192-thread CTA use 568 of 576 slots; the 512 x 2 shape
    // below would leave 45 % of its lanes without a piece (and its 128-register CTAs own the whole register file)
    if (P > 512 && P <= 576 && D1 == 8) return { 192, 3, 2 };
    if (P <= 1024) return { 512, 2, D1 / 2 };
    if (P <= 2048 && D1 == 8) return { 512, 4, 2 };
    return {};
}

MmvShape mmv_fast_pick_shape(int wtype, int K) {
    switch (wtype) {
        case T_Q4_K: return pick_shape_t<T_Q4_K>(K);
        case T_Q4_0: return pick_shape_t<T_Q4_0>(K);
        case T_Q3_K: return pick_shape_t<T_Q3_K>(K);
    }
    return {};
}

// exactly the shapes pick_shape_t<TYPE> returns are instantiated
template <int TYPE>
static void launch_type(const MmvShape & s, const WPlanes & W, const ActQ & A, float * y, int64_t y_stride, Epi epi, cudaStream_t stream) {
    static_assert(FX<TYPE>::D256 == 8 || FX<TYPE>::D256 == 4, "pick_shape_t knows ring depths 8 and 4");
    if constexpr (FX<TYPE>::D256 == 8) {                                     // Q4_K, Q4_0
        if (s.nt == 160 && s.j == 1) launch_cfg<TYPE, 160, 1, 8>(W, A, y, y_stride, epi, stream);
        else if (s.nt == 256 && s.j == 1) launch_cfg<TYPE, 256, 1, 8>(W, A, y, y_stride, epi, stream);
        else if (s.nt == 256 && s.j == 2) launch_cfg<TYPE, 256, 2, 4>(W, A, y, y_stride, epi, stream);
        else if (s.nt == 192 && s.j == 3) launch_cfg<TYPE, 192, 3, 2>(W, A, y, y_stride, epi, stream);
        else if (s.nt == 512 && s.j == 2) launch_cfg<TYPE, 512, 2, 4>(W, A, y, y_stride, epi, stream);
        else if (s.nt == 512 && s.j == 4) launch_cfg<TYPE, 512, 4, 2>(W, A, y, y_stride, epi, stream);
        else B200_ASSERT(!"mmv_fast: no kernel for this launch shape");
    } else {                                                                 // Q3_K
        if (s.nt == 128 && s.j == 1) launch_cfg<TYPE, 128, 1, 4>(W, A, y, y_stride, epi, stream);
        else if (s.nt == 256 && s.j == 1) launch_cfg<TYPE, 256, 1, 4>(W, A, y, y_stride, epi, stream);
        else if (s.nt == 512 && s.j == 1) launch_cfg<TYPE, 512, 1, 4>(W, A, y, y_stride, epi, stream);
        else if (s.nt == 512 && s.j == 2) launch_cfg<TYPE, 512, 2, 2>(W, A, y, y_stride, epi, stream);
        else B200_ASSERT(!"mmv_fast: no kernel for this launch shape");
    }
}

// returns false if the shape / type is not covered (the caller then uses the generic ring kernel of mmv.cu)
bool launch_mmv_fast(const WPlanes & W, const ActQ & A, float * y, int64_t y_stride, MmvEpilogue e, cudaStream_t stream) {
    Epi epi{};
    epi.kind = e.kind; epi.r1 = e.r1; epi.r2 = e.r2; epi.late_wait = e.late_wait;
    if (e.qout && e.qctr) {
        B200_ASSERT(A.N == 1 && W.M % 256 == 0 && e.qout->K == W.M && (e.qout->type == T_Q8_K || e.qout->type == T_Q8_0));
        epi.qA = *e.qout; epi.qctr = e.qctr;
    }
    const MmvShape s = mmv_fast_pick_shape(W.type, W.K);
    if (!s.nt) return false;
    switch (W.type) {
        case T_Q4_K: launch_type<T_Q4_K>(s, W, A, y, y_stride, epi, stream); break;
        case T_Q4_0: launch_type<T_Q4_0>(s, W, A, y, y_stride, epi, stream); break;
        case T_Q3_K: launch_type<T_Q3_K>(s, W, A, y, y_stride, epi, stream); break;
    }
    return true;
}
// Which (type, K) the fused single-stream decode path of engine.cu may rely on.  Q3_K has a fast mat-vec (used through
// launch_mmv) but is NOT listed: its kernel is issue-bound, and the two-stream per-node path, which runs the attention and
// MLP branches' mat-vecs concurrently, is faster for it (Falcon-40B).
bool mmv_fast_supports(int wtype, int K) {
    return (wtype == T_Q4_K || wtype == T_Q4_0) && K <= 64 * 1024;
}
// true when the shape chosen for W (3 CTAs of 192 threads at 96 registers) leaves no room on an SM for a side-stream kernel:
// the decode step then schedules wo BEFORE this mat-vec (engine.cu).  The 512-thread shapes leave ~14k registers: one attention CTA fits.
bool mmv_fast_fills_sm(const WPlanes & W) {
    if (W.type != T_Q4_K && W.type != T_Q4_0) return false;
    const int P = W.K / 32;
    return P > 512 && P <= 576;
}
