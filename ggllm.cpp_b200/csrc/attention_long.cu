// attention_long.cu -- the tensor-core tier of the split-KV decode attention (attn_split.cuh), used above attention_long_threshold() keys.
//
// At thousands of keys attention.cu's kernels stop being hidden beside ffn_up / ffn_down; here the work is laid out differently:
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
// Against the oracle the tiny-model evals stay at the 1e-8 * S level.  Short contexts gain nothing; the decode graphs of engine.cu are
// captured per tier.
// An fp16 cache (template parameter E = __half) is already an exact mma operand: K and V rows go into the B fragments as they are, the
// split falls away on the cache side -- scores Q_hi K + Q_lo K (2 mma instead of 3), values e V (1 mma instead of 2).  Nothing is
// dropped beyond what the fp32 cache's split drops already (its lo x lo term), so the error bound of the tier is unchanged.
#include <type_traits>
#include "attn_split.cuh"

__device__ __forceinline__ void cp_async16(void * smem, const void * g) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(smem_u32(smem)), "l"(g) : "memory"); }
__device__ __forceinline__ void cp_async4(void * smem, const void * g) { asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" :: "r"(smem_u32(smem)), "l"(g) : "memory"); }
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N) : "memory"); }

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
// Ring row strides in elements.  f32: K 64 + 8 keeps the B-fragment LDS.64s of a half-warp on distinct banks, V 64 + 4 does the same for
// the LDS.32s of the second product.  fp16 (128-byte rows): K 64 + 8 puts the 32-bit word (gid, 8 t + tig) of a lane on bank
// 4 gid + tig + 8 t -- 32 distinct banks; V 64 + 8 puts the 16-bit loads (keys 2 tig (+1), dim 8 nt + gid) on banks 8 tig + gid / 2
// (+ 4), distinct per tig, lanes gid = 2 m, 2 m + 1 sharing a word; and 144-byte rows keep the 16-byte cp.async destinations aligned.
template <typename E> struct AlRing;
template <> struct AlRing<float>  { static constexpr int KS = 72, VS = 68; using E2 = float2; };
template <> struct AlRing<__half> { static constexpr int KS = 72, VS = 72; using E2 = __half2; };
__device__ __forceinline__ float al_cvt(float x, float *) { return x; }
__device__ __forceinline__ __half al_cvt(float x, __half *) { return __float2half_rn(x); }
// 8-key blocks of a split go round-robin to the warps: block b = stage * SPLIT_WARPS + warp
__device__ __forceinline__ int warp_blocks(int nk, int warp) { const int nb = (nk + AL_KB - 1) / AL_KB; return nb > warp ? (nb - warp + SPLIT_WARPS - 1) / SPLIT_WARPS : 0; }

template <typename E>
__global__ void __launch_bounds__(SPLIT_THREADS, 4) attn_long_scores_kernel(const SplitArgs a) {
    constexpr int KS = AlRing<E>::KS, CP = 16 / sizeof(E);                     // CP: elements per 16-byte copy
    __shared__ float wmax[SPLIT_WARPS][SPLIT_G];
    __shared__ __align__(16) E ring[SPLIT_WARPS][AL_KR][AL_KB][KS];           // 18 KB (f32) / 9 KB (fp16): K rows in flight
    __shared__ __align__(16) float qs[SPLIT_G][64];                           // this position's query rows, rotated
    __shared__ __align__(16) E knew_s[KS];                                    // this position's key row, rotated (not in the cache yet), as the cache holds it
    const int split = blockIdx.x, kvh = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int h0 = kvh * a.G + blockIdx.z * SPLIT_G, G = min(SPLIT_G, a.G - (int) blockIdx.z * SPLIT_G);      // this CTA's query heads: h0 .. h0 + G - 1
    const int n_past = a.n_past_dev ? *a.n_past_dev : a.n_past, T = n_past + 1;
    int k_lo, k_hi; split_range(T, a.n_splits, split, k_lo, k_hi);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // the values kernel may take its place on the SMs now (it waits for this grid to finish)
    // RoPE work of thread t: pair i = t % 32 (elements i, i + 32) of heads t / 32 + 4 r and, for t < 32, of the key row.  The rows do not
    // depend on n_past: their loads are in flight while the device scalar arrives.
    const int ri = tid & 31, rh = tid >> 5;
    float qa[SPLIT_G / SPLIT_WARPS], qb[SPLIT_G / SPLIT_WARPS];
#pragma unroll
    for (int r = 0; r < SPLIT_G / SPLIT_WARPS; r++) {
        const int h = rh + SPLIT_WARPS * r;
        const float * src = a.qkv + (size_t) (h0 + min(h, G - 1)) * 64;
        qa[r] = src[ri]; qb[r] = src[ri + 32];
    }
    const float * ksrc = a.qkv + (size_t) (a.n_head + kvh) * 64;
    const float ka = ksrc[ri], kb_ = ksrc[ri + 32];
    if (k_lo >= k_hi) return;                                   // a split without keys (short context): nothing to score, nobody reads its pmax
    const int nk = k_hi - k_lo, nst = warp_blocks(nk, warp);
    const int j_new = a.fuse_rope ? n_past - k_lo : -1;           // this position's key is not in the cache yet (another CTA may be writing it right now)
    const size_t kv_row = (size_t) a.n_head_kv * 64;
    const int gid = lane >> 2, tig = lane & 3;
    const E * kp = kv_k<E>(a.kv) + (size_t) kvh * 64 + 16 * tig + (size_t) k_lo * kv_row;
    auto issue = [&](int i) {                                     // lane copies dims 16 tig .. 16 tig + 15 of key gid of the block
        if (i < nst) {
            const int jj = (i * SPLIT_WARPS + warp) * AL_KB + gid;
            if (jj < nk && jj != j_new) {
                E * dst = &ring[warp][i % AL_KR][gid][16 * tig];
                const E * src = kp + (size_t) jj * kv_row;
#pragma unroll
                for (int c = 0; c < 16 / CP; c++) cp_async16(dst + CP * c, src + CP * c);
            }
        }
        cp_async_commit();
    };
#pragma unroll
    for (int i = 0; i < AL_KR - 1; i++) issue(i);                // the first rows travel while RoPE runs
    // Fused RoPE + KV append (libfalcon.cpp:2229-2281)
    {
        float c = 1.f, sn = 0.f;
        if (a.fuse_rope) {
            const float th = rope_theta(n_past, ri, a.theta_scale);
            c = cosf(th); sn = sinf(th);
        }
        auto rot = [&](float x0, float x1, float & y0, float & y1) {
            if (a.fuse_rope) { const float2 r = rope_rotate(x0, x1, c, sn); y0 = r.x; y1 = r.y; }
            else { y0 = x0; y1 = x1; }
        };
#pragma unroll
        for (int r = 0; r < SPLIT_G / SPLIT_WARPS; r++) {
            const int h = rh + SPLIT_WARPS * r;
            float y0, y1; rot(qa[r], qb[r], y0, y1);
            qs[h][ri] = h < G ? y0 : 0.f; qs[h][ri + 32] = h < G ? y1 : 0.f;
        }
        if (a.fuse_rope && warp == 0) {
            float y0, y1; rot(ka, kb_, y0, y1);
            knew_s[ri] = al_cvt(y0, (E *) nullptr); knew_s[ri + 32] = al_cvt(y1, (E *) nullptr);
            if (blockIdx.z == 0 && n_past >= k_lo && n_past < k_hi) {                                                  // one warp appends K and V to the cache
                const size_t o = ((size_t) n_past * a.n_head_kv + kvh) * 64;
                const float * vsrc = a.qkv + (size_t) (a.n_head + a.n_head_kv + kvh) * 64;
                const float v0 = vsrc[ri], v1 = vsrc[ri + 32];
                kv_put_k(a.kv, o + ri, y0); kv_put_k(a.kv, o + ri + 32, y1);
                kv_put_v(a.kv, o + ri, kvh, ri, n_past, v0); kv_put_v(a.kv, o + ri + 32, kvh, ri + 32, n_past, v1);
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
        const int jj0 = (i * SPLIT_WARPS + warp) * AL_KB;
        const E * krow = jj0 + gid == j_new ? knew_s : &ring[warp][i % AL_KR][gid][0];     // B column gid = key jj0 + gid
        float c[4] = { 0.f, 0.f, 0.f, 0.f };
#pragma unroll
        for (int t = 0; t < 4; t++) {
            if constexpr (std::is_same<E, float>::value) {
                const float2 p0 = *reinterpret_cast<const float2 *>(krow + 16 * t + 2 * tig), p1 = *reinterpret_cast<const float2 *>(krow + 16 * t + 2 * tig + 8);
                uint32_t bh0, bl0, bh1, bl1;
                split_h2(p0.x, p0.y, bh0, bl0); split_h2(p1.x, p1.y, bh1, bl1);
                mma_16816(c, ah[t], bh0, bh1); mma_16816(c, ah[t], bl0, bl1); mma_16816(c, al[t], bh0, bh1);
            } else {
                const uint32_t b0 = *reinterpret_cast<const uint32_t *>(krow + 16 * t + 2 * tig), b1 = *reinterpret_cast<const uint32_t *>(krow + 16 * t + 2 * tig + 8);
                mma_16816(c, ah[t], b0, b1); mma_16816(c, al[t], b0, b1);
            }
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
        for (int w = 1; w < SPLIT_WARPS; w++) mx = fmaxf(mx, wmax[w][tid]);
        a.pmax[(size_t) (h0 + tid) * SPLIT_MAX + split] = mx;
    }
}

template <typename E>
__global__ void __launch_bounds__(SPLIT_THREADS, 4) attn_long_values_kernel(const SplitArgs a) {
    constexpr int VS = AlRing<E>::VS, CP = 16 / sizeof(E);
    using E2 = typename AlRing<E>::E2;
    // V rows in flight; once a warp has consumed its rows the same memory holds its partial outputs [head][64] (sized for the larger use)
    constexpr int RING2 = AL_KR * AL_KB * VS * (int) sizeof(E) / 8, WS = RING2 > SPLIT_G * 32 ? RING2 : SPLIT_G * 32;
    __shared__ __align__(16) float2 vring[SPLIT_WARPS][WS];
    __shared__ float sring[SPLIT_WARPS][AL_KR][32][4];                // the scores of those rows, lane-private: (gid, 2 tig), (gid, 2 tig + 1), (gid + 8, ..)
    __shared__ float gmax[SPLIT_G];
    __shared__ double dsum[SPLIT_WARPS][SPLIT_G];
    const int split = blockIdx.x, kvh = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int h0 = kvh * a.G + blockIdx.z * SPLIT_G, G = min(SPLIT_G, a.G - (int) blockIdx.z * SPLIT_G);
    const int n_past = a.n_past_dev ? *a.n_past_dev : a.n_past, T = n_past + 1;
    int k_lo, k_hi; split_range(T, a.n_splits, split, k_lo, k_hi);
    const int nk = k_hi - k_lo, nst = warp_blocks(nk, warp);
    const size_t kv_row = (size_t) a.n_head_kv * 64;
    const int n_used = splits_used(T, a.n_splits);                // splits 0 .. n_used - 1 hold keys
    const int j_new = n_past - k_lo;                              // this position's V row is appended by the scores kernel: read after the wait
    const int gid = lane >> 2, tig = lane & 3;
    const E * vp = kv_v<E>(a.kv) + (size_t) kvh * 64 + 16 * tig + (size_t) k_lo * kv_row;
    const float * S0 = a.S + (size_t) (h0 + min(gid, G - 1)) * a.n_ctx + k_lo, * S1 = a.S + (size_t) (h0 + min(gid + 8, G - 1)) * a.n_ctx + k_lo;
    E (*vr)[AL_KB][VS] = reinterpret_cast<E (*)[AL_KB][VS]>(vring[warp]);
    auto issue = [&](int i, bool v, bool s) {
        if (i < nst) {
            const int jj0 = (i * SPLIT_WARPS + warp) * AL_KB;
            if (v) {                                              // lane copies dims 16 tig .. + 15 of key gid; rows past the end are zeroed (0 x garbage could be NaN)
                const int jj = jj0 + gid;
                E * dst = &vr[i % AL_KR][gid][16 * tig];
                if (jj < nk && jj != j_new) {
                    const E * src = vp + (size_t) jj * kv_row;
#pragma unroll
                    for (int c = 0; c < 16 / CP; c++) cp_async16(dst + CP * c, src + CP * c);
                } else if (jj >= nk) {
#pragma unroll
                    for (int c = 0; c < 16 / CP; c++) *reinterpret_cast<float4 *>(dst + CP * c) = make_float4(0.f, 0.f, 0.f, 0.f);
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
    E2 vnew{};
    if (has_new) vnew = *reinterpret_cast<const E2 *>(kv_v<E>(a.kv) + (size_t) kvh * 64 + 2 * lane + (size_t) (k_lo + j_new) * kv_row);
    if (tid < SPLIT_G) {
        float mx = -INFINITY;
        if (tid < G) for (int s = 0; s < n_used; s++) mx = fmaxf(mx, a.pmax[(size_t) (h0 + tid) * SPLIT_MAX + s]);
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
        const int jj0 = (i * SPLIT_WARPS + warp) * AL_KB, st = i % AL_KR;
        if (has_new && j_new >= jj0 && j_new < jj0 + AL_KB) {     // this position's V row goes into its ring row now
            *reinterpret_cast<E2 *>(&vr[st][j_new - jj0][2 * lane]) = vnew;
            __syncwarp();
        }
        // e = table_exp_f16[f16(s - max)] (ggml.c:12427-12440), produced directly in A-fragment layout: a0 = (gid; keys 2 tig, + 1), a1 = (gid + 8; ..)
        float e[4];
#pragma unroll
        for (int u = 0; u < 2; u++) {
            const bool live = jj0 + 2 * tig + u < nk;
            e[u]     = live && gid < G     ? exp_f16lut(__fsub_rn(sring[warp][st][lane][u], gm0)) : 0.f;
            e[2 + u] = live && gid + 8 < G ? exp_f16lut(__fsub_rn(sring[warp][st][lane][2 + u], gm1)) : 0.f;
        }
        lsum0 += (double) e[0] + (double) e[1]; lsum1 += (double) e[2] + (double) e[3];
        const __half2 e0h = __floats2half2_rn(e[0], e[1]), e1h = __floats2half2_rn(e[2], e[3]);       // exact: e is an fp16 value
        const uint32_t a0 = *reinterpret_cast<const uint32_t *>(&e0h), a1 = *reinterpret_cast<const uint32_t *>(&e1h);
#pragma unroll
        for (int nt = 0; nt < 8; nt++) {                                         // B column gid = dim 8 nt + gid, rows = keys 2 tig, 2 tig + 1
            if constexpr (std::is_same<E, float>::value) {
                uint32_t bh, bl;
                split_h2(vr[st][2 * tig][8 * nt + gid], vr[st][2 * tig + 1][8 * nt + gid], bh, bl);
                mma_1688(acc[nt], a0, a1, bh); mma_1688(acc[nt], a0, a1, bl);
            } else {
                const __half2 b = __halves2half2(vr[st][2 * tig][8 * nt + gid], vr[st][2 * tig + 1][8 * nt + gid]);
                mma_1688(acc[nt], a0, a1, *reinterpret_cast<const uint32_t *>(&b));
            }
        }
        __syncwarp();                                             // all reads of this stage are done before the next iteration refills it
    }
    cp_async_wait<0>();
    lsum0 += __shfl_xor_sync(0xffffffffu, lsum0, 1); lsum0 += __shfl_xor_sync(0xffffffffu, lsum0, 2);
    lsum1 += __shfl_xor_sync(0xffffffffu, lsum1, 1); lsum1 += __shfl_xor_sync(0xffffffffu, lsum1, 2);
    if (tig == 0) { dsum[warp][gid] = lsum0; dsum[warp][gid + 8] = lsum1; }
    __syncwarp();                                                              // every lane is done with the ring: it becomes the warp's partial-output block [head][64]
#pragma unroll
    for (int nt = 0; nt < 8; nt++) {
        vring[warp][gid * 32 + 4 * nt + tig] = make_float2(acc[nt][0], acc[nt][1]);
        vring[warp][(gid + 8) * 32 + 4 * nt + tig] = make_float2(acc[nt][2], acc[nt][3]);
    }
    __syncthreads();
    }   // nk > 0
    split_combine(a, vring, dsum, a.n_splits, n_used, nk, split, h0, G);
}

static int g_long_launches = 0;
extern "C" int b200_attention_long_launches(void) { return g_long_launches; }       // diagnostics / tests: launches (eager or captured) of this tier

void launch_attention_long(SplitArgs a, cudaStream_t stream) {
    // one wave: as many key splits as SMs divided by the (KV head, head group) pairs -- Falcon-40B 18, 180B 9, 7B 29
    a.n_splits = num_sms() / (a.n_head_kv * ((a.G + SPLIT_G - 1) / SPLIT_G));
    a.n_splits = a.n_splits < 4 ? 4 : a.n_splits > SPLIT_MAX ? SPLIT_MAX : a.n_splits;
    static bool set = false;
    if (!set) {
        for (const void * k : { (const void *) attn_long_scores_kernel<float>, (const void *) attn_long_values_kernel<float>,
                                (const void *) attn_long_scores_kernel<__half>, (const void *) attn_long_values_kernel<__half> })
            B200_CUDA_CHECK(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, B200_CARVEOUT));
        set = true;
    }
    g_long_launches++;
    if (kv_f16(a.kv)) split_launch(attn_long_scores_kernel<__half>, attn_long_values_kernel<__half>, a, 0, stream);
    else split_launch(attn_long_scores_kernel<float>, attn_long_values_kernel<float>, a, 0, stream);
}
