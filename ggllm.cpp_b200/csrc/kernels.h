// kernels.h -- internal launcher declarations (C++ linkage) shared by the C ABI, the ggml_cuda_* surface and the engine.
#pragma once
#include "formats.cuh"

// ---- weights.cu
size_t wplanes_layout(WPlanes & W, int type, int K, int M);
void   wplanes_upload(WPlanes & W, int type, int K, int M, const void * host_raw, cudaStream_t stream);
void   wplanes_alloc_random(WPlanes & W, int type, int K, int M, uint64_t seed, cudaStream_t stream);
// the two halves of the above, for planes that live in memory the caller provides: place a laid-out matrix at `base`, then fill it
void   wplanes_place(WPlanes & W, uint8_t * base);
void   wplanes_fill(const WPlanes & W, const void * host_raw, cudaStream_t stream);
void   wplanes_fill_random(const WPlanes & W, uint64_t seed, cudaStream_t stream);
void   launch_repack_rows(const WPlanes & W, const void * stage_dev, int64_t row0, int64_t nrows, cudaStream_t stream);   // raw blocks of rows [row0, row0 + nrows) -> planes
void   wplanes_free(WPlanes & W);
void   launch_dequant_rows(const WPlanes & W, const int32_t * rows_dev, int nrows, float * dst, int64_t dst_stride, cudaStream_t stream);

// ---- actquant.cu
size_t actq_bytes(int act_type, int K, int N);
void   actq_bind(ActQ & A, int act_type, int K, int N, void * base);          // carve a caller-provided buffer
void   launch_quantize_act(const float * x, int64_t x_stride, const ActQ & A, cudaStream_t stream);
void   launch_actq_to_f16(const ActQ & A, __half * dst, int64_t dst_stride, cudaStream_t stream);  // d*q -> fp16: b200_actq_to_f16, the reference for A.h

// ---- mmv.cu : y[n][m] = sum_k W[m][k] * xq[n][k], N small (decode), integer dots on quantised activations
enum { EPI_NONE = 0, EPI_GELU = 1, EPI_ADD2 = 2 };
struct MmvEpilogue { int kind; const float * r1; const float * r2;         // ADD2: y = (dot + r1[m]) + r2[m]
    // optional (fast kernel, N == 1, M % 256 == 0): the output row is also quantised for the NEXT mat-mul (its INIT pass,
    // ggml.c:11462-11476) by whichever CTA completes a 256-value chunk; qctr = M / 256 zero-initialised, self-resetting counters
    const ActQ * qout; unsigned * qctr;
    // The kernel in front of this one in the stream produces NOTHING this one reads, and everything it reads was complete AND flushed before
    // that kernel's main body ran (ffn_up behind qkv: both read the LayerNorm's output): with programmatic dependent launch the rows then
    // stream from the moment the CTAs are resident, and griddepcontrol.wait moves to the END of the kernel, where it only keeps the chain
    // of completions intact (whoever waits for this grid has thereby waited for the one in front of it)
    int late_wait; };
void   launch_mmv(const WPlanes & W, const ActQ & A, float * y, int64_t y_stride, MmvEpilogue epi, cudaStream_t stream);
void   launch_mmv_f(const WPlanes & W, const float * x, int64_t x_stride, int N, float * y, int64_t y_stride, cudaStream_t stream); // f16/f32 weights

// mmv_fast.cu: the tuned kernel (Q4_K, Q4_0, Q3_K); false = type / K not covered, nothing launched
bool   launch_mmv_fast(const WPlanes & W, const ActQ & A, float * y, int64_t y_stride, MmvEpilogue e, cudaStream_t stream);
struct MmvShape { int nt, j, d; };                  // NT threads per CTA, J pieces per thread, ring depth D; nt == 0: generic kernel
MmvShape mmv_fast_pick_shape(int wtype, int K);     // the shape launch_mmv_fast launches
bool   mmv_fast_supports(int wtype, int K);
bool   mmv_fast_fills_sm(const WPlanes & W);       // its CTAs leave no registers for a side-stream kernel beside them
// ---- c_api.cu
cudaStream_t b200_current_stream();                 // the stream the C ABI's calls run on

// ---- ops.cu
unsigned ew_grid(int64_t n);                        // grid of the 256-thread grid-stride elementwise kernels: one thread per value, at most 132 * 16 CTAs
void   launch_layernorm(const float * x, int64_t x_stride, const float * g, const float * b, float * y, int64_t y_stride,
                        int n, int rows, cudaStream_t stream);              // y = norm(x)*g + b ; g,b may be null (plain ggml_norm)
// [x = (ra + rb) + x, written back] ; A1 = Q(norm(x)*g1+b1) ; A2 = Q(norm(x)*g2+b2) (optional) ; with y: rows r >= y_row0 also
// store norm(x)*g1+b1 in fp32 at y + (r - y_row0) * y_stride (16-byte aligned rows)
void   launch_layernorm_q(float * x, int64_t x_stride, const float * ra, const float * rb, int64_t r_stride,
                          const float * g1, const float * b1, const ActQ * A1,
                          const float * g2, const float * b2, const ActQ * A2, int n, int rows, cudaStream_t stream,
                          float * y = nullptr, int64_t y_stride = 0, int y_row0 = 0);
void   launch_argmax_hist(const float * x, int n, int32_t * out, int32_t * hist, int * step, cudaStream_t stream);  // greedy: lowest index on ties; hist[(*step)++] = id (graph-replayable)
void   launch_gelu(const float * x, float * y, int64_t n, cudaStream_t stream);
void   launch_f32_to_f16(const float * x, __half * y, int64_t n, cudaStream_t stream);     // the fp16 activation rows of an F16-weight mat-mul
void   launch_add(const float * a, const float * b, float * y, int64_t n, cudaStream_t stream);
void   launch_add3(const float * a, const float * b, const float * c, float * y, int64_t n, cudaStream_t stream);   // (a+b)+c
void   launch_mul_bcast(const float * a, const float * b, float * y, int64_t n, int64_t nb, cudaStream_t stream);  // y[i] = a[i]*b[i%nb]
void   launch_add_bcast(const float * a, const float * b, float * y, int64_t n, int64_t nb, cudaStream_t stream);
void   launch_scale(const float * a, float s, float * y, int64_t n, cudaStream_t stream);
// dst[c * ld_dst + r] = src[r * ld_src + c] for r < rows, c < cols (tiled through shared memory, coalesced on both sides)
void   launch_transpose_f32(const float * src, int64_t ld_src, int rows, int cols, float * dst, int64_t ld_dst, cudaStream_t stream);
struct RopeParams { int n_past; int head_dim; float theta_scale; };
float  rope_theta_scale_host(int head_dim, int n_ctx_rope, int dynamic_mode, float ntk_alpha, int freq_base);
float  falcon_rope_theta_scale(int head_dim, int n_ctx_rope, int n_ctx);   // Falcon's settings (libfalcon.cpp:2229-2234); n_ctx_rope 0: n_ctx
// rotates x[t][h][head_dim] in place (token stride tok_stride, head stride head_dim), position = *n_past_dev + t (or n_past if dev ptr null)
void   launch_rope_neox(float * x, int n_tok, int n_head, int head_dim, int64_t tok_stride, int n_past, const int * n_past_dev,
                        float theta_scale, cudaStream_t stream);

// ---- attention: attention.cu picks the kernel (attention_long.cu, attention_ws.cu and attention_prefill.cu hold the others)
// One layer's KV cache, passed by value from the engine down to every attention kernel.  Null planes do not exist.  The element type
// is fp16 exactly when v16 is set (kv_f16): k16 / v16 are then the cache and k / v are null.  Otherwise k / v are the cache and k16
// (with vt16) is its fp16 shadow for the prompt kernel (attention_ws.cu), or null.  Rows of k / v / k16 / v16: [n_ctx][n_head_kv][head_dim].
struct KvCache {
    float * k, * v;             // f32 cache
    __half * k16, * v16;        // fp16 K (the cache itself, or the f32 cache's shadow) and fp16 V (fp16 cache only)
    __half * vt16;              // V^T [n_head_kv][64][ctx_pad] for the prompt kernel, or null
    int ctx_pad;                // attention_ctx_pad(n_ctx)
};
__host__ __device__ __forceinline__ bool kv_f16(const KvCache & c) { return c.v16 != nullptr; }
// the cache planes as element type E (float: the f32 cache, __half: the fp16 one)
template <typename E> __host__ __device__ __forceinline__ const E * kv_k(const KvCache & c) { if constexpr (sizeof(E) == 4) return c.k; else return c.k16; }
template <typename E> __host__ __device__ __forceinline__ const E * kv_v(const KvCache & c) { if constexpr (sizeof(E) == 4) return c.v; else return c.v16; }
struct AttnParams {
    int n_head, n_head_kv, head_dim;
    int n_tok;                  // new tokens (queries)
    int n_past;                 // tokens already in the cache (host value; ignored if n_past_dev != null)
    const int * n_past_dev;     // optional device scalar (CUDA-graph replay; one token)
    int n_ctx;                  // KV capacity (row count of the cache)
    int64_t qkv_stride;         // floats between consecutive tokens in the fused QKV buffer
    const ActQ * qout;          // optional: also emit the output row quantised for the wo mat-mul (its INIT pass)
    // This layer's cache.  rope_kv_append keeps every plane in step.  An fp16 cache rounds rows when they are appended
    // (__float2half_rn, ggml_fp32_to_fp16 on an F16C host) and every reader widens them exactly.
    KvCache kv;
    // RoPE(Q, K) with rope_theta_scale and the KV append are part of launch_attention.  fuse_rope (decode): the split-KV scores kernel
    // may do them itself, on qkv's rows in registers, instead of a kernel of their own -- qkv is then NOT rotated in place.
    int fuse_rope; float rope_theta_scale;
    // decode with n_past in a device scalar (graph replay): the caller's promise that this launch only serves contexts longer than
    // attention_long_threshold() keys, so the long-context kernels (attention_long.cu) may be captured; with a host n_past the launcher
    // decides by itself
    int long_ctx;
};
// The one writer of a cache element (row offset o): every plane that exists gets it -- the fp32 row, the fp16 rows (k16 / v16), V^T
// (vt16, position pos, dim d of KV head kvh).  An fp16 plane stores __float2half_rn(x): beyond +-65504 that is +-Inf.
__device__ __forceinline__ void kv_put_k(const KvCache & c, size_t o, float x) {
    if (c.k) c.k[o] = x;
    if (c.k16) c.k16[o] = __float2half_rn(x);
}
__device__ __forceinline__ void kv_put_v_rows(const KvCache & c, size_t o, float x) {      // the V rows only, not V^T
    if (c.v) c.v[o] = x;
    if (c.v16) c.v16[o] = __float2half_rn(x);
}
__device__ __forceinline__ void kv_put_v(const KvCache & c, size_t o, int kvh, int d, int pos, float x) {
    kv_put_v_rows(c, o, x);
    if (c.vt16) c.vt16[((size_t) kvh * 64 + d) * c.ctx_pad + pos] = __float2half_rn(x);
}
// a cache element widened to f32 (exact for fp16)
__device__ __forceinline__ float kv_ld(const float * p) { return *p; }
__device__ __forceinline__ float kv_ld(const __half * p) { return __half2float(*p); }
// two consecutive elements (8-byte / 4-byte aligned), read-only path
__device__ __forceinline__ float2 kv_ld2(const float * p) { return __ldg(reinterpret_cast<const float2 *>(p)); }
__device__ __forceinline__ float2 kv_ld2(const __half * p) { return __half22float2(__ldg(reinterpret_cast<const __half2 *>(p))); }
// the same for a row the kernel in front of this one may just have written (not through the read-only path)
__device__ __forceinline__ float2 kv_ld2_new(const float * p) { return *reinterpret_cast<const float2 *>(p); }
__device__ __forceinline__ float2 kv_ld2_new(const __half * p) { return __half22float2(*reinterpret_cast<const __half2 *>(p)); }
// elements 4 i .. 4 i + 3 of a row (16-byte / 8-byte aligned)
__device__ __forceinline__ float4 kv_ld4(const float * p, int i) { return reinterpret_cast<const float4 *>(p)[i]; }
__device__ __forceinline__ float4 kv_ld4(const __half * p, int i) {
    const uint2 u = reinterpret_cast<const uint2 *>(p)[i];
    const float2 a = __half22float2(*reinterpret_cast<const __half2 *>(&u.x)), b = __half22float2(*reinterpret_cast<const __half2 *>(&u.y));
    return make_float4(a.x, a.y, b.x, b.y);
}
// what a reader of the cache sees of a value that has just been appended
__device__ __forceinline__ float kv_seen(float x, const float *) { return x; }
__device__ __forceinline__ float kv_seen(float x, const __half *) { return __half2float(__float2half_rn(x)); }
// The attention scratch starts with this many bytes of split-KV arrival counters.  Their owner zeroes them once; they re-arm themselves.
#define ATTN_CTR_BYTES 4096
int    attention_long_threshold();          // keys above which decode attention switches to attention_long.cu
// fused: rope(Q), rope(K) with p.rope_theta_scale -> K cache append, V cache append      (libfalcon.cpp:2229-2281)
void   launch_rope_kv_append(float * qkv, const AttnParams & p, cudaStream_t stream);
// RoPE + KV append, then out[t][h*head_dim + i] = softmax(scale * Q K^T + causal mask) V   (libfalcon.cpp:2229-2366), and p.qout.
// scratch: attention_scratch_bytes(p) bytes (null when that is 0).  Returns the number of kernels launched; folded (optional): whether
// p.qout was written by the attention kernels themselves rather than by a quantize_act of its own; rope_in_place (optional): whether
// Q and K were rotated in qkv itself (false when the split-KV kernels did RoPE in registers, p.fuse_rope).
int    launch_attention(float * qkv, float * out, int64_t out_stride, const AttnParams & p, float * scratch, cudaStream_t stream,
                        bool * folded = nullptr, bool * rope_in_place = nullptr);
size_t attention_scratch_bytes(const AttnParams & p);                // one token: enough for either decode tier at any position
int    attention_ctx_pad(int n_ctx);
size_t attention_shadow_halves(int n_head_kv, int n_ctx);           // halves per layer, for k16 and for vt16 each
// cache rows [pos, pos + n) -> the shadow planes of c, if it has them: vt16, and k16 of an f32 cache
void   launch_kv_shadow_refresh(const KvCache & c, int n_head_kv, int pos, int n, cudaStream_t stream);

// ---- gemm.cu : mat-mul dispatch, Y[n][m] = sum_k W[m][k] * X[n][k].  N <= MMV_MAX_N: the mat-vec; above: the prompt GEMM.
// The launchers return the launches the engine counts: one per mat-vec, quantiser, GELU or GEMM (a GEMM runs in chunks of 512 rows
// but counts once).
constexpr int MMV_MAX_N = 8;
// quantised activations already in A (A.N is set to N); N > MMV_MAX_N needs the fp16 GEMM operand in A.h
int    launch_mul_mat_q(const WPlanes & W, const ActQ & A, int N, float * y, int64_t y_stride, int epi, cudaStream_t stream);
// fp32 activation rows: F32 / F16 weights take them as they are (launch_mmv_f, then GELU if asked); quantised weights get them
// quantised into `scratch` (mul_mat_scratch_bytes(W, N) bytes), fp16 operand included, then launch_mul_mat_q
int    launch_mul_mat(const WPlanes & W, const float * x, int64_t x_stride, int N, float * y, int64_t y_stride, int epi, void * scratch,
                      cudaStream_t stream);
size_t mul_mat_scratch_bytes(const WPlanes & W, int N);
// the prompt GEMM on fp16 activations: wgmma (gemm_tc.cu) where it covers the shape, the CUDA-core kernel (gemm_simt.cu) elsewhere
void   launch_mmq_gemm(const WPlanes & W, const __half * X, int64_t x_stride, int N, float * Y, int64_t y_stride, int epi_gelu, cudaStream_t stream);
void   launch_gemm_simt(const WPlanes & W, const __half * X, int64_t x_stride, int N, float * Y, int64_t y_stride, int epi_gelu, cudaStream_t stream);
bool   launch_gemm_tc(const WPlanes & W, const __half * X, int64_t x_stride, int N, float * Y, int64_t y_stride, int epi_gelu, cudaStream_t stream);   // false: shape not covered
// what launch_gemm_tc launches: bn token-tile width (64 / 128 / 256), ksplit CTAs over K (1 / 2), producer the fast dequantiser's
// type (T_Q4_K, T_Q4_0, T_Q3_K) or -1 for the generic one; bn == 0: not covered (N outside 1..512, K % 64, x_stride % 8, X not
// 16-byte aligned), nothing launched
struct GemmTcShape { int bn, ksplit, producer; };
GemmTcShape gemm_tc_pick_shape(int type, int64_t K, int64_t M, int N, int64_t x_stride, bool x_aligned, int epi_gelu);

// ---- quant_gpu.cu: ggml_quantize_chunk (ggml.c:19479-19560) over consecutive chunks of `chunk` values, the last one shorter, for
// every falcon_quantize output type but F32.  Only the carried types (make_qkx1_quants: Q2_K, Q4_K, Q5_K) see the chunks: one chain
// per full chunk, and the short tail a second launch; every other type is one launch over the whole buffer.  hist_dev (16 counters,
// or null) accumulates the legacy types' code histograms.  Returns the bytes written, 0 for any other type, -1 for a bad shape.
int64_t launch_quantize_chunks(int ggml_type, const float * x, void * dst, int64_t n, int64_t chunk, unsigned long long * hist_dev,
                               cudaStream_t s);

// ---- sampling.cu: falcon_main's sampling chain on the device (logit bias, repetition / frequency / presence penalties, top-k,
// tail-free, typical, top-p, temperature, mirostat 1 / 2, MT19937 draw)
#define B200_SAMPLER_MAX_WINDOW 256
#define B200_SAMPLER_MAX_BIAS 64
struct SamplerParams {
    int top_k;                          // <= 0: whole vocabulary (1..1024: block arg-max rounds, otherwise a radix sort of the row)
    float top_p; float temp; float repeat_penalty;
    float tfs_z, typical_p, frequency_penalty, presence_penalty;
    int mirostat; float mirostat_tau, mirostat_eta;
    int n_bias; int32_t bias_id[B200_SAMPLER_MAX_BIAS]; float bias_value[B200_SAMPLER_MAX_BIAS];   // unused entries zero (memcmp-comparable)
};
struct SamplerState;
SamplerState * sampler_state_alloc();
void   sampler_state_free(SamplerState * s);
size_t sampler_work_floats(int n_vocab);                       // size of launch_sample's `work` scratch
float  sampler_mu(const SamplerState * s);                     // synchronous read of the mirostat state
void   launch_sampler_init(SamplerState * s, uint32_t seed, const int32_t * window_dev, int n, int cap, float mu, cudaStream_t stream);
// tap: null, or sampler_tap_bytes(n_vocab) bytes that receive the candidate list after every stage (b200_sampler_tap)
void   launch_sample(const float * logits, int n_vocab, const SamplerParams & p, SamplerState * st, float * work, int32_t * out, int32_t * hist, int * step,
                     float * tap, cudaStream_t stream);
size_t sampler_tap_bytes(int n_vocab);
bool   sampler_tap_read(const float * tap, int n_vocab, const char * stage, const char * field, void * host, size_t bytes);
// falcon_perplexity's per-token term -log(softmax(row)[target]) of rows [0, n_rows) (row r at logits + r * row_stride): target -1
// skips the row (nll[r] unwritten), a target outside [0, n_vocab) writes NaN (b200_token_nll)
void   launch_token_nll(const float * logits, int n_vocab, int n_rows, int64_t row_stride, const int32_t * targets, float * nll, cudaStream_t stream);

// ---- engine.cu (internal, C++ linkage): adopt a matrix that is already resident in the planar layout (no copy, not freed by the engine)
struct b200_falcon;
bool   falcon_adopt_matrix(b200_falcon * f, const char * ggcc_name, const WPlanes & W);
int    falcon_eval_begin(b200_falcon * f, const int32_t * tokens, int n_tokens, int n_past, int n_ctx_rope, int all_logits);   // enqueue only (b200_falcon_eval's checks and return codes)
void   falcon_eval_finish(b200_falcon * f, float * logits, float * embedding = nullptr);    // wait; logits (optional) receive what begin asked for, embedding (optional, embeddings on) the n_embd floats of b200_falcon_embeddings
// The KV section of the reference's session state (falcon_copy_state_data / falcon_set_state_data, libfalcon.cpp:4280-4330), host side:
// positions [0, n) of every local layer in f32, K as n rows of n_head_kv * 64 floats, V transposed: n_head_kv * 64 columns of n positions,
// column stride v_ld.  Local layer l's K starts k_layer floats after layer l - 1's, its V v_layer floats after.  Either plane may be null.
// V goes through a device staging buffer and the tiled transpose; each byte crosses PCIe once.  Import also refreshes the fp16 shadow of
// [0, n).  f32 caches only: returns 0, or 1 for an fp16 cache or n outside [0, n_ctx].
struct RefKvLayout { size_t k_layer, v_ld, v_layer; };
int    falcon_ref_kv_export(b200_falcon * f, int n, float * k, float * v, const RefKvLayout & L);
int    falcon_ref_kv_import(b200_falcon * f, int n, const float * k, const float * v, const RefKvLayout & L);
