// engine.cu -- part B of include/ggml_b200.h: the Falcon eval path, device-resident.
//
// What the reference spreads over libfalcon.cpp (loader upload :1196-1270, VRAM planner :1764-1886, KV cache
// :1335-1385, graph builder falcon_eval_internal :2011-2588) plus one H2D + kernel + D2H + cudaDeviceSynchronize
// round trip per MUL_MAT node (ggml-cuda.cu:2520-2820, 241 per 40B token) becomes:
//   * weights uploaded once into planar device layout; KV cache and every activation live in HBM
//   * a prompt eval (N > 1) = ~9 kernels per layer on two streams (attention branch || MLP branch, which Falcon's
//     parallel block makes independent, libfalcon.cpp:2166-2188 / 2382-2401); only token ids go H2D and logits D2H
//   * decode (N == 1) is captured once into a CUDA graph and replayed; n_past and the token id are read from
//     device scalars so the same graph serves every position.  For the types with a register-resident mat-vec the
//     four mat-vecs of a layer run back to back on one stream, chained by programmatic dependent launch, with the
//     small attention kernels beside ffn_up on the second stream (enqueue_decode_fused; DESIGN.md section 4.5)
//   * multi-GPU = contiguous layer ranges, one process per GPU; the residual stream [N x n_embd] f32 crosses each
//     boundary with a single ncclSend/ncclRecv on the compute stream (replaces the row-split tensor parallelism of
//     ggml-cuda.cu:2594-2601, 2719-2725, 2779-2788)
#include "kernels.h"
#include "ggcc_file.h"
#include "../../include/ggml_b200.h"
#include <nccl.h>
#include <dlfcn.h>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#include <algorithm>
#include <array>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

// ------------------------------------------------------------------------------------------------ NCCL (loaded lazily)
struct NcclApi {
    void * lib = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*Send)(const void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    const char * (*GetErrorString)(ncclResult_t) = nullptr;
};
static NcclApi & nccl() {
    static NcclApi api;
    if (!api.lib) {
        api.lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!api.lib) { fprintf(stderr, "b200: cannot load libnccl.so.2 (%s); multi-GPU pipeline unavailable\n", dlerror()); exit(1); }
#define L(name) *(void **) (&api.name) = dlsym(api.lib, "nccl" #name); B200_ASSERT(api.name != nullptr)
        L(GetUniqueId); L(CommInitRank); L(Send); L(Recv); L(CommDestroy); L(GetErrorString);
#undef L
    }
    return api;
}
#define B200_NCCL_CHECK(expr) do { ncclResult_t r_ = (expr); if (r_ != ncclSuccess) { \
    fprintf(stderr, "b200: NCCL error %d (%s) at %s:%d\n", (int) r_, nccl().GetErrorString(r_), __FILE__, __LINE__); exit(1); } } while (0)

// ------------------------------------------------------------------------------------------------ model
struct Layer {
    WPlanes wqkv{}, wo{}, up{}, down{};
    float * ln_attn_g = nullptr, * ln_attn_b = nullptr, * ln_mlp_g = nullptr, * ln_mlp_b = nullptr;
};

enum { G_DEVICE, G_HOST, G_GEN };               // the decode step graphs, see b200_falcon::graph

struct b200_falcon {
    b200_falcon_params hp;
    int E, H, HKV, D, QKV, FF, V, NL;          // NL = local layers
    bool first, last;
    std::vector<Layer> layers;
    WPlanes tok_emb{}, lm_head{};
    float * lnf_g = nullptr, * lnf_b = nullptr;
    // the KV cache (f32, or fp16 from b200_falcon_create_kv), every layer in one allocation per plane: layer 0's view (kv_layer).  The
    // prompt kernel's V^T, and an f32 cache's fp16 K shadow, exist only when n_batch > 8.  shadow_layer: halves per layer of each fp16 plane
    KvCache kv{}; size_t shadow_layer = 0;
    // activation arena
    float * inp = nullptr, * qkv = nullptr, * att = nullptr, * ao = nullptr, * up = nullptr, * dn = nullptr, * logits = nullptr;
    void * actq_mem = nullptr; ActQ xa{}, xm{}, xatt{}, xup{}, xf{};
    __half * xh_a = nullptr, * xh_b = nullptr, * xh_m = nullptr;      // fp16 GEMM operands (d * q), written by the kernels that quantise: attention branch, MLP branch, MLP input
    DevScratch attn_scratch;                       // prompt attention
    float * attn_dec_scratch = nullptr;            // decode attention: zeroed before the decode graphs are captured
    int32_t * tokens_dev = nullptr; int * n_past_dev = nullptr;
    int32_t * tokens_h = nullptr; int * n_past_h = nullptr; float * logits_h = nullptr; size_t logits_h_floats = 0;
    int32_t * score_tg = nullptr, * score_tg_h = nullptr; float * score_nll = nullptr, * score_nll_h = nullptr;    // b200_falcon_score's targets / terms [n_batch]
    cudaStream_t s_main = nullptr, s_mlp = nullptr;
    cudaEvent_t e_fork = nullptr, e_join = nullptr, e_t0 = nullptr, e_t1 = nullptr;
    // decode step graphs [tier][which], each with the RoPE theta scale it was captured for.  tier 1: captured with the long-context
    // attention kernels (attention_long.cu), used above attention_long_threshold() keys.  which: G_DEVICE token id and logits stay on
    // the device; G_HOST token H2D and logits D2H nodes inside; G_GEN generation step, G_DEVICE plus the sampler (in a pipeline the
    // sampled id travels last rank -> rank 0 by ncclSend / ncclRecv)
    struct { cudaGraphExec_t exec = nullptr; float theta = -1.f; } graph[2][3];
    int graph_launches = 0, cur_tier = 0;
    bool ring_mode = false;                     // set while the generation-step graph is being captured
    int32_t * tok_next = nullptr, * gen_hist = nullptr; int * gen_step = nullptr;   // sampled id, ids so far, step counter (device)
    SamplerState * sampler = nullptr; SamplerParams sampler_p{}; bool use_sampler = false; float * sampler_work = nullptr;   // generation with the sampling chain (sampling.cu)
    int act_type = -1;                // the ONE activation format every layer matrix takes (fast paths), -1: see generic_layers
    // Files the reference evaluates but the fused paths do not cover: F16 / F32 matrices (an unquantised model, or lm_head kept in F16
    // by --leave-output-tensor, libfalcon.cpp:3609) and legacy + K-quant types mixed in one model.  They run through enqueue_eval_generic:
    // one fp32 LayerNorm per norm, activations quantised per matrix for ITS type (what ggml's MUL_MAT INIT pass does, ggml.c:11462-11476).
    bool classified = false, generic_layers = false, generic_head = false;
    float * gen_na = nullptr, * gen_nm = nullptr; void * gen_mm = nullptr;     // gen_mm: the activations of one matrix, in its format
    unsigned * q_ctr = nullptr;                 // chunk counters of the quantise-on-completion epilogue (ffn_up -> ffn_down)
    ncclComm_t comm = nullptr;
    int launches = 0; float last_ms = 0.f;
    size_t weight_bytes = 0;
    double load_seconds = 0.0; size_t load_bytes = 0;   // b200_falcon_load_ggcc
    size_t pending_floats = 0;                  // logits of the eval in flight (falcon_eval_begin / finish)
    // falcon_context_params.embedding (b200_falcon_set_embeddings): the final LayerNorm's last head row ("result_norm") of every
    // b200_falcon_eval goes to the pinned emb_h.  The fused head's LayerNorm kernel stores it in emb_dev, the generic head leaves it in
    // gen_na; emb_src is the one the last head read.  emb_valid: emb_h holds the row of the most recent eval call.
    bool emb_on = false, emb_valid = false;
    float * emb_dev = nullptr, * emb_h = nullptr; const float * emb_src = nullptr;
    std::vector<const void *> borrowed;         // device planes adopted from another owner (ggml_cuda_transform_tensor): never freed here
    // test tap (b200_falcon_tap / _tap_layers): while mem is set, every eval copies its intermediates into mem -- one slice of layer_bytes
    // per tapped local layer at the end of that layer, then one slice after the head.  Node offsets are the same in every layer slice.
    struct TapNode { std::string name; const void * src; size_t row_bytes, off; bool all_rows; };    // all_rows: N rows, else the head's rows
    struct Tap { uint8_t * mem = nullptr; std::vector<TapNode> layer, head; size_t layer_bytes = 0; int rows = 0, head_rows = 0, n_slices = 0;
                 std::vector<int> rotated, slice; } tap;         // rotated[l]: RoPE ran in place on qkv (not inside the attention kernels);
                                                                 // slice[l]: local layer l's slice, -1 when it is not tapped
    // Streamed layers (b200_falcon_create_streamed): their matrices live in pinned host images, in the device's planar bytes, and every
    // eval copies each one into device slot rank % 2 on s_copy shortly before the layer runs.  A slot has one region per matrix role
    // (wqkv, wo, up, down), sized to the largest streamed matrix of that role; a streamed WPlanes points into its slot for good, so
    // the captured graphs bake in fixed addresses.  rank[l]: local layer l's position among the streamed layers, -1 when resident.
    struct Streamed { std::vector<int> layers, rank; std::vector<std::array<uint8_t *, 4>> image;
                      uint8_t * slot[2] = {}; size_t region[4] = {}, region_off[4] = {}, slot_bytes = 0;
                      cudaStream_t s_copy = nullptr; cudaEvent_t e_fork = nullptr, e_join = nullptr, ready[2] = {}, free[2] = {}; } st;
};

// Local layer l's slice of the KV cache (kernels.h's KvCache): f32 rows of kv_row() floats, fp16 planes shadow_layer halves apart.
static size_t kv_row(const b200_falcon * f) { return (size_t) f->HKV * f->D; }
static KvCache kv_layer(const b200_falcon * f, int l) {
    KvCache c = f->kv;
    const size_t off = (size_t) l * f->hp.n_ctx * kv_row(f), off16 = (size_t) l * f->shadow_layer;
    if (c.k) { c.k += off; c.v += off; }
    if (c.k16) c.k16 += off16;
    if (c.v16) c.v16 += off16;
    if (c.vt16) c.vt16 += off16;
    return c;
}
// f32 host rows <-> a cache plane (kv_read / kv_write)
static void kv_d2h(float * dst, const float * src, size_t n) { B200_CUDA_CHECK(cudaMemcpy(dst, src, n * 4, cudaMemcpyDeviceToHost)); }
static void kv_d2h(float * dst, const __half * src, size_t n) {
    std::vector<__half> h(n);
    B200_CUDA_CHECK(cudaMemcpy(h.data(), src, n * 2, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < n; i++) dst[i] = __half2float(h[i]);
}
static void kv_h2d(float * dst, const float * src, size_t n) { B200_CUDA_CHECK(cudaMemcpy(dst, src, n * 4, cudaMemcpyHostToDevice)); }
static void kv_h2d(__half * dst, const float * src, size_t n) {
    std::vector<__half> h(n);
    for (size_t i = 0; i < n; i++) h[i] = __float2half_rn(src[i]);
    B200_CUDA_CHECK(cudaMemcpy(dst, h.data(), n * 2, cudaMemcpyHostToDevice));
}

template <typename E>
__global__ void fill_kernel(E * p, int64_t n, float base, float amp, uint64_t seed) {
    for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) {
        uint64_t x = seed + (uint64_t) i * 0x9E3779B97F4A7C15ULL; x ^= x >> 31; x *= 0xBF58476D1CE4E5B9ULL; x ^= x >> 29;
        const float v = base + amp * ((float) (x & 0xffffff) / 8388608.f - 1.f);
        if constexpr (sizeof(E) == 2) p[i] = __float2half_rn(v); else p[i] = v;
    }
}

static size_t algorithmic_bytes(int type, int64_t K, int64_t M) {
    const TypeSpec ts = type_spec(type);
    return (size_t) (K / ts.blk_elems) * ts.blk_bytes * (size_t) M;
}

// The model's tensor slots and the GGCC names that address them (libfalcon.cpp:1764, 1793-1796, 1847-1861).  Shapes are [M][K]; a
// slot without M is a LayerNorm vector of K floats.  The embedding table lives on the first rank, the final LayerNorm and lm_head on
// the last, a layer's tensors on the rank whose layer range holds it.
enum SlotKind { S_EMB, S_LNF_G, S_LNF_B, S_LM_HEAD, S_LN_ATTN_G, S_LN_ATTN_B, S_LN_MLP_G, S_LN_MLP_B, S_QKV, S_WO, S_UP, S_DOWN };
enum SlotOwner { OWN_FIRST, OWN_LAST, OWN_LAYER };
using FalconDim = int b200_falcon::*;
struct SlotDesc { const char * name; SlotKind kind; SlotOwner owner; FalconDim K, M; };
static const SlotDesc SLOTS[] = {                // OWN_LAYER names follow "transformer.h.<layer>."
    { "transformer.word_embeddings.weight",    S_EMB,       OWN_FIRST, &b200_falcon::E,  &b200_falcon::V   },
    { "transformer.ln_f.weight",               S_LNF_G,     OWN_LAST,  &b200_falcon::E,  nullptr           },
    { "transformer.ln_f.bias",                 S_LNF_B,     OWN_LAST,  &b200_falcon::E,  nullptr           },
    { "lm_head.weight",                        S_LM_HEAD,   OWN_LAST,  &b200_falcon::E,  &b200_falcon::V   },
    { "ln_attn.weight",                        S_LN_ATTN_G, OWN_LAYER, &b200_falcon::E,  nullptr           },
    { "ln_attn.bias",                          S_LN_ATTN_B, OWN_LAYER, &b200_falcon::E,  nullptr           },
    { "ln_mlp.weight",                         S_LN_MLP_G,  OWN_LAYER, &b200_falcon::E,  nullptr           },
    { "ln_mlp.bias",                           S_LN_MLP_B,  OWN_LAYER, &b200_falcon::E,  nullptr           },
    { "input_layernorm.weight",                S_LN_MLP_G,  OWN_LAYER, &b200_falcon::E,  nullptr           },   // Falcon-7B's name
    { "input_layernorm.bias",                  S_LN_MLP_B,  OWN_LAYER, &b200_falcon::E,  nullptr           },
    { "self_attention.query_key_value.weight", S_QKV,       OWN_LAYER, &b200_falcon::E,  &b200_falcon::QKV },
    { "self_attention.dense.weight",           S_WO,        OWN_LAYER, &b200_falcon::E,  &b200_falcon::E   },
    { "mlp.dense_h_to_4h.weight",              S_UP,        OWN_LAYER, &b200_falcon::E,  &b200_falcon::FF  },
    { "mlp.dense_4h_to_h.weight",              S_DOWN,      OWN_LAYER, &b200_falcon::FF, &b200_falcon::E   },
};
struct Slot { const SlotDesc * d; int layer; };  // layer: -1 for the model-level slots
static bool find_slot(const std::string & name, Slot & s) {
    const std::string pre = "transformer.h.";
    std::string key = name;
    s.layer = -1;
    if (name.compare(0, pre.size(), pre) == 0) {
        const size_t dot = name.find('.', pre.size());
        if (dot == std::string::npos) return false;
        s.layer = atoi(name.substr(pre.size(), dot - pre.size()).c_str());
        key = name.substr(dot + 1);
    }
    for (const SlotDesc & d : SLOTS)
        if (key == d.name && (d.owner == OWN_LAYER) == (s.layer >= 0)) { s.d = &d; return true; }
    return false;
}
static bool is_matrix(const Slot & s) { return s.d->M != nullptr; }
static int64_t slot_K(const b200_falcon * f, const Slot & s) { return f->*s.d->K; }
static int64_t slot_M(const b200_falcon * f, const Slot & s) { return is_matrix(s) ? f->*s.d->M : 1; }
static bool owns(const b200_falcon * f, const Slot & s) {
    if (s.d->owner == OWN_LAYER) return s.layer >= f->hp.layer_first && s.layer < f->hp.layer_last;
    return s.d->owner == OWN_FIRST ? f->first : f->last;
}
struct SlotDest { WPlanes * W; float ** v; };   // where the slot's tensor lives: exactly one of the two is set
static SlotDest slot_dest(b200_falcon * f, const Slot & s) {
    Layer * L = s.layer >= 0 ? &f->layers[s.layer - f->hp.layer_first] : nullptr;
    switch (s.d->kind) {
        case S_EMB:       return { &f->tok_emb, nullptr };
        case S_LNF_G:     return { nullptr, &f->lnf_g };
        case S_LNF_B:     return { nullptr, &f->lnf_b };
        case S_LM_HEAD:   return { &f->lm_head, nullptr };
        case S_LN_ATTN_G: return { nullptr, &L->ln_attn_g };
        case S_LN_ATTN_B: return { nullptr, &L->ln_attn_b };
        case S_LN_MLP_G:  return { nullptr, &L->ln_mlp_g };
        case S_LN_MLP_B:  return { nullptr, &L->ln_mlp_b };
        case S_QKV:       return { &L->wqkv, nullptr };
        case S_WO:        return { &L->wo, nullptr };
        case S_UP:        return { &L->up, nullptr };
        case S_DOWN:      return { &L->down, nullptr };
    }
    return { nullptr, nullptr };
}

// the instantiated decode graphs bake in device pointers (weights, LayerNorm vectors, the pinned logits buffer):
// whenever one of those is replaced the graphs are dropped and rebuilt by the next decode
static void invalidate_graphs(b200_falcon * f) {
    for (auto & tier : f->graph)
        for (auto & g : tier) if (g.exec) {
            B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
            B200_CUDA_CHECK(cudaGraphExecDestroy(g.exec)); g.exec = nullptr; g.theta = -1.f;
        }
}

// Which path the model's matrices allow (re-derived after every tensor change).  The reference's quantiser writes every 2-D weight with
// one type (libfalcon.cpp:3606-3624), so its files take the fast paths; anything else still evaluates, through the generic path.
static void classify(b200_falcon * f) {
    int at = -2; bool uniform = true;
    for (const auto & L : f->layers)
        for (const WPlanes * W : { &L.wqkv, &L.wo, &L.up, &L.down }) {
            if (!W->p[0]) continue;
            const int a = act_type_for(W->type);
            if (at == -2) at = a; else if (a != at) uniform = false;
        }
    const int nat = (uniform && at >= 0) ? at : -1;
    if (nat != f->act_type && f->actq_mem) { B200_CUDA_CHECK(cudaDeviceSynchronize()); B200_CUDA_CHECK(cudaFree(f->actq_mem)); f->actq_mem = nullptr; }
    f->act_type = nat;
    f->generic_layers = f->NL > 0 && nat < 0;
    f->generic_head = f->last && f->lm_head.p[0] && (f->generic_layers || (f->NL > 0 && act_type_for(f->lm_head.type) != nat));
    if (f->NL == 0 && f->last && f->lm_head.p[0]) { f->act_type = act_type_for(f->lm_head.type); f->generic_head = f->act_type < 0; }
    f->classified = true;
}

// ---- streamed layers (b200_falcon::Streamed)
static const WPlanes & role_matrix(const Layer & L, int r) { return r == 0 ? L.wqkv : r == 1 ? L.wo : r == 2 ? L.up : L.down; }
static WPlanes & role_matrix(Layer & L, int r) { return const_cast<WPlanes &>(role_matrix((const Layer &) L, r)); }
static int matrix_role(const Slot & s) {
    switch (s.d->kind) { case S_QKV: return 0; case S_WO: return 1; case S_UP: return 2; case S_DOWN: return 3; default: return -1; }
}
static int stream_rank(const b200_falcon * f, int l) { return f->st.rank.empty() ? -1 : f->st.rank[l]; }
static bool is_streamed(const b200_falcon * f, const Slot & s) {
    return s.layer >= 0 && matrix_role(s) >= 0 && stream_rank(f, s.layer - f->hp.layer_first) >= 0;
}
static bool in_slot(const b200_falcon * f, const void * p) {
    for (const uint8_t * s : f->st.slot) if (s && p >= s && p < s + f->st.slot_bytes) return true;
    return false;
}
// Sizes the two slots for the streamed matrices laid out so far (reallocated only when a region changes size, which drops the graphs)
// and points every one of them into its slot.
static void stream_slots(b200_falcon * f) {
    auto & S = f->st;
    size_t need[4] = {};
    for (int l : S.layers) for (int r = 0; r < 4; r++) need[r] = std::max(need[r], role_matrix(f->layers[l], r).bytes);
    if (memcmp(need, S.region, sizeof(need)) != 0) {
        invalidate_graphs(f);
        B200_CUDA_CHECK(cudaDeviceSynchronize());
        for (auto & p : S.slot) { B200_CUDA_CHECK(cudaFree(p)); p = nullptr; }
        S.slot_bytes = 0;
        for (int r = 0; r < 4; r++) { S.region[r] = need[r]; S.region_off[r] = S.slot_bytes; S.slot_bytes += need[r]; }
        if (S.slot_bytes) for (auto & p : S.slot) B200_CUDA_CHECK(cudaMalloc(&p, S.slot_bytes));
    }
    for (size_t j = 0; j < S.layers.size(); j++)
        for (int r = 0; r < 4; r++) {
            WPlanes & W = role_matrix(f->layers[S.layers[j]], r);
            if (W.bytes) wplanes_place(W, S.slot[j % 2] + S.region_off[r]);
        }
}
// The planes of streamed matrix `s`, just built in its slot region, become its pinned host image.
static void stream_store(b200_falcon * f, const Slot & s, const WPlanes & W, cudaStream_t st) {
    uint8_t *& img = f->st.image[stream_rank(f, s.layer - f->hp.layer_first)][matrix_role(s)];
    B200_ASSERT(!img);
    B200_CUDA_CHECK(cudaHostAlloc(&img, W.bytes, cudaHostAllocDefault));
    B200_CUDA_CHECK(cudaMemcpyAsync(img, W.p[0], W.bytes, cudaMemcpyDeviceToHost, st));
    B200_CUDA_CHECK(cudaStreamSynchronize(st));
}
// The schedule on s_copy.  Streamed layer j's copy waits until layer j - 2 has released slot j % 2, then brings the four images over
// and records ready[j % 2]; the first two copies go out when s_copy is forked from s_main at the start of the eval, beside the resident
// layers in front of them.  A resident engine enqueues none of this.
static void stream_copy(b200_falcon * f, int j) {
    auto & S = f->st;
    if (j >= 2) B200_CUDA_CHECK(cudaStreamWaitEvent(S.s_copy, S.free[j % 2], 0));
    const Layer & L = f->layers[S.layers[j]];
    for (int r = 0; r < 4; r++) {
        const WPlanes & W = role_matrix(L, r);
        if (S.image[j][r]) B200_CUDA_CHECK(cudaMemcpyAsync(W.p[0], S.image[j][r], W.bytes, cudaMemcpyHostToDevice, S.s_copy));
    }
    B200_CUDA_CHECK(cudaEventRecord(S.ready[j % 2], S.s_copy));
}
static void stream_fork(b200_falcon * f) {
    auto & S = f->st;
    if (S.layers.empty()) return;
    B200_CUDA_CHECK(cudaEventRecord(S.e_fork, f->s_main));
    B200_CUDA_CHECK(cudaStreamWaitEvent(S.s_copy, S.e_fork, 0));
    for (int j = 0; j < (int) S.layers.size() && j < 2; j++) stream_copy(f, j);
}
static void stream_join(b200_falcon * f) {
    auto & S = f->st;
    if (S.layers.empty()) return;
    B200_CUDA_CHECK(cudaEventRecord(S.e_join, S.s_copy));
    B200_CUDA_CHECK(cudaStreamWaitEvent(f->s_main, S.e_join, 0));
}
// acquire: `st`, which is about to read local layer l's matrices, waits until they are in their slot.  release: every read of them has
// been issued on s_main (the branches joined), so the slot may take the streamed layer after next.
static void stream_acquire(b200_falcon * f, int l, cudaStream_t st) {
    const int j = stream_rank(f, l);
    if (j >= 0) B200_CUDA_CHECK(cudaStreamWaitEvent(st, f->st.ready[j % 2], 0));
}
static void stream_release(b200_falcon * f, int l) {
    const int j = stream_rank(f, l);
    if (j < 0) return;
    B200_CUDA_CHECK(cudaEventRecord(f->st.free[j % 2], f->s_main));
    if (j + 2 < (int) f->st.layers.size()) stream_copy(f, j + 2);
}

extern "C" {

b200_falcon * b200_falcon_create(const b200_falcon_params * p) { return b200_falcon_create_kv(p, T_F32); }
b200_falcon * b200_falcon_create_kv(const b200_falcon_params * p, int kv_ggml_type) {
    if (kv_ggml_type != T_F32 && kv_ggml_type != T_F16) return nullptr;
    b200_falcon * f = new b200_falcon();
    f->hp = *p;
    B200_ASSERT(p->n_embd % p->n_head == 0 && p->n_head % p->n_head_kv == 0);
    f->E = p->n_embd; f->H = p->n_head; f->HKV = p->n_head_kv; f->D = p->n_embd / p->n_head;
    f->QKV = (f->H + 2 * f->HKV) * f->D; f->FF = 4 * f->E; f->V = p->n_vocab;
    if (f->hp.world <= 0) { f->hp.world = 1; f->hp.rank = 0; }
    if (f->hp.layer_last <= 0) { f->hp.layer_first = 0; f->hp.layer_last = p->n_layer; }
    f->NL = f->hp.layer_last - f->hp.layer_first;
    f->first = f->hp.rank == 0; f->last = f->hp.rank == f->hp.world - 1;
    f->layers.resize(f->NL);
    B200_CUDA_CHECK(cudaStreamCreateWithFlags(&f->s_main, cudaStreamNonBlocking));
    B200_CUDA_CHECK(cudaStreamCreateWithFlags(&f->s_mlp, cudaStreamNonBlocking));
    B200_CUDA_CHECK(cudaEventCreateWithFlags(&f->e_fork, cudaEventDisableTiming));
    B200_CUDA_CHECK(cudaEventCreateWithFlags(&f->e_join, cudaEventDisableTiming));
    B200_CUDA_CHECK(cudaEventCreate(&f->e_t0)); B200_CUDA_CHECK(cudaEventCreate(&f->e_t1));
    const size_t NB = (size_t) (p->n_batch > 0 ? p->n_batch : 1);
    const bool shadow = p->n_batch > MMV_MAX_N && f->D == 64 && f->NL > 0;      // the prompt kernel's fp16 planes
    auto alloc16 = [&](__half ** d) {
        const size_t sb = (size_t) f->NL * f->shadow_layer * sizeof(__half);
        B200_CUDA_CHECK(cudaMalloc(d, sb ? sb : 4)); B200_CUDA_CHECK(cudaMemset(*d, 0, sb));
    };
    f->kv.ctx_pad = attention_ctx_pad(p->n_ctx);
    if (kv_ggml_type == T_F16) {                 // the cache is the fp16 K plane and V rows (rows padded to a multiple of 64 like the planes)
        f->shadow_layer = (size_t) f->kv.ctx_pad * kv_row(f);
        alloc16(&f->kv.k16); alloc16(&f->kv.v16);
        if (shadow) alloc16(&f->kv.vt16);
    } else {
        const size_t kv = (size_t) f->NL * p->n_ctx * kv_row(f) * sizeof(float);
        B200_CUDA_CHECK(cudaMalloc(&f->kv.k, kv ? kv : 4)); B200_CUDA_CHECK(cudaMalloc(&f->kv.v, kv ? kv : 4));
        B200_CUDA_CHECK(cudaMemset(f->kv.k, 0, kv)); B200_CUDA_CHECK(cudaMemset(f->kv.v, 0, kv));
        if (shadow) { f->shadow_layer = attention_shadow_halves(f->HKV, p->n_ctx); alloc16(&f->kv.k16); alloc16(&f->kv.vt16); }
    }
    B200_CUDA_CHECK(cudaMalloc(&f->inp, NB * f->E * 4)); B200_CUDA_CHECK(cudaMalloc(&f->qkv, NB * f->QKV * 4));
    B200_CUDA_CHECK(cudaMalloc(&f->att, NB * f->E * 4)); B200_CUDA_CHECK(cudaMalloc(&f->ao, NB * f->E * 4));
    B200_CUDA_CHECK(cudaMalloc(&f->up, NB * f->FF * 4)); B200_CUDA_CHECK(cudaMalloc(&f->dn, NB * f->E * 4));
    B200_CUDA_CHECK(cudaMalloc(&f->logits, NB * f->V * 4));
    B200_CUDA_CHECK(cudaMalloc(&f->tokens_dev, NB * 4)); B200_CUDA_CHECK(cudaMalloc(&f->n_past_dev, 4));
    B200_CUDA_CHECK(cudaMalloc(&f->tok_next, 4)); B200_CUDA_CHECK(cudaMalloc(&f->gen_step, 4));
    B200_CUDA_CHECK(cudaMalloc(&f->gen_hist, (size_t) (p->n_ctx > 0 ? p->n_ctx : 1) * 4));
    B200_CUDA_CHECK(cudaMallocHost(&f->tokens_h, NB * 4)); B200_CUDA_CHECK(cudaMallocHost(&f->n_past_h, 4));
    B200_CUDA_CHECK(cudaMalloc(&f->score_tg, NB * 4)); B200_CUDA_CHECK(cudaMalloc(&f->score_nll, NB * 4));
    B200_CUDA_CHECK(cudaMallocHost(&f->score_tg_h, NB * 4)); B200_CUDA_CHECK(cudaMallocHost(&f->score_nll_h, NB * 4));
    f->logits_h_floats = (size_t) f->V; B200_CUDA_CHECK(cudaMallocHost(&f->logits_h, f->logits_h_floats * 4));
    return f;
}
b200_falcon * b200_falcon_create_streamed(const b200_falcon_params * p, int kv_ggml_type, const int32_t * streamed_layers, int n_streamed) {
    if (n_streamed == 0) return b200_falcon_create_kv(p, kv_ggml_type);
    if (n_streamed < 0 || !streamed_layers || p->world > 1) return nullptr;
    const int lf = p->layer_last <= 0 ? 0 : p->layer_first, ll = p->layer_last <= 0 ? p->n_layer : p->layer_last;
    std::vector<int> layers;
    for (int i = 0; i < n_streamed; i++) {
        const int l = streamed_layers[i];
        if (l < lf || l >= ll || std::find(layers.begin(), layers.end(), l - lf) != layers.end()) return nullptr;
        layers.push_back(l - lf);
    }
    b200_falcon * f = b200_falcon_create_kv(p, kv_ggml_type);
    if (!f) return nullptr;
    auto & S = f->st;
    std::sort(layers.begin(), layers.end());
    S.layers = layers;
    S.rank.assign(f->NL, -1);
    for (size_t j = 0; j < layers.size(); j++) S.rank[layers[j]] = (int) j;
    S.image.assign(layers.size(), {});
    B200_CUDA_CHECK(cudaStreamCreateWithFlags(&S.s_copy, cudaStreamNonBlocking));
    for (cudaEvent_t * e : { &S.e_fork, &S.e_join, &S.ready[0], &S.ready[1], &S.free[0], &S.free[1] })
        B200_CUDA_CHECK(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    return f;
}
int b200_falcon_stream_info(const b200_falcon * f, int32_t * layers_out, size_t * host_bytes, size_t * slot_bytes, size_t * copy_bytes) {
    const auto & S = f->st;
    size_t host = 0, copy = 0;
    for (size_t j = 0; j < S.layers.size(); j++) {
        if (layers_out) layers_out[j] = f->hp.layer_first + S.layers[j];
        for (int r = 0; r < 4; r++) {
            const size_t b = role_matrix(f->layers[S.layers[j]], r).bytes;
            copy += b; if (S.image[j][r]) host += b;
        }
    }
    if (host_bytes) *host_bytes = host;
    if (slot_bytes) *slot_bytes = S.slot[0] ? 2 * S.slot_bytes : 0;
    if (copy_bytes) *copy_bytes = copy;
    return (int) S.layers.size();
}

static void ensure_actq(b200_falcon * f) {
    if (!f->attn_dec_scratch) {
        AttnParams ap = { f->H, f->HKV, f->D, 1, 0, nullptr, f->hp.n_ctx, (int64_t) f->QKV };
        const size_t sb = attention_scratch_bytes(ap);
        if (sb) { B200_CUDA_CHECK(cudaMalloc(&f->attn_dec_scratch, sb)); B200_CUDA_CHECK(cudaMemset(f->attn_dec_scratch, 0, sb)); }
    }
    if (!f->q_ctr) { B200_CUDA_CHECK(cudaMalloc(&f->q_ctr, (size_t) (f->FF / 256 + 1) * sizeof(unsigned))); B200_CUDA_CHECK(cudaMemset(f->q_ctr, 0, (size_t) (f->FF / 256 + 1) * sizeof(unsigned))); }
    if (!f->classified) classify(f);
    const int NB = f->hp.n_batch > 0 ? f->hp.n_batch : 1;
    if ((f->generic_layers || f->generic_head) && !f->gen_na) {
        B200_CUDA_CHECK(cudaMalloc(&f->gen_na, (size_t) NB * f->E * 4)); B200_CUDA_CHECK(cudaMalloc(&f->gen_nm, (size_t) NB * f->E * 4));
        size_t ab = 0;
        for (int t : { T_Q8_0, T_Q8_1, T_Q8_K }) { const size_t b = actq_bytes(t, f->FF, NB); if (b > ab) ab = b; }
        B200_CUDA_CHECK(cudaMalloc(&f->gen_mm, ab + (size_t) NB * f->FF * 2));           // codes, then the fp16 GEMM operand
    }
    if (f->actq_mem || f->act_type < 0) return;
    const int at = f->act_type;
    const size_t bE = actq_bytes(at, f->E, NB), bF = actq_bytes(at, f->FF, NB);
    B200_CUDA_CHECK(cudaMalloc(&f->actq_mem, 4 * bE + bF));
    uint8_t * p = (uint8_t *) f->actq_mem;
    actq_bind(f->xa, at, f->E, NB, p); p += bE; actq_bind(f->xm, at, f->E, NB, p); p += bE;
    actq_bind(f->xatt, at, f->E, NB, p); p += bE; actq_bind(f->xf, at, f->E, NB, p); p += bE;
    actq_bind(f->xup, at, f->FF, NB, p);
    if (NB > MMV_MAX_N && !f->xh_a) {
        B200_CUDA_CHECK(cudaMalloc(&f->xh_a, (size_t) NB * f->E * 2)); B200_CUDA_CHECK(cudaMalloc(&f->xh_b, (size_t) NB * f->FF * 2));
        B200_CUDA_CHECK(cudaMalloc(&f->xh_m, (size_t) NB * f->E * 2));
    }
}

static void free_matrix(b200_falcon * f, WPlanes & W) {
    for (const void * b : f->borrowed) if (b == (const void *) W.p[0]) { W = WPlanes{}; return; }      // adopted: its owner frees it
    if (in_slot(f, W.p[0])) { W = WPlanes{}; return; }                                                 // streamed: the slots are shared
    wplanes_free(W);
}

// Empties matrix slot `s` for a new matrix of `type`, which the caller puts there: frees the old one, keeps weight_bytes (every
// matrix but the embedding table, which is gathered from, not streamed) in step and has the model's path re-derived.
static WPlanes & replace_matrix(b200_falcon * f, const Slot & s, int type) {
    invalidate_graphs(f);
    WPlanes & W = *slot_dest(f, s).W;
    const bool counted = s.d->kind != S_EMB;
    if (W.p[0]) { if (counted) f->weight_bytes -= algorithmic_bytes(W.type, W.K, W.M); free_matrix(f, W); }
    if (is_streamed(f, s)) {
        uint8_t *& img = f->st.image[stream_rank(f, s.layer - f->hp.layer_first)][matrix_role(s)];
        if (img) { B200_CUDA_CHECK(cudaFreeHost(img)); img = nullptr; }
    }
    if (counted) f->weight_bytes += algorithmic_bytes(type, slot_K(f, s), slot_M(f, s));
    f->classified = false;
    return W;
}

// A weight matrix that is already resident in this library's planar layout (uploaded by ggml_cuda_transform_tensor for the reference's
// loader, ggml_surface.cu) becomes the engine's matrix `name` without another copy.  Returns false for an unknown name / wrong shape /
// a matrix of another rank or of a streamed layer.
extern "C++" bool falcon_adopt_matrix(b200_falcon * f, const char * name, const WPlanes & W) {
    Slot s;
    if (!find_slot(name, s) || !is_matrix(s) || !owns(f, s) || is_streamed(f, s)) return false;
    if (W.K != slot_K(f, s) || W.M != slot_M(f, s)) return false;
    replace_matrix(f, s, W.type) = W;
    f->borrowed.push_back((const void *) W.p[0]);
    return true;
}

static double wall_seconds() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

static void place_tensor(b200_falcon * f, const Slot & s, int type, const void * host_data, bool random, uint64_t seed) {
    if (!owns(f, s)) return;
    const int64_t K = slot_K(f, s), M = slot_M(f, s);
    cudaStream_t st = f->s_main;
    if (is_matrix(s)) {
        WPlanes & W = replace_matrix(f, s, type);
        if (is_streamed(f, s)) {                    // built in its slot region, kept in its host image
            wplanes_layout(W, type, (int) K, (int) M);
            stream_slots(f);
            if (random) wplanes_fill_random(W, seed, st); else wplanes_fill(W, host_data, st);
            stream_store(f, s, W, st);
        } else if (random) wplanes_alloc_random(W, type, (int) K, (int) M, seed, st);
        else wplanes_upload(W, type, (int) K, (int) M, host_data, st);
    } else {
        invalidate_graphs(f);
        float *& v = *slot_dest(f, s).v;
        if (v) B200_CUDA_CHECK(cudaFree(v));
        B200_CUDA_CHECK(cudaMalloc(&v, (size_t) K * 4));
        if (random) {                               // LayerNorm gamma around 1, beta around 0
            const bool gamma = s.d->kind == S_LNF_G || s.d->kind == S_LN_ATTN_G || s.d->kind == S_LN_MLP_G;
            fill_kernel<<<32, 256, 0, st>>>(v, K, gamma ? 1.f : 0.f, gamma ? 0.1f : 0.01f, seed); B200_CUDA_CHECK(cudaGetLastError());
        } else {
            B200_ASSERT(type == T_F32);
            B200_CUDA_CHECK(cudaMemcpyAsync(v, host_data, (size_t) K * 4, cudaMemcpyHostToDevice, st));
        }
    }
    B200_CUDA_CHECK(cudaStreamSynchronize(st));
}

void b200_falcon_set_tensor(b200_falcon * f, const char * name, int type, int n_dims, const int64_t * ne, const void * data) {
    Slot s;
    if (!find_slot(name, s)) { fprintf(stderr, "b200: unknown tensor '%s'\n", name); abort(); }
    B200_ASSERT(ne[0] == slot_K(f, s) && (n_dims == 1 ? slot_M(f, s) == 1 : ne[1] == slot_M(f, s)));
    place_tensor(f, s, type, data, false, 0);
}
void b200_falcon_set_tensor_random(b200_falcon * f, const char * name, int type, uint64_t seed) {
    Slot s;
    if (!find_slot(name, s)) { fprintf(stderr, "b200: unknown tensor '%s'\n", name); abort(); }
    place_tensor(f, s, type, nullptr, true, seed);
}

// ---- GGCC v10 files are read by ggcc_file.h.  The file is untrusted input: a malformed file makes the loaders return -1 (no assert,
// no leak).
static int ggcc_header(Cursor & c, b200_falcon_params * out) {
    GgccHeader h;
    if (!ggcc_read_header(c, h)) return -1;
    out->n_vocab = (int32_t) h.n_vocab; out->n_embd = (int32_t) h.n_embd; out->n_head = (int32_t) h.n_head; out->n_head_kv = (int32_t) h.n_head_kv;
    out->n_layer = (int32_t) h.n_layer; out->falcon_type = (int32_t) h.falcon_type;
    return 0;
}
int b200_ggcc_read_hparams(const char * path, b200_falcon_params * out) {
    FILE * fp = fopen(path, "rb");
    if (!fp) return -1;
    uint8_t buf[40]; const size_t n = fread(buf, 1, sizeof(buf), fp); fclose(fp);
    if (n < 40) return -1;
    Cursor c = { buf, 0, n, false };
    return ggcc_header(c, out);
}

// GPU-direct weight path (SURVEY 8f-1; replaces the loader's per-tensor blocking cudaMemcpy, libfalcon.cpp:1196-1270 +
// ggml-cuda.cu:3030-3073): the file is mapped, every matrix's planes are allocated up front, then LOAD_THREADS host threads stream row
// chunks  page cache -> pinned ring buffer -> cudaMemcpyAsync -> repack kernel (AoS blocks -> planar layout, formats.cuh)  each on its
// own stream with two buffers in flight, so the host copy of chunk i+1 overlaps the DMA and repack of chunk i; one synchronize at the end.
struct LoadItem { WPlanes * W; const uint8_t * src; int64_t row0, nrows; size_t bytes; };
static constexpr size_t LOAD_BUF = 32u << 20;
static constexpr int LOAD_THREADS = 6, LOAD_SLOTS = 2;

static void load_worker(int dev, const std::vector<LoadItem> * items, std::atomic<size_t> * next) {
    B200_CUDA_CHECK(cudaSetDevice(dev));
    cudaStream_t st; B200_CUDA_CHECK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    uint8_t * pin[LOAD_SLOTS], * stage[LOAD_SLOTS]; cudaEvent_t done[LOAD_SLOTS]; bool used[LOAD_SLOTS] = {};
    for (int k = 0; k < LOAD_SLOTS; k++) {
        B200_CUDA_CHECK(cudaMallocHost(&pin[k], LOAD_BUF)); B200_CUDA_CHECK(cudaMalloc(&stage[k], LOAD_BUF));
        B200_CUDA_CHECK(cudaEventCreateWithFlags(&done[k], cudaEventDisableTiming));
    }
    for (int n = 0;; n++) {
        const size_t i = next->fetch_add(1);
        if (i >= items->size()) break;
        const LoadItem & it = (*items)[i];
        const int k = n % LOAD_SLOTS;
        if (used[k]) B200_CUDA_CHECK(cudaEventSynchronize(done[k]));          // the DMA that read this pinned buffer (and the repack behind it) is finished
        memcpy(pin[k], it.src, it.bytes);                                      // page cache / mmap -> pinned
        B200_CUDA_CHECK(cudaMemcpyAsync(stage[k], pin[k], it.bytes, cudaMemcpyHostToDevice, st));
        launch_repack_rows(*it.W, stage[k], it.row0, it.nrows, st);
        B200_CUDA_CHECK(cudaEventRecord(done[k], st)); used[k] = true;
    }
    B200_CUDA_CHECK(cudaStreamSynchronize(st));
    for (int k = 0; k < LOAD_SLOTS; k++) { cudaFreeHost(pin[k]); cudaFree(stage[k]); cudaEventDestroy(done[k]); }
    cudaStreamDestroy(st);
}

int b200_falcon_load_ggcc(b200_falcon * f, const char * path) {
    const int fd = open(path, O_RDONLY);
    if (fd < 0) { fprintf(stderr, "b200: cannot open %s\n", path); return -1; }
    struct stat sb;
    if (fstat(fd, &sb) != 0 || sb.st_size < 40) { close(fd); return -1; }
    void * map = mmap(nullptr, (size_t) sb.st_size, PROT_READ, MAP_PRIVATE, fd, 0);
    close(fd);
    if (map == MAP_FAILED) return -1;
    auto fail = [&](const char * why) { fprintf(stderr, "b200: %s: %s\n", path, why); munmap(map, (size_t) sb.st_size); return -1; };
    Cursor c = { (const uint8_t *) map, 0, (size_t) sb.st_size, false };
    b200_falcon_params hp{};
    if (ggcc_header(c, &hp) != 0) return fail("not a GGCC v10 file");
    if (hp.n_vocab != f->hp.n_vocab || hp.n_embd != f->hp.n_embd || hp.n_head != f->hp.n_head || hp.n_head_kv != f->hp.n_head_kv || hp.n_layer != f->hp.n_layer)
        return fail("hyper-parameters differ from the engine's");
    GgccHeader gh{}; gh.n_vocab = (uint32_t) hp.n_vocab;
    if (!ggcc_skip_vocab(c, gh)) return fail("truncated vocabulary");
    const double t0 = wall_seconds();
    struct StreamItem { Slot s; const uint8_t * src; size_t row_bytes; };
    std::vector<LoadItem> items;
    std::vector<StreamItem> streamed;
    size_t total = 0;
    for (;;) {
        GgccTensor t; const char * why = nullptr;
        const int got = ggcc_next_tensor(c, t, &why);
        if (got < 0) return fail(why);
        if (got == 0) break;
        const std::string & name = t.name; const uint32_t n_dims = t.n_dims, type = t.type; const int64_t * ne = t.ne;
        const size_t row_bytes = t.row_bytes, nbytes = t.nbytes;
        const TypeSpec ts = type_spec((int) type);
        Slot s;
        if (!find_slot(name, s)) return fail("unknown tensor name");
        const int64_t M = slot_M(f, s);
        if (ne[0] != slot_K(f, s) || (n_dims == 1 ? M != 1 : ne[1] != M)) return fail("tensor shape does not match the hyper-parameters");
        const uint8_t * data = t.data;
        if (!is_matrix(s) || ts.n_planes == 1) {                                // LayerNorm vectors, f16 / f32 matrices: the plain path
            if (!is_matrix(s) && type != T_F32) return fail("1-D tensors must be f32");
            place_tensor(f, s, (int) type, data, false, 0);
            continue;
        }
        if (!owns(f, s)) continue;
        const int64_t chunk = (int64_t) (LOAD_BUF / row_bytes);
        if (chunk < 1) return fail("a row does not fit the staging buffer");
        WPlanes * W = &replace_matrix(f, s, (int) type);
        total += nbytes;
        if (is_streamed(f, s)) {                                                   // laid out now, filled through a slot below
            wplanes_layout(*W, (int) type, (int) ne[0], (int) M);
            streamed.push_back({ s, data, row_bytes });
            continue;
        }
        wplanes_upload(*W, (int) type, (int) ne[0], (int) M, nullptr, f->s_main);  // planes allocated and laid out, filled below
        for (int64_t r0 = 0; r0 < M; r0 += chunk) {
            const int64_t nr = r0 + chunk <= M ? chunk : M - r0;
            items.push_back({ W, data + (size_t) r0 * row_bytes, r0, nr, (size_t) nr * row_bytes });
        }
    }
    int dev; B200_CUDA_CHECK(cudaGetDevice(&dev));
    std::atomic<size_t> next(0);
    std::vector<std::thread> th;
    for (int t = 0; t < LOAD_THREADS; t++) th.emplace_back(load_worker, dev, &items, &next);
    for (auto & t : th) t.join();
    // streamed matrices, one at a time through their slot region: raw rows H2D, the repack, the planes D2H into the host image
    if (!streamed.empty()) {
        stream_slots(f);
        uint8_t * stage = nullptr;
        B200_CUDA_CHECK(cudaMalloc(&stage, LOAD_BUF));
        for (const StreamItem & it : streamed) {
            const WPlanes & W = *slot_dest(f, it.s).W;
            const int64_t chunk = (int64_t) (LOAD_BUF / it.row_bytes);
            for (int64_t r0 = 0; r0 < W.M; r0 += chunk) {
                const int64_t nr = std::min(chunk, (int64_t) W.M - r0);
                B200_CUDA_CHECK(cudaMemcpyAsync(stage, it.src + (size_t) r0 * it.row_bytes, (size_t) nr * it.row_bytes, cudaMemcpyHostToDevice, f->s_main));
                launch_repack_rows(W, stage, r0, nr, f->s_main);
            }
            stream_store(f, it.s, W, f->s_main);
        }
        B200_CUDA_CHECK(cudaFree(stage));
    }
    munmap(map, (size_t) sb.st_size);
    f->load_seconds = wall_seconds() - t0; f->load_bytes = total;
    if (getenv("B200_VERBOSE")) fprintf(stderr, "b200: %s: %.2f GB of quantised matrices in %.2f s (%.1f GB/s)\n", path, total / 1e9, f->load_seconds, total / 1e9 / f->load_seconds);
    return 0;
}
double b200_falcon_load_seconds(const b200_falcon * f, size_t * bytes) { if (bytes) *bytes = f->load_bytes; return f->load_seconds; }

size_t b200_falcon_weight_bytes(const b200_falcon * f) { return f->weight_bytes; }

void b200_nccl_unique_id(void * id128) { ncclUniqueId id; B200_NCCL_CHECK(nccl().GetUniqueId(&id)); memcpy(id128, &id, sizeof(id)); }
void b200_falcon_init_pipeline(b200_falcon * f, const void * id128) {
    if (f->hp.world <= 1) return;
    ncclUniqueId id; memcpy(&id, id128, sizeof(id));
    B200_NCCL_CHECK(nccl().CommInitRank(&f->comm, f->hp.world, id, f->hp.rank));
}

void b200_falcon_free(b200_falcon * f) {
    if (!f) return;
    cudaDeviceSynchronize();
    for (auto & L : f->layers) { free_matrix(f, L.wqkv); free_matrix(f, L.wo); free_matrix(f, L.up); free_matrix(f, L.down);
        cudaFree(L.ln_attn_g); cudaFree(L.ln_attn_b); cudaFree(L.ln_mlp_g); cudaFree(L.ln_mlp_b); }
    free_matrix(f, f->tok_emb); free_matrix(f, f->lm_head);
    for (auto & img : f->st.image) for (uint8_t * p : img) cudaFreeHost(p);
    cudaFree(f->st.slot[0]); cudaFree(f->st.slot[1]);
    if (f->st.s_copy) {
        cudaStreamDestroy(f->st.s_copy);
        for (cudaEvent_t e : { f->st.e_fork, f->st.e_join, f->st.ready[0], f->st.ready[1], f->st.free[0], f->st.free[1] }) cudaEventDestroy(e);
    }
    cudaFree(f->lnf_g); cudaFree(f->lnf_b); cudaFree(f->kv.k); cudaFree(f->kv.v); cudaFree(f->kv.k16); cudaFree(f->kv.v16); cudaFree(f->kv.vt16);
    cudaFree(f->inp); cudaFree(f->qkv); cudaFree(f->att); cudaFree(f->ao); cudaFree(f->up); cudaFree(f->dn); cudaFree(f->logits);
    f->attn_scratch.release(); cudaFree(f->actq_mem); cudaFree(f->gen_na); cudaFree(f->gen_nm); cudaFree(f->gen_mm); cudaFree(f->xh_a); cudaFree(f->xh_b); cudaFree(f->xh_m);
    cudaFree(f->tokens_dev); cudaFree(f->n_past_dev); cudaFree(f->q_ctr); cudaFree(f->attn_dec_scratch); cudaFree(f->tap.mem);
    cudaFreeHost(f->tokens_h); cudaFreeHost(f->n_past_h); cudaFreeHost(f->logits_h);
    cudaFree(f->emb_dev); cudaFreeHost(f->emb_h);
    cudaFree(f->score_tg); cudaFree(f->score_nll); cudaFreeHost(f->score_tg_h); cudaFreeHost(f->score_nll_h);
    for (auto & tier : f->graph) for (auto & g : tier) if (g.exec) cudaGraphExecDestroy(g.exec);
    cudaFree(f->tok_next); cudaFree(f->gen_hist); cudaFree(f->gen_step); cudaFree(f->sampler_work); sampler_state_free(f->sampler);
    if (f->comm) nccl().CommDestroy(f->comm);
    cudaEventDestroy(f->e_fork); cudaEventDestroy(f->e_join); cudaEventDestroy(f->e_t0); cudaEventDestroy(f->e_t1);
    cudaStreamDestroy(f->s_main); cudaStreamDestroy(f->s_mlp);
    delete f;
}

} // extern "C"

// ------------------------------------------------------------------------------------------------ eval
static void mmv(b200_falcon * f, const WPlanes & W, const ActQ & A, float * y, int64_t y_stride, const MmvEpilogue & e, cudaStream_t st) {
    launch_mmv(W, A, y, y_stride, e, st); f->launches++;
}

// Y = W x for ANY weight type, from fp32 activation rows (stride K), the format made on the spot (launch_mul_mat).  F16 weights above
// MMV_MAX_N tokens take fp16-rounded rows (ggml_compute_forward_mul_mat_f16_f32, ggml.c:11232-11251) and the GEMM.  Slow path: see
// b200_falcon::generic_layers.
static void mm_any(b200_falcon * f, const WPlanes & W, const float * x, int N, float * y, int64_t y_stride, bool gelu, cudaStream_t st) {
    if (W.type == T_F16 && N > MMV_MAX_N) {
        __half * xh = (__half *) f->gen_mm;
        launch_f32_to_f16(x, xh, (int64_t) N * W.K, st);
        launch_mmq_gemm(W, xh, W.K, N, y, y_stride, 0, st); f->launches += 2;
        if (gelu) { B200_ASSERT(y_stride == W.M); launch_gelu(y, y, (int64_t) N * W.M, st); f->launches++; }            // ggml.c:10298-10337
    } else f->launches += launch_mul_mat(W, x, W.K, N, y, y_stride, gelu ? EPI_GELU : EPI_NONE, f->gen_mm, st);
}

// Test tap: D2D copies on s_main, after everything that writes the tapped buffers and before anything overwrites them.  Off (no mem):
// nothing is enqueued.
static void tap_copy(b200_falcon * f, const std::vector<b200_falcon::TapNode> & nodes, uint8_t * dst) {
    for (const auto & n : nodes)
        B200_CUDA_CHECK(cudaMemcpyAsync(dst + n.off, n.src, n.row_bytes * (n.all_rows ? f->tap.rows : f->tap.head_rows), cudaMemcpyDeviceToDevice, f->s_main));
}
static void tap_layer(b200_falcon * f, int l, int N) {
    if (!f->tap.mem) return;
    f->tap.rows = N;
    if (f->tap.slice[l] >= 0) tap_copy(f, f->tap.layer, f->tap.mem + (size_t) f->tap.slice[l] * f->tap.layer_bytes);
}
static void tap_head(b200_falcon * f, int N, int nr) {
    if (!f->tap.mem) return;
    f->tap.rows = N; f->tap.head_rows = nr;
    tap_copy(f, f->tap.head, f->tap.mem + (size_t) f->tap.n_slices * f->tap.layer_bytes);
}

// final LayerNorm + lm_head over rows x[0 .. nr) of the residual stream: libfalcon.cpp:2422-2440.  ra / rb (optional, quantised head
// only): the last layer's branch outputs, which the LayerNorm kernel adds to x first (x = (ra + rb) + x, written back).  With embeddings
// on, the quantised head's LayerNorm also stores its last row in fp32 (the row falcon_eval_internal copies, libfalcon.cpp:2551-2557).
static void enqueue_head(b200_falcon * f, float * x, int nr, const float * ra, const float * rb, cudaStream_t sa) {
    const int E = f->E;
    if (f->generic_head) {
        launch_layernorm(x, E, f->lnf_g, f->lnf_b, f->gen_na, E, E, nr, sa); f->launches++;
        mm_any(f, f->lm_head, f->gen_na, nr, f->logits, f->V, false, sa);
        f->emb_src = f->gen_na + (size_t) (nr - 1) * E;
        return;
    }
    ActQ xfr = f->xf; xfr.N = nr;
    if (nr > MMV_MAX_N) xfr.h = f->xh_a;
    launch_layernorm_q(x, E, ra, rb, ra ? E : 0, f->lnf_g, f->lnf_b, &xfr, nullptr, nullptr, nullptr, E, nr, sa,
                       f->emb_on ? f->emb_dev : nullptr, E, nr - 1); f->launches++;
    f->launches += launch_mul_mat_q(f->lm_head, xfr, nr, f->logits, f->V, EPI_NONE, sa);
    f->emb_src = f->emb_dev;
}
// the head's "result_norm" row to the host, behind the logits copy of the same eval (a node of the G_HOST decode graph for one token)
static void enqueue_embedding_copy(b200_falcon * f) {
    if (f->emb_on) B200_CUDA_CHECK(cudaMemcpyAsync(f->emb_h, f->emb_src, (size_t) f->E * 4, cudaMemcpyDeviceToHost, f->s_main));
}

// Generation step (graph G_GEN): where the token id comes from and where the sampled one goes.
//   rank 0 of a pipeline receives the id the last rank sampled in the previous step (one 4-byte ncclRecv, in-graph, eval_input);
//   the last rank samples from its logits on the device, records the id and sends it to rank 0 (single GPU: writes it
//   straight into the embedding gather's input).  No logits and no token id touch the host between steps.
static void ring_token_out(b200_falcon * f) {
    if (!f->ring_mode) return;
    int32_t * dst = f->hp.world > 1 ? f->tok_next : f->tokens_dev;
    if (f->use_sampler) launch_sample(f->logits, f->V, f->sampler_p, f->sampler, f->sampler_work, dst, f->gen_hist, f->gen_step, nullptr, f->s_main);
    else launch_argmax_hist(f->logits, f->V, dst, f->gen_hist, f->gen_step, f->s_main);
    f->launches++;
    if (f->hp.world > 1) B200_NCCL_CHECK(nccl().Send(f->tok_next, 1, ncclInt32, 0, f->comm, f->s_main));
}

// The residual stream's rows at the start of an eval: the embedding gather of the token ids on the first rank (libfalcon.cpp:2120),
// the rows the previous rank sent on every other one.  The streamed layers' copies start here.
static void eval_input(b200_falcon * f, int N) {
    stream_fork(f);
    if (f->first) {
        if (f->ring_mode && f->hp.world > 1) B200_NCCL_CHECK(nccl().Recv(f->tokens_dev, 1, ncclInt32, f->hp.world - 1, f->comm, f->s_main));
        launch_dequant_rows(f->tok_emb, f->tokens_dev, N, f->inp, f->E, f->s_main); f->launches++;
    } else B200_NCCL_CHECK(nccl().Recv(f->inp, (size_t) N * f->E, ncclFloat, f->hp.rank - 1, f->comm, f->s_main));
}
// The end of an eval: the residual adds of the last local layer (:2399-2400), then on the last rank the head over rows
// [logits_rows_from, N) (none when logits_rows_from == N: a scoring batch without a scored row) and, in the generation-step graph,
// the sampled id; on every other rank the rows go on to the next one.
// fold_add: a quantised head's LayerNorm kernel does the adds (one kernel less on the decode step)
static void eval_output(b200_falcon * f, int N, int logits_rows_from, bool fold_add) {
    stream_join(f);
    const bool fold = fold_add && f->last && !f->generic_head && f->NL > 0;
    if (f->NL > 0 && !fold) { launch_add3(f->dn, f->ao, f->inp, f->inp, (int64_t) N * f->E, f->s_main); f->launches++; }
    if (!f->last) { B200_NCCL_CHECK(nccl().Send(f->inp, (size_t) N * f->E, ncclFloat, f->hp.rank + 1, f->comm, f->s_main)); return; }
    if (logits_rows_from < N)
        enqueue_head(f, f->inp + (size_t) logits_rows_from * f->E, N - logits_rows_from, fold ? f->dn : nullptr, fold ? f->ao : nullptr, f->s_main);
    tap_head(f, N, N - logits_rows_from);
    ring_token_out(f);
}

// AttnParams of local layer l for N new tokens.  graph_mode: n_past is read from the device scalar, and the tier the graph is captured
// for (cur_tier) says whether the long-context kernels may be captured.
static AttnParams attn_params(const b200_falcon * f, int l, int N, int n_past, float theta_scale, bool graph_mode) {
    AttnParams ap = { f->H, f->HKV, f->D, N, n_past, graph_mode ? f->n_past_dev : nullptr, f->hp.n_ctx, (int64_t) f->QKV };
    ap.long_ctx = graph_mode ? f->cur_tier : 0;
    ap.rope_theta_scale = theta_scale;
    ap.kv = kv_layer(f, l);
    return ap;
}
// RoPE + KV append of layer l's new rows (:2229-2281), then the attention qkv -> att (:2285-2366).  Prompts run eagerly, on s_main
// like their attention: a scratch that has to grow waits for the previous user.
static void enqueue_attention(b200_falcon * f, int l, const AttnParams & ap, cudaStream_t st) {
    float * scratch = ap.n_tok > 1 ? (float *) f->attn_scratch.get(attention_scratch_bytes(ap), st) : f->attn_dec_scratch;
    bool rotated = true;
    f->launches += launch_attention(f->qkv, f->att, f->E, ap, scratch, st, nullptr, &rotated);
    if (f->tap.mem) f->tap.rotated[l] = rotated;
}

static bool fused_decode_ok(const b200_falcon * f) {
    if (getenv("B200_NO_FUSED_DECODE")) return false;
    for (const auto & L : f->layers)
        if (!mmv_fast_supports(L.wo.type, L.wo.K) || !mmv_fast_supports(L.down.type, L.down.K) ||
            !mmv_fast_supports(L.up.type, L.up.K) || !mmv_fast_supports(L.wqkv.type, L.wqkv.K)) return false;
    return f->act_type >= 0 && f->FF % 256 == 0;
}
// ---- decode (N == 1) on the register-resident mat-vecs, 7 kernels per layer: one LayerNorm kernel (the previous layer's residual adds +
// LayerNorm(s) + activation quantisation), the four mat-vecs, and the two split-KV attention kernels, which do RoPE + the KV append and
// quantise wo's input.
static void enqueue_decode_fused(b200_falcon * f, int n_past, float theta_scale, bool graph_mode) {
    cudaStream_t sa = f->s_main, sb = f->s_mlp;
    const int E = f->E;
    const bool dual = f->hp.falcon_type == 40;
    ensure_actq(f);
    ActQ xa = f->xa, xm = f->xm, xup = f->xup, xatt = f->xatt; xa.N = xm.N = xup.N = xatt.N = 1;
    eval_input(f, 1);
    const MmvEpilogue none = { EPI_NONE, nullptr, nullptr, nullptr, nullptr };
    // ffn_up applies GELU and, chunk by chunk as CTAs finish, quantises its output row for ffn_down (no INIT pass, no prologue work there)
    MmvEpilogue gelu = { EPI_GELU, nullptr, nullptr, &xup, f->q_ctr };
    // ffn_up reads the LayerNorm's output, which was complete and flushed before qkv's rows started: nothing it reads comes from the kernel in
    // front of it (MmvEpilogue::late_wait).  wo does NOT get it although it reads nothing of ffn_down's either: its input comes from the
    // attention kernels of the OTHER stream, and inside the captured graph that join may be a programmatic edge too -- only
    // griddepcontrol.wait then guarantees that their stores are visible (one wrong eval in ~12 runs of a tiny model with a late wait there).
    MmvEpilogue wo_epi = none;
    gelu.late_wait = 1;
    // All four mat-vecs of a layer go back to back on ONE stream (each is launched with programmatic dependent launch,
    // so its weight prefetch overlaps the previous one's tail); the small attention kernels run beside ffn_up on the
    // second stream:   s_main: LN -> qkv -> ffn_up(+GELU) -> ffn_down -> wo   (7B: wo -> ffn_down)     s_mlp: attention (RoPE + KV append inside)
    for (int l = 0; l < f->NL; l++) {
        const Layer & L = f->layers[l];
        const float * ra = l > 0 ? f->dn : nullptr, * rb = l > 0 ? f->ao : nullptr;
        if (dual) launch_layernorm_q(f->inp, E, ra, rb, E, L.ln_attn_g, L.ln_attn_b, &xa, L.ln_mlp_g, L.ln_mlp_b, &xm, E, 1, sa);
        else      launch_layernorm_q(f->inp, E, ra, rb, E, L.ln_mlp_g, L.ln_mlp_b, &xm, nullptr, nullptr, nullptr, E, 1, sa);
        f->launches++;
        stream_acquire(f, l, sa);
        mmv(f, L.wqkv, dual ? xa : xm, f->qkv, f->QKV, none, sa);                                                // libfalcon.cpp:2192
        B200_CUDA_CHECK(cudaEventRecord(f->e_fork, sa));
        B200_CUDA_CHECK(cudaStreamWaitEvent(sb, f->e_fork, 0));
        AttnParams ap = attn_params(f, l, 1, n_past, theta_scale, graph_mode);
        ap.fuse_rope = 1;
        ap.qout = &xatt;                       // wo's activation quantisation, off the critical path
        enqueue_attention(f, l, ap, sb);
        B200_CUDA_CHECK(cudaEventRecord(f->e_join, sb));
        mmv(f, L.up, xm, f->up, f->FF, gelu, sa);                                                                // :2389-2392
        // The attention kernels of the side stream run BESIDE ffn_up, and beside ffn_down too when its CTAs leave them registers
        // (Falcon-40B / 180B: at long contexts the attention outlasts ffn_up, and this order beat wo first).
        // Falcon-7B's ffn_down shape fills the SMs: attention work still pending when ffn_up ends would be shut out until it had
        // drained, so there wo (which has to wait for the attention anyway) goes first.
        const bool wo_first = mmv_fast_fills_sm(L.down);
        if (!wo_first) mmv(f, L.down, xup, f->dn, E, none, sa);                                                 // :2394
        B200_CUDA_CHECK(cudaStreamWaitEvent(sa, f->e_join, 0));
        mmv(f, L.wo, xatt, f->ao, E, wo_epi, sa);                                                                // :2370
        if (wo_first) mmv(f, L.down, xup, f->dn, E, none, sa);
        stream_release(f, l);
        tap_layer(f, l, 1);
    }
    eval_output(f, 1, 0, true);                                                      // :2399-2400, 2422-2440
}

// The eval for models the fused paths do not cover (see b200_falcon::generic_layers): one stream, one kernel per graph node of
// libfalcon.cpp:2120-2440, activations kept in fp32 between the nodes exactly as ggml keeps them.
static void enqueue_eval_generic(b200_falcon * f, int N, int n_past, float theta_scale, bool graph_mode, int logits_rows_from) {
    cudaStream_t sa = f->s_main;
    const int E = f->E, FF = f->FF;
    const bool dual = f->hp.falcon_type == 40;
    eval_input(f, N);
    for (int l = 0; l < f->NL; l++) {
        const Layer & L = f->layers[l];
        if (l > 0) { launch_add3(f->dn, f->ao, f->inp, f->inp, (int64_t) N * E, sa); f->launches++; }                 // :2399-2400
        launch_layernorm(f->inp, E, L.ln_mlp_g, L.ln_mlp_b, f->gen_nm, E, E, N, sa); f->launches++;                     // :2166-2185
        if (dual) { launch_layernorm(f->inp, E, L.ln_attn_g, L.ln_attn_b, f->gen_na, E, E, N, sa); f->launches++; }
        stream_acquire(f, l, sa);
        mm_any(f, L.wqkv, dual ? f->gen_na : f->gen_nm, N, f->qkv, f->QKV, false, sa);                                   // :2192
        enqueue_attention(f, l, attn_params(f, l, N, n_past, theta_scale, graph_mode), sa);
        mm_any(f, L.wo, f->att, N, f->ao, E, false, sa);                                                                 // :2370
        mm_any(f, L.up, f->gen_nm, N, f->up, FF, true, sa);                                                              // :2389-2392
        mm_any(f, L.down, f->up, N, f->dn, E, false, sa);                                                                // :2394
        stream_release(f, l);
        tap_layer(f, l, N);
    }
    eval_output(f, N, logits_rows_from, false);
}

// Enqueue one eval of N tokens on (s_main, s_mlp).  Device scalars carry n_past when `graph_mode`.
static void enqueue_eval(b200_falcon * f, int N, int n_past, float theta_scale, bool graph_mode, int logits_rows_from) {
    ensure_actq(f);
    if (f->generic_layers) { enqueue_eval_generic(f, N, n_past, theta_scale, graph_mode, logits_rows_from); return; }
    if (N == 1 && fused_decode_ok(f)) { enqueue_decode_fused(f, n_past, theta_scale, graph_mode); return; }
    cudaStream_t sa = f->s_main, sb = f->s_mlp;
    const int E = f->E, FF = f->FF;
    const bool dual = f->hp.falcon_type == 40;
    B200_ASSERT(f->act_type >= 0);
    ActQ xa = f->xa, xm = f->xm, xatt = f->xatt, xup = f->xup;
    xa.N = xm.N = xatt.N = xup.N = N;
    if (N > MMV_MAX_N) { xa.h = f->xh_a; xm.h = f->xh_m; xatt.h = f->xh_a; xup.h = f->xh_b; }     // GEMM path: fp16 operands come with the codes
    eval_input(f, N);
    for (int l = 0; l < f->NL; l++) {
        const Layer & L = f->layers[l];
        // residual adds of the previous layer + LayerNorm(s) + activation quantisation, one kernel
        const float * ra = l > 0 ? f->dn : nullptr, * rb = l > 0 ? f->ao : nullptr;
        if (dual) launch_layernorm_q(f->inp, E, ra, rb, E, L.ln_attn_g, L.ln_attn_b, &xa, L.ln_mlp_g, L.ln_mlp_b, &xm, E, N, sa);
        else      launch_layernorm_q(f->inp, E, ra, rb, E, L.ln_mlp_g, L.ln_mlp_b, &xm, nullptr, nullptr, nullptr, E, N, sa);
        f->launches++;
        // fork: MLP branch on s_mlp
        B200_CUDA_CHECK(cudaEventRecord(f->e_fork, sa));
        B200_CUDA_CHECK(cudaStreamWaitEvent(sb, f->e_fork, 0));
        stream_acquire(f, l, sb);
        f->launches += launch_mul_mat_q(L.up, xm, N, f->up, FF, EPI_GELU, sb);                                   // libfalcon.cpp:2389-2392
        launch_quantize_act(f->up, FF, xup, sb); f->launches++;
        f->launches += launch_mul_mat_q(L.down, xup, N, f->dn, E, EPI_NONE, sb);                                 // :2394
        B200_CUDA_CHECK(cudaEventRecord(f->e_join, sb));
        // attention branch on s_main
        stream_acquire(f, l, sa);
        f->launches += launch_mul_mat_q(L.wqkv, dual ? xa : xm, N, f->qkv, f->QKV, EPI_NONE, sa);                // :2192
        AttnParams ap = attn_params(f, l, N, n_past, theta_scale, graph_mode);
        ap.fuse_rope = N == 1;                                                                                   // decode: RoPE + KV append inside the attention kernels
        enqueue_attention(f, l, ap, sa);
        launch_quantize_act(f->att, E, xatt, sa); f->launches++;
        f->launches += launch_mul_mat_q(L.wo, xatt, N, f->ao, E, EPI_NONE, sa);                                  // :2370
        B200_CUDA_CHECK(cudaStreamWaitEvent(sa, f->e_join, 0));                                                  // join
        stream_release(f, l);
        tap_layer(f, l, N);
    }
    eval_output(f, N, logits_rows_from, false);
}

__global__ void set_i32_kernel(int * p, int v) { *p = v; }

static int tier_of(int n_past) { return n_past + 1 > attention_long_threshold() ? 1 : 0; }
static void build_decode_graph(b200_falcon * f, int which, float theta_scale, int tier) {
    auto & dg = f->graph[tier][which];
    if (dg.exec) { B200_CUDA_CHECK(cudaGraphExecDestroy(dg.exec)); dg.exec = nullptr; }
    f->cur_tier = tier;
    auto host_inputs = [&] {                   // G_HOST: position and token id come from the pinned host scalars
        if (which != G_HOST) return;
        B200_CUDA_CHECK(cudaMemcpyAsync(f->n_past_dev, f->n_past_h, 4, cudaMemcpyHostToDevice, f->s_main));
        if (f->first) B200_CUDA_CHECK(cudaMemcpyAsync(f->tokens_dev, f->tokens_h, 4, cudaMemcpyHostToDevice, f->s_main));
    };
    // one eager pass first: sets the kernels' shared-memory attributes and allocates the activation arena outside
    // the capture (it recomputes the same token at the same position, which the replay then overwrites identically)
    host_inputs();
    enqueue_eval(f, 1, 0, theta_scale, true, 0);
    B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
    cudaGraph_t g;
    f->launches = 0;
    B200_CUDA_CHECK(cudaStreamBeginCapture(f->s_main, cudaStreamCaptureModeThreadLocal));
    host_inputs();
    f->ring_mode = which == G_GEN;                 // (the eager pass above ran without it: every rank must issue the same NCCL calls there)
    enqueue_eval(f, 1, 0, theta_scale, true, 0);
    f->ring_mode = false;
    if (which == G_HOST && f->last) {
        B200_CUDA_CHECK(cudaMemcpyAsync(f->logits_h, f->logits, (size_t) f->V * 4, cudaMemcpyDeviceToHost, f->s_main));
        enqueue_embedding_copy(f);
    }
    B200_CUDA_CHECK(cudaStreamEndCapture(f->s_main, &g));
    B200_CUDA_CHECK(cudaGraphInstantiate(&dg.exec, g, 0));
    B200_CUDA_CHECK(cudaGraphDestroy(g));
    dg.theta = theta_scale; f->graph_launches = f->launches; f->cur_tier = 0;
}
// the decode step graph (which, tier) for RoPE theta scale `theta`, built first unless it exists for that theta; a build runs the step
// once eagerly, on the device inputs the caller has set
static cudaGraphExec_t decode_graph(b200_falcon * f, int which, int tier, float theta) {
    if (!f->graph[tier][which].exec || f->graph[tier][which].theta != theta) build_decode_graph(f, which, theta, tier);
    return f->graph[tier][which].exec;
}

// b200_falcon_eval's argument checks: 0, 1 (batch or positions outside the engine's n_batch / n_ctx), 2 (a token id outside the vocabulary)
static int eval_args(const b200_falcon * f, const int32_t * tokens, int n_tokens, int n_past) {
    if (n_tokens <= 0 || n_past < 0 || n_past + n_tokens > f->hp.n_ctx || n_tokens > (f->hp.n_batch > 0 ? f->hp.n_batch : 1)) return 1;
    if (f->first) {                                  // token ids index the embedding matrix: reject anything outside it (ggml_get_rows asserts, ggml.c:11990)
        if (!tokens) return 1;
        for (int i = 0; i < n_tokens; i++) if (tokens[i] < 0 || tokens[i] >= f->V) return 2;
    }
    return 0;
}

// One batch of b200_falcon_score / b200_falcon_perplexity on s_main, tokens already in tokens_dev: the eval of N tokens at n_past, then
// the scoring kernel over the rows whose device target is not -1, terms into nll_dev.  scored: some target is not -1; the head then runs
// over all N rows, the rows b200_falcon_eval(all_logits = 1) runs it over (the mat-vec head up to MMV_MAX_N rows, the GEMM above: a
// suffix of the rows could take the other path and round differently), otherwise not at all.  One token replays the decode step graph
// as b200_falcon_eval does, minus its logits copy.
static void enqueue_score_batch(b200_falcon * f, int N, int n_past, float theta, const int32_t * targets_dev, float * nll_dev, bool scored) {
    if (N == 1) {
        set_i32_kernel<<<1, 1, 0, f->s_main>>>(f->n_past_dev, n_past);
        const cudaGraphExec_t g = decode_graph(f, G_DEVICE, tier_of(n_past), theta);
        B200_CUDA_CHECK(cudaGraphLaunch(g, f->s_main));
        f->launches = f->graph_launches;
    } else {
        f->launches = 0;
        enqueue_eval(f, N, n_past, theta, false, scored ? 0 : N);
    }
    if (scored) { launch_token_nll(f->logits, f->V, N, f->V, targets_dev, nll_dev, f->s_main); f->launches++; }
}

extern "C" {

// The eval in two halves: enqueue everything (returns at once: the GPU works while the caller does something else) / wait and hand the
// logits over.  b200_falcon_eval is begin + finish; the operator hook (ggml_surface.cu) calls begin at the graph's first ROPE node and
// finish at "result_lm_head", so the reference's walk over its remaining ~2000 graph nodes overlaps the device work.
extern "C++" int falcon_eval_begin(b200_falcon * f, const int32_t * tokens, int n_tokens, int n_past, int n_ctx_rope, int all_logits) {
    const int rc = eval_args(f, tokens, n_tokens, n_past);
    if (rc != 0) return rc;
    const float theta = falcon_rope_theta_scale(f->D, n_ctx_rope, f->hp.n_ctx);         // libfalcon.cpp:2229-2234
    if (n_tokens == 1) {
        f->tokens_h[0] = tokens ? tokens[0] : 0; *f->n_past_h = n_past;
        const cudaGraphExec_t g = decode_graph(f, G_HOST, tier_of(n_past), theta);
        B200_CUDA_CHECK(cudaEventRecord(f->e_t0, f->s_main));
        B200_CUDA_CHECK(cudaGraphLaunch(g, f->s_main));
        B200_CUDA_CHECK(cudaEventRecord(f->e_t1, f->s_main));
        f->launches = f->graph_launches;
        f->pending_floats = f->last ? (size_t) f->V : 0;
    } else {
        const int r0 = all_logits ? 0 : n_tokens - 1;
        f->launches = 0;
        if (f->first) { memcpy(f->tokens_h, tokens, (size_t) n_tokens * 4);
            B200_CUDA_CHECK(cudaMemcpyAsync(f->tokens_dev, f->tokens_h, (size_t) n_tokens * 4, cudaMemcpyHostToDevice, f->s_main)); }
        B200_CUDA_CHECK(cudaEventRecord(f->e_t0, f->s_main));
        enqueue_eval(f, n_tokens, n_past, theta, false, r0);
        B200_CUDA_CHECK(cudaEventRecord(f->e_t1, f->s_main));
        f->pending_floats = 0;
        if (f->last) {
            const size_t nfl = (size_t) (n_tokens - r0) * f->V;
            if (nfl > f->logits_h_floats) {          // the G_HOST graphs copy its logits row into this buffer: rebuild it around the new one
                invalidate_graphs(f);
                B200_CUDA_CHECK(cudaFreeHost(f->logits_h)); f->logits_h_floats = nfl; B200_CUDA_CHECK(cudaMallocHost(&f->logits_h, nfl * 4));
            }
            B200_CUDA_CHECK(cudaMemcpyAsync(f->logits_h, f->logits, nfl * 4, cudaMemcpyDeviceToHost, f->s_main));
            enqueue_embedding_copy(f);
            f->pending_floats = nfl;
        }
    }
    f->emb_valid = f->emb_on;
    return 0;
}
extern "C++" void falcon_eval_finish(b200_falcon * f, float * logits, float * embedding) {
    B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
    if (logits && f->pending_floats) memcpy(logits, f->logits_h, f->pending_floats * 4);
    if (embedding) { B200_ASSERT(f->emb_valid); memcpy(embedding, f->emb_h, (size_t) f->E * 4); }
    B200_CUDA_CHECK(cudaEventElapsedTime(&f->last_ms, f->e_t0, f->e_t1));
}
int b200_falcon_eval(b200_falcon * f, const int32_t * tokens, int n_tokens, int n_past, int n_ctx_rope, float * logits, int all_logits) {
    const int rc = falcon_eval_begin(f, tokens, n_tokens, n_past, n_ctx_rope, all_logits);
    if (rc != 0) return rc;
    falcon_eval_finish(f, logits);
    return 0;
}

int b200_falcon_set_embeddings(b200_falcon * f, int on) {
    if (!f->last) return 1;
    if ((on != 0) != f->emb_on) invalidate_graphs(f);          // the decode graphs hold the LayerNorm kernel's output and the copy, or neither
    f->emb_on = on != 0;
    if (f->emb_on && !f->emb_dev) {
        B200_CUDA_CHECK(cudaMalloc(&f->emb_dev, (size_t) f->E * 4)); B200_CUDA_CHECK(cudaMallocHost(&f->emb_h, (size_t) f->E * 4));
    }
    if (!f->emb_on) f->emb_valid = false;
    return 0;
}
const float * b200_falcon_embeddings(const b200_falcon * f) { return f->emb_valid ? f->emb_h : nullptr; }

int b200_falcon_score(b200_falcon * f, const int32_t * tokens, int n_tokens, int n_past, int n_ctx_rope, const int32_t * targets, float * nll) {
    if (f->hp.world > 1) return 1;
    const int rc = eval_args(f, tokens, n_tokens, n_past);
    if (rc != 0) return rc;
    if (!targets) return 3;
    bool scored = false;
    for (int i = 0; i < n_tokens; i++) {
        if (targets[i] < -1 || targets[i] >= f->V) return 3;
        scored = scored || targets[i] >= 0;
    }
    if (scored && !nll) return 1;
    f->emb_valid = false;
    const float theta = falcon_rope_theta_scale(f->D, n_ctx_rope, f->hp.n_ctx);
    const size_t bytes = (size_t) n_tokens * 4;
    memcpy(f->tokens_h, tokens, bytes); memcpy(f->score_tg_h, targets, bytes);
    B200_CUDA_CHECK(cudaMemcpyAsync(f->tokens_dev, f->tokens_h, bytes, cudaMemcpyHostToDevice, f->s_main));
    B200_CUDA_CHECK(cudaMemcpyAsync(f->score_tg, f->score_tg_h, bytes, cudaMemcpyHostToDevice, f->s_main));
    B200_CUDA_CHECK(cudaEventRecord(f->e_t0, f->s_main));
    enqueue_score_batch(f, n_tokens, n_past, theta, f->score_tg, f->score_nll, scored);
    B200_CUDA_CHECK(cudaEventRecord(f->e_t1, f->s_main));
    if (scored) B200_CUDA_CHECK(cudaMemcpyAsync(f->score_nll_h, f->score_nll, bytes, cudaMemcpyDeviceToHost, f->s_main));
    B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
    for (int i = 0; i < n_tokens; i++) if (targets[i] >= 0) nll[i] = f->score_nll_h[i];
    B200_CUDA_CHECK(cudaEventElapsedTime(&f->last_ms, f->e_t0, f->e_t1));
    return 0;
}

// falcon_perplexity's loop (falcon_perplexity.cpp:28-123) over b200_falcon_score's batches.  The token ids and the per-row targets
// (-1 outside the scored range) go H2D once; every batch copies its ids D2D into the eval's input; the terms stay on the device until
// the end, and the host sums them in double in the reference's order.
int b200_falcon_perplexity(b200_falcon * f, const int32_t * tokens, int n_tokens, int n_ctx, double * ppl, float * nll) {
    if (f->hp.world > 1 || n_ctx < 2 || n_ctx > f->hp.n_ctx || n_tokens < 0 || (n_tokens > 0 && !tokens)) return -1;
    for (int i = 0; i < n_tokens; i++) if (tokens[i] < 0 || tokens[i] >= f->V) return -1;
    const int n_chunk = n_tokens / n_ctx;
    if (n_chunk == 0) return 0;
    f->emb_valid = false;
    const int n_batch = f->hp.n_batch > 0 ? f->hp.n_batch : 1, first = std::min(512, n_ctx / 2);
    const size_t n_used = (size_t) n_chunk * n_ctx;
    std::vector<int32_t> tg(n_used, -1);
    for (size_t c = 0; c < (size_t) n_chunk; c++)
        for (int k = first; k < n_ctx - 1; k++) tg[c * n_ctx + k] = tokens[c * n_ctx + k + 1];
    int32_t * tok_d = nullptr, * tg_d = nullptr; float * terms_d = nullptr;
    B200_CUDA_CHECK(cudaMalloc(&tok_d, n_used * 4)); B200_CUDA_CHECK(cudaMalloc(&tg_d, n_used * 4)); B200_CUDA_CHECK(cudaMalloc(&terms_d, n_used * 4));
    B200_CUDA_CHECK(cudaMemcpyAsync(tok_d, tokens, n_used * 4, cudaMemcpyHostToDevice, f->s_main));
    B200_CUDA_CHECK(cudaMemcpyAsync(tg_d, tg.data(), n_used * 4, cudaMemcpyHostToDevice, f->s_main));
    const float theta = falcon_rope_theta_scale(f->D, n_ctx, f->hp.n_ctx);          // the reference's context is made with n_ctx
    int launches = 0;
    B200_CUDA_CHECK(cudaEventRecord(f->e_t0, f->s_main));
    for (size_t c = 0; c < (size_t) n_chunk; c++)
        for (int p0 = 0; p0 < n_ctx; p0 += n_batch) {
            const int N = std::min(n_ctx - p0, n_batch);
            const size_t off = c * n_ctx + p0;
            B200_CUDA_CHECK(cudaMemcpyAsync(f->tokens_dev, tok_d + off, (size_t) N * 4, cudaMemcpyDeviceToDevice, f->s_main));
            enqueue_score_batch(f, N, p0, theta, tg_d + off, terms_d + off, std::max(p0, first) < std::min(p0 + N, n_ctx - 1));
            launches += f->launches;
        }
    B200_CUDA_CHECK(cudaEventRecord(f->e_t1, f->s_main));
    std::vector<float> terms(n_used);
    B200_CUDA_CHECK(cudaMemcpyAsync(terms.data(), terms_d, n_used * 4, cudaMemcpyDeviceToHost, f->s_main));
    B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
    B200_CUDA_CHECK(cudaEventElapsedTime(&f->last_ms, f->e_t0, f->e_t1));
    f->launches = launches;
    cudaFree(tok_d); cudaFree(tg_d); cudaFree(terms_d);
    double sum = 0.0; size_t count = 0;
    for (size_t c = 0; c < (size_t) n_chunk; c++) {
        for (int k = first; k < n_ctx - 1; k++) {
            const float t = terms[c * n_ctx + k];
            sum += t;                                                       // nll += -std::log(prob)
            if (nll) nll[count] = t;
            count++;
        }
        if (ppl) ppl[c] = std::exp(sum / (double) count);
    }
    return n_chunk;
}

int b200_falcon_decode_dev(b200_falcon * f, const int32_t * token_dev, int n_past, int n_ctx_rope) {
    if (n_past < 0 || n_past >= f->hp.n_ctx) return 1;                       // the KV append would leave this layer's cache slice
    f->emb_valid = false;
    const float theta = falcon_rope_theta_scale(f->D, n_ctx_rope, f->hp.n_ctx);
    const int tier = tier_of(n_past);
    // position and token id are device scalars the graph (and a build's eager pass) reads; both are set stream-ordered (the position
    // travels as a kernel argument, so the host may run ahead by any number of steps)
    set_i32_kernel<<<1, 1, 0, f->s_main>>>(f->n_past_dev, n_past);
    if (f->first && token_dev) B200_CUDA_CHECK(cudaMemcpyAsync(f->tokens_dev, token_dev, 4, cudaMemcpyDeviceToDevice, f->s_main));
    const cudaGraphExec_t g = decode_graph(f, G_DEVICE, tier, theta);
    if (getenv("B200_NO_GRAPH")) { f->launches = 0; f->cur_tier = tier; enqueue_eval(f, 1, 0, theta, true, 0); f->cur_tier = 0; return 0; }   // the same step, launched eagerly
    B200_CUDA_CHECK(cudaGraphLaunch(g, f->s_main));
    f->launches = f->graph_launches;
    return 0;
}
const float * b200_falcon_logits_dev(const b200_falcon * f) { return f->logits; }

// Greedy generation without the host in the loop.  After every decode step the last rank takes the arg-max of its logits on
// the device (lowest index on ties, like a sequential scan) and hands the id to the embedding gather of the next step -- directly
// on one GPU, through one 4-byte ncclSend/ncclRecv (last rank -> rank 0) in a layer pipeline -- so no logits and no token id cross
// PCIe between steps: this is the strict autoregressive single-stream rate.  First slice of SURVEY 8f-2 (the reference samples on
// the host from a 260 KB logits row per token, falcon_main.cpp:897-980 with top_k = 1 / temp <= 0 -> llama_sample_token_greedy,
// libfalcon.cpp:3464-3473).  Every rank of a pipeline calls it with the same arguments; tokens_out is written on the last rank.
static int generate_impl(b200_falcon * f, int32_t first_token, int n_past, int n_steps, int n_ctx_rope, int32_t * tokens_out);
int b200_falcon_generate_greedy(b200_falcon * f, int32_t first_token, int n_past, int n_steps, int n_ctx_rope, int32_t * tokens_out) {
    if (f->use_sampler) { f->use_sampler = false; invalidate_graphs(f); }       // the generation-step graph bakes the sampler kernel in
    return generate_impl(f, first_token, n_past, n_steps, n_ctx_rope, tokens_out);
}
// Generation with falcon_main's sampling chain on the device (sampling.cu): logit bias, repetition / frequency / presence penalties
// over the last repeat_last_n ids (seeded with last_tokens[0..n_last), oldest first), then greedy, mirostat 1 / 2 or top-k ->
// tail-free -> typical -> top-p -> temperature and the MT19937-driven draw of llama_sample_token (falcon_main.cpp:896-987).
// The sampler state (window, MT19937, mirostat's mu = 2 * tau at the start of every call) is reset here and then lives on the device
// across the graph replays.  Returns 0 on success, 1 on a bad argument (see sampler_params_of, positions outside the context).
b200_sampling_chain sampler_chain_of(const b200_sampling_params & sp);                          // c_api.cu
bool sampler_params_of(const b200_sampling_chain * c, int n_vocab, SamplerParams * out);
int b200_falcon_generate_chain(b200_falcon * f, const b200_sampling_chain * c, const int32_t * last_tokens, int n_last,
                               int32_t first_token, int n_past, int n_steps, int n_ctx_rope, int32_t * tokens_out) {
    SamplerParams np;
    if (!sampler_params_of(c, f->V, &np) || n_last < 0 || (n_last > 0 && !last_tokens)) return 1;
    if (np.top_k > f->V) np.top_k = f->V;
    if (!f->use_sampler || memcmp(&np, &f->sampler_p, sizeof(np)) != 0) { invalidate_graphs(f); f->sampler_p = np; f->use_sampler = true; }
    if (f->last) {
        if (!f->sampler) { f->sampler = sampler_state_alloc(); B200_CUDA_CHECK(cudaMalloc(&f->sampler_work, sampler_work_floats(f->V) * 4)); }
        int32_t * w = nullptr;
        if (n_last > 0) { B200_CUDA_CHECK(cudaMalloc(&w, (size_t) n_last * 4)); B200_CUDA_CHECK(cudaMemcpyAsync(w, last_tokens, (size_t) n_last * 4, cudaMemcpyHostToDevice, f->s_main)); }
        launch_sampler_init(f->sampler, c->seed, w, n_last, c->repeat_last_n, 2.0f * c->mirostat_tau, f->s_main);
        B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
        if (w) B200_CUDA_CHECK(cudaFree(w));
    }
    return generate_impl(f, first_token, n_past, n_steps, n_ctx_rope, tokens_out);
}
// The default chain (b200_sampling_params: top_k 1..1024, no extras).
int b200_falcon_generate(b200_falcon * f, const b200_sampling_params * sp, const int32_t * last_tokens, int n_last,
                         int32_t first_token, int n_past, int n_steps, int n_ctx_rope, int32_t * tokens_out) {
    if (!sp || sp->top_k < 1 || sp->top_k > 1024 || sp->repeat_last_n < 0 || sp->repeat_last_n > B200_SAMPLER_MAX_WINDOW || n_last < 0) return 1;
    const b200_sampling_chain c = sampler_chain_of(*sp);
    return b200_falcon_generate_chain(f, &c, last_tokens, n_last, first_token, n_past, n_steps, n_ctx_rope, tokens_out);
}
static int generate_impl(b200_falcon * f, int32_t first_token, int n_past, int n_steps, int n_ctx_rope, int32_t * tokens_out) {
    if (n_steps <= 0 || n_past < 0 || n_past + n_steps > f->hp.n_ctx || first_token < 0 || first_token >= f->V) return 1;
    f->emb_valid = false;
    const float theta = falcon_rope_theta_scale(f->D, n_ctx_rope, f->hp.n_ctx);
    cudaStream_t st = f->s_main;
    set_i32_kernel<<<1, 1, 0, st>>>(f->n_past_dev, n_past);
    if (f->first) { set_i32_kernel<<<1, 1, 0, st>>>((int *) f->tokens_dev, first_token); }
    // both step graphs on every rank, built in the same order (each build runs one eager pass with the pipeline's send / recv pairs)
    // (a generation that crosses the long-context threshold needs both tiers)
    for (int tier = tier_of(n_past); tier <= tier_of(n_past + n_steps - 1); tier++)
        for (int which : { G_DEVICE, G_GEN }) decode_graph(f, which, tier, theta);
    set_i32_kernel<<<1, 1, 0, st>>>(f->n_past_dev, n_past);
    set_i32_kernel<<<1, 1, 0, st>>>(f->gen_step, 0);
    if (f->first) { set_i32_kernel<<<1, 1, 0, st>>>((int *) f->tokens_dev, first_token); }
    B200_CUDA_CHECK(cudaEventRecord(f->e_t0, st));
    for (int i = 0; i < n_steps; i++) {
        set_i32_kernel<<<1, 1, 0, st>>>(f->n_past_dev, n_past + i);
        // rank 0 of a pipeline takes its first id from the caller and every later one from the last rank
        const int which = (f->last || (f->first && i > 0)) ? G_GEN : G_DEVICE;
        B200_CUDA_CHECK(cudaGraphLaunch(f->graph[tier_of(n_past + i)][which].exec, st));
    }
    if (f->first && f->hp.world > 1) B200_NCCL_CHECK(nccl().Recv(f->tokens_dev, 1, ncclInt32, f->hp.world - 1, f->comm, st));   // the id sampled after the last step
    B200_CUDA_CHECK(cudaEventRecord(f->e_t1, st));
    if (f->last && tokens_out) B200_CUDA_CHECK(cudaMemcpyAsync(tokens_out, f->gen_hist, (size_t) n_steps * 4, cudaMemcpyDeviceToHost, st));
    B200_CUDA_CHECK(cudaStreamSynchronize(st));
    B200_CUDA_CHECK(cudaEventElapsedTime(&f->last_ms, f->e_t0, f->e_t1));
    f->launches = f->graph_launches;
    return 0;
}
// ---- KV cache access (session state, SURVEY 8f-4).  The reference serialises its KV cache with the context
// (falcon_copy_state_data / falcon_set_state_data, libfalcon.cpp:4313-4490: n_tokens x n_embd_kv floats per layer for K and V);
// here the cache is device-resident [layer][n_ctx][n_head_kv][head_dim] f32 or fp16 and rows are copied straight out of / into HBM.  The
// host rows are f32 for either engine: an fp16 cache's values are widened exactly on the way out and rounded (to nearest even) on the way in.
int b200_falcon_kv_read(b200_falcon * f, int layer, int pos, int n, float * k_out, float * v_out) {
    if (layer < f->hp.layer_first || layer >= f->hp.layer_last || pos < 0 || n < 0 || pos + n > f->hp.n_ctx) return 1;
    const KvCache c = kv_layer(f, layer - f->hp.layer_first);
    const size_t row = kv_row(f), o = (size_t) pos * row, cnt = (size_t) n * row;
    B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
    auto get = [&](float * dst, const auto * src) { if (dst) kv_d2h(dst, src + o, cnt); };
    if (kv_f16(c)) { get(k_out, c.k16); get(v_out, c.v16); } else { get(k_out, c.k); get(v_out, c.v); }
    return 0;
}
// the fp16 planes the prompt kernel reads (attention_ws.cu), positions [pos, pos + n) of `layer`: k16_out [n][n_head_kv][head_dim] (an fp16
// engine's K cache itself), vt16_out [n_head_kv][head_dim][n].  The range may reach attention_ctx_pad(n_ctx), so that the padding can be inspected.
int b200_falcon_kv_shadow_read(b200_falcon * f, int layer, int pos, int n, uint16_t * k16_out, uint16_t * vt16_out) {
    const int ctx_pad = f->kv.ctx_pad;
    if (!f->kv.k16 || (vt16_out && !f->kv.vt16) || layer < f->hp.layer_first || layer >= f->hp.layer_last || pos < 0 || n < 0 || pos + n > ctx_pad) return 1;
    const KvCache c = kv_layer(f, layer - f->hp.layer_first);
    const size_t row = kv_row(f);
    B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
    if (k16_out && n) B200_CUDA_CHECK(cudaMemcpy(k16_out, c.k16 + (size_t) pos * row, (size_t) n * row * 2, cudaMemcpyDeviceToHost));
    if (vt16_out && n) B200_CUDA_CHECK(cudaMemcpy2D(vt16_out, (size_t) n * 2, c.vt16 + pos, (size_t) ctx_pad * 2, (size_t) n * 2, row, cudaMemcpyDeviceToHost));
    return 0;
}
int b200_falcon_kv_write(b200_falcon * f, int layer, int pos, int n, const float * k_in, const float * v_in) {
    if (layer < f->hp.layer_first || layer >= f->hp.layer_last || pos < 0 || n < 0 || pos + n > f->hp.n_ctx) return 1;
    const KvCache c = kv_layer(f, layer - f->hp.layer_first);
    const size_t row = kv_row(f), o = (size_t) pos * row, cnt = (size_t) n * row;
    B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
    auto put = [&](auto * dst, const float * src) { if (src) kv_h2d(dst + o, src, cnt); };
    if (kv_f16(c)) { put(c.k16, k_in); put(c.v16, v_in); } else { put(c.k, k_in); put(c.v, v_in); }
    launch_kv_shadow_refresh(c, f->HKV, pos, n, f->s_main);
    B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
    return 0;
}
// the reference's session-state layout (kernels.h).  The cache rows of a layer are [n_ctx][E]: K rows copy straight across, V rows
// are [position][E] and the state's V is [E][position]
static bool ref_kv_args(const b200_falcon * f, int n, const void * v, const RefKvLayout & L) {
    return !kv_f16(f->kv) && n >= 0 && n <= f->hp.n_ctx && (!v || L.v_ld >= (size_t) n);
}
extern "C++" int falcon_ref_kv_export(b200_falcon * f, int n, float * k, float * v, const RefKvLayout & L) {
    if (!ref_kv_args(f, n, v, L)) return 1;
    const size_t E = kv_row(f), lay = (size_t) f->hp.n_ctx * E;
    if (n > 0 && k) B200_CUDA_CHECK(cudaMemcpy2DAsync(k, L.k_layer * 4, f->kv.k, lay * 4, (size_t) n * E * 4, f->NL, cudaMemcpyDeviceToHost, f->s_main));
    float * stage = nullptr;
    if (n > 0 && v) B200_CUDA_CHECK(cudaMalloc(&stage, (size_t) n * E * 4));
    for (int l = 0; stage && l < f->NL; l++) {
        launch_transpose_f32(kv_layer(f, l).v, (int64_t) E, n, (int) E, stage, n, f->s_main);
        B200_CUDA_CHECK(cudaMemcpy2DAsync(v + l * L.v_layer, L.v_ld * 4, stage, (size_t) n * 4, (size_t) n * 4, E, cudaMemcpyDeviceToHost, f->s_main));
    }
    B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
    if (stage) B200_CUDA_CHECK(cudaFree(stage));
    return 0;
}
extern "C++" int falcon_ref_kv_import(b200_falcon * f, int n, const float * k, const float * v, const RefKvLayout & L) {
    if (!ref_kv_args(f, n, v, L)) return 1;
    const size_t E = kv_row(f), lay = (size_t) f->hp.n_ctx * E;
    if (n > 0 && k) B200_CUDA_CHECK(cudaMemcpy2DAsync(f->kv.k, lay * 4, k, L.k_layer * 4, (size_t) n * E * 4, f->NL, cudaMemcpyHostToDevice, f->s_main));
    float * stage = nullptr;
    if (n > 0 && v) B200_CUDA_CHECK(cudaMalloc(&stage, (size_t) n * E * 4));
    for (int l = 0; l < f->NL && n > 0; l++) {
        const KvCache c = kv_layer(f, l);
        if (v) {
            B200_CUDA_CHECK(cudaMemcpy2DAsync(stage, (size_t) n * 4, v + l * L.v_layer, L.v_ld * 4, (size_t) n * 4, E, cudaMemcpyHostToDevice, f->s_main));
            launch_transpose_f32(stage, n, (int) E, n, c.v, (int64_t) E, f->s_main);
        }
        launch_kv_shadow_refresh(c, f->HKV, 0, n, f->s_main);
    }
    B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
    if (stage) B200_CUDA_CHECK(cudaFree(stage));
    return 0;
}
// random K / V rows generated on the device for positions [pos, pos + n) of every local layer: pre-fills a long context
// for throughput runs (BASELINE config 5: decode at 8k context) without evaluating 8k tokens first
int b200_falcon_kv_fill_random(b200_falcon * f, int pos, int n, uint64_t seed) {
    if (pos < 0 || n < 0 || pos + n > f->hp.n_ctx) return 1;
    const size_t row = kv_row(f);
    for (int l = 0; l < f->NL; l++) {
        const KvCache c = kv_layer(f, l);
        const int64_t cnt = (int64_t) ((size_t) n * row);
        auto fill = [&](auto * dst, uint64_t s) { fill_kernel<<<296, 256, 0, f->s_main>>>(dst + (size_t) pos * row, cnt, 0.f, 1.f, s); };
        if (kv_f16(c)) { fill(c.k16, seed + 2 * l); fill(c.v16, seed + 2 * l + 1); }      // the same values, rounded to the cache's fp16
        else { fill(c.k, seed + 2 * l); fill(c.v, seed + 2 * l + 1); }
        launch_kv_shadow_refresh(c, f->HKV, pos, n, f->s_main);
    }
    B200_CUDA_CHECK(cudaGetLastError());
    B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
    return 0;
}
// Session file over the device KV cache: what falcon_save_session_file / falcon_load_session_file (libfalcon.cpp:4490-4563) keep of
// the KV state, written straight from / read straight into HBM through a bounded pinned buffer.  Own container (the reference's
// serialises its transposed, ping-ponged host V buffers, which do not exist here):
//   u32 magic 'b2kv', u32 version 1, i32 layer_first, layer_last, n_head_kv, head_dim, n_tokens; then per local layer: K rows, V rows (f32)
// for either cache type (kv_read / kv_write: an fp16 engine's file round-trips bit for bit, an f32 file loaded into it is rounded)
// save: returns 0 / -1.  load: returns the number of positions restored (the caller continues at that n_past), -1 on any mismatch.
int b200_falcon_save_kv(b200_falcon * f, const char * path, int n_tokens) {
    if (n_tokens < 0 || n_tokens > f->hp.n_ctx) return -1;
    FILE * fp = fopen(path, "wb");
    if (!fp) return -1;
    const int32_t hdr[7] = { 0x766b3262, 1, f->hp.layer_first, f->hp.layer_last, f->HKV, f->D, n_tokens };
    bool ok = fwrite(hdr, sizeof(hdr), 1, fp) == 1;
    const size_t bytes = (size_t) n_tokens * kv_row(f) * 4;
    std::vector<float> k(bytes / 4 + 1), v(bytes / 4 + 1);
    for (int l = 0; l < f->NL && ok; l++) {
        b200_falcon_kv_read(f, f->hp.layer_first + l, 0, n_tokens, k.data(), v.data());
        ok = bytes == 0 || (fwrite(k.data(), bytes, 1, fp) == 1 && fwrite(v.data(), bytes, 1, fp) == 1);
    }
    ok = (fclose(fp) == 0) && ok;
    return ok ? 0 : -1;
}
int b200_falcon_load_kv(b200_falcon * f, const char * path) {
    FILE * fp = fopen(path, "rb");
    if (!fp) return -1;
    int32_t hdr[7];
    if (fread(hdr, sizeof(hdr), 1, fp) != 1 || hdr[0] != 0x766b3262 || hdr[1] != 1 || hdr[2] != f->hp.layer_first || hdr[3] != f->hp.layer_last ||
        hdr[4] != f->HKV || hdr[5] != f->D || hdr[6] < 0 || hdr[6] > f->hp.n_ctx) { fclose(fp); return -1; }
    const int n = hdr[6];
    const size_t bytes = (size_t) n * kv_row(f) * 4;
    std::vector<float> k(bytes / 4 + 1), v(bytes / 4 + 1);
    for (int l = 0; l < f->NL; l++) {
        if (bytes && (fread(k.data(), bytes, 1, fp) != 1 || fread(v.data(), bytes, 1, fp) != 1)) { fclose(fp); return -1; }
        if (b200_falcon_kv_write(f, f->hp.layer_first + l, 0, n, k.data(), v.data()) != 0) { fclose(fp); return -1; }     // also refreshes the fp16 planes
    }
    fclose(fp);
    return n;
}
// Test tap: see include/ggml_b200.h.  The node list follows what ensure_actq allocated for this model (tensors must be set first).
static void tap_add(std::vector<b200_falcon::TapNode> & v, size_t & total, const std::string & name, const void * src, size_t row_bytes,
                    int NB, bool all_rows = true) {
    if (!src) return;
    v.push_back({ name, src, row_bytes, total, all_rows });
    total += ((size_t) NB * row_bytes + 255) & ~(size_t) 255;
}
static void tap_add_actq(std::vector<b200_falcon::TapNode> & v, size_t & total, const std::string & name, const ActQ & A, int NB, bool all_rows = true) {
    if (!A.q) return;
    tap_add(v, total, name + ".q", A.q, (size_t) A.K, NB, all_rows);
    tap_add(v, total, name + ".d", A.d, (size_t) (A.K / act_block(A.type)) * 4, NB, all_rows);
    tap_add(v, total, name + ".s", A.s, (size_t) (A.K / 32) * 4, NB, all_rows);
    tap_add(v, total, name + ".bs", A.bs, (size_t) (A.K / (A.type == T_Q8_K ? 16 : 32)) * 2, NB, all_rows);
}
// slice[l] >= 0 for the local layers that get a slice (tap on), or slice empty (tap off)
static void tap_setup(b200_falcon * f, const std::vector<int> & slice) {
    invalidate_graphs(f);                                 // the captured decode graphs hold the copies (or their absence)
    B200_CUDA_CHECK(cudaDeviceSynchronize());
    B200_CUDA_CHECK(cudaFree(f->tap.mem));
    f->tap = b200_falcon::Tap{};
    if (slice.empty()) return;
    ensure_actq(f);
    const int NB = f->hp.n_batch > 0 ? f->hp.n_batch : 1;
    const size_t E4 = (size_t) f->E * 4;
    auto & T = f->tap;
    size_t lb = 0, hb = 0;
    tap_add(T.layer, lb, "inp", f->inp, E4, NB); tap_add(T.layer, lb, "qkv", f->qkv, (size_t) f->QKV * 4, NB);
    tap_add(T.layer, lb, "att", f->att, E4, NB); tap_add(T.layer, lb, "up", f->up, (size_t) f->FF * 4, NB);
    tap_add(T.layer, lb, "dn", f->dn, E4, NB);   tap_add(T.layer, lb, "ao", f->ao, E4, NB);
    if (f->act_type >= 0) {
        tap_add_actq(T.layer, lb, "xa", f->xa, NB); tap_add_actq(T.layer, lb, "xm", f->xm, NB);
        tap_add_actq(T.layer, lb, "xatt", f->xatt, NB); tap_add_actq(T.layer, lb, "xup", f->xup, NB);
        tap_add(T.layer, lb, "xh_a", f->xh_a, (size_t) f->E * 2, NB); tap_add(T.layer, lb, "xh_b", f->xh_b, (size_t) f->FF * 2, NB);
        tap_add(T.layer, lb, "xh_m", f->xh_m, (size_t) f->E * 2, NB);
    }
    if (f->generic_layers) { tap_add(T.layer, lb, "gen_na", f->gen_na, E4, NB); tap_add(T.layer, lb, "gen_nm", f->gen_nm, E4, NB); }
    if (f->last) {
        tap_add(T.head, hb, "inp", f->inp, E4, NB);
        if (f->generic_head) tap_add(T.head, hb, "gen_na", f->gen_na, E4, NB, false);
        else tap_add_actq(T.head, hb, "xf", f->xf, NB, false);
        tap_add(T.head, hb, "logits", f->logits, (size_t) f->V * 4, NB, false);
    }
    T.layer_bytes = lb;
    T.slice = slice;
    for (int s : slice) T.n_slices += s >= 0;
    B200_CUDA_CHECK(cudaMalloc(&T.mem, lb * T.n_slices + hb + 256));
    T.rotated.assign(f->NL, 0);
}
int b200_falcon_tap(b200_falcon * f, int on) {
    std::vector<int> slice;
    for (int l = 0; on && l < f->NL; l++) slice.push_back(l);
    tap_setup(f, slice);
    return 0;
}
int b200_falcon_tap_layers(b200_falcon * f, const int * layers, int n) {
    std::vector<int> slice(f->NL, -1);
    bool ok = n > 0 && layers;
    for (int i = 0; ok && i < n; i++) {
        const int l = layers[i] - f->hp.layer_first;
        ok = l >= 0 && l < f->NL && slice[l] < 0;
        if (ok) slice[l] = i;
    }
    tap_setup(f, ok ? slice : std::vector<int>());
    return ok ? 0 : 1;
}
int b200_falcon_tap_read(const b200_falcon * f, int layer, const char * node, void * host, size_t bytes) {
    const auto & T = f->tap;
    if (!T.mem || !node || !host) return 1;
    const bool head = layer == -1;
    const int l = layer - f->hp.layer_first;
    if (head ? !f->last : (l < 0 || l >= f->NL || T.slice[l] < 0)) return 1;
    if (!head && !strcmp(node, "qkv_rotated")) {
        if (bytes != sizeof(int)) return 1;
        memcpy(host, &T.rotated[l], sizeof(int));
        return 0;
    }
    for (const auto & n : head ? T.head : T.layer) {
        if (n.name != node) continue;
        if (bytes != n.row_bytes * (n.all_rows ? T.rows : T.head_rows)) return 1;
        B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
        B200_CUDA_CHECK(cudaMemcpy(host, T.mem + (size_t) (head ? T.n_slices : T.slice[l]) * T.layer_bytes + n.off, bytes, cudaMemcpyDeviceToHost));
        return 0;
    }
    return 1;
}

int b200_falcon_kv_type(const b200_falcon * f) { return kv_f16(f->kv) ? T_F16 : T_F32; }
size_t b200_falcon_kv_device_bytes(const b200_falcon * f) {
    const size_t planes16 = (f->kv.k16 ? 1 : 0) + (f->kv.v16 ? 1 : 0) + (f->kv.vt16 ? 1 : 0);
    return (f->kv.k ? 2 * (size_t) f->NL * f->hp.n_ctx * kv_row(f) * sizeof(float) : 0) + planes16 * f->NL * f->shadow_layer * sizeof(__half);
}
int b200_falcon_last_launches(const b200_falcon * f) { return f->launches; }
float b200_falcon_last_ms(const b200_falcon * f) { return f->last_ms; }
void * b200_falcon_stream(b200_falcon * f) { return (void *) f->s_main; }

// Times the dominant kernel in isolation on the model's own matrices: every local quantised mat-vec of the resident layers (4 per
// layer; a streamed layer's matrices are in HBM only while an eval runs it) + lm_head launched back to back on the eval stream, `reps` passes, CUDA events around the whole region.  Each
// launch reads a different matrix and one pass touches weight_bytes >> L2, so every launch streams cold HBM.
// Returns the total milliseconds; *n_launches and *bytes describe the region (bytes = algorithmic weight bytes).
float b200_falcon_profile_matvec(b200_falcon * f, int reps, int * n_launches, size_t * bytes) {
    B200_ASSERT(f->act_type >= 0);
    ensure_actq(f);
    cudaStream_t st = f->s_main;
    ActQ xe = f->xm, xff = f->xup; xe.N = 1; xff.N = 1;
    B200_CUDA_CHECK(cudaMemsetAsync(f->inp, 0, (size_t) f->E * 4, st));
    launch_quantize_act(f->inp, f->E, xe, st);
    B200_CUDA_CHECK(cudaMemsetAsync(f->up, 0, (size_t) f->FF * 4, st));
    launch_quantize_act(f->up, f->FF, xff, st);
    MmvEpilogue e = { EPI_NONE, nullptr, nullptr };
    int n = 0; size_t b = 0;
    auto pass = [&](bool count) {
        for (int l = 0; l < f->NL; l++) {
            if (stream_rank(f, l) >= 0) continue;
            const Layer & L = f->layers[l];
            launch_mmv(L.wqkv, xe, f->qkv, f->QKV, e, st); launch_mmv(L.wo, xe, f->ao, f->E, e, st);
            launch_mmv(L.up, xe, f->up, f->FF, e, st); launch_mmv(L.down, xff, f->dn, f->E, e, st);
            if (count) { n += 4; b += algorithmic_bytes(L.wqkv.type, L.wqkv.K, L.wqkv.M) + algorithmic_bytes(L.wo.type, L.wo.K, L.wo.M)
                                    + algorithmic_bytes(L.up.type, L.up.K, L.up.M) + algorithmic_bytes(L.down.type, L.down.K, L.down.M); }
        }
        if (f->last && f->lm_head.p[0]) { launch_mmv(f->lm_head, xe, f->logits, f->V, e, st);
            if (count) { n += 1; b += algorithmic_bytes(f->lm_head.type, f->lm_head.K, f->lm_head.M); } }
    };
    pass(false);                                                       // warm-up
    B200_CUDA_CHECK(cudaEventRecord(f->e_t0, st));
    for (int r = 0; r < reps; r++) pass(r == 0);
    B200_CUDA_CHECK(cudaEventRecord(f->e_t1, st));
    B200_CUDA_CHECK(cudaStreamSynchronize(st));
    float ms = 0.f; B200_CUDA_CHECK(cudaEventElapsedTime(&ms, f->e_t0, f->e_t1));
    if (n_launches) *n_launches = n * reps;
    if (bytes) *bytes = b * (size_t) reps;
    return ms;
}

} // extern "C"
