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
#include "../../include/ggml_b200.h"
#include <nccl.h>
#include <dlfcn.h>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#include <atomic>
#include <chrono>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

cudaStream_t b200_current_stream();

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
    float * k_cache = nullptr, * v_cache = nullptr;
    __half * k16 = nullptr, * vt16 = nullptr; size_t shadow_layer = 0;      // fp16 shadow of the cache for the prompt kernel (attention_ws.cu); only when n_batch > 8
    // activation arena
    float * inp = nullptr, * qkv = nullptr, * att = nullptr, * ao = nullptr, * up = nullptr, * dn = nullptr, * logits = nullptr;
    void * actq_mem = nullptr; ActQ xa{}, xm{}, xatt{}, xup{}, xf{};
    __half * xh_a = nullptr, * xh_b = nullptr, * xh_m = nullptr;      // fp16 GEMM operands (d * q), written by the kernels that quantise: attention branch, MLP branch, MLP input
    float * attn_scratch = nullptr; size_t attn_scratch_bytes = 0;     // prompt attention (grown on demand)
    float * attn_dec_scratch = nullptr;            // decode attention: zeroed before the decode graphs are captured
    int32_t * tokens_dev = nullptr; int * n_past_dev = nullptr;
    int32_t * tokens_h = nullptr; int * n_past_h = nullptr; float * logits_h = nullptr; size_t logits_h_floats = 0;
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
    float * gen_na = nullptr, * gen_nm = nullptr; void * gen_actq = nullptr; __half * gen_xh = nullptr;
    unsigned * q_ctr = nullptr;                 // chunk counters of the quantise-on-completion epilogue (ffn_up -> ffn_down)
    ncclComm_t comm = nullptr;
    int launches = 0; float last_ms = 0.f;
    size_t weight_bytes = 0;
    double load_seconds = 0.0; size_t load_bytes = 0;   // b200_falcon_load_ggcc
    size_t pending_floats = 0;                  // logits of the eval in flight (falcon_eval_begin / finish)
    std::vector<const void *> borrowed;         // device planes adopted from another owner (ggml_cuda_transform_tensor): never freed here
    // test tap (b200_falcon_tap): while mem is set, every eval copies its intermediates into mem -- one slice of layer_bytes per local
    // layer at the end of that layer, then one slice after the head.  Node offsets are the same in every layer slice.
    struct TapNode { std::string name; const void * src; size_t row_bytes, off; bool all_rows; };    // all_rows: N rows, else the head's rows
    struct Tap { uint8_t * mem = nullptr; std::vector<TapNode> layer, head; size_t layer_bytes = 0; int rows = 0, head_rows = 0;
                 std::vector<int> rotated; } tap;                // rotated[l]: RoPE ran in place on qkv (not inside the attention kernels)
};

// Local layer l's slice of the KV cache.  k / v: [n_ctx][n_head_kv][head_dim] f32, rows of kv_row() floats.  k16 / vt16: its fp16
// shadow in the layout of AttnParams::k16 / vt16, null when the engine keeps none.
struct KvLayer { float * k, * v; __half * k16, * vt16; };
static size_t kv_row(const b200_falcon * f) { return (size_t) f->HKV * f->D; }
static KvLayer kv_layer(const b200_falcon * f, int l) {
    const size_t off = (size_t) l * f->hp.n_ctx * kv_row(f);
    KvLayer c = { f->k_cache + off, f->v_cache + off, nullptr, nullptr };
    if (f->k16) { c.k16 = f->k16 + (size_t) l * f->shadow_layer; c.vt16 = f->vt16 + (size_t) l * f->shadow_layer; }
    return c;
}

__global__ void fill_f32_kernel(float * p, int64_t n, float base, float amp, uint64_t seed) {
    for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) {
        uint64_t x = seed + (uint64_t) i * 0x9E3779B97F4A7C15ULL; x ^= x >> 31; x *= 0xBF58476D1CE4E5B9ULL; x ^= x >> 29;
        p[i] = base + amp * ((float) (x & 0xffffff) / 8388608.f - 1.f);
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

extern "C" {

b200_falcon * b200_falcon_create(const b200_falcon_params * p) {
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
    const size_t kv = (size_t) f->NL * p->n_ctx * kv_row(f) * sizeof(float);
    B200_CUDA_CHECK(cudaMalloc(&f->k_cache, kv ? kv : 4)); B200_CUDA_CHECK(cudaMalloc(&f->v_cache, kv ? kv : 4));
    B200_CUDA_CHECK(cudaMemset(f->k_cache, 0, kv)); B200_CUDA_CHECK(cudaMemset(f->v_cache, 0, kv));
    if (p->n_batch > b200_mmv_max_n() && f->D == 64 && f->NL > 0) {
        f->shadow_layer = attention_shadow_halves(f->HKV, p->n_ctx);
        const size_t sb = (size_t) f->NL * f->shadow_layer * sizeof(__half);
        B200_CUDA_CHECK(cudaMalloc(&f->k16, sb)); B200_CUDA_CHECK(cudaMalloc(&f->vt16, sb));
        B200_CUDA_CHECK(cudaMemset(f->k16, 0, sb)); B200_CUDA_CHECK(cudaMemset(f->vt16, 0, sb));
    }
    B200_CUDA_CHECK(cudaMalloc(&f->inp, NB * f->E * 4)); B200_CUDA_CHECK(cudaMalloc(&f->qkv, NB * f->QKV * 4));
    B200_CUDA_CHECK(cudaMalloc(&f->att, NB * f->E * 4)); B200_CUDA_CHECK(cudaMalloc(&f->ao, NB * f->E * 4));
    B200_CUDA_CHECK(cudaMalloc(&f->up, NB * f->FF * 4)); B200_CUDA_CHECK(cudaMalloc(&f->dn, NB * f->E * 4));
    B200_CUDA_CHECK(cudaMalloc(&f->logits, NB * f->V * 4));
    B200_CUDA_CHECK(cudaMalloc(&f->tokens_dev, NB * 4)); B200_CUDA_CHECK(cudaMalloc(&f->n_past_dev, 4));
    B200_CUDA_CHECK(cudaMalloc(&f->tok_next, 4)); B200_CUDA_CHECK(cudaMalloc(&f->gen_step, 4));
    B200_CUDA_CHECK(cudaMalloc(&f->gen_hist, (size_t) (p->n_ctx > 0 ? p->n_ctx : 1) * 4));
    B200_CUDA_CHECK(cudaMallocHost(&f->tokens_h, NB * 4)); B200_CUDA_CHECK(cudaMallocHost(&f->n_past_h, 4));
    f->logits_h_floats = (size_t) f->V; B200_CUDA_CHECK(cudaMallocHost(&f->logits_h, f->logits_h_floats * 4));
    return f;
}

static void ensure_actq(b200_falcon * f) {
    if (!f->attn_dec_scratch) {
        AttnParams ap = { f->H, f->HKV, f->D, 1, 0, nullptr, f->hp.n_ctx, (int64_t) f->QKV, nullptr };
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
        B200_CUDA_CHECK(cudaMalloc(&f->gen_actq, ab));
        B200_CUDA_CHECK(cudaMalloc(&f->gen_xh, (size_t) NB * f->FF * 2));
    }
    if (f->actq_mem || f->act_type < 0) return;
    const int at = f->act_type;
    const size_t bE = actq_bytes(at, f->E, NB), bF = actq_bytes(at, f->FF, NB);
    B200_CUDA_CHECK(cudaMalloc(&f->actq_mem, 4 * bE + bF));
    uint8_t * p = (uint8_t *) f->actq_mem;
    actq_bind(f->xa, at, f->E, NB, p); p += bE; actq_bind(f->xm, at, f->E, NB, p); p += bE;
    actq_bind(f->xatt, at, f->E, NB, p); p += bE; actq_bind(f->xf, at, f->E, NB, p); p += bE;
    actq_bind(f->xup, at, f->FF, NB, p);
    if (NB > b200_mmv_max_n() && !f->xh_a) {
        B200_CUDA_CHECK(cudaMalloc(&f->xh_a, (size_t) NB * f->E * 2)); B200_CUDA_CHECK(cudaMalloc(&f->xh_b, (size_t) NB * f->FF * 2));
        B200_CUDA_CHECK(cudaMalloc(&f->xh_m, (size_t) NB * f->E * 2));
    }
}

static void free_matrix(b200_falcon * f, WPlanes & W) {
    for (const void * b : f->borrowed) if (b == (const void *) W.p[0]) { W = WPlanes{}; return; }      // adopted: its owner frees it
    wplanes_free(W);
}

// Empties matrix slot `s` for a new matrix of `type`, which the caller puts there: frees the old one, keeps weight_bytes (every
// matrix but the embedding table, which is gathered from, not streamed) in step and has the model's path re-derived.
static WPlanes & replace_matrix(b200_falcon * f, const Slot & s, int type) {
    invalidate_graphs(f);
    WPlanes & W = *slot_dest(f, s).W;
    const bool counted = s.d->kind != S_EMB;
    if (W.p[0]) { if (counted) f->weight_bytes -= algorithmic_bytes(W.type, W.K, W.M); free_matrix(f, W); }
    if (counted) f->weight_bytes += algorithmic_bytes(type, slot_K(f, s), slot_M(f, s));
    f->classified = false;
    return W;
}

// A weight matrix that is already resident in this library's planar layout (uploaded by ggml_cuda_transform_tensor for the reference's
// loader, ggml_surface.cu) becomes the engine's matrix `name` without another copy.  Returns false for an unknown name / wrong shape /
// a matrix of another rank.
extern "C++" bool falcon_adopt_matrix(b200_falcon * f, const char * name, const WPlanes & W) {
    Slot s;
    if (!find_slot(name, s) || !is_matrix(s) || !owns(f, s)) return false;
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
        if (random) wplanes_alloc_random(W, type, (int) K, (int) M, seed, st);
        else wplanes_upload(W, type, (int) K, (int) M, host_data, st);
    } else {
        invalidate_graphs(f);
        float *& v = *slot_dest(f, s).v;
        if (v) B200_CUDA_CHECK(cudaFree(v));
        B200_CUDA_CHECK(cudaMalloc(&v, (size_t) K * 4));
        if (random) {                               // LayerNorm gamma around 1, beta around 0
            const bool gamma = s.d->kind == S_LNF_G || s.d->kind == S_LN_ATTN_G || s.d->kind == S_LN_MLP_G;
            fill_f32_kernel<<<32, 256, 0, st>>>(v, K, gamma ? 1.f : 0.f, gamma ? 0.1f : 0.01f, seed); B200_CUDA_CHECK(cudaGetLastError());
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

// ---- GGCC v10 reader (libfalcon.cpp:770-973): header, vocab, merges, then {n_dims, name_len, type, ne[], name, pad32, data}.
// The file is untrusted input: every read is bounds-checked and a malformed file makes the loaders return -1 (no assert, no leak).
struct Cursor { const uint8_t * p; size_t off, size; bool bad;
    uint32_t u32() { if (off + 4 > size) { bad = true; return 0; } uint32_t v; memcpy(&v, p + off, 4); off += 4; return v; }
    void skip(size_t n) { if (n > size - off) bad = true; else off += n; } };
static int ggcc_header(Cursor & c, b200_falcon_params * out) {
    if (c.u32() != 0x67676363u || c.u32() != 10u || c.bad) return -1;
    out->n_vocab = (int32_t) c.u32(); out->n_embd = (int32_t) c.u32(); out->n_head = (int32_t) c.u32(); out->n_head_kv = (int32_t) c.u32();
    out->n_layer = (int32_t) c.u32(); out->falcon_type = (int32_t) c.u32();
    c.u32(); /* ftype */ c.u32(); /* n_bpe_merges */
    return c.bad ? -1 : 0;
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
    for (int i = 0; i < hp.n_vocab && !c.bad; i++) { const uint32_t len = c.u32(); c.skip((size_t) len + 4); }
    const uint32_t n_merges = c.u32();
    for (uint32_t i = 0; i < 2 * n_merges && !c.bad; i++) { const uint32_t len = c.u32(); c.skip(len); }
    if (c.bad) return fail("truncated vocabulary");
    const double t0 = wall_seconds();
    std::vector<LoadItem> items;
    size_t total = 0;
    while (c.off < c.size) {
        const uint32_t n_dims = c.u32(), name_len = c.u32(), type = c.u32();
        if (c.bad || n_dims < 1 || n_dims > 2 || name_len > 256) return fail("malformed tensor header");
        int64_t ne[2] = { 1, 1 };
        for (uint32_t d = 0; d < n_dims; d++) ne[d] = c.u32();
        if (c.bad || name_len > c.size - c.off) return fail("truncated tensor header");
        const std::string name((const char *) c.p + c.off, name_len); c.off += name_len;
        c.skip((size_t) (-(int64_t) c.off & 31));
        const TypeSpec ts = type_spec((int) type);
        if (c.bad || ts.blk_elems <= 0 || ne[0] <= 0 || ne[1] <= 0 || ne[0] % ts.blk_elems != 0) return fail("bad tensor type / shape");
        const size_t row_bytes = (size_t) (ne[0] / ts.blk_elems) * ts.blk_bytes, nbytes = row_bytes * (size_t) ne[1];
        if (nbytes > c.size - c.off) return fail("tensor data runs past the end of the file");
        Slot s;
        if (!find_slot(name, s)) return fail("unknown tensor name");
        const int64_t M = slot_M(f, s);
        if (ne[0] != slot_K(f, s) || (n_dims == 1 ? M != 1 : ne[1] != M)) return fail("tensor shape does not match the hyper-parameters");
        const uint8_t * data = c.p + c.off;
        c.off += nbytes;
        if (!is_matrix(s) || ts.n_planes == 1) {                                // LayerNorm vectors, f16 / f32 matrices: the plain path
            if (!is_matrix(s) && type != T_F32) return fail("1-D tensors must be f32");
            place_tensor(f, s, (int) type, data, false, 0);
            continue;
        }
        if (!owns(f, s)) continue;
        WPlanes * W = &replace_matrix(f, s, (int) type);
        wplanes_upload(*W, (int) type, (int) ne[0], (int) M, nullptr, f->s_main);  // planes allocated and laid out, filled below
        const int64_t chunk = (int64_t) (LOAD_BUF / row_bytes);
        if (chunk < 1) return fail("a row does not fit the staging buffer");
        for (int64_t r0 = 0; r0 < M; r0 += chunk) {
            const int64_t nr = r0 + chunk <= M ? chunk : M - r0;
            items.push_back({ W, data + (size_t) r0 * row_bytes, r0, nr, (size_t) nr * row_bytes });
        }
        total += nbytes;
    }
    int dev; B200_CUDA_CHECK(cudaGetDevice(&dev));
    std::atomic<size_t> next(0);
    std::vector<std::thread> th;
    for (int t = 0; t < LOAD_THREADS; t++) th.emplace_back(load_worker, dev, &items, &next);
    for (auto & t : th) t.join();
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
    cudaFree(f->lnf_g); cudaFree(f->lnf_b); cudaFree(f->k_cache); cudaFree(f->v_cache); cudaFree(f->k16); cudaFree(f->vt16);
    cudaFree(f->inp); cudaFree(f->qkv); cudaFree(f->att); cudaFree(f->ao); cudaFree(f->up); cudaFree(f->dn); cudaFree(f->logits);
    cudaFree(f->attn_scratch); cudaFree(f->actq_mem); cudaFree(f->gen_na); cudaFree(f->gen_nm); cudaFree(f->gen_actq); cudaFree(f->gen_xh); cudaFree(f->xh_a); cudaFree(f->xh_b); cudaFree(f->xh_m);
    cudaFree(f->tokens_dev); cudaFree(f->n_past_dev); cudaFree(f->q_ctr); cudaFree(f->attn_dec_scratch); cudaFree(f->tap.mem);
    cudaFreeHost(f->tokens_h); cudaFreeHost(f->n_past_h); cudaFreeHost(f->logits_h);
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

// Y = W x: quantised activations already in A.  mat-vec for small N, tensor-core GEMM otherwise.
static void mm(b200_falcon * f, const WPlanes & W, const ActQ & A, int N, float * y, int64_t y_stride, int epi, __half * xh, cudaStream_t st) {
    ActQ a = A; a.N = N;
    if (N <= b200_mmv_max_n()) mmv(f, W, a, y, y_stride, { epi, nullptr, nullptr }, st);
    else {
        B200_ASSERT(epi != EPI_ADD2);
        if (a.h) xh = a.h;                                     // the producer of the codes already wrote the fp16 operand
        else { launch_actq_to_f16(a, xh, W.K, st); f->launches++; }
        launch_mmq_gemm(W, xh, W.K, N, y, y_stride, epi == EPI_GELU, st); f->launches++;
    }
}

// Y = W x for ANY weight type, from fp32 activation rows (stride K): the activation format is made on the spot for this matrix --
// Q8_0 / Q8_1 / Q8_K codes for a quantised one (the INIT pass of ggml's MUL_MAT, ggml.c:11462-11476), fp16-rounded rows for F16
// weights (ggml_compute_forward_mul_mat_f16_f32, ggml.c:11232-11251), the rows themselves for F32.  Slow path: see b200_falcon::generic_layers.
static void mm_any(b200_falcon * f, const WPlanes & W, const float * x, int N, float * y, int64_t y_stride, bool gelu, cudaStream_t st) {
    const int at = act_type_for(W.type);
    if (at >= 0) {
        ActQ a; actq_bind(a, at, W.K, N, f->gen_actq);
        if (N > b200_mmv_max_n()) a.h = f->gen_xh;
        launch_quantize_act(x, W.K, a, st); f->launches++;
        mm(f, W, a, N, y, y_stride, gelu ? EPI_GELU : EPI_NONE, f->gen_xh, st);
        return;
    }
    if (W.type == T_F16 && N > b200_mmv_max_n()) {
        launch_f32_to_f16(x, f->gen_xh, (int64_t) N * W.K, st);
        launch_mmq_gemm(W, f->gen_xh, W.K, N, y, y_stride, 0, st); f->launches += 2;
    } else { launch_mmv_f(W, x, W.K, N, y, y_stride, st); f->launches++; }
    if (gelu) { B200_ASSERT(y_stride == W.M); launch_gelu(y, y, (int64_t) N * W.M, st); f->launches++; }                // ggml.c:10298-10337
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
    tap_copy(f, f->tap.layer, f->tap.mem + (size_t) l * f->tap.layer_bytes);
}
static void tap_head(b200_falcon * f, int N, int nr) {
    if (!f->tap.mem) return;
    f->tap.rows = N; f->tap.head_rows = nr;
    tap_copy(f, f->tap.head, f->tap.mem + (size_t) f->NL * f->tap.layer_bytes);
}

// final LayerNorm + lm_head over rows x[0 .. nr) of the residual stream: libfalcon.cpp:2422-2440.  ra / rb (optional, quantised head
// only): the last layer's branch outputs, which the LayerNorm kernel adds to x first (x = (ra + rb) + x, written back)
static void enqueue_head(b200_falcon * f, float * x, int nr, const float * ra, const float * rb, cudaStream_t sa) {
    const int E = f->E;
    if (f->generic_head) {
        launch_layernorm(x, E, f->lnf_g, f->lnf_b, f->gen_na, E, E, nr, sa); f->launches++;
        mm_any(f, f->lm_head, f->gen_na, nr, f->logits, f->V, false, sa);
        return;
    }
    ActQ xfr = f->xf; xfr.N = nr;
    if (nr > b200_mmv_max_n()) xfr.h = f->xh_a;
    launch_layernorm_q(x, E, ra, rb, ra ? E : 0, f->lnf_g, f->lnf_b, &xfr, nullptr, nullptr, nullptr, E, nr, sa); f->launches++;
    mm(f, f->lm_head, xfr, nr, f->logits, f->V, EPI_NONE, f->xh_a, sa);
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
// the rows the previous rank sent on every other one
static void eval_input(b200_falcon * f, int N) {
    if (f->first) {
        if (f->ring_mode && f->hp.world > 1) B200_NCCL_CHECK(nccl().Recv(f->tokens_dev, 1, ncclInt32, f->hp.world - 1, f->comm, f->s_main));
        launch_dequant_rows(f->tok_emb, f->tokens_dev, N, f->inp, f->E, f->s_main); f->launches++;
    } else B200_NCCL_CHECK(nccl().Recv(f->inp, (size_t) N * f->E, ncclFloat, f->hp.rank - 1, f->comm, f->s_main));
}
// The end of an eval: the residual adds of the last local layer (:2399-2400), then on the last rank the head over rows
// [logits_rows_from, N) and, in the generation-step graph, the sampled id; on every other rank the rows go on to the next one.
// fold_add: a quantised head's LayerNorm kernel does the adds (one kernel less on the decode step)
static void eval_output(b200_falcon * f, int N, int logits_rows_from, bool fold_add) {
    const bool fold = fold_add && f->last && !f->generic_head && f->NL > 0;
    if (f->NL > 0 && !fold) { launch_add3(f->dn, f->ao, f->inp, f->inp, (int64_t) N * f->E, f->s_main); f->launches++; }
    if (!f->last) { B200_NCCL_CHECK(nccl().Send(f->inp, (size_t) N * f->E, ncclFloat, f->hp.rank + 1, f->comm, f->s_main)); return; }
    enqueue_head(f, f->inp + (size_t) logits_rows_from * f->E, N - logits_rows_from, fold ? f->dn : nullptr, fold ? f->ao : nullptr, f->s_main);
    tap_head(f, N, N - logits_rows_from);
    ring_token_out(f);
}

// AttnParams of local layer l for N new tokens.  graph_mode: n_past is read from the device scalar, and the tier the graph is captured
// for (cur_tier) says whether the long-context kernels may be captured.
static AttnParams attn_params(const b200_falcon * f, int l, int N, int n_past, float theta_scale, bool graph_mode) {
    AttnParams ap = { f->H, f->HKV, f->D, N, n_past, graph_mode ? f->n_past_dev : nullptr, f->hp.n_ctx, (int64_t) f->QKV, nullptr };
    ap.long_ctx = graph_mode ? f->cur_tier : 0;
    ap.rope_theta_scale = theta_scale;
    const KvLayer kv = kv_layer(f, l);
    ap.k16 = kv.k16; ap.vt16 = kv.vt16;
    return ap;
}
// RoPE + KV append of layer l's new rows (:2229-2281), then the attention qkv -> att (:2285-2366).  Prompts run eagerly, on s_main
// like their attention: a scratch that has to grow waits for the previous user.
static void enqueue_attention(b200_falcon * f, int l, const AttnParams & ap, cudaStream_t st) {
    const KvLayer kv = kv_layer(f, l);
    float * scratch = f->attn_dec_scratch;
    if (ap.n_tok > 1) {
        const size_t need = attention_scratch_bytes(ap);
        if (need > f->attn_scratch_bytes) {
            B200_CUDA_CHECK(cudaStreamSynchronize(st)); B200_CUDA_CHECK(cudaFree(f->attn_scratch));
            B200_CUDA_CHECK(cudaMalloc(&f->attn_scratch, need)); f->attn_scratch_bytes = need;
        }
        scratch = f->attn_scratch;
    }
    bool rotated = true;
    f->launches += launch_attention(f->qkv, kv.k, kv.v, f->att, f->E, ap, scratch, st, nullptr, &rotated);
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
    // debugging aid for timing experiments only (results are wrong when anything is skipped): B200_DBG_SKIP=ln,qkv,attn,up,down,wo
    const char * dbg = getenv("B200_DBG_SKIP");
    auto skip = [&](const char * what) { return dbg && strstr(dbg, what) != nullptr; };
    // All four mat-vecs of a layer go back to back on ONE stream (each is launched with programmatic dependent launch,
    // so its weight prefetch overlaps the previous one's tail); the small attention kernels run beside ffn_up on the
    // second stream:   s_main: LN -> qkv -> ffn_up(+GELU) -> ffn_down -> wo   (7B: wo -> ffn_down)     s_mlp: attention (RoPE + KV append inside)
    for (int l = 0; l < f->NL; l++) {
        const Layer & L = f->layers[l];
        const float * ra = l > 0 ? f->dn : nullptr, * rb = l > 0 ? f->ao : nullptr;
        if (!skip("ln")) {
            if (dual) launch_layernorm_q(f->inp, E, ra, rb, E, L.ln_attn_g, L.ln_attn_b, &xa, L.ln_mlp_g, L.ln_mlp_b, &xm, E, 1, sa);
            else      launch_layernorm_q(f->inp, E, ra, rb, E, L.ln_mlp_g, L.ln_mlp_b, &xm, nullptr, nullptr, nullptr, E, 1, sa);
            f->launches++;
        }
        if (!skip("qkv")) mmv(f, L.wqkv, dual ? xa : xm, f->qkv, f->QKV, none, sa);                             // libfalcon.cpp:2192
        B200_CUDA_CHECK(cudaEventRecord(f->e_fork, sa));
        B200_CUDA_CHECK(cudaStreamWaitEvent(sb, f->e_fork, 0));
        if (!skip("attn")) {
            AttnParams ap = attn_params(f, l, 1, n_past, theta_scale, graph_mode);
            ap.fuse_rope = 1;
            ap.qout = &xatt;                   // wo's activation quantisation, off the critical path
            enqueue_attention(f, l, ap, sb);
        }
        B200_CUDA_CHECK(cudaEventRecord(f->e_join, sb));
        if (!skip("up")) mmv(f, L.up, xm, f->up, f->FF, gelu, sa);                                               // :2389-2392
        // The attention kernels of the side stream run BESIDE ffn_up, and beside ffn_down too when its CTAs leave them registers
        // (Falcon-40B / 180B: at long contexts the attention outlasts ffn_up, and this order beat wo first).
        // Falcon-7B's ffn_down shape fills the SMs: attention work still pending when ffn_up ends would be shut out until it had
        // drained, so there wo (which has to wait for the attention anyway) goes first.
        const bool wo_first = mmv_fast_fills_sm(L.down);
        if (!wo_first && !skip("down")) mmv(f, L.down, xup, f->dn, E, none, sa);                                // :2394
        B200_CUDA_CHECK(cudaStreamWaitEvent(sa, f->e_join, 0));
        if (!skip("wo")) mmv(f, L.wo, xatt, f->ao, E, wo_epi, sa);                                            // :2370
        if (wo_first && !skip("down")) mmv(f, L.down, xup, f->dn, E, none, sa);
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
        mm_any(f, L.wqkv, dual ? f->gen_na : f->gen_nm, N, f->qkv, f->QKV, false, sa);                                   // :2192
        enqueue_attention(f, l, attn_params(f, l, N, n_past, theta_scale, graph_mode), sa);
        mm_any(f, L.wo, f->att, N, f->ao, E, false, sa);                                                                 // :2370
        mm_any(f, L.up, f->gen_nm, N, f->up, FF, true, sa);                                                              // :2389-2392
        mm_any(f, L.down, f->up, N, f->dn, E, false, sa);                                                                // :2394
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
    if (N > b200_mmv_max_n()) { xa.h = f->xh_a; xm.h = f->xh_m; xatt.h = f->xh_a; xup.h = f->xh_b; }     // GEMM path: fp16 operands come with the codes
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
        mm(f, L.up, xm, N, f->up, FF, EPI_GELU, f->xh_b, sb);                                                   // libfalcon.cpp:2389-2392
        launch_quantize_act(f->up, FF, xup, sb); f->launches++;
        mm(f, L.down, xup, N, f->dn, E, EPI_NONE, f->xh_b, sb);                                                 // :2394
        B200_CUDA_CHECK(cudaEventRecord(f->e_join, sb));
        // attention branch on s_main
        mm(f, L.wqkv, dual ? xa : xm, N, f->qkv, f->QKV, EPI_NONE, f->xh_a, sa);                                   // :2192
        AttnParams ap = attn_params(f, l, N, n_past, theta_scale, graph_mode);
        ap.fuse_rope = N == 1;                                                                                   // decode: RoPE + KV append inside the attention kernels
        enqueue_attention(f, l, ap, sa);
        launch_quantize_act(f->att, E, xatt, sa); f->launches++;
        mm(f, L.wo, xatt, N, f->ao, E, EPI_NONE, f->xh_a, sa);                                                  // :2370
        B200_CUDA_CHECK(cudaStreamWaitEvent(sa, f->e_join, 0));                                                  // join
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
    if (which == G_HOST && f->last) B200_CUDA_CHECK(cudaMemcpyAsync(f->logits_h, f->logits, (size_t) f->V * 4, cudaMemcpyDeviceToHost, f->s_main));
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

extern "C" {

// The eval in two halves: enqueue everything (returns at once: the GPU works while the caller does something else) / wait and hand the
// logits over.  b200_falcon_eval is begin + finish; the operator hook (ggml_surface.cu) calls begin at the graph's first ROPE node and
// finish at "result_lm_head", so the reference's walk over its remaining ~2000 graph nodes overlaps the device work.
extern "C++" int falcon_eval_begin(b200_falcon * f, const int32_t * tokens, int n_tokens, int n_past, int n_ctx_rope, int all_logits) {
    if (n_tokens <= 0 || n_past < 0 || n_past + n_tokens > f->hp.n_ctx || n_tokens > (f->hp.n_batch > 0 ? f->hp.n_batch : 1)) return 1;
    if (f->first) {                                  // token ids index the embedding matrix: reject anything outside it (ggml_get_rows asserts, ggml.c:11990)
        if (!tokens) return 1;
        for (int i = 0; i < n_tokens; i++) if (tokens[i] < 0 || tokens[i] >= f->V) return 2;
    }
    const float theta = rope_theta_scale_host(f->D, n_ctx_rope ? n_ctx_rope : f->hp.n_ctx, 1, 2.0f, 0);         // libfalcon.cpp:2229-2234
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
            f->pending_floats = nfl;
        }
    }
    return 0;
}
extern "C++" void falcon_eval_finish(b200_falcon * f, float * logits) {
    B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
    if (logits && f->pending_floats) memcpy(logits, f->logits_h, f->pending_floats * 4);
    B200_CUDA_CHECK(cudaEventElapsedTime(&f->last_ms, f->e_t0, f->e_t1));
}
int b200_falcon_eval(b200_falcon * f, const int32_t * tokens, int n_tokens, int n_past, int n_ctx_rope, float * logits, int all_logits) {
    const int rc = falcon_eval_begin(f, tokens, n_tokens, n_past, n_ctx_rope, all_logits);
    if (rc != 0) return rc;
    falcon_eval_finish(f, logits);
    return 0;
}

int b200_falcon_decode_dev(b200_falcon * f, const int32_t * token_dev, int n_past, int n_ctx_rope) {
    if (n_past < 0 || n_past >= f->hp.n_ctx) return 1;                       // the KV append would leave this layer's cache slice
    const float theta = rope_theta_scale_host(f->D, n_ctx_rope ? n_ctx_rope : f->hp.n_ctx, 1, 2.0f, 0);
    const int tier = tier_of(n_past);
    // position and token id are device scalars the graph (and a build's eager pass) reads; both are set stream-ordered (the position
    // travels as a kernel argument, so the host may run ahead by any number of steps)
    set_i32_kernel<<<1, 1, 0, f->s_main>>>(f->n_past_dev, n_past);
    if (f->first && token_dev) B200_CUDA_CHECK(cudaMemcpyAsync(f->tokens_dev, token_dev, 4, cudaMemcpyDeviceToDevice, f->s_main));
    const cudaGraphExec_t g = decode_graph(f, G_DEVICE, tier, theta);
    if (getenv("B200_NO_GRAPH")) { f->launches = 0; f->cur_tier = tier; enqueue_eval(f, 1, 0, theta, true, 0); f->cur_tier = 0; return 0; }   // timing experiments: eager launches
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
    const float theta = rope_theta_scale_host(f->D, n_ctx_rope ? n_ctx_rope : f->hp.n_ctx, 1, 2.0f, 0);
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
// here the cache is device-resident [layer][n_ctx][n_head_kv][head_dim] f32 and rows are copied straight out of / into HBM.
int b200_falcon_kv_read(b200_falcon * f, int layer, int pos, int n, float * k_out, float * v_out) {
    if (layer < f->hp.layer_first || layer >= f->hp.layer_last || pos < 0 || n < 0 || pos + n > f->hp.n_ctx) return 1;
    const KvLayer c = kv_layer(f, layer - f->hp.layer_first);
    const size_t row = kv_row(f);
    B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
    if (k_out) B200_CUDA_CHECK(cudaMemcpy(k_out, c.k + (size_t) pos * row, (size_t) n * row * 4, cudaMemcpyDeviceToHost));
    if (v_out) B200_CUDA_CHECK(cudaMemcpy(v_out, c.v + (size_t) pos * row, (size_t) n * row * 4, cudaMemcpyDeviceToHost));
    return 0;
}
// the fp16 shadow the prompt kernel reads (attention_ws.cu), positions [pos, pos + n) of `layer`: k16_out [n][n_head_kv][head_dim],
// vt16_out [n_head_kv][head_dim][n].  The range may reach attention_ctx_pad(n_ctx), so that the padding columns can be inspected.
int b200_falcon_kv_shadow_read(b200_falcon * f, int layer, int pos, int n, uint16_t * k16_out, uint16_t * vt16_out) {
    const int ctx_pad = attention_ctx_pad(f->hp.n_ctx);
    if (!f->k16 || layer < f->hp.layer_first || layer >= f->hp.layer_last || pos < 0 || n < 0 || pos + n > ctx_pad) return 1;
    const KvLayer c = kv_layer(f, layer - f->hp.layer_first);
    const size_t row = kv_row(f);
    B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
    if (k16_out && n) B200_CUDA_CHECK(cudaMemcpy(k16_out, c.k16 + (size_t) pos * row, (size_t) n * row * 2, cudaMemcpyDeviceToHost));
    if (vt16_out && n) B200_CUDA_CHECK(cudaMemcpy2D(vt16_out, (size_t) n * 2, c.vt16 + pos, (size_t) ctx_pad * 2, (size_t) n * 2, row, cudaMemcpyDeviceToHost));
    return 0;
}
int b200_falcon_kv_write(b200_falcon * f, int layer, int pos, int n, const float * k_in, const float * v_in) {
    if (layer < f->hp.layer_first || layer >= f->hp.layer_last || pos < 0 || n < 0 || pos + n > f->hp.n_ctx) return 1;
    const KvLayer c = kv_layer(f, layer - f->hp.layer_first);
    const size_t row = kv_row(f);
    B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
    if (k_in) B200_CUDA_CHECK(cudaMemcpy(c.k + (size_t) pos * row, k_in, (size_t) n * row * 4, cudaMemcpyHostToDevice));
    if (v_in) B200_CUDA_CHECK(cudaMemcpy(c.v + (size_t) pos * row, v_in, (size_t) n * row * 4, cudaMemcpyHostToDevice));
    if (c.k16) {
        launch_kv_shadow_refresh(c.k, c.v, c.k16, c.vt16, f->HKV, f->hp.n_ctx, pos, n, f->s_main);
        B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
    }
    return 0;
}
// random K / V rows generated on the device for positions [pos, pos + n) of every local layer: pre-fills a long context
// for throughput runs (BASELINE config 5: decode at 8k context) without evaluating 8k tokens first
int b200_falcon_kv_fill_random(b200_falcon * f, int pos, int n, uint64_t seed) {
    if (pos < 0 || n < 0 || pos + n > f->hp.n_ctx) return 1;
    const size_t row = kv_row(f);
    for (int l = 0; l < f->NL; l++) {
        const KvLayer c = kv_layer(f, l);
        fill_f32_kernel<<<296, 256, 0, f->s_main>>>(c.k + (size_t) pos * row, (int64_t) ((size_t) n * row), 0.f, 1.f, seed + 2 * l);
        fill_f32_kernel<<<296, 256, 0, f->s_main>>>(c.v + (size_t) pos * row, (int64_t) ((size_t) n * row), 0.f, 1.f, seed + 2 * l + 1);
        if (c.k16) launch_kv_shadow_refresh(c.k, c.v, c.k16, c.vt16, f->HKV, f->hp.n_ctx, pos, n, f->s_main);
    }
    B200_CUDA_CHECK(cudaGetLastError());
    B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
    return 0;
}
// Session file over the device KV cache: what falcon_save_session_file / falcon_load_session_file (libfalcon.cpp:4490-4563) keep of
// the KV state, written straight from / read straight into HBM through a bounded pinned buffer.  Own container (the reference's
// serialises its transposed, ping-ponged host V buffers, which do not exist here):
//   u32 magic 'b2kv', u32 version 1, i32 layer_first, layer_last, n_head_kv, head_dim, n_tokens; then per local layer: K rows, V rows (f32)
// save: returns 0 / -1.  load: returns the number of positions restored (the caller continues at that n_past), -1 on any mismatch.
int b200_falcon_save_kv(b200_falcon * f, const char * path, int n_tokens) {
    if (n_tokens < 0 || n_tokens > f->hp.n_ctx) return -1;
    FILE * fp = fopen(path, "wb");
    if (!fp) return -1;
    const int32_t hdr[7] = { 0x766b3262, 1, f->hp.layer_first, f->hp.layer_last, f->HKV, f->D, n_tokens };
    bool ok = fwrite(hdr, sizeof(hdr), 1, fp) == 1;
    const size_t bytes = (size_t) n_tokens * kv_row(f) * 4;
    std::vector<float> buf(bytes / 4 + 1);
    B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
    for (int l = 0; l < f->NL && ok; l++)
        for (const float * base : { kv_layer(f, l).k, kv_layer(f, l).v }) {
            B200_CUDA_CHECK(cudaMemcpy(buf.data(), base, bytes, cudaMemcpyDeviceToHost));
            ok = ok && (bytes == 0 || fwrite(buf.data(), bytes, 1, fp) == 1);
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
        if (b200_falcon_kv_write(f, f->hp.layer_first + l, 0, n, k.data(), v.data()) != 0) { fclose(fp); return -1; }     // also refreshes the fp16 shadow
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
int b200_falcon_tap(b200_falcon * f, int on) {
    invalidate_graphs(f);                                 // the captured decode graphs hold the copies (or their absence)
    B200_CUDA_CHECK(cudaDeviceSynchronize());
    B200_CUDA_CHECK(cudaFree(f->tap.mem));
    f->tap = b200_falcon::Tap{};
    if (!on) return 0;
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
    B200_CUDA_CHECK(cudaMalloc(&T.mem, lb * f->NL + hb + 256));
    T.rotated.assign(f->NL, 0);
    return 0;
}
int b200_falcon_tap_read(const b200_falcon * f, int layer, const char * node, void * host, size_t bytes) {
    const auto & T = f->tap;
    if (!T.mem || !node || !host) return 1;
    const bool head = layer == -1;
    const int l = layer - f->hp.layer_first;
    if (head ? !f->last : (l < 0 || l >= f->NL)) return 1;
    if (!head && !strcmp(node, "qkv_rotated")) {
        if (bytes != sizeof(int)) return 1;
        memcpy(host, &T.rotated[l], sizeof(int));
        return 0;
    }
    for (const auto & n : head ? T.head : T.layer) {
        if (n.name != node) continue;
        if (bytes != n.row_bytes * (n.all_rows ? T.rows : T.head_rows)) return 1;
        B200_CUDA_CHECK(cudaStreamSynchronize(f->s_main));
        B200_CUDA_CHECK(cudaMemcpy(host, T.mem + (head ? (size_t) f->NL * T.layer_bytes : (size_t) l * T.layer_bytes) + n.off, bytes, cudaMemcpyDeviceToHost));
        return 0;
    }
    return 1;
}

int b200_falcon_last_launches(const b200_falcon * f) { return f->launches; }
float b200_falcon_last_ms(const b200_falcon * f) { return f->last_ms; }
void * b200_falcon_stream(b200_falcon * f) { return (void *) f->s_main; }

// Times the dominant kernel in isolation on the model's own matrices: every local quantised mat-vec (4 per layer +
// lm_head) launched back to back on the eval stream, `reps` passes, CUDA events around the whole region.  Each
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
        for (auto & L : f->layers) {
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
