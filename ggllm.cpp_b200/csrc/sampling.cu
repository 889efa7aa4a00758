// sampling.cu -- falcon_main's whole sampling chain on the device (SURVEY 8f-2), so that only a token id leaves the GPU per step.
//
// What falcon_main does on the host with the 260 KB logits row of every token (examples/falcon/falcon_main.cpp:896-987):
//   logit bias                       (:899-902)                 row[id] += value (applied here to the work copy; the logits stay intact)
//   llama_sample_repetition_penalty  (libfalcon.cpp:3281-3308)  logits of ids in the last-n window: l <= 0 ? l * penalty : l / penalty
//   llama_sample_frequency_and_presence_penalties (:3310-3339)  l -= float(count) * alpha_f + float(count > 0) * alpha_p
//   temp <= 0 : llama_sample_token_greedy (:3433-3447)          first maximum
//   mirostat 1: temperature -> llama_sample_token_mirostat (:3342-3389): softmax over the whole vocabulary, s_hat from the top 100,
//               k = powf(...), top_k(int(k)), draw, mu -= eta * (surprise - tau)
//   mirostat 2: temperature -> llama_sample_token_mirostat_v2 (:3391-3431): softmax, cut at -log2f(p) > mu, softmax, draw, mu update
//   otherwise   llama_sample_top_k (:3094-3118) -> tail_free (:3154-3203) -> typical (:3206-3267) -> top_p (:3121-3150, including its
//               "last_idx = i" cut, which drops the candidate that crosses p) -> temperature (:3269-3279) -> llama_sample_token
//               (:3449-3468): softmax in fp32, then std::discrete_distribution over the probabilities driven by the context's std::mt19937
// is restated here, INCLUDING the random draw: the kernel carries the MT19937 state (seeded like std::mt19937(seed)), builds the
// double-precision cumulative table of libstdc++'s discrete_distribution (normalise by the double sum, partial sums, last entry
// forced to 1.0), draws generate_canonical<double, 53> from two 32-bit outputs and takes the lower bound.
//
// Arithmetic: the reference is compiled with g++ -O3 -std=c++11 -march=x86-64-v3 (oracle/Makefile), where ISO mode turns fp
// contraction off -- except that its objdump shows three fused multiply-adds, all in mirostat: sum_ti_bi and sum_ti_sq
// (vfmadd231ss) and the mu update (vfnmadd213ss).  Those three use fmaf here; everything else is written with __f*_rn so that nvcc
// cannot fuse it.  Every fp32 sum runs sequentially in the reference's order (softmax sums stop early once a term cannot change
// the sum, see seq_sum_desc).
//
// Transcendentals: expf / logf / log2f / powf are evaluated in double and rounded once (ref_expf ...), i.e. correctly rounded
// except within ~2^-29 relative of a float rounding boundary.  glibc's float functions are NOT correctly rounded: on an x86-64 host
// with FMA (glibc 2.39) logf differs from the correctly rounded value on 0.73 % of probabilities in (0, 1), log2f on 0.56 %, expf
// on 0.06 % of arguments in (-40, 0], powf on 0.06 % of pairs.  So the device is bit for bit with an exact restatement of the
// chain over correctly rounded functions (tests/sampler_twin.py, checked stage by stage through the tap below), and the reference
// differs from that restatement in the last bit of a probability, typical's entropy and scores, or mirostat's s_hat and mu
// wherever glibc rounds differently.  An id changes only when such an ulp moves a value across a boundary (a draw, a cut or
// mirostat 1's int(k)); over the 1,558 fixed-seed steps of tests/test_sampler_stages_gpu.py that count is zero.
// Matching glibc bit for bit would mean carrying its float functions' tables onto the device, which this file does not do.
//
// Ordering: top-k with 1 <= k <= 1024 (the default chain) takes k rounds of block arg-max as before; mirostat, top_k <= 0 and
// top_k > 1024 sort the whole row with a stable LSD radix sort (4 passes of 8 bits over an L2-resident scratch), descending logits
// with equal logits by ascending id.  Typical reorders its candidates by the same sort (ascending shifted score, ties by position).
// The reference sorts with std::sort, which leaves equal keys in an unspecified order; ids can only differ from it on exact ties.
// One CTA of 1024 threads; every sequential part runs on thread 0.
#include "kernels.h"
#include <climits>
#include <cstring>

struct SamplerState {                   // device resident
    uint32_t mt[624]; int mti;
    int32_t window[B200_SAMPLER_MAX_WINDOW]; int wlen, wcap;      // the last-n ids the penalties look at (oldest first)
    int wpos;
    float mu;                                                      // mirostat's running target surprise (starts at 2 * tau)
};

namespace {

constexpr int NT = 1024;

__device__ uint32_t mt_next(SamplerState * s) {                       // MT19937 (std::mt19937): regenerate every 624 outputs, then temper
    if (s->mti >= 624) {
        for (int i = 0; i < 624; i++) {
            const uint32_t y = (s->mt[i] & 0x80000000u) | (s->mt[(i + 1) % 624] & 0x7fffffffu);
            s->mt[i] = s->mt[(i + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
        }
        s->mti = 0;
    }
    uint32_t y = s->mt[s->mti++];
    y ^= y >> 11; y ^= (y << 7) & 0x9d2c5680u; y ^= (y << 15) & 0xefc60000u; y ^= y >> 18;
    return y;
}

__global__ void sampler_init_kernel(SamplerState * s, uint32_t seed, const int32_t * window, int n, int cap, float mu) {
    s->mt[0] = seed;
    for (int i = 1; i < 624; i++) s->mt[i] = 1812433253u * (s->mt[i - 1] ^ (s->mt[i - 1] >> 30)) + (uint32_t) i;
    s->mti = 624;
    s->wcap = cap; s->wlen = n < cap ? n : cap; s->wpos = 0;
    for (int i = 0; i < s->wlen; i++) s->window[i] = window[n - s->wlen + i];
    if (s->wlen == cap) s->wpos = 0; else s->wpos = s->wlen;          // next slot to write
    s->mu = mu;
}

// correctly rounded float transcendentals (double evaluation, rounded once); glibc's float functions differ in the last bit at times
__device__ __forceinline__ float ref_expf(float x) { return (float) exp((double) x); }
__device__ __forceinline__ float ref_logf(float x) { return (float) log((double) x); }
__device__ __forceinline__ float ref_log2f(float x) { return (float) log2((double) x); }
__device__ __forceinline__ float ref_powf(float x, float y) { return (float) pow((double) x, (double) y); }

// int(k) as x86 compiles it (cvttss2si): NaN and anything outside int32 give INT_MIN, not a saturated value
__device__ __forceinline__ int x86_float_to_int(float x) {
    return (x > -2147483904.0f && x < 2147483648.0f) ? (int) x : INT_MIN;
}

// the fp32 sum of x[0..n) in index order, bit for bit.  x must be non-negative and non-increasing up to a factor of 2 (softmax
// terms in descending-logit order): once x[i] < ulp(S)/4, every later term is < ulp(S)/2 and rounds away, so the loop stops there.
__device__ float seq_sum_desc(const float * x, int n) {
    float S = 0.f;
    for (int i = 0; i < n; i++) {
        const float e = x[i];
        if (S > 0.f) {
            const float ulp = __int_as_float((__float_as_int(S) & 0x7f800000) ) * 1.1920928955078125e-07f;   // 2^(exp(S) - 23)
            if (e < __fmul_rn(ulp, 0.25f)) break;
        }
        S = __fadd_rn(S, e);
    }
    return S;
}

// llama_sample_softmax over cl[0..n) (already in the order the reference holds them): max = cl[0], p = expf(l - max) / sum.
// desc: cl is in descending order, so the sum may stop early; after typical's reordering it may not.
__device__ void block_softmax(const float * cl, float * cp, int n, float * s_f, bool desc = true) {
    const float mx = cl[0];
    for (int i = threadIdx.x; i < n; i += NT) cp[i] = ref_expf(__fsub_rn(cl[i], mx));
    __syncthreads();
    if (threadIdx.x == 0) {
        if (desc) s_f[0] = seq_sum_desc(cp, n);
        else { float sum = 0.f; for (int i = 0; i < n; i++) sum = __fadd_rn(sum, cp[i]); s_f[0] = sum; }
    }
    __syncthreads();
    const float S = s_f[0];
    for (int i = threadIdx.x; i < n; i += NT) cp[i] = __fdiv_rn(cp[i], S);
    __syncthreads();
}

// llama_sample_token's draw over the probabilities cp[0..n): std::discrete_distribution (double table) with the context's
// std::mt19937.  Returns the drawn position (every thread).  n < 2 draws nothing, as libstdc++'s empty table does.
// Up to 4096 entries the table is summed sequentially like libstdc++; beyond that in 1024 contiguous chunks (double sums of fp32
// probabilities, then a sequential pass over the chunk sums): the partial sums then differ from the sequential ones by at most
// about n * 2^-53 relative (7e-12 at n = 65024), five orders below the spacing of the fp32 terms they are built from.
__device__ int block_draw(const float * cp, int n, SamplerState * st, double * s_d, int * s_i) {
    const int tid = threadIdx.x;
    if (n < 2) return 0;
    if (tid == 0) {
        const uint32_t x0 = mt_next(st), x1 = mt_next(st);
        double u = ((double) x0 + (double) x1 * 4294967296.0) / 18446744073709551616.0;      // generate_canonical<double, 53>
        if (u >= 1.0) u = 0.99999999999999988898;                      // nextafter(1.0, 0.0)
        s_d[NT] = u;
        if (n <= 4096) {
            double sum = 0.0;
            for (int i = 0; i < n; i++) sum += (double) cp[i];
            double acc = 0.0;
            int pick = n - 1;
            for (int i = 0; i < n; i++) {
                acc += (double) cp[i] / sum;
                const double c = i == n - 1 ? 1.0 : acc;               // the table's last entry is forced to 1.0
                if (!(c < u)) { pick = i; break; }                     // std::lower_bound: first entry >= u
            }
            s_i[0] = pick;
        }
    }
    __syncthreads();
    if (n <= 4096) { const int pick = s_i[0]; __syncthreads(); return pick; }
    const double u = s_d[NT];
    const int chunk = (n + NT - 1) / NT, b = tid * chunk, e = min(n, b + chunk);
    double cs = 0.0;
    for (int i = b; i < e; i++) cs += (double) cp[i];
    s_d[tid] = cs;
    __syncthreads();
    if (tid == 0) { double sum = 0.0; for (int t = 0; t < NT; t++) sum += s_d[t]; s_d[NT + 1] = sum; s_i[0] = n - 1; }
    __syncthreads();
    const double sum = s_d[NT + 1];
    double q = 0.0;
    for (int i = b; i < e; i++) q += (double) cp[i] / sum;
    __syncthreads();
    s_d[tid] = q;
    __syncthreads();
    if (tid == 0) { double run = 0.0; for (int t = 0; t < NT; t++) { const double c = s_d[t]; s_d[t] = run; run += c; } }
    __syncthreads();
    double acc = s_d[tid];
    for (int i = b; i < e; i++) {
        acc += (double) cp[i] / sum;
        const double c = i == n - 1 ? 1.0 : acc;
        if (!(c < u)) { atomicMin(s_i, i); break; }
    }
    __syncthreads();
    const int pick = s_i[0];
    __syncthreads();
    return pick;
}

__device__ __forceinline__ uint32_t key_asc(float f) {                 // order-preserving: a < b  <=>  key(a) < key(b); -0 == +0
    if (f == 0.f) f = 0.f;
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// stable LSD radix sort of (k0, v0)[0..n) by ascending key, 4 passes of 8 bits; ka/va are scratch of n entries.  Result in k0/v0.
// Stability inside a 1024-element tile: ranks from __match_any_sync within a warp, then per-digit offsets over the warps in order.
__device__ void block_radix_sort(uint32_t * k0, int32_t * v0, uint32_t * ka, int32_t * va, int n, int (*s_cnt)[256], int * s_base) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int i = tid; i < 32 * 256; i += NT) (&s_cnt[0][0])[i] = 0;
    for (int pass = 0; pass < 4; pass++) {
        const int shift = pass * 8;
        uint32_t * ks = (pass & 1) ? ka : k0; int32_t * vs = (pass & 1) ? va : v0;
        uint32_t * kd = (pass & 1) ? k0 : ka; int32_t * vd = (pass & 1) ? v0 : va;
        if (tid < 256) s_base[tid] = 0;
        __syncthreads();
        for (int i = tid; i < n; i += NT) atomicAdd(&s_base[(ks[i] >> shift) & 255], 1);
        __syncthreads();
        if (tid == 0) { int run = 0; for (int d = 0; d < 256; d++) { const int c = s_base[d]; s_base[d] = run; run += c; } }
        __syncthreads();
        for (int t0 = 0; t0 < n; t0 += NT) {
            const int i = t0 + tid;
            const bool valid = i < n;
            const uint32_t key = valid ? ks[i] : 0u; const int32_t val = valid ? vs[i] : 0;
            const int d = valid ? (int) ((key >> shift) & 255) : 256;
            const unsigned peers = __match_any_sync(0xffffffffu, d);
            const int rank = __popc(peers & ((1u << lane) - 1u));
            if (valid && lane == __ffs(peers) - 1) s_cnt[warp][d] = __popc(peers);
            __syncthreads();
            if (tid < 256) {
                int run = s_base[tid];
                for (int w = 0; w < 32; w++) { const int c = s_cnt[w][tid]; s_cnt[w][tid] = run; run += c; }
                s_base[tid] = run;
            }
            __syncthreads();
            if (valid) { const int pos = s_cnt[warp][d] + rank; kd[pos] = key; vd[pos] = val; }
            __syncthreads();
            for (int j = tid; j < 32 * 256; j += NT) (&s_cnt[0][0])[j] = 0;
            __syncthreads();
        }
    }
}

enum { TAP_ORDER, TAP_TFS, TAP_TYPICAL, TAP_TOP_P, TAP_TEMP, TAP_FINAL, TAP_STAGES };
struct TapHead { int n[TAP_STAGES]; int pick, id, k; float entropy, mu; double u; };      // n = -1: the stage did not run
constexpr int TAP_HEAD_FLOATS = 64;
static_assert(sizeof(TapHead) <= TAP_HEAD_FLOATS * 4, "tap head");

struct Scratch {                        // sampler_work_floats(n) floats, carved into n-entry arrays
    float * work; uint32_t * k0; uint32_t * ka; int32_t * v0; int32_t * va; int32_t * cid; float * cl; float * cp; float * tmp;
};
__device__ __forceinline__ Scratch carve(float * w, int n) {
    Scratch s; s.work = w; s.k0 = (uint32_t *) (w + (size_t) n); s.ka = (uint32_t *) (w + 2 * (size_t) n);
    s.v0 = (int32_t *) (w + 3 * (size_t) n); s.va = (int32_t *) (w + 4 * (size_t) n); s.cid = (int32_t *) (w + 5 * (size_t) n);
    s.cl = w + 6 * (size_t) n; s.cp = w + 7 * (size_t) n; s.tmp = w + 8 * (size_t) n;
    return s;
}

// test tap (b200_sampler_tap): a copy of the candidate list after every stage, in the order the reference holds it.  Layout
// (sampler_tap_bytes): the TapHead, then the row after bias and penalties [n_vocab], then per stage ids, logits, p [n_vocab] each.
__device__ __forceinline__ int32_t * tap_ids(float * tap, int V, int stage) { return (int32_t *) (tap + TAP_HEAD_FLOATS + V + (size_t) (3 * stage) * V); }
__device__ __forceinline__ float * tap_logits(float * tap, int V, int stage) { return tap + TAP_HEAD_FLOATS + V + (size_t) (3 * stage + 1) * V; }
__device__ __forceinline__ float * tap_p(float * tap, int V, int stage) { return tap + TAP_HEAD_FLOATS + V + (size_t) (3 * stage + 2) * V; }
// entry i is candidate perm[i] (perm null: i) of ids / l / p (p null: not written).  Called by every thread, in uniform control flow.
__device__ void tap_list(float * tap, int V, int stage, int n, const int32_t * ids, const float * l, const float * p, const int32_t * perm) {
    for (int i = threadIdx.x; i < n; i += NT) {
        const int j = perm ? perm[i] : i;
        tap_ids(tap, V, stage)[i] = ids[j]; tap_logits(tap, V, stage)[i] = l[j];
        if (p) tap_p(tap, V, stage)[i] = p[j];
    }
    if (threadIdx.x == 0) ((TapHead *) tap)->n[stage] = n;
    __syncthreads();
}

__global__ void __launch_bounds__(NT) sample_kernel(const float * __restrict__ logits, int n_vocab, SamplerParams p, SamplerState * st,
                                                    float * __restrict__ work, int32_t * out, int32_t * hist, int * step, float * tap) {
    __shared__ float sv[32]; __shared__ int si[32];
    __shared__ int32_t win[B200_SAMPLER_MAX_WINDOW]; __shared__ int s_wlen;
    __shared__ int s_cnt[32][256]; __shared__ int s_base[256];
    __shared__ double s_d[NT + 2]; __shared__ int s_i[2]; __shared__ float s_f[2];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const Scratch S = carve(work, n_vocab);
    const bool rep = p.repeat_penalty != 1.0f, fp = p.frequency_penalty != 0.0f || p.presence_penalty != 0.0f;
    if (tid == 0) s_wlen = (rep || fp) ? st->wlen : 0;
    __syncthreads();
    const int wlen = s_wlen;
    for (int i = tid; i < wlen; i += NT) win[i] = st->window[i];
    for (int i = tid; i < n_vocab; i += NT) S.work[i] = logits[i];
    if (tap && tid == 0) {
        TapHead * h = (TapHead *) tap;
        for (int s = 0; s < TAP_STAGES; s++) h->n[s] = -1;
        h->pick = -1; h->id = -1; h->k = -1; h->entropy = NAN; h->mu = st->mu; h->u = -1.0;
    }
    __syncthreads();
    // ---- logit bias (ids unique, validated on the host), then the penalties on each distinct id of the window
    if (tid < p.n_bias) S.work[p.bias_id[tid]] = __fadd_rn(S.work[p.bias_id[tid]], p.bias_value[tid]);
    __syncthreads();
    if (tid < wlen) {
        const int id = win[tid];
        bool first = true; int count = 0;
        for (int j = 0; j < wlen; j++) { if (win[j] == id) { count++; if (j < tid) first = false; } }
        if (first && id >= 0 && id < n_vocab) {
            float l = S.work[id];
            if (rep) l = l <= 0.f ? __fmul_rn(l, p.repeat_penalty) : __fdiv_rn(l, p.repeat_penalty);
            if (fp) l = __fsub_rn(l, __fadd_rn(__fmul_rn((float) count, p.frequency_penalty), __fmul_rn(count > 0 ? 1.0f : 0.0f, p.presence_penalty)));
            S.work[id] = l;
        }
    }
    __syncthreads();
    if (tap) {
        for (int i = tid; i < n_vocab; i += NT) tap[TAP_HEAD_FLOATS + i] = S.work[i];
        __syncthreads();
    }
    int n, pick = 0;
    bool reordered = false;                                            // typical left the candidates out of descending order
    const bool greedy = p.temp <= 0.f;
    if (greedy || (p.mirostat == 0 && p.top_k >= 1 && p.top_k <= NT)) {
        // ---- the k largest logits, descending (equal values: lowest id first), by k rounds of block arg-max; a taken entry becomes
        // NaN, so it cannot win again even when every entry left is -inf
        n = greedy ? 1 : min(p.top_k, n_vocab);
        for (int r = 0; r < n; r++) {
            float best = -INFINITY; int bi = 0x7fffffff;
            for (int i = tid; i < n_vocab; i += NT) { const float v = S.work[i]; if (v > best || (v == best && i < bi)) { best = v; bi = i; } }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, best, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
            }
            if (lane == 0) { sv[warp] = best; si[warp] = bi; }
            __syncthreads();
            if (warp == 0) {
                best = sv[lane]; bi = si[lane];
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    const float ov = __shfl_xor_sync(0xffffffffu, best, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
                }
                if (lane == 0) { S.cl[r] = best; S.cid[r] = bi; if (bi < n_vocab) S.work[bi] = NAN; }   // NaN loses every comparison
            }
            __syncthreads();
        }
    } else {
        // ---- the whole row in descending order (mirostat divides by the temperature first, as the reference does before its sort)
        for (int i = tid; i < n_vocab; i += NT) {
            float l = S.work[i];
            if (p.mirostat != 0) { l = __fdiv_rn(l, p.temp); S.work[i] = l; }
            S.k0[i] = ~key_asc(l); S.v0[i] = i;
        }
        __syncthreads();
        block_radix_sort(S.k0, S.v0, S.ka, S.va, n_vocab, s_cnt, s_base);
        for (int i = tid; i < n_vocab; i += NT) { const int id = S.v0[i]; S.cid[i] = id; S.cl[i] = S.work[id]; }
        __syncthreads();
        n = (p.mirostat != 0 || p.top_k <= 0 || p.top_k > n_vocab) ? n_vocab : p.top_k;
    }
    if (tap) tap_list(tap, n_vocab, TAP_ORDER, n, S.cid, S.cl, nullptr, nullptr);

    if (!greedy && p.mirostat == 1) {
        block_softmax(S.cl, S.cp, n, s_f);
        if (tid == 0) {                                                // s_hat from the m = 100 most probable, k, then top_k(int(k), 1)
            float sum_ti_bi = 0.f, sum_ti_sq = 0.f;
            for (int i = 0; i < 99 && i < n - 1; i++) {
                const float t_i = ref_logf(__fdiv_rn((float) (i + 2), (float) (i + 1)));
                const float b_i = ref_logf(__fdiv_rn(S.cp[i], S.cp[i + 1]));
                sum_ti_bi = fmaf(t_i, b_i, sum_ti_bi);
                sum_ti_sq = fmaf(t_i, t_i, sum_ti_sq);
            }
            const float s_hat = __fdiv_rn(sum_ti_bi, sum_ti_sq);
            const float eps = __fsub_rn(s_hat, 1.0f);
            const float k = ref_powf(__fdiv_rn(__fmul_rn(eps, ref_powf(2.0f, st->mu)), __fsub_rn(1.0f, ref_powf((float) n_vocab, -eps))),
                                     __fdiv_rn(1.0f, s_hat));
            int ki = x86_float_to_int(k);
            ki = max(ki, 1); ki = min(ki, n);
            s_i[1] = ki;
            if (tap) ((TapHead *) tap)->k = ki;
        }
        __syncthreads();
        n = s_i[1];
    } else if (!greedy && p.mirostat == 2) {
        block_softmax(S.cl, S.cp, n, s_f);
        if (tid == 0) s_i[1] = n;
        __syncthreads();
        const float mu = st->mu;
        for (int i = tid; i < n; i += NT) if (-ref_log2f(S.cp[i]) > mu) { atomicMin(&s_i[1], i); break; }
        __syncthreads();
        n = max(s_i[1], 1);
        __syncthreads();
    } else if (!greedy) {
        // ---- tail-free: second derivatives of the sorted probabilities, normalised, cut where their running sum passes z
        if (p.tfs_z < 1.0f && n > 2) {
            block_softmax(S.cl, S.cp, n, s_f);
            for (int i = tid; i < n - 2; i += NT) {
                const float d0 = __fsub_rn(S.cp[i], S.cp[i + 1]), d1 = __fsub_rn(S.cp[i + 1], S.cp[i + 2]);
                S.tmp[i] = fabsf(__fsub_rn(d0, d1));
            }
            __syncthreads();
            if (tid == 0) {
                float sum = 0.f;
                for (int i = 0; i < n - 2; i++) sum = __fadd_rn(sum, S.tmp[i]);
                float cum = 0.f; int last = n;
                for (int i = 0; i < n - 2; i++) {
                    cum = __fadd_rn(cum, __fdiv_rn(S.tmp[i], sum));
                    if (cum > p.tfs_z && i >= 1) { last = i; break; }
                }
                s_i[1] = last;
            }
            __syncthreads();
            n = s_i[1];
            __syncthreads();
            if (tap) tap_list(tap, n_vocab, TAP_TFS, n, S.cid, S.cl, S.cp, nullptr);
        }
        // ---- typical: candidates reordered by |-log p - entropy| (ascending), cut where their probabilities pass typical_p
        if (p.typical_p < 1.0f) {
            block_softmax(S.cl, S.cp, n, s_f);
            if (tid == 0) {
                float ent = 0.f;
                for (int i = 0; i < n; i++) ent = __fadd_rn(ent, __fmul_rn(-S.cp[i], ref_logf(S.cp[i])));
                s_f[1] = ent;
            }
            __syncthreads();
            const float ent = s_f[1];
            for (int i = tid; i < n; i += NT) { S.k0[i] = key_asc(fabsf(__fsub_rn(-ref_logf(S.cp[i]), ent))); S.v0[i] = i; }
            __syncthreads();
            block_radix_sort(S.k0, S.v0, S.ka, S.va, n, s_cnt, s_base);
            if (tid == 0) {
                float cum = 0.f; int last = n;
                for (int i = 0; i < n; i++) {
                    cum = __fadd_rn(cum, S.cp[S.v0[i]]);
                    if (cum > p.typical_p) { last = i + 1; break; }
                }
                s_i[1] = last;
            }
            __syncthreads();
            const int last = s_i[1];
            if (tap) {
                if (tid == 0) ((TapHead *) tap)->entropy = ent;
                tap_list(tap, n_vocab, TAP_TYPICAL, last, S.cid, S.cl, S.cp, S.v0);
            }
            for (int i = tid; i < last; i += NT) { const int j = S.v0[i]; S.va[i] = S.cid[j]; S.tmp[i] = S.cl[j]; }
            __syncthreads();
            for (int i = tid; i < last; i += NT) { S.cid[i] = S.va[i]; S.cl[i] = S.tmp[i]; }
            __syncthreads();
            n = last; reordered = true;
        }
        // ---- top-p: softmax (max = the first candidate, whatever order typical left), cumulative sum, cut
        if (p.top_p < 1.0f) {
            block_softmax(S.cl, S.cp, n, s_f, !reordered);
            if (tid == 0) {
                float cum = 0.f; int last = n;
                for (int i = 0; i < n; i++) {
                    cum = __fadd_rn(cum, S.cp[i]);
                    if (cum > p.top_p && i >= 1) { last = i; break; }
                }
                s_i[1] = last;
            }
            __syncthreads();
            n = s_i[1];
            __syncthreads();
            if (tap) tap_list(tap, n_vocab, TAP_TOP_P, n, S.cid, S.cl, S.cp, nullptr);
        }
        for (int i = tid; i < n; i += NT) S.cl[i] = __fdiv_rn(S.cl[i], p.temp);       // llama_sample_temperature
        __syncthreads();
        if (tap) tap_list(tap, n_vocab, TAP_TEMP, n, S.cid, S.cl, nullptr, nullptr);
    }
    if (!greedy) {
        // ---- llama_sample_token: softmax, discrete_distribution(probs)(rng); mirostat then updates mu from the drawn p
        if (n >= 2) block_softmax(S.cl, S.cp, n, s_f, !reordered);
        else if (tid == 0) S.cp[0] = 1.0f;                             // the softmax of one candidate
        __syncthreads();
        pick = block_draw(S.cp, n, st, s_d, s_i);
        if (tid == 0 && p.mirostat != 0) {
            const float e = __fsub_rn(-ref_log2f(S.cp[pick]), p.mirostat_tau);
            st->mu = fmaf(-p.mirostat_eta, e, st->mu);
        }
        if (tap && tid == 0 && n >= 2) ((TapHead *) tap)->u = s_d[NT];
    } else if (tid == 0) S.cp[0] = 1.0f;
    if (tap) {
        __syncthreads();
        tap_list(tap, n_vocab, TAP_FINAL, n, S.cid, S.cl, S.cp, nullptr);
        if (tid == 0) { TapHead * h = (TapHead *) tap; h->pick = pick; h->id = S.cid[pick]; h->mu = st->mu; }
    }
    if (tid != 0) return;
    const int id = S.cid[pick];
    *out = id;
    if (hist) { const int s = *step; hist[s] = id; *step = s + 1; }
    if (st->wcap > 0) {                                                // the window slides: drop the oldest id, append the new one
        if (st->wlen < st->wcap) st->window[st->wlen++] = id;
        else { for (int i = 1; i < st->wcap; i++) st->window[i - 1] = st->window[i]; st->window[st->wcap - 1] = id; }
    }
}

} // namespace

SamplerState * sampler_state_alloc() { SamplerState * s = nullptr; B200_CUDA_CHECK(cudaMalloc(&s, sizeof(SamplerState))); return s; }
void sampler_state_free(SamplerState * s) { if (s) B200_CUDA_CHECK(cudaFree(s)); }
size_t sampler_work_floats(int n_vocab) { return 9 * (size_t) n_vocab; }
size_t sampler_tap_bytes(int n_vocab) { return 4 * (TAP_HEAD_FLOATS + (1 + 3 * (size_t) TAP_STAGES) * n_vocab); }
// one stage of the tap (see tap_list) copied to the host; returns false for an unknown stage / field or a wrong size
bool sampler_tap_read(const float * tap, int n_vocab, const char * stage, const char * field, void * host, size_t bytes) {
    static const char * names[TAP_STAGES] = { "order", "tfs", "typical", "top_p", "temp", "final" };
    TapHead h;
    B200_CUDA_CHECK(cudaMemcpy(&h, tap, sizeof(h), cudaMemcpyDeviceToHost));
    auto scalar = [&](const void * v, size_t sz) { if (bytes != sz) return false; memcpy(host, v, sz); return true; };
    if (!strcmp(stage, "row")) {
        if (strcmp(field, "logits") || bytes != (size_t) n_vocab * 4) return false;
        B200_CUDA_CHECK(cudaMemcpy(host, tap + TAP_HEAD_FLOATS, bytes, cudaMemcpyDeviceToHost));
        return true;
    }
    int s = 0;
    while (s < TAP_STAGES && strcmp(stage, names[s])) s++;
    if (s == TAP_STAGES) return false;
    if (!strcmp(field, "n")) return scalar(&h.n[s], 4);
    if (s == TAP_TYPICAL && !strcmp(field, "entropy")) return scalar(&h.entropy, 4);
    if (s == TAP_FINAL) {
        if (!strcmp(field, "u")) return scalar(&h.u, 8);
        if (!strcmp(field, "pick")) return scalar(&h.pick, 4);
        if (!strcmp(field, "id")) return scalar(&h.id, 4);
        if (!strcmp(field, "mu")) return scalar(&h.mu, 4);
        if (!strcmp(field, "k")) return scalar(&h.k, 4);
    }
    const int arr = !strcmp(field, "ids") ? 0 : !strcmp(field, "logits") ? 1 : !strcmp(field, "p") ? 2 : -1;
    if (arr < 0 || (arr == 2 && (s == TAP_ORDER || s == TAP_TEMP)) || h.n[s] < 0 || bytes != (size_t) h.n[s] * 4) return false;
    B200_CUDA_CHECK(cudaMemcpy(host, tap + TAP_HEAD_FLOATS + n_vocab + (size_t) (3 * s + arr) * n_vocab, bytes, cudaMemcpyDeviceToHost));
    return true;
}
float sampler_mu(const SamplerState * s) {
    float mu = 0.f;
    B200_CUDA_CHECK(cudaMemcpy(&mu, &s->mu, 4, cudaMemcpyDeviceToHost));
    return mu;
}
// window: the n most recent token ids (oldest first) the penalties start from; at most `cap` (= repeat_last_n) are kept
void launch_sampler_init(SamplerState * s, uint32_t seed, const int32_t * window_dev, int n, int cap, float mu, cudaStream_t stream) {
    B200_ASSERT(cap >= 0 && cap <= B200_SAMPLER_MAX_WINDOW);
    sampler_init_kernel<<<1, 1, 0, stream>>>(s, seed, window_dev, n, cap, mu);
    B200_CUDA_CHECK(cudaGetLastError());
}
void launch_sample(const float * logits, int n_vocab, const SamplerParams & p, SamplerState * st, float * work, int32_t * out, int32_t * hist, int * step,
                   float * tap, cudaStream_t stream) {
    B200_ASSERT(p.mirostat >= 0 && p.mirostat <= 2 && p.n_bias >= 0 && p.n_bias <= B200_SAMPLER_MAX_BIAS);
    sample_kernel<<<1, NT, 0, stream>>>(logits, n_vocab, p, st, work, out, hist, step, tap);
    B200_CUDA_CHECK(cudaGetLastError());
}
