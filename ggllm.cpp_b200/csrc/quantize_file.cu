// quantize_file.cu -- falcon_quantize on the device: b200_quantize_ggcc (include/ggml_b200.h), the file-level driver of
// falcon_model_quantize_internal (libfalcon.cpp:3533-3743) around the device quantisers of quant_gpu.cu.
//
// The output is byte for byte the reference's: the header with the new ftype, the vocabulary and merges as llama_file_saver writes
// them back (libfalcon.cpp:975-1052), then every tensor in input order, quantised or copied by the reference's rules.  Tensor names
// are not engine slots here: any GGCC file is quantised by its names and shapes alone.
//
// Pipeline (one host thread, two streams).  For each tensor to quantise, in order:
//   read    mapped file -> one of N_STAGE pinned staging buffers -> H2D on s_in -> planar repack (weights.cu) into input slot k
//           (F32 / F16 input: straight into slot k); the host waits only for the staging buffer it reuses
//   convert on s_q, once slot k is complete, into the fp32 buffer: F16 widened, quantised types through dequant_rows (both bit-exact
//           with llama_convert_tensor_internal); F32 input is quantised from slot k itself
//   quantise launch_quantize_chunks on the chunk plan, then D2H of the blocks and the histogram into pinned output buffer k
//   write   the previous tensor's header and data, once its D2H is complete
// so the host reads tensor i + 1 while the device converts and quantises tensor i, and writes tensor i while it runs tensor i + 1.
// Input slots alternate (k = i % 2); s_in waits before refilling a slot until s_q has consumed it.  Device memory is sized from the
// file: two input slots of the largest quantised tensor as stored (quantised inputs in the planar layout), one fp32 buffer and one
// output buffer.
#include "kernels.h"
#include "ggcc_file.h"
#include "../../include/ggml_b200.h"
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <set>
#include <thread>
#include <vector>

namespace {

// ggml_fp16_to_fp32_row (exact widening, NaN payloads kept as __half2float keeps them)
__global__ void f16_to_f32_kernel(const __half * __restrict__ x, float * __restrict__ y, int64_t n) {
    for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) y[i] = __half2float(x[i]);
}
void launch_f16_to_f32(const __half * x, float * y, int64_t n, cudaStream_t s) {
    f16_to_f32_kernel<<<ew_grid(n), 256, 0, s>>>(x, y, n);
    B200_CUDA_CHECK(cudaGetLastError());
}

constexpr size_t STAGE_BYTES = 8u << 20;          // one pinned staging buffer
constexpr int N_STAGE = 4;
constexpr int64_t CHUNK = 32 * 512;               // falcon_model_quantize_internal's chunk_size

// enum llama_ftype -> the one ggml type every quantised tensor gets (libfalcon.cpp:3538-3560); -1: the reference throws
int ftype_to_type(int ftype) {
    switch (ftype) {
        case 0: return T_F32; case 1: return T_F16; case 2: return T_Q4_0; case 3: return T_Q4_1; case 7: return T_Q8_0;
        case 8: return T_Q5_0; case 9: return T_Q5_1; case 10: return T_Q2_K; case 11: case 12: case 13: return T_Q3_K;
        case 14: case 15: return T_Q4_K; case 16: case 17: return T_Q5_K; case 18: return T_Q6_K;
    }
    return -1;
}

struct Job {
    GgccTensor t;
    bool quantize;
    int new_type;
    int64_t n, chunk;           // values, chunk_elems of the plan
    size_t in_bytes;            // input slot bytes: planar layout, or the raw f32 values
    size_t out_bytes;
};

double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

struct Resources {
    void * map = MAP_FAILED; size_t map_size = 0;
    FILE * out = nullptr;
    cudaStream_t s_in = nullptr, s_q = nullptr;
    uint8_t * in_dev[2] = {}, * out_dev = nullptr, * stage_dev[N_STAGE] = {}, * stage_pin[N_STAGE] = {}, * out_pin[2] = {};
    float * f32_dev = nullptr;
    unsigned long long * hist_dev = nullptr, * hist_pin = nullptr;
    cudaEvent_t ev_stage[N_STAGE] = {}, ev_consumed[2] = {}, ev_done[2] = {}, ev_uploaded = nullptr;
    ~Resources() {
        if (s_in) cudaStreamSynchronize(s_in);
        if (s_q) cudaStreamSynchronize(s_q);
        for (int k = 0; k < 2; k++) { cudaFree(in_dev[k]); cudaFreeHost(out_pin[k]); if (ev_consumed[k]) cudaEventDestroy(ev_consumed[k]); if (ev_done[k]) cudaEventDestroy(ev_done[k]); }
        for (int j = 0; j < N_STAGE; j++) { cudaFree(stage_dev[j]); cudaFreeHost(stage_pin[j]); if (ev_stage[j]) cudaEventDestroy(ev_stage[j]); }
        cudaFree(out_dev); cudaFree(f32_dev); cudaFree(hist_dev); cudaFreeHost(hist_pin);
        if (ev_uploaded) cudaEventDestroy(ev_uploaded);
        if (s_in) cudaStreamDestroy(s_in);
        if (s_q) cudaStreamDestroy(s_q);
        if (out) fclose(out);
        if (map != MAP_FAILED) munmap(map, map_size);
    }
};

bool put(FILE * f, const void * p, size_t n, size_t & pos) { pos += n; return n == 0 || fwrite(p, 1, n, f) == n; }
bool put32(FILE * f, uint32_t v, size_t & pos) { return put(f, &v, 4, pos); }

// the planes of one input slot holding `t` (F16 / quantised input), rebased onto the slot
WPlanes slot_planes(const GgccTensor & t, uint8_t * base) {
    WPlanes W;
    wplanes_layout(W, (int) t.type, (int) t.ne[0], (int) t.ne[1]);
    for (int i = 0; i < type_spec((int) t.type).n_planes; i++) W.p[i] = base + reinterpret_cast<size_t>(W.p[i]);
    return W;
}

} // namespace

extern "C" int b200_quantize_ggcc(const char * path_in, const char * path_out, const b200_quantize_params * p, b200_quantize_report * rep) {
    const double t_start = now_s();
    if (!p) return -1;
    const int qtype = ftype_to_type(p->ftype);
    if (qtype < 0) { fprintf(stderr, "b200_quantize_ggcc: invalid output file type %d\n", p->ftype); return 1; }
    int nthread = p->nthread;
    if (nthread <= 0) nthread = (int) std::thread::hardware_concurrency();

    Resources R;
    {
        const int fd = open(path_in, O_RDONLY);
        if (fd < 0) { fprintf(stderr, "b200_quantize_ggcc: cannot open %s\n", path_in); return -1; }
        struct stat sb;
        if (fstat(fd, &sb) != 0 || sb.st_size < 40) { close(fd); return -1; }
        R.map_size = (size_t) sb.st_size;
        R.map = mmap(nullptr, R.map_size, PROT_READ, MAP_PRIVATE, fd, 0);
        close(fd);
        if (R.map == MAP_FAILED) return -1;
    }
    auto malformed = [&](const char * why) { fprintf(stderr, "b200_quantize_ggcc: %s: %s\n", path_in, why); return -1; };

    // ---- header, vocabulary, merges: what llama_file_saver writes back
    const uint8_t * base = (const uint8_t *) R.map;
    Cursor c = { base, 0, R.map_size, false };
    GgccHeader h;
    if (!ggcc_read_header(c, h)) return malformed("not a GGCC v10 file");
    const size_t vocab_at = c.off;
    size_t vocab_end = 0;                              // end of the tokens written back
    uint32_t n_vocab_out = h.n_vocab;
    for (uint32_t i = 0; i < h.n_vocab && !c.bad; i++) {
        const size_t tok_at = c.off;
        const uint32_t len = c.u32();
        const bool pad = i == 65024 && h.n_vocab == 65025 && len == 5 && !c.bad && c.size - c.off >= 5 && memcmp(base + c.off, "[PAD]", 5) == 0;
        c.skip((size_t) len + 4);
        if (pad) { n_vocab_out = 65024; vocab_end = tok_at; }      // the reference's "wizard hack" (libfalcon.cpp:863-868): token 65024 dropped
    }
    if (!vocab_end) vocab_end = c.off;
    const uint32_t n_merges = c.u32();
    const size_t merges_at = c.off;
    size_t merges_end = h.n_bpe_merges == 0 ? merges_at : 0;
    for (uint32_t i = 0; i < n_merges && !c.bad; i++) {
        for (int half = 0; half < 2; half++) { const uint32_t len = c.u32(); c.skip(len); }
        if (i + 1 == h.n_bpe_merges) merges_end = c.off;
    }
    if (c.bad) return malformed("truncated vocabulary");
    if (h.n_bpe_merges > n_merges) return malformed("the header counts more merges than the file holds");

    // ---- the tensor directory and the reference's decisions, before anything is written
    std::vector<Job> jobs;
    std::set<std::string> names;
    size_t in_max = 0, f32_max = 0, out_max = 0, out_host_max = 0;
    for (;;) {
        Job j{}; const char * why = nullptr;
        const int got = ggcc_next_tensor(c, j.t, &why);
        if (got < 0) return malformed(why);
        if (got == 0) break;
        if (!names.insert(j.t.name).second) return malformed("duplicate tensor name");
        const std::string & name = j.t.name;
        bool q = name.rfind("weight") == name.size() - 6;             // libfalcon.cpp:3606-3611, verbatim
        q &= j.t.n_dims == 2;
        q &= p->quantize_output_tensor != 0 || name != "lm_head.weight";
        q &= (int) j.t.type != qtype;
        j.quantize = q;
        j.new_type = q ? qtype : (int) j.t.type;
        j.n = j.t.ne[0] * j.t.ne[1];
        if (q) {
            if (qtype >= T_Q2_K && qtype <= T_Q6_K && j.t.ne[0] % 256 != 0) {
                fprintf(stderr, "b200_quantize_ggcc: tensor %s: %lld values per row are not a multiple of 256, required by k-quants\n", name.c_str(), (long long) j.t.ne[0]);
                return 1;
            }
            if (j.t.type != T_F32 && j.t.type != T_F16 && !p->allow_requantize) {
                fprintf(stderr, "b200_quantize_ggcc: tensor %s: requantizing is disabled\n", name.c_str());
                return 1;
            }
            if (qtype != T_F32 && qtype != T_F16 && j.t.ne[0] % 32 != 0) return malformed("a row the output type cannot hold");
            if (j.t.ne[0] > INT32_MAX || j.t.ne[1] > INT32_MAX || j.n > INT32_MAX) return malformed("tensor too large for the reference's int sizes");
            const int64_t nchunk = (j.n + CHUNK - 1) / CHUNK;
            const int nthread_use = nthread > 1 ? (int) std::max<int64_t>(1, std::min<int64_t>(nthread, nchunk)) : 1;
            j.chunk = nthread_use < 2 ? j.n : CHUNK;
            if (j.t.type == T_F32 || j.t.type == T_F16) j.in_bytes = j.t.nbytes;
            else {
                WPlanes W; j.in_bytes = wplanes_layout(W, (int) j.t.type, (int) j.t.ne[0], (int) j.t.ne[1]);
                if (j.t.row_bytes > STAGE_BYTES) return malformed("a row does not fit a staging buffer");
            }
            if (j.t.type != T_F32) f32_max = std::max(f32_max, (size_t) j.n * 4);
            const TypeSpec ts = type_spec(qtype);
            j.out_bytes = (size_t) (j.t.ne[0] / ts.blk_elems) * ts.blk_bytes * (size_t) j.t.ne[1];
            in_max = std::max(in_max, j.in_bytes);
            if (qtype != T_F32) out_max = std::max(out_max, j.out_bytes);
            out_host_max = std::max(out_host_max, j.out_bytes);
        } else j.out_bytes = j.t.nbytes;
        jobs.push_back(std::move(j));
    }

    // ---- device and pinned buffers
    B200_CUDA_CHECK(cudaStreamCreateWithFlags(&R.s_in, cudaStreamNonBlocking));
    B200_CUDA_CHECK(cudaStreamCreateWithFlags(&R.s_q, cudaStreamNonBlocking));
    size_t dev_bytes = 0;
    auto dmalloc = [&](void ** ptr, size_t n) { if (n) { B200_CUDA_CHECK(cudaMalloc(ptr, n)); dev_bytes += n; } };
    for (int k = 0; k < 2; k++) {
        dmalloc((void **) &R.in_dev[k], in_max);
        if (out_host_max) B200_CUDA_CHECK(cudaMallocHost((void **) &R.out_pin[k], out_host_max));
        B200_CUDA_CHECK(cudaEventCreateWithFlags(&R.ev_consumed[k], cudaEventDisableTiming));
        B200_CUDA_CHECK(cudaEventCreateWithFlags(&R.ev_done[k], cudaEventDisableTiming));
    }
    for (int s = 0; s < N_STAGE; s++) {
        dmalloc((void **) &R.stage_dev[s], STAGE_BYTES);
        B200_CUDA_CHECK(cudaMallocHost((void **) &R.stage_pin[s], STAGE_BYTES));
        B200_CUDA_CHECK(cudaEventCreateWithFlags(&R.ev_stage[s], cudaEventDisableTiming));
    }
    B200_CUDA_CHECK(cudaEventCreateWithFlags(&R.ev_uploaded, cudaEventDisableTiming));
    dmalloc((void **) &R.f32_dev, f32_max);
    dmalloc((void **) &R.out_dev, out_max);
    dmalloc((void **) &R.hist_dev, 2 * 16 * sizeof(unsigned long long));
    B200_CUDA_CHECK(cudaMallocHost((void **) &R.hist_pin, 2 * 16 * sizeof(unsigned long long)));

    R.out = fopen(path_out, "wb");
    if (!R.out) { fprintf(stderr, "b200_quantize_ggcc: cannot create %s\n", path_out); return -1; }
    setvbuf(R.out, nullptr, _IOFBF, 1u << 20);
    size_t pos = 0;
    bool ok = true;
    const uint32_t hdr[10] = { 0x67676363u, 10u, n_vocab_out, h.n_embd, h.n_head, h.n_head_kv, h.n_layer, h.falcon_type, (uint32_t) p->ftype, h.n_bpe_merges };
    ok &= put(R.out, hdr, sizeof(hdr), pos);
    ok &= put(R.out, base + vocab_at, vocab_end - vocab_at, pos);
    ok &= put32(R.out, h.n_bpe_merges, pos);
    ok &= put(R.out, base + merges_at, merges_end - merges_at, pos);

    b200_quantize_report rp{};
    auto write_tensor = [&](const Job & j, const void * data) {
        const uint32_t th[3] = { j.t.n_dims, (uint32_t) j.t.name.size(), (uint32_t) j.new_type };
        ok &= put(R.out, th, sizeof(th), pos);
        for (uint32_t d = 0; d < j.t.n_dims; d++) ok &= put32(R.out, (uint32_t) j.t.ne[d], pos);
        ok &= put(R.out, j.t.name.data(), j.t.name.size(), pos);
        static const uint8_t zeros[32] = {};
        ok &= put(R.out, zeros, (size_t) (-(int64_t) pos & 31), pos);
        ok &= put(R.out, data, j.out_bytes, pos);
        rp.size_org += j.t.nbytes; rp.size_new += j.out_bytes; rp.n_tensors++;
    };
    int pending = -1, pending_k = 0;                   // the quantised tensor whose result is still on its way back
    auto flush = [&]() {
        if (pending < 0) return;
        B200_CUDA_CHECK(cudaEventSynchronize(R.ev_done[pending_k]));
        for (int i = 0; i < 16; i++) rp.hist[i] += (int64_t) R.hist_pin[16 * pending_k + i];
        write_tensor(jobs[pending], R.out_pin[pending_k]);
        rp.n_quantized++;
        pending = -1;
    };

    bool slot_used[2] = {}, stage_used[N_STAGE] = {};
    int stage_next = 0, k = 0;
    for (size_t i = 0; i < jobs.size() && ok; i++) {
        const Job & j = jobs[i];
        if (!j.quantize) { flush(); write_tensor(j, j.t.data); continue; }
        // read: mapped file -> pinned staging -> slot k
        if (slot_used[k]) B200_CUDA_CHECK(cudaStreamWaitEvent(R.s_in, R.ev_consumed[k], 0));
        const bool f32_in = j.t.type == T_F32, raw = f32_in || j.t.type == T_F16;      // stored as they are in the file
        WPlanes W{};
        if (!raw) W = slot_planes(j.t, R.in_dev[k]);
        // pieces of at most STAGE_BYTES: whole rows for the repack, any bytes for f32 / f16 values
        const size_t piece = raw ? STAGE_BYTES : STAGE_BYTES / j.t.row_bytes * j.t.row_bytes;
        for (size_t off = 0; off < j.t.nbytes; off += piece) {
            const size_t nb = std::min(piece, j.t.nbytes - off);
            const int s = stage_next; stage_next = (stage_next + 1) % N_STAGE;
            if (stage_used[s]) B200_CUDA_CHECK(cudaEventSynchronize(R.ev_stage[s]));      // its H2D (and repack) are done
            memcpy(R.stage_pin[s], j.t.data + off, nb);
            if (raw) B200_CUDA_CHECK(cudaMemcpyAsync(R.in_dev[k] + off, R.stage_pin[s], nb, cudaMemcpyHostToDevice, R.s_in));
            else {
                B200_CUDA_CHECK(cudaMemcpyAsync(R.stage_dev[s], R.stage_pin[s], nb, cudaMemcpyHostToDevice, R.s_in));
                launch_repack_rows(W, R.stage_dev[s], (int64_t) (off / j.t.row_bytes), (int64_t) (nb / j.t.row_bytes), R.s_in);
            }
            B200_CUDA_CHECK(cudaEventRecord(R.ev_stage[s], R.s_in)); stage_used[s] = true;
        }
        B200_CUDA_CHECK(cudaEventRecord(R.ev_uploaded, R.s_in));
        B200_CUDA_CHECK(cudaStreamWaitEvent(R.s_q, R.ev_uploaded, 0));
        // convert and quantise on s_q
        const float * x = (const float *) R.in_dev[k];
        if (j.t.type == T_F16) {
            launch_f16_to_f32(reinterpret_cast<const __half *>(R.in_dev[k]), R.f32_dev, j.n, R.s_q);
            x = R.f32_dev;
        } else if (!f32_in) {
            for (int64_t r0 = 0; r0 < j.t.ne[1]; r0 += 65535) {               // the dequant grid's y extent
                WPlanes Wr = W;
                const int nr = (int) std::min<int64_t>(65535, j.t.ne[1] - r0);
                for (int pl = 0; pl < type_spec(W.type).n_planes; pl++) Wr.p[pl] = W.p[pl] + (size_t) r0 * W.stride[pl];
                Wr.M = nr;
                launch_dequant_rows(Wr, nullptr, nr, R.f32_dev + r0 * j.t.ne[0], j.t.ne[0], R.s_q);
            }
            x = R.f32_dev;
        }
        unsigned long long * hd = R.hist_dev + 16 * k;
        B200_CUDA_CHECK(cudaMemsetAsync(hd, 0, 16 * sizeof(unsigned long long), R.s_q));
        if (j.new_type == T_F32) {                                           // ggml_quantize_chunk's memcpy
            B200_CUDA_CHECK(cudaEventRecord(R.ev_consumed[k], R.s_q));
            B200_CUDA_CHECK(cudaMemcpyAsync(R.out_pin[k], x, j.out_bytes, cudaMemcpyDeviceToHost, R.s_q));
        } else {
            const int64_t got = launch_quantize_chunks(j.new_type, x, R.out_dev, j.n, j.chunk, hd, R.s_q);
            B200_ASSERT(got == (int64_t) j.out_bytes);
            B200_CUDA_CHECK(cudaEventRecord(R.ev_consumed[k], R.s_q));
            B200_CUDA_CHECK(cudaMemcpyAsync(R.out_pin[k], R.out_dev, j.out_bytes, cudaMemcpyDeviceToHost, R.s_q));
        }
        B200_CUDA_CHECK(cudaMemcpyAsync(R.hist_pin + 16 * k, hd, 16 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, R.s_q));
        B200_CUDA_CHECK(cudaEventRecord(R.ev_done[k], R.s_q));
        slot_used[k] = true;
        // write the previous tensor while this one runs
        flush();
        pending = (int) i; pending_k = k; k ^= 1;
    }
    flush();
    ok &= fflush(R.out) == 0;
    ok &= fclose(R.out) == 0; R.out = nullptr;
    if (!ok) { fprintf(stderr, "b200_quantize_ggcc: write error on %s\n", path_out); return -1; }
    rp.seconds = now_s() - t_start;
    rp.staging_bytes = STAGE_BYTES;
    rp.device_bytes = dev_bytes;
    if (rep) *rep = rp;
    return 0;
}
