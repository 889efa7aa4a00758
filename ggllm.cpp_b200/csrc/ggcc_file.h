// ggcc_file.h -- the one reader of the GGCC v10 format (libfalcon.cpp:770-973), shared by the engine's loader (engine.cu) and the file
// quantiser (quantize_file.cu): header, vocab, merges, then per tensor {n_dims, name_len, type, ne[], name, pad to 32 B, data}.
// The file is untrusted input: every read is bounds-checked and sets `bad` instead of reading past the end.
#pragma once
#include <cstdint>
#include <cstring>
#include <string>
#include "formats.cuh"

struct Cursor { const uint8_t * p; size_t off, size; bool bad;
    uint32_t u32() { if (off + 4 > size) { bad = true; return 0; } uint32_t v; memcpy(&v, p + off, 4); off += 4; return v; }
    void skip(size_t n) { if (n > size - off) bad = true; else off += n; } };

struct GgccHeader { uint32_t n_vocab, n_embd, n_head, n_head_kv, n_layer, falcon_type, ftype, n_bpe_merges; };

// magic, version and the eight hparam words; false for another format or a short file
static inline bool ggcc_read_header(Cursor & c, GgccHeader & h) {
    if (c.u32() != 0x67676363u || c.u32() != 10u || c.bad) return false;
    uint32_t * w = &h.n_vocab;
    for (int i = 0; i < 8; i++) w[i] = c.u32();
    return !c.bad;
}

// steps over the vocabulary and the merges (n_merges, optional: the merges' own count word); false if the file ends inside them
static inline bool ggcc_skip_vocab(Cursor & c, const GgccHeader & h, uint32_t * n_merges = nullptr) {
    for (uint32_t i = 0; i < h.n_vocab && !c.bad; i++) { const uint32_t len = c.u32(); c.skip((size_t) len + 4); }
    const uint32_t nm = c.u32();
    for (uint32_t i = 0; i < 2 * nm && !c.bad; i++) { const uint32_t len = c.u32(); c.skip(len); }
    if (n_merges) *n_merges = nm;
    return !c.bad;
}

struct GgccTensor {
    std::string name;
    uint32_t n_dims, type;
    int64_t ne[2];                   // ne[1] == 1 for a 1-D tensor
    const uint8_t * data;
    size_t nbytes, row_bytes;
};

// the next tensor's header and data extent: 1 and the cursor past its data, 0 at the end of the file, -1 (why set) for a malformed one
static inline int ggcc_next_tensor(Cursor & c, GgccTensor & t, const char ** why) {
    if (c.off >= c.size) return 0;
    t.n_dims = c.u32(); const uint32_t name_len = c.u32(); t.type = c.u32();
    if (c.bad || t.n_dims < 1 || t.n_dims > 2 || name_len > 256) { *why = "malformed tensor header"; return -1; }
    t.ne[0] = t.ne[1] = 1;
    for (uint32_t d = 0; d < t.n_dims; d++) t.ne[d] = c.u32();
    if (c.bad || name_len > c.size - c.off) { *why = "truncated tensor header"; return -1; }
    t.name.assign((const char *) c.p + c.off, name_len); c.off += name_len;
    c.skip((size_t) (-(int64_t) c.off & 31));
    const TypeSpec ts = type_spec((int) t.type);
    if (c.bad || ts.blk_elems <= 0 || t.ne[0] <= 0 || t.ne[1] <= 0 || t.ne[0] % ts.blk_elems != 0) { *why = "bad tensor type / shape"; return -1; }
    t.row_bytes = (size_t) (t.ne[0] / ts.blk_elems) * ts.blk_bytes; t.nbytes = t.row_bytes * (size_t) t.ne[1];
    if (t.nbytes > c.size - c.off) { *why = "tensor data runs past the end of the file"; return -1; }
    t.data = c.p + c.off;
    c.off += t.nbytes;
    return 1;
}
