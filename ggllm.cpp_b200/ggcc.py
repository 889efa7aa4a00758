"""GGCC v10 model-file reader / writer (host-side tool, numpy only).

The file format is the reference's (libfalcon.cpp:770-973 reader, 975-1052 writer):
  u32 magic 'ggcc' (0x67676363), u32 version 10                                   (libfalcon.h:36, libfalcon.cpp:813-818)
  u32 n_vocab, n_embd, n_head, n_head_kv, n_layer, n_falcon_type(7|40), ftype, n_bpe_merges   (libfalcon.cpp:826-845)
  n_vocab x { u32 len, bytes, f32 score }                                         (libfalcon.cpp:846-861)
  u32 n_merges, n_merges x { u32 len, bytes, u32 len, bytes }                     (libfalcon.cpp:869-881)
  until EOF: { u32 n_dims(1|2), u32 name_len, u32 ggml_type, u32 ne[n_dims], name, pad to 32 B, raw data }  (libfalcon.cpp:920-972)

Tensor names and shapes are those the reference loader asks for (libfalcon.cpp:1764, 1793-1796, 1847-1861).
Used to create the synthetic random-init models of BASELINE.json's configs and to feed the same bytes to
the reference (falcon_init_from_file) and to this backend (b200_falcon_* / ggml_cuda_transform_tensor).
"""
import struct
import numpy as np

GGCC_MAGIC = 0x67676363
GGCC_VERSION = 10

# enum ggml_type (ggml.h:241-262) -> (elements per block, bytes per block)
BLOCK = {0: (1, 4), 1: (1, 2), 2: (32, 18), 3: (32, 20), 6: (32, 22), 7: (32, 24), 8: (32, 34),
         10: (256, 84), 11: (256, 110), 12: (256, 144), 13: (256, 176), 14: (256, 210)}
TYPE_ID = {"f32": 0, "f16": 1, "q4_0": 2, "q4_1": 3, "q5_0": 6, "q5_1": 7, "q8_0": 8,
           "q2_K": 10, "q3_K": 11, "q4_K": 12, "q5_K": 13, "q6_K": 14}
TYPE_NAME = {v: k for k, v in TYPE_ID.items()}
# enum llama_ftype (libfalcon.h:112-131) for a uniformly quantised file of a given ggml type
FTYPE_OF_TYPE = {0: 0, 1: 1, 2: 2, 3: 3, 8: 7, 6: 8, 7: 9, 10: 10, 11: 12, 12: 15, 13: 17, 14: 18}


def tensor_nbytes(ggml_type, ne):
    per, bsz = BLOCK[ggml_type]
    n = int(np.prod(ne))
    assert ne[0] % per == 0, "row length must be a multiple of the block size"
    return n // per * bsz


def falcon_shapes(hp):
    """{tensor name: ne} for a Falcon model with hparams `hp` (libfalcon.cpp:1764-1861)."""
    E, H, HKV, L, V = hp["n_embd"], hp["n_head"], hp["n_head_kv"], hp["n_layer"], hp["n_vocab"]
    D = E // H
    out = {"transformer.word_embeddings.weight": (E, V)}
    for i in range(L):
        p = "transformer.h.%d." % i
        if hp["falcon_type"] == 40:
            for n in ("ln_mlp", "ln_attn"):
                out[p + n + ".weight"] = (E,)
                out[p + n + ".bias"] = (E,)
        else:
            out[p + "input_layernorm.weight"] = (E,)
            out[p + "input_layernorm.bias"] = (E,)
        out[p + "self_attention.query_key_value.weight"] = (E, (H + 2 * HKV) * D)
        out[p + "self_attention.dense.weight"] = (E, E)
        out[p + "mlp.dense_h_to_4h.weight"] = (E, 4 * E)
        out[p + "mlp.dense_4h_to_h.weight"] = (4 * E, E)
    out["transformer.ln_f.weight"] = (E,)
    out["transformer.ln_f.bias"] = (E,)
    out["lm_head.weight"] = (E, V)
    return out


def write_ggcc(path, hp, tensors, ftype=0):
    """tensors: {name: (ggml_type, ne tuple, ndarray holding the raw bytes / f32 values)} in file order."""
    with open(path, "wb") as f:
        f.write(struct.pack("<II", GGCC_MAGIC, GGCC_VERSION))
        f.write(struct.pack("<8I", hp["n_vocab"], hp["n_embd"], hp["n_head"], hp["n_head_kv"], hp["n_layer"],
                            hp["falcon_type"], ftype, 0))
        for i in range(hp["n_vocab"]):
            w = ("<t%d>" % i).encode()
            f.write(struct.pack("<I", len(w)))
            f.write(w)
            f.write(struct.pack("<f", 0.0))
        f.write(struct.pack("<I", 0))  # no BPE merges (accepted by the reader, libfalcon.cpp:869-881)
        for name, (t, ne, arr) in tensors.items():
            nb = name.encode()
            f.write(struct.pack("<III", len(ne), len(nb), t))
            f.write(struct.pack("<%dI" % len(ne), *ne))
            f.write(nb)
            f.write(b"\0" * (-f.tell() & 31))
            raw = np.ascontiguousarray(arr).view(np.uint8).reshape(-1)
            assert raw.size == tensor_nbytes(t, ne), (name, raw.size, tensor_nbytes(t, ne))
            raw.tofile(f)
    return path


def read_ggcc(path, mmap=True):
    """-> (hparams, {name: (ggml_type, ne, uint8 ndarray view of the raw data)})"""
    buf = np.memmap(path, dtype=np.uint8, mode="r") if mmap else np.fromfile(path, dtype=np.uint8)
    mv = memoryview(buf)
    off = 0

    def u32():
        nonlocal off
        v = struct.unpack_from("<I", mv, off)[0]
        off += 4
        return v

    magic, version = u32(), u32()
    if magic != GGCC_MAGIC or version != GGCC_VERSION:
        raise ValueError("not a GGCC v10 file: magic %08x version %d" % (magic, version))
    keys = ("n_vocab", "n_embd", "n_head", "n_head_kv", "n_layer", "falcon_type", "ftype", "n_bpe_merges")
    hp = {k: u32() for k in keys}
    for _ in range(hp["n_vocab"]):
        n = u32()
        off += n + 4          # token bytes + f32 score
    for _ in range(u32()):
        for _half in range(2):
            n = u32()
            off += n
    tensors = {}
    size = buf.size
    while off < size:
        n_dims, name_len, t = u32(), u32(), u32()
        ne = tuple(u32() for _ in range(n_dims))
        name = bytes(mv[off:off + name_len]).decode()
        off += name_len
        off += -off & 31
        nbytes = tensor_nbytes(t, ne)
        tensors[name] = (t, ne, buf[off:off + nbytes])
        off += nbytes
    return hp, tensors


def random_blocks(ggml_type, n_rows, k, rng):
    """n_rows x k weights as well-formed pseudo-random blocks of `ggml_type` (uniform quant bytes, sane fp16 scales), drawn from
    numpy's `rng`, for files the reference has to load (SURVEY.md section 8d).  Not the device's bytes: b200_weight_random hashes
    its blocks with mix32, its F16 / F32 values lie in [0, 0.04) rather than 0.02 N(0, 1), and its Q4_1 / Q5_1 mins are 4 d;
    tests/device_random.py is the byte-for-byte twin of those."""
    per, bsz = BLOCK[ggml_type]
    nb = n_rows * (k // per)
    if ggml_type == 0:
        return (0.02 * rng.standard_normal((n_rows, k))).astype(np.float32)
    if ggml_type == 1:
        return (0.02 * rng.standard_normal((n_rows, k))).astype(np.float16)
    raw = rng.integers(0, 256, size=(nb, bsz), dtype=np.uint8)
    unit = 1e-4 if per == 256 else 2e-3
    d = (unit * (1.0 + 2.0 * rng.random(nb))).astype(np.float16).view(np.uint16)
    lo, hi = (d & 0xff).astype(np.uint8), (d >> 8).astype(np.uint8)
    # byte offsets of the fp16 scale fields inside one block (ggml.c:879-916, k_quants.h:20-74)
    offs = {2: [0], 3: [0, 2], 6: [0], 7: [0, 2], 8: [0], 10: [80, 82], 11: [108], 12: [0, 2], 13: [0, 2], 14: [208]}[ggml_type]
    for o in offs:
        raw[:, o], raw[:, o + 1] = lo, hi
    return raw.reshape(n_rows, -1)
