"""A restatement of falcon_quantize (falcon_model_quantize_internal, libfalcon.cpp:3533-3743) in Python over the oracle's codecs:
the output file it writes, the per-tensor and total 16-bin histograms and the byte totals.  The tests hold it to the reference's
own file (falcon_model_quantize from oracle/_ref, called through ctypes) and the device's b200_quantize_ggcc to it.

Chunk plan: nthread <= 0 is the host's CPU count; nchunk = ceil(n / 16384); nthread_use = min(nthread, nchunk) if nthread > 1,
else 1; with nthread_use < 2 a tensor is one ggml_quantize_chunk call, otherwise one call per 16384 values, the last one shorter.
Each call is one quantize_row_q*_reference over the chunk (orc_quantize_row), so Q2_K / Q4_K / Q5_K carry their codes across it.
"""
import ctypes as C
import os
import struct
import numpy as np
import pyoracle as po

CHUNK = 32 * 512
# enum llama_ftype -> ggml type (libfalcon.cpp:3538-3560); anything else is refused
FTYPE_TYPE = {0: po.F32, 1: po.F16, 2: po.Q4_0, 3: po.Q4_1, 7: po.Q8_0, 8: po.Q5_0, 9: po.Q5_1, 10: po.Q2_K, 11: po.Q3_K,
              12: po.Q3_K, 13: po.Q3_K, 14: po.Q4_K, 15: po.Q4_K, 16: po.Q5_K, 17: po.Q5_K, 18: po.Q6_K}
LEGACY = (po.Q4_0, po.Q4_1, po.Q5_0, po.Q5_1, po.Q8_0)
KQUANTS = (po.Q2_K, po.Q3_K, po.Q4_K, po.Q5_K, po.Q6_K)


class Refused(Exception):
    """falcon_model_quantize returns 1"""


# ------------------------------------------------------------------------------------------------ the reference, through ctypes
class _QuantizeParams(C.Structure):          # llama_model_quantize_params, libfalcon.h:140-145
    _fields_ = [("nthread", C.c_int), ("ftype", C.c_int), ("allow_requantize", C.c_bool), ("quantize_output_tensor", C.c_bool)]


_falcon_ref = None


def ref_quantize_file(src, dst, ftype, nthread=1, allow_requantize=False, quantize_output_tensor=True):
    """the unmodified reference's falcon_model_quantize (oracle/_ref/libfalcon_ref.so) with every field of its parameters, after
    falcon_init_backend as examples/falcon_quantize/quantize.cpp:185 calls it (it fills the fp16 table the legacy dequantisers
    read) -> its return code: 0, or 1 where it refuses.  Its per-tensor report goes to stdout."""
    global _falcon_ref
    if _falcon_ref is None:
        L = C.CDLL(os.path.join(po.HERE, "_ref", "libfalcon_ref.so"))
        L.falcon_init_backend.argtypes, L.falcon_init_backend.restype = [], None
        L.falcon_model_quantize.argtypes = [C.c_char_p, C.c_char_p, C.POINTER(_QuantizeParams)]
        L.falcon_model_quantize.restype = C.c_int
        L.falcon_init_backend()
        _falcon_ref = L
    p = _QuantizeParams(nthread, ftype, bool(allow_requantize), bool(quantize_output_tensor))
    rc = int(_falcon_ref.falcon_model_quantize(src.encode(), dst.encode(), C.byref(p)))
    C.CDLL(None).fflush(None)                # its printf report, before a caller reads the captured stdout
    return rc


def ref_quantize_chunk(t, x, start, n, hist):
    """ggml_quantize_chunk exported by oracle/_ref/libggml_ref.so on float32 x: adds to hist (int64[16]) and returns (bytes, the
    blocks of values [start, start + n) as uint8)"""
    L = po.ref().L                             # ggml_init has filled the fp16 table
    L.ggml_quantize_chunk.restype = C.c_size_t
    L.ggml_quantize_chunk.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    x = np.ascontiguousarray(x, dtype=np.float32)
    assert hist.dtype == np.int64 and hist.size == 16
    dst = np.zeros(x.size * 4 + 64, np.uint8)
    nb = int(L.ggml_quantize_chunk(t, po._fp(x), po._fp(dst), start, n, po._fp(hist)))
    off = start // po.BLOCK_ELEMS[t] * po.BLOCK_BYTES[t]
    return nb, dst[off:off + nb].copy()


def legacy_hist(t, blocks):
    """the 16 bins ggml_quantize_q4_0 / q4_1 / q5_0 / q5_1 / q8_0 add for `blocks` (uint8 [nblocks][block bytes]), ggml.c:19352-19477.
    q5_*: value j/2's low nibble takes bit j of qh, its high nibble (qh & (1u << (j + 16))) >> (j + 12); the compiled reference
    shifts by the count modulo 32 (x86), which is what is done here for j >= 16."""
    b = np.ascontiguousarray(blocks, np.uint8).reshape(-1, po.BLOCK_BYTES[t])
    if t == po.Q8_0:
        v = b[:, 2:].view(np.int8).astype(np.int32)
        return np.bincount((np.trunc(v / 16).astype(np.int32) + 8).ravel(), minlength=16).astype(np.int64)
    if t in (po.Q4_0, po.Q4_1):
        qs = b[:, 2 if t == po.Q4_0 else 4:]
        return np.bincount(np.concatenate([(qs & 15).ravel(), (qs >> 4).ravel()]), minlength=16).astype(np.int64)
    qo = 2 if t == po.Q5_0 else 4
    qh = b[:, qo:qo + 4].copy().view("<u4")[:, 0].astype(np.uint64)
    qs = b[:, qo + 4:qo + 20].astype(np.uint64)
    bins = []
    for j in range(0, 32, 2):
        vh0 = ((qh >> np.uint64(j)) & np.uint64(1)) << np.uint64(4)
        vh1 = ((qh & np.uint64(1 << ((j + 16) & 31))) >> np.uint64((j + 12) & 31)) & np.uint64(0xff)
        bins.append(((qs[:, j // 2] & np.uint64(15)) | vh0) // np.uint64(2))
        bins.append((((qs[:, j // 2] >> np.uint64(4)) | vh1) & np.uint64(0xff)) // np.uint64(2))
    return np.bincount(np.concatenate(bins).astype(np.int64), minlength=16).astype(np.int64)


def quantize_chunks(t, x, chunk):
    """ggml_quantize_chunk on consecutive chunks of `chunk` values of float32 x -> (uint8 blocks, int64[16] histogram)"""
    o = po.orc()
    x = np.ascontiguousarray(x, np.float32).ravel()
    if t == po.F32:
        return x.view(np.uint8).copy(), np.zeros(16, np.int64)
    out = np.zeros(po.row_bytes(t, x.size), np.uint8)
    be, bb = po.BLOCK_ELEMS[t], po.BLOCK_BYTES[t]
    for s in range(0, x.size, chunk):
        n = min(chunk, x.size - s)
        assert o.L.orc_quantize_row(t, po._fp(x[s:]), po._fp(out[s // be * bb:]), n) == 0
    hist = legacy_hist(t, out) if t in LEGACY else np.zeros(16, np.int64)
    return out, hist


def to_f32(t, raw, ne):
    """llama_convert_tensor_internal: F16 widening or dequantize_row_q (row by row is the same as whole-tensor: blocks are independent)"""
    if t == po.F32:
        return np.asarray(raw).view(np.float32).reshape(-1)
    if t == po.F16:
        return np.asarray(raw).view(np.float16).astype(np.float32).reshape(-1)
    return po.orc().dequantize(t, np.asarray(raw).reshape(ne[1], -1), ne[0]).reshape(-1)


def plan_chunk(n, nthread):
    if nthread <= 0:
        nthread = os.cpu_count()
    nchunk = (n + CHUNK - 1) // CHUNK
    use = max(1, min(nthread, nchunk)) if nthread > 1 else 1
    return n if use < 2 else CHUNK


def quantize_file(src, dst, ftype, nthread=1, allow_requantize=False, quantize_output_tensor=True):
    """writes dst as falcon_quantize would; -> dict(size_org, size_new, hist (int64[16] total), per_tensor {name: int64[16]},
    n_tensors).  Raises Refused where the reference returns 1."""
    if ftype not in FTYPE_TYPE:
        raise Refused("invalid output file type %d" % ftype)
    qtype = FTYPE_TYPE[ftype]
    buf = np.fromfile(src, np.uint8)
    mv = memoryview(buf)
    off = 0

    def u32():
        nonlocal off
        v = struct.unpack_from("<I", mv, off)[0]
        off += 4
        return v

    hdr = [u32() for _ in range(10)]
    assert hdr[0] == 0x67676363 and hdr[1] == 10
    n_vocab, n_bpe = hdr[2], hdr[9]
    vocab_at = off
    vocab_end = None
    for i in range(n_vocab):
        at = off
        n = u32()
        if i == 65024 and n_vocab == 65025 and bytes(mv[off:off + n]) == b"[PAD]":
            vocab_end, hdr[2] = at, 65024          # libfalcon.cpp:863-868
        off += n + 4
    vocab_end = off if vocab_end is None else vocab_end
    n_merges = u32()
    merges_at = off
    merges_end = off if n_bpe == 0 else None
    for i in range(n_merges):
        for _ in range(2):
            off += u32()
        if i + 1 == n_bpe:
            merges_end = off
    hdr[8] = ftype
    out = bytearray(struct.pack("<10I", *hdr))
    out += bytes(mv[vocab_at:vocab_end])
    out += struct.pack("<I", n_bpe) + bytes(mv[merges_at:merges_end])

    rep = dict(size_org=0, size_new=0, hist=np.zeros(16, np.int64), per_tensor={}, n_tensors=0)
    while off < buf.size:
        n_dims, name_len, t = u32(), u32(), u32()
        ne = [u32() for _ in range(n_dims)]
        name = bytes(mv[off:off + name_len]).decode()
        off += name_len
        off += -off & 31
        nbytes = po.row_bytes(t, ne[0]) * (ne[1] if n_dims == 2 else 1)
        raw = buf[off:off + nbytes]
        off += nbytes
        q = name.endswith("weight") or len(name) == 5    # rfind("weight") == size() - 6, size_t arithmetic included
        q = q and n_dims == 2 and (quantize_output_tensor or name != "lm_head.weight") and t != qtype
        new_t, data = t, bytes(raw)
        if q:
            if qtype in KQUANTS and ne[0] % 256:
                raise Refused("k-quants need rows of a multiple of 256: %s %s" % (name, ne))
            if t not in (po.F32, po.F16) and not allow_requantize:
                raise Refused("requantizing from type %d is disabled" % t)
            x = to_f32(t, raw, ne)
            blocks, h = quantize_chunks(qtype, x, plan_chunk(x.size, nthread))
            new_t, data = qtype, blocks.tobytes()
            rep["hist"] += h
            rep["per_tensor"][name] = h
        out += struct.pack("<3I", n_dims, name_len, new_t) + struct.pack("<%dI" % n_dims, *ne) + name.encode()
        out += b"\0" * (-len(out) & 31)
        out += data
        rep["size_org"] += nbytes
        rep["size_new"] += len(data)
        rep["n_tensors"] += 1
    with open(dst, "wb") as f:
        f.write(out)
    return rep


# ------------------------------------------------------------------------------------------------ test models
# 40B-type, n_embd 768 (16384 is not a multiple of it: chunks split rows) and an odd vocabulary (the last chunk is partial)
MODEL_A = dict(n_vocab=1001, n_embd=768, n_head=12, n_head_kv=2, n_layer=1, falcon_type=40)
# embedding and head of 256 x 64 = 16384 values: one chunk, so nthread 4 still takes the single-call branch for them
MODEL_B = dict(n_vocab=64, n_embd=256, n_head=4, n_head_kv=1, n_layer=1, falcon_type=40)


def write_model(path, hp, wtype=po.F16, seed=7, shapes=None):
    """A GGCC file of i.i.d. N(0, 0.02) weights: 2-D tensors as `wtype` (F32, F16, or quantised row by row by the oracle), 1-D as f32.
    i.i.d. data on purpose: the reference starts every Q2_K / Q4_K / Q5_K chunk from uninitialised stack codes where the device
    starts from zeros, and the two agree unless a sub-block's first-round codes happen to equal the stale ones, which random
    data practically never produces."""
    import ggllm_cpp_b200.ggcc as ggcc
    rng = np.random.default_rng(seed)
    tensors = {}
    for name, ne in (shapes or ggcc.falcon_shapes(hp)).items():
        if len(ne) == 1:
            tensors[name] = (po.F32, ne, (1.0 + 0.1 * rng.standard_normal(ne[0])).astype(np.float32))
            continue
        x = (0.02 * rng.standard_normal((ne[1], ne[0]))).astype(np.float32)
        if wtype == po.F32:
            tensors[name] = (po.F32, ne, x)
        elif wtype == po.F16:
            tensors[name] = (po.F16, ne, x.astype(np.float16))
        else:
            tensors[name] = (wtype, ne, po.orc().quantize(wtype, x))
    ggcc.write_ggcc(path, hp, tensors, ftype=ggcc.FTYPE_OF_TYPE.get(wtype, 1))
    return path


def parse_printed_hists(text):
    """falcon_quantize's per-tensor "| hist: f f f ..." lines -> list of 16-float lists, in tensor order"""
    out = []
    for line in text.splitlines():
        if "| hist:" in line and "[" in line:
            vals = line.split("| hist:")[1].split()
            if vals:
                out.append([float(v) for v in vals])
    return out
