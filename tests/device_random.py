"""Host twin of the synthetic data the device makes for bench.py's models, byte for byte.

  * weights: fill_random_kernel (weights.cu) hashes every (block, plane, 4-byte word) with mix32 straight into the planar layout,
    masks the expanded 6-bit scale planes (PlaneSpec kind 1 / kind 2), then overwrites each block's fp16 scale fields.  The twin
    generates the same planes and inverts the upload's repack (repack_kernel: kind 0 copies, kind 1 expands the 12-byte packed 6-bit
    field, kind 2 stores the signed Q3_K scales) to give the reference's block bytes, which orc.dequantize reads.
  * LayerNorm vectors and KV rows: fill_kernel (engine.cu), in f32 or fp16.

Everything is row-local (block index idx = r * nb + b), so any subset of a 65024-row matrix is built without the rest.

Contraction.  nvcc builds engine.cu and weights.cu with FMA contraction on; the SASS of fill_kernel<float> and fill_kernel<__half>
computes base + amp * t with one FFMA, and fill_random_kernel computes dsm * 10.f - 0.02f with one FFMA (cuobjdump -sass of
engine.o / weights.o).  The twin follows the binary: it forms both in float64, where the product and the sum are exact (t has 24
significant bits, amp and dsm 24, and the sums stay within 53 bits), and rounds once to fp32, which is what an FMA does.

Seeds follow binding.Falcon.set_random: tensor i of ggcc.falcon_shapes(hp) (in that order) gets seed * 1000003 + i; 2-D tensors
are `wtype` blocks, 1-D ones f32 LayerNorm vectors (gamma around 1, beta around 0).  b200_falcon_kv_fill_random(pos, n, seed) fills
layer l's K rows with seed + 2 l and its V rows with seed + 2 l + 1, the hash index starting at 0 at row pos.
"""
import numpy as np

F32, F16, Q4_0, Q4_1, Q5_0, Q5_1, Q8_0, Q2_K, Q3_K, Q4_K, Q5_K, Q6_K = 0, 1, 2, 3, 6, 7, 8, 10, 11, 12, 13, 14
TYPES = (F32, F16, Q4_0, Q4_1, Q5_0, Q5_1, Q8_0, Q2_K, Q3_K, Q4_K, Q5_K, Q6_K)

# type_spec (formats.cuh): blk_elems, blk_bytes, planes (src_off, bytes, kind); plane 0 is the main quant plane
TYPE_SPEC = {
    F32: (1, 4, [(0, 4, 0)]),
    F16: (1, 2, [(0, 2, 0)]),
    Q4_0: (32, 18, [(2, 16, 0), (0, 2, 0)]),
    Q4_1: (32, 20, [(4, 16, 0), (0, 4, 0)]),
    Q5_0: (32, 22, [(6, 16, 0), (2, 4, 0), (0, 2, 0)]),
    Q5_1: (32, 24, [(8, 16, 0), (4, 4, 0), (0, 4, 0)]),
    Q8_0: (32, 34, [(2, 32, 0), (0, 2, 0)]),
    Q2_K: (256, 84, [(16, 64, 0), (0, 16, 0), (80, 4, 0)]),
    Q3_K: (256, 110, [(32, 64, 0), (0, 32, 0), (96, 16, 2), (108, 2, 0)]),
    Q4_K: (256, 144, [(16, 128, 0), (4, 16, 1), (0, 4, 0)]),
    Q5_K: (256, 176, [(48, 128, 0), (16, 32, 0), (4, 16, 1), (0, 4, 0)]),
    Q6_K: (256, 210, [(0, 128, 0), (128, 64, 0), (192, 16, 0), (208, 2, 0)]),
}
# fill_random_kernel's fp16 overwrites: (plane, byte offset in the plane's block, "d" = fp16(dsm) or "m" = fp16(4 dsm));
# F16 / F32 write dsm * 10 - 0.02 into the whole element instead
SCALE_FIELDS = {Q4_0: [(1, 0, "d")], Q8_0: [(1, 0, "d")], Q4_1: [(1, 0, "d"), (1, 2, "m")], Q5_0: [(2, 0, "d")],
                Q5_1: [(2, 0, "d"), (2, 2, "m")], Q2_K: [(2, 0, "d"), (2, 2, "d")], Q3_K: [(3, 0, "d")],
                Q4_K: [(2, 0, "d"), (2, 2, "d")], Q5_K: [(3, 0, "d"), (3, 2, "d")], Q6_K: [(3, 0, "d")]}

def _u64(v):
    return np.uint64(v & 0xFFFFFFFFFFFFFFFF)


def mix32(x):
    """weights.cu mix32 (the murmur3 finaliser, low 32 bits) of uint64 values, wrapping like the device"""
    x = np.asarray(x, np.uint64)
    x = x ^ (x >> np.uint64(33))
    x = x * _u64(0xff51afd7ed558ccd)
    x = x ^ (x >> np.uint64(33))
    x = x * _u64(0xc4ceb9fe1a85ec53)
    x = x ^ (x >> np.uint64(33))
    return (x & np.uint64(0xFFFFFFFF)).astype(np.uint32)


def row_bytes(t, K):
    per, bsz, _ = TYPE_SPEC[t]
    return K // per * bsz


# ------------------------------------------------------------------------------------------------ weights
def weight_planes(t, K, rows, seed):
    """the device planes fill_random_kernel writes for `rows` of a K-wide matrix: a list of uint8 [len(rows)][nb][plane bytes]"""
    per, _, planes = TYPE_SPEC[t]
    nb = K // per
    rows = np.asarray(rows, np.int64)
    idx = (rows[:, None] * nb + np.arange(nb, dtype=np.int64)[None]).astype(np.uint64)          # [R][nb]
    s = _u64(seed)
    out = []
    for p, (_, nbytes, kind) in enumerate(planes):
        words = (nbytes + 3) // 4
        i = np.arange(words, dtype=np.uint64) * np.uint64(4)
        v = mix32(s ^ ((idx * np.uint64(8) + np.uint64(p)) << np.uint64(20))[..., None] ^ i)       # [R][nb][words]
        if kind == 1:
            v = v & np.uint32(0x3f3f3f3f)
        elif kind == 2:
            v = (((v & np.uint32(0x3f3f3f3f)) | np.uint32(0x80808080)) - np.uint32(0x20202020)) ^ np.uint32(0x80808080)
        out.append(np.ascontiguousarray(v.astype("<u4")).view(np.uint8).reshape(len(rows), nb, words * 4)[..., :nbytes].copy())
    h = mix32(s ^ _u64(0x9e3779b97f4a7c15) ^ idx)
    unit = np.float32(1e-4 if per == 256 else 2e-3)
    dsm = unit * (np.float32(1) + np.float32(2) * (h & np.uint32(0xffff)).astype(np.float32) / np.float32(65536))
    dsm = dsm.astype(np.float32)
    if t in (F32, F16):
        v = (dsm.astype(np.float64) * 10.0 + np.float64(np.float32(-0.02))).astype(np.float32)        # one FFMA
        out[0][...] = (v if t == F32 else v.astype(np.float16)).view(np.uint8).reshape(out[0].shape)
        return out
    fields = {"d": dsm.astype(np.float16).view(np.uint8).reshape(len(rows), nb, 2),
              "m": (dsm * np.float32(4)).astype(np.float16).view(np.uint8).reshape(len(rows), nb, 2)}
    for p, off, which in SCALE_FIELDS[t]:
        out[p][..., off:off + 2] = fields[which]
    return out


def _pack_sm6(sc, mn):
    """pack_sm6 (formats.cuh) for j = 0..7 in order: 8 six-bit scales and mins [..][8] -> the 12-byte field [..][12]"""
    q = np.zeros(sc.shape[:-1] + (12,), np.uint8)
    for j in range(8):
        ls, lm = sc[..., j].astype(np.uint8), mn[..., j].astype(np.uint8)
        if j < 4:
            q[..., j] = ls
            q[..., j + 4] = lm
        else:
            q[..., j + 4] = (ls & 0xF) | ((lm & 0xF) << 4)
            q[..., j - 4] |= (ls >> 4) << 6
            q[..., j] |= (lm >> 4) << 6
    return q


def _unpack_sm6(f):
    """get_scale_min_k4 of every j: the 12-byte field [..][12] -> (scales, mins) [..][8]"""
    f = f.astype(np.int32)
    sc, mn = np.zeros(f.shape[:-1] + (8,), np.int32), np.zeros(f.shape[:-1] + (8,), np.int32)
    for j in range(8):
        if j < 4:
            sc[..., j], mn[..., j] = f[..., j] & 63, f[..., j + 4] & 63
        else:
            sc[..., j] = (f[..., j + 4] & 0xF) | ((f[..., j - 4] >> 6) << 4)
            mn[..., j] = (f[..., j + 4] >> 4) | ((f[..., j] >> 6) << 4)
    return sc, mn


def _q3_pos(j):
    """byte of the expanded Q3_K scale plane that holds scale j (q3_scale16)"""
    return 4 * (2 * (j >> 3) + (j & 1)) + ((j >> 1) & 3)


def _pack_q3(sc6):
    """16 six-bit Q3_K scales (bias 32 included) [..][16] -> the 12-byte field q3_scale reads"""
    s = np.zeros(sc6.shape[:-1] + (12,), np.uint8)
    sc6 = sc6.astype(np.uint8)
    for j in range(16):
        if j < 8:
            s[..., j] |= sc6[..., j] & 0xF
        else:
            s[..., j - 8] |= (sc6[..., j] & 0xF) << 4
        s[..., 8 + (j & 3)] |= ((sc6[..., j] >> 4) & 3) << (2 * (j >> 2))
    return s


def _q3_scales(f):
    """q3_scale of every j: the 12-byte field [..][12] -> [..][16] with the bias kept"""
    f = f.astype(np.int32)
    out = np.zeros(f.shape[:-1] + (16,), np.int32)
    for j in range(16):
        lo = (f[..., j] & 0xF) if j < 8 else (f[..., j - 8] >> 4)
        hi = (f[..., 8 + (j & 3)] >> (2 * (j >> 2))) & 3
        out[..., j] = lo | (hi << 4)
    return out


def planes_to_blocks(t, planes):
    """the inverse of repack_kernel: device planes [R][nb][plane bytes] -> the reference's blocks, uint8 [R][nb * blk_bytes]"""
    _, bsz, spec = TYPE_SPEC[t]
    R, nb = planes[0].shape[:2]
    blk = np.zeros((R, nb, bsz), np.uint8)
    for (off, nbytes, kind), pl in zip(spec, planes):
        if kind == 0:
            blk[..., off:off + nbytes] = pl
        elif kind == 1:                    # {sc[2p], sc[2p+1], m[2p], m[2p+1]} for p = 0..3
            e = pl.reshape(R, nb, 4, 4)
            sc = e[..., :2].reshape(R, nb, 8)
            mn = e[..., 2:].reshape(R, nb, 8)
            blk[..., off:off + 12] = _pack_sm6(sc, mn)
        else:                              # signed scale - 32 at q3_pos(j)
            sc = np.stack([pl[..., _q3_pos(j)].view(np.int8).astype(np.int32) + 32 for j in range(16)], -1)
            blk[..., off:off + 12] = _pack_q3(sc)
    return blk.reshape(R, nb * bsz)


def blocks_to_planes(t, blocks):
    """host model of repack_kernel: the reference's blocks uint8 [R][row bytes] -> the device planes"""
    _, bsz, spec = TYPE_SPEC[t]
    blk = np.ascontiguousarray(blocks, np.uint8).reshape(len(blocks), -1, bsz)
    R, nb = blk.shape[:2]
    out = []
    for off, nbytes, kind in spec:
        if kind == 0:
            out.append(blk[..., off:off + nbytes].copy())
        elif kind == 1:
            sc, mn = _unpack_sm6(blk[..., off:off + 12])
            e = np.zeros((R, nb, 4, 4), np.uint8)
            e[..., 0], e[..., 1] = sc[..., 0::2], sc[..., 1::2]
            e[..., 2], e[..., 3] = mn[..., 0::2], mn[..., 1::2]
            out.append(e.reshape(R, nb, 16))
        else:
            s = _q3_scales(blk[..., off:off + 12])
            e = np.zeros((R, nb, 16), np.uint8)
            for j in range(16):
                e[..., _q3_pos(j)] = (s[..., j] - 32).astype(np.int8).view(np.uint8)
            out.append(e)
    return out


def weight_rows(t, K, rows, seed):
    """rows of the matrix b200_weight_random(t, K, M, seed) / set_tensor_random makes, as the reference stores them: uint8 blocks
    [len(rows)][row bytes] for quantised types, float32 / float16 [len(rows)][K] for F32 / F16"""
    blocks = planes_to_blocks(t, weight_planes(t, K, rows, seed))
    if t == F32:
        return blocks.view(np.float32)
    if t == F16:
        return blocks.view(np.float16)
    return blocks


# ------------------------------------------------------------------------------------------------ fill_kernel
def fill_values(n, base, amp, seed, dtype=np.float32):
    """fill_kernel<E>(p, n, base, amp, seed): element i = base + amp * (hash(seed, i) / 2^23 - 1), one FFMA, stored as `dtype`"""
    i = np.arange(n, dtype=np.uint64)
    x = _u64(seed) + i * _u64(0x9E3779B97F4A7C15)
    x = x ^ (x >> np.uint64(31))
    x = x * _u64(0xBF58476D1CE4E5B9)
    x = x ^ (x >> np.uint64(29))
    u = (x & np.uint64(0xffffff)).astype(np.float32) / np.float32(8388608) - np.float32(1)           # exact
    v = (np.float64(np.float32(amp)) * u.astype(np.float64) + np.float64(np.float32(base))).astype(np.float32)
    return v if dtype == np.float32 else v.astype(np.float16)


def layernorm_vector(name, n, seed):
    """a 1-D tensor of set_tensor_random: LayerNorm gamma (base 1, amplitude 0.1) or beta (base 0, amplitude 0.01), f32"""
    gamma = name.endswith(".weight")
    return fill_values(n, 1.0 if gamma else 0.0, 0.1 if gamma else 0.01, seed)


def kv_rows(layer, pos, n, width, seed, f16=False):
    """(K, V) float32 [n][width] that b200_falcon_kv_fill_random(pos, n, seed) writes to rows [pos, pos + n) of local layer `layer`,
    as kv_read returns them (an fp16 cache: the values rounded to fp16, widened)"""
    dt = np.float16 if f16 else np.float32
    k = fill_values(n * width, 0.0, 1.0, seed + 2 * layer, dt).astype(np.float32).reshape(n, width)
    v = fill_values(n * width, 0.0, 1.0, seed + 2 * layer + 1, dt).astype(np.float32).reshape(n, width)
    return k, v


def tensor_seeds(shapes, seed):
    """{name: seed} of Falcon.set_random(shapes, wtype, seed)"""
    return {name: seed * 1000003 + i for i, name in enumerate(shapes)}
