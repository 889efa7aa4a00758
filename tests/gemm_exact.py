"""Exactly representable operands for the prompt GEMM (gemm_tc.cu, gemm_simt.cu) and a numpy model of its output, with injected faults.

Grid weights: ggcc.random_blocks rows whose scale fields are rewritten so that every dequantised weight is an integer multiple of G.
Block scales d and mins dmin are G or 2 G (alternating between neighbouring blocks, super-blocks and rows, d and dmin out of step),
sub-block scales and mins are small integers that differ between neighbouring sub-blocks, and the codes keep random_blocks' uniform
bytes, so they cover their full range.  Every product in the fp32 dequantiser is then exact, every weight is below 2048 G and so
exact in fp16, and the producers' single fp16 rounding rounds nothing.  F16 weights are small integers times G or 2 G.
Grid activations: small non-zero integers (+-1, +-2) in fp16.

Then every product w x and every partial sum, in any order, is a multiple of G; the tests hold each output to
sum_k |w_k x_k| <= HEADROOM * G.  Below that, every fp32 accumulation order -- the CUDA-core FMA chain, wgmma, the two-way atomic K
split -- gives exactly the fp64 result (2^24 G would do for plain fp32 adds; the extra 4 bits cover tensor-core adders that keep fewer
bits below the largest term of an MMA group), so the GPU tests compare bits, not tolerances.  On an H100 (sm_90a) the fp16 wgmma with
fp32 accumulation met this on every case of the parametrisation below.

gemm_model computes that result in float64 and can inject the faults a producer or the K split typically has (FAULT_DOC).
"""
import numpy as np
import pyoracle as po
import mmv_exact as mx

G = 2.0 ** -10
HEADROOM = 2.0 ** 20
BK, BM, ST, N_MAX = 64, 128, 4, 512          # gemm_tc.cu's K block, weight tile, ring depth and tokens per call
FAST = (po.Q4_K, po.Q4_0, po.Q3_K)           # types with a dedicated producer; the others go through the generic one
GRID_TYPES = po.WEIGHT_TYPES + [po.F16]
# bytes of the 4-bit code plane whose low / high nibbles hold different elements
NIBBLES = {po.Q4_0: (2, 16), po.Q4_1: (4, 16), po.Q5_0: (6, 16), po.Q5_1: (8, 16), po.Q4_K: (16, 128), po.Q5_K: (48, 128), po.Q6_K: (0, 128)}
FAULT_DOC = {
    "d_next": "every block takes its scale d from the next block of the row (a single-block row: from the next row)",
    "min_next": "every block takes its min (dmin, or m of Q4_1 / Q5_1) from the next block",
    "kb+1": "every 64-wide K block takes the weights of K block kb + 1 (the last one those of kb - 1)",
    "kb-1": "every 64-wide K block takes the weights of K block kb - 1 (the first one those of kb + 1)",
    "chunk": "8-weight chunk h of every K block swapped with chunk h ^ 1",
    "nibbles": "low and high nibbles of every code byte swapped",
    "q3_hbit": "Q3_K codes take their high bit from the other 128-value half of the super-block",
    "row_next": "output row m computed from weight row m + 1",
    "tok_next": "token n computed from activation row n + 1",
    "drop0": "the last K block of split half 0 dropped",
    "drop1": "the last K block of split half 1 dropped",
    "twice0": "split half 0 added twice",
    "twice1": "split half 1 added twice",
}


def _f16_bytes(v):
    return np.asarray(v, np.float16)[..., None].view(np.uint8)


def _pack_k4(sc, m):
    """8 scales and 8 mins < 16 -> the 12 bytes get_scale_min_k4 (k_quants.c:592-601) unpacks them from"""
    out = np.zeros(sc.shape[:-1] + (12,), np.uint8)
    out[..., 0:4] = sc[..., 0:4]
    out[..., 4:8] = m[..., 0:4]
    out[..., 8:12] = sc[..., 4:8] | (m[..., 4:8] << 4)
    return out


def _pack_q3(s6):
    """16 six-bit Q3_K scales (stored value, scale + 32) -> the 12 packed bytes (k_quants.c dequantize_row_q3_K's aux unpacking):
    low nibbles in bytes 0..7 (j < 8 low, j >= 8 high nibble of byte j - 8), high two bits at bits 2 (j / 4) of byte 8 + j % 4"""
    out = np.zeros(s6.shape[:-1] + (12,), np.uint8)
    for j in range(16):
        lo, hi = s6[..., j] & 15, s6[..., j] >> 4
        out[..., j % 8] |= (lo << (4 * (j // 8))).astype(np.uint8)
        out[..., 8 + j % 4] |= (hi << (2 * (j // 4))).astype(np.uint8)
    return out


def sub_scales(t, M, nb):
    """[M][nb][sub-blocks] the sub-block scales (and mins) the grid builder writes: small integers, neighbours differ"""
    r = np.arange(M)[:, None, None]
    b = np.arange(nb)[None, :, None]
    j = np.arange(16)[None, None, :]
    if t in (po.Q4_K, po.Q5_K, po.Q2_K):
        n = 8 if t != po.Q2_K else 16
        return (1 + (j + r + b) % 3)[..., :n].astype(np.uint8), ((j + 2 * r + b) % 4)[..., :n].astype(np.uint8)
    if t in (po.Q3_K, po.Q6_K):
        return np.array([1, -1, 2, -2])[(j + r + b) % 4].astype(np.int8), None
    return None, None


def grid_weights(t, M, K, rng):
    """M x K grid weights of type t: raw blocks (uint8 [M][row bytes]), or float16 [M][K] for F16"""
    r = np.arange(M)[:, None]
    if t == po.F16:
        e = (r + np.arange(K)[None, :] // 32) % 2
        k = rng.integers(-48, 49, (M, K))
        return (k * G * 2.0 ** e).astype(np.float16)
    import ggllm_cpp_b200.ggcc as ggcc
    wq = ggcc.random_blocks(t, M, K, rng)
    nb, bb = K // mx.BE[t], po.BLOCK_BYTES[t]
    v = wq.reshape(M, nb, bb)
    b = np.arange(nb)[None, :]
    v[:, :, mx.D_OFF[t]:mx.D_OFF[t] + 2] = _f16_bytes(G * 2.0 ** ((r + b) % 2))
    if t in (po.Q4_1, po.Q5_1):                       # w = q d + m: m a signed small multiple of G
        v[:, :, 2:4] = _f16_bytes((1 + (r + 2 * b) % 3) * G * np.where(b % 2, -1.0, 1.0))
    elif t in mx.M_OFF:
        v[:, :, mx.M_OFF[t]:mx.M_OFF[t] + 2] = _f16_bytes(G * 2.0 ** ((r + b + 1) % 2))
    sc, m = sub_scales(t, M, nb)
    if t in (po.Q4_K, po.Q5_K):
        v[:, :, 4:16] = _pack_k4(sc, m)
    elif t == po.Q2_K:
        v[:, :, 0:16] = sc | (m << 4)
    elif t == po.Q3_K:
        v[:, :, 96:108] = _pack_q3((sc.astype(np.int16) + 32).astype(np.uint8))
    elif t == po.Q6_K:
        v[:, :, 192:208] = sc.view(np.uint8)
    return v.reshape(M, -1)


def grid_acts(N, K, rng):
    """N x K activations: +-1, +-2 in fp16"""
    return (rng.integers(1, 3, (N, K)) * rng.choice([-1, 1], (N, K))).astype(np.float16)


def grid_acts_q8(wtype, N, K, rng):
    """fp32 rows that b200_mul_mat's activation quantiser turns into themselves: grid_acts with one +-127 per 32-value block (Q8_0 /
    Q8_1: d = amax / 127 = 1) or one +-128 per 256-value block (Q8_K: iscale = -128 / max = -+1), so fp16(d q) == x everywhere"""
    x = grid_acts(N, K, rng).astype(np.float32)
    blk, top = (256, 128.0) if po.VEC_DOT_TYPE[wtype] == po.Q8_K else (32, 127.0)
    v = x.reshape(N, K // blk, blk)
    pos = rng.integers(0, blk, (N, K // blk))
    np.put_along_axis(v, pos[..., None], (top * rng.choice([-1.0, 1.0], (N, K // blk)))[..., None], axis=2)
    return v.reshape(N, K)


def dequant(t, wq, K):
    """float64 [rows][K] weights through the oracle's dequantiser"""
    if t == po.F16:
        return np.asarray(wq, np.float16).astype(np.float64)
    return po.orc().dequantize(t, wq, K).astype(np.float64)


def _field_from_next_block(t, wq, off):
    nb = wq.shape[1] // po.BLOCK_BYTES[t]
    v = wq.reshape(wq.shape[0], nb, -1).copy()
    if nb > 1:
        v[:, :-1, off:off + 2] = v[:, 1:, off:off + 2]
        v[:, -1, off:off + 2] = v[:, -2, off:off + 2]
    else:
        v[:, 0, off:off + 2] = np.roll(v[:, 0, off:off + 2], -1, axis=0)
    return v.reshape(wq.shape)


def _faulty_weights(t, wq, K, fault):
    if fault == "d_next":
        wq = _field_from_next_block(t, wq, mx.D_OFF[t])
    elif fault == "min_next":
        wq = _field_from_next_block(t, wq, mx.M_OFF[t])
    elif fault == "nibbles":
        o, n = NIBBLES[t]
        v = wq.reshape(wq.shape[0], -1, po.BLOCK_BYTES[t]).copy()
        q = v[:, :, o:o + n]
        v[:, :, o:o + n] = ((q & 0x0F) << 4) | (q >> 4)
        wq = v.reshape(wq.shape)
    elif fault == "q3_hbit":
        v = wq.reshape(wq.shape[0], -1, 110).copy()
        h = v[:, :, 0:32]
        v[:, :, 0:32] = ((h & 0x0F) << 4) | (h >> 4)
        wq = v.reshape(wq.shape)
    w = dequant(t, wq, K)
    if fault in ("kb+1", "kb-1"):
        kbt = K // BK
        kb = np.arange(kbt)
        src = kb + (1 if fault == "kb+1" else -1)
        src = np.where((src < 0) | (src >= kbt), 2 * kb - src, src)
        w = w.reshape(w.shape[0], kbt, BK)[:, src].reshape(w.shape)
    elif fault == "chunk":
        w = w.reshape(w.shape[0], K // BK, 8, 8)[:, :, np.arange(8) ^ 1].reshape(w.shape)
    return w


def halves(K, ksplit):
    """[(kb0, KB)] the K blocks each CTA of a split owns (gemm_tc_kernel: kb0 = KBT z / ksplit)"""
    kbt = K // BK
    return [(kbt * z // ksplit, kbt * (z + 1) // ksplit - kbt * z // ksplit) for z in range(ksplit)]


def faults_for(t, ksplit, K):
    """the faults that apply to a weight type and launch: scale / min / code faults where the type has that field, K-block faults
    where there is a neighbouring K block, split faults where K is split"""
    f = ["chunk", "row_next", "tok_next", "drop0"]
    if t != po.F16:
        f.append("d_next")
    if t in mx.M_OFF:
        f.append("min_next")
    if t in NIBBLES:
        f.append("nibbles")
    if t == po.Q3_K:
        f.append("q3_hbit")
    if K // BK > 1:
        f += ["kb+1", "kb-1"]
    if ksplit == 2:
        f += ["drop1", "twice0", "twice1"]
    return f


def gemm_model(t, wq, K, x, ksplit=1, fault=None, rows=None, toks=None, mag=False, chunk=256):
    """Y[n][m] = sum_k w[m][k] x[n][k] in float64 (exact on grid operands) for tokens `toks` and weight rows `rows` (default: all),
    with one fault of FAULT_DOC injected (ksplit: the K split the drop / twice faults refer to).
    mag=True also returns sum_k |w x| per output."""
    M, N = wq.shape[0], x.shape[0]
    rows = np.arange(M) if rows is None else np.asarray(rows)
    toks = np.arange(N) if toks is None else np.asarray(toks)
    rsel = (rows + 1) % M if fault == "row_next" else rows
    tsel = (toks + 1) % N if fault == "tok_next" else toks
    X = np.asarray(x, np.float64)[tsel]
    Y = np.zeros((len(toks), len(rows)))
    A = np.zeros_like(Y) if mag else None
    for c0 in range(0, len(rsel), chunk):
        w = _faulty_weights(t, np.asarray(wq)[rsel[c0:c0 + chunk]], K, fault)
        y = X @ w.T
        if fault and fault[:-1] in ("drop", "twice"):
            kb0, kb = halves(K, ksplit)[int(fault[-1])]
            lo, hi = (kb0 + kb - 1) * BK if fault.startswith("drop") else kb0 * BK, (kb0 + kb) * BK
            part = X[:, lo:hi] @ w[:, lo:hi].T
            y = y - part if fault.startswith("drop") else y + part
        Y[:, c0:c0 + chunk] = y
        if mag:
            A[:, c0:c0 + chunk] = np.abs(X) @ np.abs(w).T
    return (Y, A) if mag else Y


# ------------------------------------------------------------------------------------------------ the GPU parametrisation
# (type, K, M, N): b200_mul_mat_f16 with impl 1 (wgmma) and impl 0 (CUDA core).  Every (producer, BN, ksplit); K blocks per CTA 1, 2,
# 3, ST and ST + 1; odd K-block counts split unevenly (9 -> 4 + 5, 71 -> 35 + 36); Q3_K / Q4_K / Q2_K halves starting inside a
# super-block (K = 768, 1280: kb0 = 6, 10); M % 128 = 1, <= 64 and > 64; N % BN != 0; Falcon-40B / 180B widths on both sides of the
# K-split decision (K = 8192 at M = 12800 fills 100 tiles: no split).
TC = [
    (po.Q4_0, 64, 129, 40), (po.Q4_0, 128, 200, 33), (po.Q4_0, 192, 300, 100), (po.Q4_0, 320, 77, 300), (po.Q4_0, 8192, 12800, 9),
    (po.Q4_0, 4544, 200, 40), (po.Q4_0, 576, 130, 128), (po.Q4_0, 32768, 129, 300),
    (po.Q4_K, 256, 300, 9), (po.Q4_K, 256, 77, 128), (po.Q4_K, 256, 129, 257), (po.Q4_K, 768, 200, 64), (po.Q4_K, 14848, 130, 100),
    (po.Q4_K, 8192, 300, 512),
    (po.Q3_K, 256, 129, 64), (po.Q3_K, 256, 300, 65), (po.Q3_K, 256, 200, 512), (po.Q3_K, 32768, 77, 20), (po.Q3_K, 768, 300, 100),
    (po.Q3_K, 1280, 130, 300),
    (po.Q4_1, 64, 129, 40), (po.Q5_0, 128, 300, 100), (po.Q5_1, 192, 77, 300), (po.Q8_0, 4544, 200, 40), (po.Q2_K, 768, 130, 128),
    (po.Q5_K, 1280, 300, 300), (po.Q6_K, 256, 129, 64), (po.F16, 576, 200, 257), (po.F16, 320, 130, 100), (po.Q5_K, 256, 77, 200),
    (po.Q6_K, 2048, 300, 128), (po.Q2_K, 256, 300, 512), (po.Q4_1, 4544, 77, 64), (po.Q5_0, 1024, 129, 300), (po.Q5_1, 576, 200, 9),
    (po.Q8_0, 256, 300, 130), (po.Q2_K, 8192, 130, 40),
]
# GEMM + GELU (never split): (type, K, M, N), both kernels
GELU = [(po.Q4_K, 14848, 130, 100), (po.Q4_0, 4544, 300, 300), (po.Q3_K, 8192, 77, 64), (po.Q6_K, 1024, 129, 128), (po.F16, 512, 200, 40)]
# b200_mul_mat (activation quantiser + dispatcher): N > 512 in chunks of 512, K % 64 == 32 on the CUDA-core kernel
MUL_MAT = [(po.Q4_K, 1024, 300, 513), (po.Q4_0, 4576, 200, 1000), (po.Q3_K, 2048, 129, 1025), (po.Q5_1, 1056, 77, 1000),
           (po.Q6_K, 512, 130, 1025), (po.Q8_0, 1056, 129, 513)]


def case_id(c):
    return "%s-K%d-M%d-N%d" % (po.TYPE_NAMES[c[0]], c[1], c[2], c[3])


def case_seed(c):
    return 7919 * c[0] + 31 * c[1] + 7 * c[2] + c[3]


def chunks(N):
    """token counts of the calls launch_mmq_gemm makes"""
    return [min(N_MAX, N - n0) for n0 in range(0, N, N_MAX)]


def launches(c, gelu=False):
    """[(shape or None, N of the call)] for every GEMM call the case makes (b200_gemm_launch_shape; None: the CUDA-core kernel)"""
    import ggllm_cpp_b200.binding as b
    t, K, M, N = c
    return [(b.gemm_launch_shape(t, K, M, n, K, gelu), n) for n in chunks(N)]
