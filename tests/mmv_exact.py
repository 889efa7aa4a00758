"""Exact-arithmetic restatement of the decode mat-vec kernels (numpy, float64) and a per-output error bound.

Every quantised kernel splits a row into 16-byte "pieces" (16 or 32 weights) and forms one fp32 term per piece from an exact
integer dot: (d_w d_x) isum - (dmin_w d_x) msum, or the type's equivalent (mmv.cu MV<>::dot, mmv_fast.cuh FX<>::dot).  Here the
integer dots are computed as integers and everything else in float64, from the raw weight blocks and the quantised activation
exactly as the device stores it (codes q, scales d, Q8_1 sums s).  The integer codes times their sub-block scales come from the
oracle's dequantiser with the block's scale field set to 1 and its min field to 0 (and the min part from scale 0, min 1): every
such value is a small integer, so the dequantiser's fp32 arithmetic is exact.

Bound, per output:  (r + depth) u sum_pieces (|A| + |B|),  u = 2^-24 (to first order; gamma_k = k u / (1 - k u) is used)
  A, B    the two fp32 products of a piece term, A = (d_w d_x) isum, B = (dmin_w d_x) msum (B = 0 for types without a min)
  r       roundings inside one piece term: d_w * d_x, * isum (2); for a min: dmin_w * d_x, * msum, and the subtraction (3)
  depth   the longest chain of fp32 additions a piece term passes through on its way to the output (see `depth`)
Epilogues: ADD2 adds two roundings of |y| + |r1| + |r2|; GELU is compared on its fp16 grid (`gelu_ok`).
"""
import numpy as np
import pyoracle as po

U = 2.0 ** -24

# per type: elements per block, pieces per block, roundings r of one piece term, byte offsets of the fp16 scale and min fields
BE = {po.Q4_0: 32, po.Q4_1: 32, po.Q5_0: 32, po.Q5_1: 32, po.Q8_0: 32, po.Q2_K: 256, po.Q3_K: 256, po.Q4_K: 256, po.Q5_K: 256, po.Q6_K: 256}
PPB = {po.Q4_0: 1, po.Q4_1: 1, po.Q5_0: 1, po.Q5_1: 1, po.Q8_0: 2, po.Q2_K: 4, po.Q3_K: 4, po.Q4_K: 8, po.Q5_K: 8, po.Q6_K: 8}
R = {po.Q4_0: 2, po.Q4_1: 3, po.Q5_0: 2, po.Q5_1: 3, po.Q8_0: 2, po.Q2_K: 3, po.Q3_K: 2, po.Q4_K: 3, po.Q5_K: 3, po.Q6_K: 2}
D_OFF = {po.Q4_0: 0, po.Q4_1: 0, po.Q5_0: 0, po.Q5_1: 0, po.Q8_0: 0, po.Q2_K: 80, po.Q3_K: 108, po.Q4_K: 0, po.Q5_K: 0, po.Q6_K: 208}
M_OFF = {po.Q4_1: 2, po.Q5_1: 2, po.Q2_K: 82, po.Q4_K: 2, po.Q5_K: 2}
# generic kernel (mmv.cu): blocks per work unit, MV<TYPE>::CH
CH = {po.Q4_K: 32, po.Q5_K: 16, po.Q6_K: 16, po.Q3_K: 32, po.Q2_K: 32, po.Q4_0: 256, po.Q4_1: 256, po.Q5_0: 128, po.Q5_1: 128, po.Q8_0: 128}


def swept_weights(t, M, K, rng, n_swept=8):
    """ggcc.random_blocks rows; the first n_swept rows have their block scales d swept over 2^-4 .. 2^3 (by row and by block)"""
    import ggllm_cpp_b200.ggcc as ggcc
    wq = ggcc.random_blocks(t, M, K, rng)
    nb, bb = K // BE[t], po.BLOCK_BYTES[t]
    v = wq.reshape(M, nb, bb)
    n = min(n_swept, M)
    d = v[:n, :, D_OFF[t]:D_OFF[t] + 2].copy().view(np.float16)[..., 0].astype(np.float32)
    e = (np.arange(n)[:, None] + 3 * np.arange(nb)[None, :]) % 8 - 4
    v[:n, :, D_OFF[t]:D_OFF[t] + 2] = (d * np.exp2(e)).astype(np.float16)[..., None].view(np.uint8)
    return v.reshape(M, -1)


def swept_acts(t, N, K, rng):
    """activation rows whose 32-value (legacy types) or 256-value (K-quants) blocks have magnitudes swept over 2^-8 .. 2^8; the first
    and the last block sit at the loud end, so that a mistake in a row's head or ragged tail is not hidden by louder blocks"""
    blk = 256 if BE[t] == 256 else 32
    e = rng.uniform(-8, 8, (N, K // blk))
    e[:, 0] = e[:, -1] = 8
    return (rng.standard_normal((N, K)) * np.repeat(np.exp2(e), blk, 1)).astype(np.float32)


def _piece_elems(t):
    """[PPB][weights per piece] element offsets (inside a block) that piece pc of a block multiplies"""
    a = np.arange(16)
    if t in (po.Q4_K, po.Q5_K):      # mmv_fast.cuh:47-49, mmv.cu:64-65, 90-91: low nibbles at e0, high nibbles at e0 + 32
        return np.array([np.r_[64 * (pc >> 1) + 16 * (pc & 1) + a, 64 * (pc >> 1) + 16 * (pc & 1) + 32 + a] for pc in range(8)])
    if t == po.Q6_K:                 # mmv.cu:124-127
        el = [128 * (pc >> 2) + (32 if pc & 2 else 0) + 16 * (pc & 1) for pc in range(8)]
        return np.array([np.r_[e + a, e + 64 + a] for e in el])
    if t in (po.Q3_K, po.Q2_K):      # mmv_fast.cuh:181-185, mmv.cu:158-163, 190-196: four 16-value quads
        return np.array([np.concatenate([128 * (pc >> 1) + 32 * qd + 16 * (pc & 1) + a for qd in range(4)]) for pc in range(4)])
    if t == po.Q8_0:                 # mmv.cu:308: 16 codes per piece
        return np.array([a, 16 + a])
    return np.arange(32)[None, :]    # legacy 4/5-bit types: one piece is the whole block


def _set_f16(blocks, t, off, value):
    b = blocks.reshape(-1, po.BLOCK_BYTES[t]).copy()
    b[:, off:off + 2] = np.frombuffer(np.float16(value).tobytes(), np.uint8)
    return b.reshape(blocks.shape)


def _f16_field(blocks, t, off):
    b = blocks.reshape(blocks.shape[0], -1, po.BLOCK_BYTES[t])
    return b[:, :, off:off + 2].copy().view(np.float16)[..., 0].astype(np.float64)


def act_from_blocks(wtype, raw, K):
    """orc.quantize_act's blocks -> (q [N][K] int8, d [N][K/blk] fp32, s [N][K/32] fp32, bs) as ActQ.download() returns them"""
    at = po.VEC_DOT_TYPE[wtype]
    N = raw.shape[0]
    r = raw.reshape(N, K // po.BLOCK_ELEMS[at], po.BLOCK_BYTES[at])
    if at == po.Q8_K:
        q = r[:, :, 4:260].copy().view(np.int8).reshape(N, K)
        d = r[:, :, 0:4].copy().view(np.float32).reshape(N, -1)
        return q, d, np.zeros((N, K // 32), np.float32), r[:, :, 260:292].copy().view(np.int16).reshape(N, -1)
    if at == po.Q8_0:
        q = r[:, :, 2:34].copy().view(np.int8).reshape(N, K)
        d = r[:, :, 0:2].copy().view(np.float16).astype(np.float32).reshape(N, -1)
        return q, d, np.zeros((N, K // 32), np.float32), q.reshape(N, -1, 32).astype(np.int32).sum(-1).astype(np.int16)
    q = r[:, :, 8:40].copy().view(np.int8).reshape(N, K)
    d = r[:, :, 0:4].copy().view(np.float32).reshape(N, -1)
    s = r[:, :, 4:8].copy().view(np.float32).reshape(N, -1)
    return q, d, s, q.reshape(N, -1, 32).astype(np.int32).sum(-1).astype(np.int16)


def depth(t, K, kernel):
    """longest fp32 addition chain from a piece term to the stored output.
    kernel: ("fast", NT, J) -- mmv_fast.cuh:322-324 J - 1 sequential adds per thread, :232-260 transpose_reduce's 5 butterfly levels,
            :346-348 NT / 32 - 1 adds of the fixed-order sum over warps (v starts at 0: its first add is exact);
            ("generic",) -- mmv.cu:419-421 the per-lane acc += over every piece the lane takes in every unit of the row (acc starts
            at 0, mmv.cu:410 / 435), plus warp_sum's 5 levels (common.cuh:69-72)"""
    if kernel[0] == "fast":
        _, nt, j = kernel
        return (j - 1) + 5 + (nt // 32 - 1)
    assert kernel[0] == "generic"
    nb = K // BE[t]
    per_lane = 0
    for b0 in range(0, nb, CH[t]):                 # lane 0 takes the most pieces of every unit
        per_lane += -(-min(CH[t], nb - b0) * PPB[t] // 32)
    return per_lane - 1 + 5


def gamma(k):
    return k * U / (1 - k * U)


def reference(t, wq, K, q, d, s, kernel, rows=None, chunk_elems=1 << 23, xd_piece=None, drop=None, d_from_next_row=None,
              swap_mins=False, q3_hbit_other_half=False):
    """One activation row: wq uint8 [M][row bytes] raw blocks of type t, q [K] int8 codes, d / s its scales / Q8_1 sums.
    -> (y, bound, mag, pieces) float64 [M]: the exact output, its error bound for `kernel` (see `depth`), sum (|A| + |B|), and the
    piece terms are not kept (pieces is None) unless rows is given, which also restricts the evaluation to those rows.
    Mutations the sensitivity tests use to show the bound can fail:
      xd_piece=g            piece position g of every row takes the activation scale of the next block (the previous for the last)
      drop=("piece"|"unit", row)   that row (every row for None) loses its last piece / its last work unit of the generic kernel
      d_from_next_row=(row, blk)   that block takes its weight scale d from the same block of the next row
      swap_mins             Q4_K / Q5_K: every piece uses m1 for its low nibbles and m0 for its high nibbles
      q3_hbit_other_half    Q3_K: every code takes its high bit from the other 128-value half of the block (hmask bit 4 n + j <-> 4 (1-n) + j)"""
    wq = np.ascontiguousarray(wq, np.uint8)
    M = wq.shape[0]
    nb, be, ppb = K // BE[t], BE[t], PPB[t]
    orc = po.orc()
    elems = _piece_elems(t)
    qx = np.asarray(q, np.int64).reshape(nb, be)
    xd = np.asarray(d, np.float64)
    if t in (po.Q2_K, po.Q3_K, po.Q4_K, po.Q5_K, po.Q6_K):
        xdb = xd                                                     # one Q8_K scale per 256 weights
    else:
        xdb = xd[:nb]                                                # one Q8_0 / Q8_1 scale per 32 weights
    xd_p = np.repeat(xdb[:, None], ppb, 1)                           # [nb][ppb]: activation scale each piece uses
    if xd_piece is not None:
        b = xd_piece // ppb
        xd_p[b, xd_piece % ppb] = xdb[b + 1 if b + 1 < nb else b - 1]
    row_ids = np.arange(M) if rows is None else np.asarray(rows)
    if d_from_next_row is not None:
        wq = wq.copy()
        rr, bb = d_from_next_row
        o = bb * po.BLOCK_BYTES[t] + D_OFF[t]
        wq[rr, o:o + 2] = wq[(rr + 1) % M, o:o + 2]
    if q3_hbit_other_half:
        assert t == po.Q3_K
        v = wq.reshape(M, nb, 110).copy()
        h = v[:, :, 0:32]
        v[:, :, 0:32] = ((h & 0x0F) << 4) | (h >> 4)
        wq = v.reshape(M, -1)
    y = np.zeros(len(row_ids))
    mag = np.zeros(len(row_ids))
    keep = [] if rows is not None else None
    step = max(1, chunk_elems // K)
    for c0 in range(0, len(row_ids), step):
        ids = row_ids[c0:c0 + step]
        blk = wq[ids]
        # A: codes times sub-block scales, as integers (scale field 1, min field 0)
        bA = _set_f16(blk, t, D_OFF[t], 1.0)
        if t in M_OFF:
            bA = _set_f16(bA, t, M_OFF[t], 0.0)
        cA = orc.dequantize(t, bA, K).astype(np.int64).reshape(len(ids), nb, be)
        iA = (cA * qx[None]).take(elems, axis=2).sum(-1)              # [rows][nb][ppb] exact integer dots
        sA = _f16_field(blk, t, D_OFF[t])                             # [rows][nb] weight scale d
        A = sA[:, :, None] * xd_p[None] * iA
        B = np.zeros_like(A)
        if t in (po.Q2_K, po.Q4_K, po.Q5_K):
            bB = _set_f16(_set_f16(blk, t, D_OFF[t], 0.0), t, M_OFF[t], 1.0)
            cB = orc.dequantize(t, bB, K).astype(np.int64).reshape(len(ids), nb, be)       # - min of each element's sub-block
            if swap_mins:
                cB = cB.reshape(len(ids), nb, 4, 2, 32)[:, :, :, ::-1].reshape(len(ids), nb, be)
            iB = (cB * qx[None]).take(elems, axis=2).sum(-1)
            B = _f16_field(blk, t, M_OFF[t])[:, :, None] * xd_p[None] * iB
        elif t in (po.Q4_1, po.Q5_1):                                 # + m_w * s_x, the Q8_1 block sum (mmv.cu:248, 292)
            B = _f16_field(blk, t, M_OFF[t])[:, :, None] * np.asarray(s, np.float64)[None, :nb, None]
        terms = (A + B).reshape(len(ids), nb * ppb)
        mags = (np.abs(A) + np.abs(B)).reshape(len(ids), nb * ppb)
        if drop is not None:
            what, dr = drop
            hit = np.arange(len(ids)) if dr is None else np.nonzero(ids == dr)[0]
            cut = 1 if what == "piece" else ((nb - 1) % CH[t] + 1) * ppb
            terms[hit, -cut:] = 0.0
        y[c0:c0 + len(ids)] = terms.sum(1)
        mag[c0:c0 + len(ids)] = mags.sum(1)
        if keep is not None:
            keep.append((A.reshape(len(ids), -1), B.reshape(len(ids), -1)))
    bound = gamma(R[t] + depth(t, K, kernel)) * mag + 1e-38
    pieces = None if keep is None else (np.concatenate([k[0] for k in keep]), np.concatenate([k[1] for k in keep]))
    return y, bound, mag, pieces


def cpu_bound(t, K, pieces_A, pieces_B, iA_lanes=None):
    """Error bound of orc.mul_mat (the CPU's sequential vec_dot order, ggml_oracle.c dot_legacy / dot_kquant) for the rows whose
    piece terms `reference(..., rows=...)` returned.  Legacy types: one term per block, r roundings, nb sequential adds.
    K-quants: the CPU forms eight lane sums per block (acc[i & 7]) instead of pieces; `iA_lanes` gives sum |d_w d_x acc_l| per row,
    which replaces sum |A|; the lane terms pass through 2 roundings, nb - 1 lane adds and 8 final adds, the min terms through
    2 roundings, nb sequential subtractions and the same 8 adds (Q2_K: one term per block, 3 roundings, nb adds)."""
    nb = K // BE[t]
    if t in (po.Q3_K, po.Q4_K, po.Q5_K, po.Q6_K):
        mag = iA_lanes + np.abs(pieces_B).sum(1)
        return gamma(nb + 11) * mag + 1e-38
    return gamma(R[t] + nb) * (np.abs(pieces_A) + np.abs(pieces_B)).sum(1) + 1e-38


def cpu_lane_magnitude(t, wq, K, q, d):
    """sum over blocks and the eight CPU lanes l of |d_w d_x sum_{e in block, e % 8 == l} c_e q_e| (K-quants with lanes)"""
    orc = po.orc()
    nb = K // 256
    bA = _set_f16(wq, t, D_OFF[t], 1.0)
    if t in M_OFF:
        bA = _set_f16(bA, t, M_OFF[t], 0.0)
    cA = orc.dequantize(t, bA, K).astype(np.int64).reshape(wq.shape[0], nb, 32, 8)
    lanes = (cA * np.asarray(q, np.int64).reshape(nb, 32, 8)[None]).sum(2)          # [rows][nb][8]
    sA = _f16_field(wq, t, D_OFF[t]) * np.asarray(d, np.float64)[None, :nb]
    return np.abs(sA[:, :, None] * lanes).sum((1, 2))


def f_reference(t, w, x):
    """F16 / F32 weights (mmv.cu:489-522): w [M][K] float32 (F16 values already widened), x [K] fp32 activation.
    -> (y, bound).  F16: x is rounded to fp16 and each pair of products (exact in fp32) is summed once, r = 1 on |w x| + |w' x'|;
    the lane walks K / 256 steps of 4 pairs.  F32: four products summed left to right per step (<= 4 roundings per product term),
    K / 128 steps per lane.  Both end with warp_sum (5 levels)."""
    K = w.shape[1]
    x64 = np.asarray(x, np.float64)
    if t == po.F16:
        x64 = x64.astype(np.float16).astype(np.float64)
        chain, r = 4 * (-(-K // 256)), 1
    else:
        chain, r = -(-K // 128), 4
    y, mag = np.zeros(w.shape[0]), np.zeros(w.shape[0])
    for r0 in range(0, w.shape[0], 4096):                            # row chunks: float64 copies stay small at lm_head width
        w64 = np.asarray(w[r0:r0 + 4096], np.float64)
        y[r0:r0 + 4096], mag[r0:r0 + 4096] = w64 @ x64, np.abs(w64) @ np.abs(x64)
    return y, gamma(r + chain - 1 + 5) * mag + 1e-38


def _nearest_midpoint(x):
    """distance from x to the nearest fp16 rounding midpoint, and the fp16 value on the other side of it"""
    h = np.asarray(x, np.float64).astype(np.float16)
    with np.errstate(over="ignore", invalid="ignore"):
        up, dn = np.nextafter(h, np.float16(np.inf)), np.nextafter(h, np.float16(-np.inf))
        h64, up64, dn64 = h.astype(np.float64), up.astype(np.float64), dn.astype(np.float64)
        du, dd = (h64 + up64) / 2 - x, x - (h64 + dn64) / 2
    use_up = du < dd
    return np.where(use_up, du, dd), np.where(use_up, up64, dn64)


def _gelu_outputs(f):
    """fp16 input f -> (the fp16 output of the LUT formula in exact arithmetic, the neighbouring fp16 output where the kernel's fp32
    formula (tanhf within 2 ulp, about six roundings) may land on the other side of an fp16 midpoint, else the same value)"""
    c = 0.79788456080286535587989211986876
    arg = c * f * (1.0 + 0.044715 * f * f)
    th = np.tanh(arg)
    g = 0.5 * f * (1.0 + th)
    err = 0.5 * np.abs(f) * (8 * U + 8 * U * np.abs(arg) * (1 - th * th)) + 8 * U * np.abs(g) + 1e-45
    dist, alt = _nearest_midpoint(g)
    out = g.astype(np.float16).astype(np.float64)
    return out, np.where(dist <= err, alt, out)


def gelu_ok(got, y, bound):
    """True where the kernel's GELU output `got` is one the exact pre-GELU value y (error <= bound) allows: exactly gelu(f16(y)),
    or, where y lies within the bound of an fp16 midpoint, gelu of the neighbouring fp16 input (attn_exact's "flip" term)"""
    dist, alt_in = _nearest_midpoint(y)
    f0 = np.asarray(y, np.float64).astype(np.float16).astype(np.float64)
    f1 = np.where(dist <= bound, alt_in, f0)
    got = np.asarray(got, np.float64)
    ok = np.zeros(got.shape, bool)
    for f in (f0, f1):
        a, b = _gelu_outputs(f)
        ok |= (got == a) | (got == b)
    return ok


def add2_bound(y, bound, r1, r2):
    """ADD2: out = (y + r1) + r2 in fp32, two roundings of |y| + |r1| + |r2| on top of the mat-vec's own bound"""
    return bound * (1 + 4 * U) + gamma(2) * (np.abs(y) + bound + np.abs(r1) + np.abs(r2))
