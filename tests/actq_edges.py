"""Edge rows for the activation quantisers (Q8_0 / Q8_1 / Q8_K): the inputs on which their rounding and tie rules decide the codes.

The device must produce the same codes, scales and block sums as the reference's quantize_row_q8_0 (x86 AVX2 body),
quantize_row_q8_1 (AVX2 body) and quantize_row_q8_K, because the mat-vec computes the CPU's integer block dots from them.
Random fp32 rows never reach the rules that matter, so every block here is built for one rule and asserts, in numpy float32,
that it really exercises it (a tie that is not on the block maximum tests nothing):

  E1  sign tie on the block maximum: +a before -a and -a before +a, inside one lane's 8 values, across lanes at every xor distance
      of the block reductions (1, 2 for 32-blocks; 1, 2, 4, 8, 16 for 256-blocks), across the two 16-value segments one Q4_K
      mat-vec piece multiplies (32 values apart), with the earlier element in the lower and in the higher lane.  For Q8_K the first
      element of largest magnitude sets the sign of d and which element is clamped; Q8_0 / Q8_1 only read the magnitude.
  E2  repeated equal magnitudes of the same sign on the fp16 grid (what fp16-grid producers such as GELU hand over).
  E3  products v * id (Q8_0 / Q8_1) or iscale * v (Q8_K) that are exactly k + 1/2, both parities and both signs, where
      round-half-even and round-half-away differ: Q8_K blocks have maximum +-2^e so iscale = -+2^(7-e) is exact, Q8_0 / Q8_1
      blocks maximum 127 * 2^e so id = 2^-e is exact.  Also blocks of fp16-grid GELU outputs that contain such products naturally.
  E4  Q8_K clamp: -vmax is present, its product is +128 and its code must be 127 (and the block sums must count 127).
  E5  zero blocks: all zero, one non-zero value, +0.0 / -0.0 mixes.
  E6  block maxima of 2^-100 and 2^100 (about 1e-30 and 1e30; Q8_0 keeps d in fp16, so its large maximum is 127 * 2^15), with
      values that round to code 0.

Out of scope: NaN and Inf inputs, and block maxima below about 127 / FLT_MAX (3.7e-37).  There 127 / amax overflows, and x86
cvtps saturation, the oracle's magic-number rounding and __float2int_rn all disagree; no producer sees such rows from a model.

Every value is a float32 with at most 7 significant bits unless it comes from the fp16 grid (E2 uses 3, GELU rows 11), so rows
can also be produced exactly by a mat-vec with selector weights (representable()).
"""
import numpy as np
import pyoracle as po

ATYPES = (po.Q8_0, po.Q8_1, po.Q8_K)
WTYPE_OF = {po.Q8_0: po.Q4_0, po.Q8_1: po.Q4_1, po.Q8_K: po.Q4_K}      # a weight type whose vec_dot_type it is
BLK = {po.Q8_0: 32, po.Q8_1: 32, po.Q8_K: 256}
FAMILIES = {po.Q8_0: ("E1", "E2", "E3", "E5", "E6"), po.Q8_1: ("E1", "E2", "E3", "E5", "E6"),
            po.Q8_K: ("E1", "E2", "E3", "E4", "E5", "E6")}
F32 = np.float32

# E1 pair positions (earlier, later) inside a block, with what they exercise
E1_PAIRS = {32: [((1, 6), "lane"), ((3, 9), "xor1"), ((2, 17), "xor2"), ((12, 27), "xor2 lanes 1/3"), ((10, 20), "xor3")],
            256: [((1, 6), "lane"), ((3, 9), "xor1"), ((2, 17), "xor2"), ((5, 37), "xor4 / q4k one lane, two segments"),
                  ((7, 70), "xor8"), ((4, 133), "xor16"), ((43, 170), "xor16 lanes 5/21"), ((100, 250), "xor3 lanes 12/31"),
                  ((20, 40), "q4k earlier in higher lane"), ((84, 104), "q4k earlier in higher lane, p 1"),
                  ((16, 64), "q4k xor2"), ((0, 128), "q4k xor4"), ((50, 99), "q4k xor3")]}


def _coarse(x, bits=6):
    """x rounded to `bits` significant bits (exact float32)"""
    m, e = np.frexp(np.asarray(x, np.float64))
    return np.ldexp(np.round(m * 2.0 ** bits) / 2.0 ** bits, e).astype(F32)


def _fill(rng, n, amax):
    """filler values strictly below amax in magnitude, 6 significant bits, never zero"""
    v = _coarse(rng.uniform(0.05, 0.9, n) * float(amax)) * rng.choice(F32([-1, 1]), n)
    return v.astype(F32)


# ------------------------------------------------------------------------------------------------ numpy float32 restatement
def scale_of(at, b):
    """the per-block multiplier the quantiser applies: id = 127 / amax (Q8_0 / Q8_1) or iscale = -128 / vmax (Q8_K, vmax = the
    first element of largest magnitude); None for an all-zero block"""
    a = np.abs(b)
    if a.max() == 0:
        return None
    if at == po.Q8_K:
        return F32(-128) / b[int(np.argmax(a))]
    return F32(127) / a.max()


def products(at, b):
    s = scale_of(at, b)
    return np.zeros_like(b) if s is None else (b * s).astype(F32)


def halfway(at, b):
    p = products(at, b)
    return (p - np.floor(p)) == 0.5


def representable(b, bits=7):
    """every value is j * 2^t with |j| < 2^bits (or zero)"""
    m, _ = np.frexp(np.asarray(b, np.float64))
    return bool(np.all(m * 2.0 ** bits == np.round(m * 2.0 ** bits)))


def premise(at, fam, label, b, period=None):
    """the property the block was built for, in numpy float32; raises AssertionError when it does not hold.  period: the block
    repeats a template of that length (the E1 pair then recurs in every copy; the first copy's pair is the one under test)"""
    b = np.asarray(b, F32)
    a = np.abs(b)
    assert b.size == BLK[at] and np.all(np.isfinite(b)), label
    copies = BLK[at] // (period or BLK[at])
    if fam == "E1":
        i, j = [int(t) for t in label.split()[1].split("/")]
        top = np.flatnonzero(a == a.max())
        assert top.size == 2 * copies and list(top[:2]) == [i, j], label
        assert b[i] == -b[j] and b[i] != 0, label
        assert (b[i] > 0) == ("+-" in label), label
        if at == po.Q8_K:
            p = products(at, b)
            assert p[i] == -128 and p[j] == 128, label                   # the earlier one sets the sign; the later one clamps
    elif fam == "E2":
        top = np.flatnonzero(a == a.max())
        assert top.size >= 3 and np.all(b[top] == b[top[0]]), label
        assert np.array_equal(b, b.astype(np.float16).astype(F32)), label
    elif fam == "E3":
        h = halfway(at, b)
        assert h.any(), label
        if not label.startswith("E3 gelu"):
            p = products(at, b)[h]
            kinds = {(int(np.floor(v)) % 2, bool(v > 0)) for v in p}
            assert kinds == {(0, True), (1, True), (0, False), (1, False)}, (label, kinds)
        else:
            assert np.array_equal(b, b.astype(np.float16).astype(F32)), label
    elif fam == "E4":
        p = products(at, b)
        assert at == po.Q8_K and np.any(p == 128) and not np.any(p > 128), label
    elif fam == "E5":
        nz = np.count_nonzero(b)
        if "one" in label:
            assert nz == copies, label
        else:
            assert nz == 0, label
        if "+-0" in label:
            assert np.signbit(b[b == 0]).any() and (~np.signbit(b[b == 0])).any(), label
    elif fam == "E6":
        amax = float(a.max())
        assert amax >= 2.0 ** 21 or amax <= 2.0 ** -99, label
        s = scale_of(at, b)
        assert np.isfinite(s) and s != 0, label
        if at == po.Q8_0:
            assert np.isfinite(np.float16(amax / 127)), label            # d is stored in fp16
        else:
            assert np.isfinite(F32(1) / s), label
        p = products(at, b)
        assert np.any((np.abs(p) < 0.5) & (b != 0)), label               # values that round to code 0
    elif fam != "fill":
        raise AssertionError("unknown family " + fam)


# ------------------------------------------------------------------------------------------------ block builders
def _e1(at, period, rng):
    out = []
    for (i, j), what in E1_PAIRS[32 if at != po.Q8_K else 256]:
        if j >= period:
            continue
        for first in (1, -1):
            a = F32(1.5 * 2.0 ** int(rng.integers(-6, 7)))
            t = _fill(rng, period, a)
            t[i], t[j] = first * a, -first * a
            out.append(("E1", "E1 %d/%d %s %s" % (i, j, "+-" if first > 0 else "-+", what), t))
    return out


def _e2(at, period, rng):
    out = []
    for sign in (1, -1):
        e = int(rng.integers(-4, 5))
        mags = F32([1.75, 1.5, 1.25, 1.0, 0.75, 0.5, 0.375, 0.25]) * F32(2.0 ** e)
        t = (rng.choice(mags[1:], period) * rng.choice(F32([-1, 1]), period)).astype(F32)
        pos = np.sort(rng.choice(period, 5, replace=False))
        t[pos] = sign * mags[0]
        out.append(("E2", "E2 repeated %s" % ("+" if sign > 0 else "-"), t))
    return out


def _e3(at, period, rng):
    out = []
    for wide in (False, True):
        for sign in (1, -1):
            e = int(rng.integers(-3, 4))
            if at == po.Q8_K:
                top = F32(sign * 2.0 ** e)                             # iscale = -sign * 2^(7-e): products -sign * (k + 1/2)
                ks = np.arange(-128, 128) if wide else np.arange(-64, 64)
                vals = ((ks + 0.5) * 2.0 ** e / 128).astype(F32)
            else:
                top = F32(sign * 127 * 2.0 ** e)                       # id = 2^-e: products k + 1/2
                ks = np.arange(-127, 127) if wide else np.arange(-64, 64)
                vals = ((ks + 0.5) * 2.0 ** e).astype(F32)
            t = np.empty(period, F32)
            t[0] = top
            pick = rng.choice(vals.size, period - 1, replace=vals.size < period - 1)
            t[1:] = vals[pick]
            out.append(("E3", "E3 %s %s" % ("wide" if wide else "7-bit", "+" if sign > 0 else "-"), t))
    return out


def _gelu_blocks(at, period, rng, want=4):
    """fp16-grid GELU outputs of N(0, 4) inputs (the ffn_down activations), blocks that contain a half-way product"""
    x = (2.0 * rng.standard_normal(period * 16384)).astype(np.float16).astype(np.float64)
    g = (0.5 * x * (1.0 + np.tanh(0.7978845608028654 * x * (1.0 + 0.044715 * x * x)))).astype(np.float16).astype(F32)
    out = []
    for t in g.reshape(-1, period):
        blk = np.tile(t, BLK[at] // period)
        if halfway(at, blk).any():
            out.append(("E3", "E3 gelu", t.copy()))
            if len(out) == want:
                break
    assert len(out) == want
    return out


def _e4(at, period, rng):
    out = []
    for sign in (1, -1):
        a = F32(1.25 * 2.0 ** int(rng.integers(-5, 6)))
        t = _fill(rng, period, a)
        i, j = sorted(rng.choice(np.arange(1, period), 2, replace=False))
        t[i], t[j] = sign * a, -sign * a
        t[int(rng.integers(0, i))] = 0.0
        out.append(("E4", "E4 clamp %s" % ("+" if sign > 0 else "-"), t))
    return out


def _e5(at, period, rng):
    z = np.zeros(period, F32)
    one_p, one_n, mix, mix1 = z.copy(), z.copy(), z.copy(), z.copy()
    one_p[period // 3] = 0.75
    one_n[period - 1] = -0.75
    mix[::3] = -0.0
    mix1[1::2] = -0.0
    mix1[period // 2] = -3.0
    return [("E5", "E5 zero", z), ("E5", "E5 one +", one_p), ("E5", "E5 one -", one_n), ("E5", "E5 +-0", mix),
            ("E5", "E5 one +-0", mix1)]


def _e6(at, period, rng):
    out = []
    tops = (2.0 ** -100, 127 * 2.0 ** 15) if at == po.Q8_0 else (2.0 ** -100, 2.0 ** 100)
    for top in tops:
        for sign in (1, -1):
            a = F32(sign * top)
            t = _fill(rng, period, abs(a))
            t[period // 2:] = _fill(rng, period - period // 2, abs(a) * 2.0 ** -9)       # these round to code 0
            t[int(rng.integers(0, period // 2))] = a
            out.append(("E6", "E6 %s%g" % ("+" if sign > 0 else "-", top), t))
    return out


def edge_blocks(at, period=None, seed=0):
    """[(family, label, block)] for activation type `at`.  period (a divisor of the block, 64 for the attention hand-over, whose
    output repeats each 64-value head): every block is a template of that length tiled over the block."""
    blk = BLK[at]
    period = period or blk
    assert blk % period == 0
    rng = np.random.default_rng(1000 * at + period + seed)
    out = _e1(at, period, rng) + _e2(at, period, rng) + _e3(at, period, rng) + _gelu_blocks(at, period, rng)
    if at == po.Q8_K:
        out += _e4(at, period, rng)
    out += _e5(at, period, rng) + _e6(at, period, rng)
    res = []
    for fam, label, t in out:
        b = np.tile(t, blk // period).astype(F32)
        premise(at, fam, label, b, period)
        res.append((fam, label, b))
    return res


def edge_rows(at, K, period=None, min_rows=1, seed=0, only=None):
    """the edge blocks laid out in rows of K values (K a multiple of the block), padded with 6-bit N(0, 1) filler blocks.
    only: a predicate on (family, label, block) selecting which edge blocks to use.  -> (rows [R][K] float32, labels [R][K/blk])"""
    blk = BLK[at]
    assert K % blk == 0
    blocks = [t for t in edge_blocks(at, period, seed) if only is None or only(*t)]
    per = K // blk
    R = max(min_rows, -(-len(blocks) // per))
    rng = np.random.default_rng(7 + at + K + seed)
    rows = np.empty((R * per, blk), F32)
    labels = []
    for i in range(R * per):
        if i < len(blocks):
            rows[i] = blocks[i][2]
            labels.append(blocks[i][1])
        else:
            rows[i] = _coarse(rng.standard_normal(blk))
            labels.append("fill")
    return rows.reshape(R, K), np.array(labels, dtype=object).reshape(R, per)


def family_of(label):
    return label.split()[0]


# ------------------------------------------------------------------------------------------------ reading quantised rows
def parse(at, raw, K):
    """raw blocks of the oracle / reference quantiser [R][row bytes] -> (q [R][K] int8, d [R][K/blk] float32, s [R][K/32] float32
    or None, bs [R][K/16 (Q8_K) or K/32] int16) in the device's ActQ layout; Q8_0 / Q8_1 sums are those of the codes"""
    raw = np.ascontiguousarray(raw, np.uint8).reshape(-1, po.row_bytes(at, K))
    R, blk, bb = raw.shape[0], BLK[at], po.BLOCK_BYTES[at]
    r = raw.reshape(R, K // blk, bb)
    if at == po.Q8_K:                                  # {f32 d; int8 qs[256]; int16 bsums[16]}
        d = r[:, :, 0:4].copy().view(F32).reshape(R, -1)
        q = r[:, :, 4:260].copy().view(np.int8).reshape(R, K)
        bs = r[:, :, 260:292].copy().view(np.int16).reshape(R, -1)
        return q, d, None, bs
    if at == po.Q8_0:                                  # {f16 d; int8 qs[32]}
        d = r[:, :, 0:2].copy().view(np.float16).astype(F32).reshape(R, -1)
        q = r[:, :, 2:34].copy().view(np.int8).reshape(R, K)
        s = None
    else:                                              # {f32 d; f32 s; int8 qs[32]}
        d = r[:, :, 0:4].copy().view(F32).reshape(R, -1)
        s = r[:, :, 4:8].copy().view(F32).reshape(R, -1)
        q = r[:, :, 8:40].copy().view(np.int8).reshape(R, K)
    bs = q.reshape(R, -1, 32).astype(np.int32).sum(-1).astype(np.int16)
    return q, d, s, bs


def f16_plane(at, q, d):
    """the prompt GEMM's operand: fp16(float32(d) * float32(q)) per value"""
    blk = BLK[at]
    dd = np.repeat(np.asarray(d, F32), blk, axis=-1)
    with np.errstate(over="ignore"):                   # E6's large scales overflow fp16 to +-inf, on the device too
        return (dd * q.astype(F32)).astype(np.float16)
