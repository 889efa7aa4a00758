"""-m gpu: every activation-quantisation producer against the oracle's quantize_row_q8_0 (x86 body) / q8_1 / q8_K, bit for bit, on the
edge rows of tests/actq_edges.py (sign ties on the block maximum, half-way products, the Q8_K clamp, zero blocks, extreme scales):
codes, d, s (Q8_1), block sums and, where the producer writes it, the fp16 GEMM operand fp16(d * q).

How each producer is fed a chosen row:
  standalone      quantize_act on the rows directly (N = 1, 9, 40, x_stride > K)
  LayerNorm       gamma = 0, beta = the row: norm(x) * 0 is +-0 and +-0 + beta = beta, so the row to quantise is beta exactly
                  (every variant: cluster, register CH = 1 / 2, shared memory; single and dual; with and without the residual adds)
  chain           an input whose quantisation is exact (Q8_K blocks of maximum -128 * 2^a, Q8_0 blocks of maximum 127 * 2^a) and
                  selector weights with power-of-two scales make y equal the designed row; a_out is then checked against it
  attention       n_past = 0: one key of weight exactly 1.  The split-KV kernel's output is then the new V row (asserted, by value:
                  -0.0 comes out as +0.0) repeated over the group's heads.  The long-context kernel's is not bit for bit, so its codes
                  are compared with the quantisation of its own output row; ties within a head survive its identical per-element
                  arithmetic
"""
import numpy as np
import pytest
import pyoracle as po
import actq_edges as ae

gpu_mark = pytest.mark.gpu
F32 = np.float32

STANDALONE_N = [1, 9, 40]
# name -> (n, rows, environment switch); which kernel launch_layernorm_q picks (ops.cu)
LN_VARIANTS = {"cluster": (8192, 1, None), "reg1": (8192, 3, None), "reg1_rows1": (8192, 1, "B200_LN_NOCLUSTER"),
               "reg2": (14848, 2, None), "smem": (18432, 2, None), "smem_env": (4096, 3, "B200_LN_SMEM")}
LN_KERNEL = {"cluster": "ln_cluster", "reg1": "ln_reg1", "reg1_rows1": "ln_reg1", "reg2": "ln_reg2", "smem": "ln_smem", "smem_env": "ln_smem"}
CHAIN = {po.Q4_K: ((-100, 0, 95), 12288), po.Q4_0: ((-12, 0, 12), 1024)}      # input block exponents, output length M
ATTN = [(16, 8, po.Q4_K), (71, 2, po.Q4_0), (8, 8, po.Q4_1)]                   # (G, n_head_kv, weight type)
ATTN_TIERS = ["split", "long"]
ALL_AT = list(ae.ATYPES)


# ------------------------------------------------------------------------------------------------ rows each test feeds
def standalone_rows(at):
    return ae.edge_rows(at, 2048)


def ln_rows(at, variant):
    return ae.edge_rows(at, LN_VARIANTS[variant][0])


def attn_rows(G, hkv, wt, tier):
    """the long-context kernel forms P * V from fp16 hi / lo splits of V (attention_long.cu): values beyond fp16's range (E6) are
    outside its domain, as they are outside any model's V rows"""
    at = po.VEC_DOT_TYPE[wt]
    return ae.edge_rows(at, 64 * hkv, period=64 if at == po.Q8_K else None, only=(lambda f, l, b: f != "E6") if tier == "long" else None)


def _chain_source(wt, exps):
    """the chain's input row: every code once per exponent a, scaled by 2^a, in blocks whose quantisation is exact.
    -> (x [K], {(a, code): k})"""
    rng = np.random.default_rng(wt)
    parts, where, k0 = [], {}, 0
    for a in exps:
        if wt == po.Q4_K:                                # one Q8_K block: -128 .. 127, vmax = -128 * 2^a: iscale = 2^-a, d = 2^a
            codes = rng.permutation(np.arange(-128, 128))
        else:                                            # nine Q8_0 blocks, each led by 127: id = 2^-a, d = 2^a (fp16-exact)
            rest = np.concatenate([np.arange(-127, 127), np.zeros(9 * 31 - 254, np.int64)])
            rest = rng.permutation(rest).reshape(9, 31)
            codes = np.concatenate([np.full((9, 1), 127), rest], axis=1).reshape(-1)
        for i, c in enumerate(codes):
            where.setdefault((a, int(c)), k0 + i)
        parts.append(np.ldexp(codes.astype(np.float64), a).astype(F32))
        k0 += codes.size
    return np.concatenate(parts), where


def _decompose(v, exps):
    """v == code * 2^(p + a) with |code| <= 127, a in exps and 2^p an fp16 value -> (a, code, p), or None"""
    if v == 0:
        return (exps[0], 0, 0)
    m, e = np.frexp(np.float64(v))
    c = m * 128
    if c != np.round(c):
        return None
    t = int(e) - 7
    for a in exps:
        if -24 <= t - a <= 15:
            return (a, int(c), t - a)
    return None


def chain_rows(wt):
    exps, M = CHAIN[wt]
    at = po.VEC_DOT_TYPE[wt]
    return ae.edge_rows(at, M, only=lambda fam, label, b: all(_decompose(v, exps) is not None for v in b))


def reached():
    """{(producer, activation type): set of edge families its tests feed}: the coverage the parametrisation below reaches"""
    out = {}

    def add(key, labels):
        out.setdefault(key, set()).update(ae.family_of(l) for l in np.asarray(labels).reshape(-1) if l != "fill")
    for at in ALL_AT:
        add(("standalone", at), standalone_rows(at)[1])
        add(("plane standalone", at), standalone_rows(at)[1])
        for v in LN_VARIANTS:
            add((LN_KERNEL[v], at), ln_rows(at, v)[1])
            if LN_VARIANTS[v][1] > 1:
                add(("plane " + LN_KERNEL[v], at), ln_rows(at, v)[1])
    for wt in CHAIN:
        add(("chain", po.VEC_DOT_TYPE[wt]), chain_rows(wt)[1])
    for G, hkv, wt in ATTN:
        for tier in ATTN_TIERS:
            add(("attn " + tier, po.VEC_DOT_TYPE[wt]), attn_rows(G, hkv, wt, tier)[1])
    return out


# ------------------------------------------------------------------------------------------------ comparison
def _want(orc, at, x):
    x = np.asarray(x, F32)
    return ae.parse(at, orc.quantize_act(ae.WTYPE_OF[at], x.reshape(-1, x.shape[-1])), x.shape[-1])


def _check(at, A, want, labels, what):
    """A's codes / scales / sums (as many rows as `want` has) == the oracle's, bit for bit; names the first mismatching block's edge label"""
    q, d, s, bs = A.download()
    wq, wd, ws, wbs = want
    R = wq.shape[0]
    q, d, s, bs = q[:R], d[:R], s[:R], bs[:R]
    blk = ae.BLK[at]
    lab = np.asarray(labels).reshape(R, -1) if labels is not None else None

    def where(bad_blocks):
        i = np.argwhere(bad_blocks)[0]
        return (what, tuple(int(t) for t in i), lab[tuple(i)] if lab is not None else None)
    assert np.array_equal(q, wq), where((q != wq).reshape(R, -1, blk).any(-1))
    assert np.array_equal(d.view(np.uint32), wd.view(np.uint32)), where(d.view(np.uint32) != wd.view(np.uint32))
    if at == po.Q8_1:
        assert np.array_equal(s.view(np.uint32), ws.view(np.uint32)), where(s.view(np.uint32) != ws.view(np.uint32))
    if at == po.Q8_K:                                   # the reference leaves the bsums of an all-zero block unwritten; the device writes 0
        nz = np.repeat(wd != 0, 16, axis=1)
        assert np.array_equal(bs[nz], wbs[nz]) and np.all(bs[~nz] == 0), where((bs != wbs).reshape(R, -1, 16).any(-1))
    else:
        assert np.array_equal(bs, wbs), where(bs != wbs)
    return q, d


def _check_plane(gpu, at, A, q, d, what):
    """the fp16 plane == fp16(float32(d) * float32(q)) of the producer's own codes == actq_to_f16 of those codes"""
    h = A.download_f16()[:q.shape[0]]
    want = ae.f16_plane(at, q, d)
    assert np.array_equal(h.view(np.uint16), want.view(np.uint16)), (what, np.argwhere(h.view(np.uint16) != want.view(np.uint16))[:4])
    buf = gpu.DevBuf(A.N * A.K * 2)
    A.to_f16(buf)
    sep = buf.download(np.uint16, (A.N, A.K))[:q.shape[0]]
    assert np.array_equal(sep, want.view(np.uint16)), what


# ------------------------------------------------------------------------------------------------ standalone
@gpu_mark
@pytest.mark.parametrize("N", STANDALONE_N)
@pytest.mark.parametrize("at", ALL_AT)
def test_standalone_quantiser(gpu, orc, at, N):
    rows, labels = standalone_rows(at)
    K, stride = rows.shape[1], rows.shape[1] + 96
    batches = [[r] for r in range(rows.shape[0])] if N == 1 else [[i % rows.shape[0] for i in range(N)]]
    for idx in batches:
        x = np.zeros((N, stride), F32)
        x[:, :K] = rows[idx]
        x[:, K:] = np.nan                                # outside the row: never read
        xd = gpu.DevBuf(src=x)
        A = gpu.ActQ(ae.WTYPE_OF[at], K, N, f16=True)
        A.quantize(xd.ptr, stride)
        q, d = _check(at, A, _want(orc, at, rows[idx]), labels[idx], "standalone N %d" % N)
        _check_plane(gpu, at, A, q, d, "standalone N %d" % N)


# ------------------------------------------------------------------------------------------------ LayerNorm producers
def _ln_launch(gpu, n, rows, x, resid, g1, b1, A1, g2, b2, A2):
    xd = gpu.DevBuf(src=x)
    rng = np.random.default_rng(rows)
    ra = gpu.DevBuf(src=(0.3 * rng.standard_normal((rows, n))).astype(F32)) if resid else None
    rb = gpu.DevBuf(src=(0.2 * rng.standard_normal((rows, n))).astype(F32)) if resid else None
    bufs = [gpu.DevBuf(src=v) if v is not None else None for v in (g1, b1, g2, b2)]
    p = [b.ptr if b is not None else None for b in bufs]
    gpu.lib().b200_layernorm_q(xd.ptr, n, ra.ptr if resid else None, rb.ptr if resid else None, p[0], p[1], A1.h, p[2], p[3],
                               A2.h if A2 is not None else None, n, rows)
    return xd, ra, rb


@gpu_mark
@pytest.mark.parametrize("dual_resid", [False, True])
@pytest.mark.parametrize("variant", list(LN_VARIANTS))
@pytest.mark.parametrize("at", ALL_AT)
def test_layernorm_quantiser_on_edge_rows(gpu, orc, monkeypatch, at, variant, dual_resid):
    """gamma = 0, beta = edge row: every row of the output must be Q(beta) (and Q(-beta) for the second pair)"""
    n, R, env = LN_VARIANTS[variant]
    if env:
        monkeypatch.setenv(env, "1")
    wt = ae.WTYPE_OF[at]
    rows, labels = ln_rows(at, variant)
    rng = np.random.default_rng(n + at)
    zero = np.zeros(n, F32)
    for r in range(rows.shape[0]):
        beta = rows[r]
        x = (rng.standard_normal((R, n)) * 2 + 0.5).astype(F32)
        A1 = gpu.ActQ(wt, n, R, f16=R > 1)
        A2 = gpu.ActQ(wt, n, R, f16=R > 1) if dual_resid else None
        _ln_launch(gpu, n, R, x, dual_resid, zero, beta, A1, zero if dual_resid else None, -beta if dual_resid else None, A2)
        for A, b, sign in ((A1, beta, "+"), (A2, -beta, "-"))[:2 if dual_resid else 1]:
            what = "%s %s row %d %sbeta" % (variant, po.TYPE_NAMES[at], r, sign)
            want = _want(orc, at, np.tile(b, (R, 1)))
            q, d = _check(at, A, want, np.tile(labels[r], (R, 1)), what)
            if R > 1:
                _check_plane(gpu, at, A, q, d, what)


@gpu_mark
@pytest.mark.parametrize("variant", list(LN_VARIANTS))
@pytest.mark.parametrize("at", ALL_AT)
def test_layernorm_quantiser_real_gamma_beta(gpu, orc, monkeypatch, at, variant):
    """real gamma / beta and the residual adds, both pairs, against the oracle's LayerNorm + quantiser (as test_layernorm_q_node)"""
    n, R, env = LN_VARIANTS[variant]
    if env:
        monkeypatch.setenv(env, "1")
    wt = ae.WTYPE_OF[at]
    rng = np.random.default_rng(3 * n + at)
    x = rng.standard_normal((R, n)).astype(F32)
    g1, g2 = [(1.0 + 0.1 * rng.standard_normal(n)).astype(F32) for _ in range(2)]
    b1, b2 = [(0.01 * rng.standard_normal(n)).astype(F32) for _ in range(2)]
    A1, A2 = gpu.ActQ(wt, n, R, f16=True), gpu.ActQ(wt, n, R, f16=True)
    xd, ra, rb = _ln_launch(gpu, n, R, x, True, g1, b1, A1, g2, b2, A2)
    xs = (ra.download(F32, (R, n)) + rb.download(F32, (R, n))) + x
    assert np.array_equal(xd.download(F32, (R, n)), xs)
    for A, g, b in ((A1, g1, b1), (A2, g2, b2)):
        q, d = _check(at, A, _want(orc, at, orc.layernorm(xs, g, b)), None, "%s %s real" % (variant, po.TYPE_NAMES[at]))
        _check_plane(gpu, at, A, q, d, "%s real" % variant)


# ------------------------------------------------------------------------------------------------ chain hand-over
def selector_blocks(wt, K, src, dexp=None):
    """raw Q4_K / Q4_0 blocks of M = len(src) rows: row m is +1 (times 2^dexp[m]) at k = src[m] and exactly 0 elsewhere.
    Q4_K: d = 2^dexp, dmin = 0, every sub-block scale 1 and min 0, code 1 at k, 0 elsewhere; blocks not holding k have d = 0.
    Q4_0: d = 2^dexp, codes 8 (zero) except 9 at k; other blocks have d = 0."""
    M = len(src)
    src = np.asarray(src)
    dexp = np.zeros(M, np.int64) if dexp is None else np.asarray(dexp)
    dh = np.ldexp(1.0, dexp).astype(np.float16).view(np.uint8).reshape(M, 2)
    rows = np.arange(M)
    if wt == po.Q4_K:
        nb = K // 256
        b = np.zeros((M, nb, 144), np.uint8)
        b[:, :, 4:8] = 1                                 # scales[0..3]: sub-blocks 0-3 scale 1, scales[4..7]: mins 0
        b[:, :, 12:16] = 1                               # scales[8..11]: sub-blocks 4-7 scale 1 (low nibble), min 0
        bi, e = src // 256, src % 256
        b[rows, bi, 0] = dh[:, 0]
        b[rows, bi, 1] = dh[:, 1]
        sb, i = e // 32, e % 32
        b[rows, bi, 16 + 32 * (sb // 2) + i] = (1 << (4 * (sb % 2))).astype(np.uint8)
    else:
        nb = K // 32
        b = np.zeros((M, nb, 18), np.uint8)
        b[:, :, 2:] = 0x88
        bi, i = src // 32, src % 32
        b[rows, bi, 0] = dh[:, 0]
        b[rows, bi, 1] = dh[:, 1]
        b[rows, bi, 2 + i % 16] = np.where(i < 16, 0x89, 0x98).astype(np.uint8)
    return b.reshape(M, -1)


@gpu_mark
@pytest.mark.parametrize("wt", list(CHAIN))
def test_chain_handover_on_edge_rows(gpu, orc, wt):
    exps, M = CHAIN[wt]
    at = po.VEC_DOT_TYPE[wt]
    x, where = _chain_source(wt, exps)
    K = x.size
    A_in = gpu.ActQ(wt, K, 1)
    xd = gpu.DevBuf(src=x)
    A_in.quantize(xd.ptr)
    qi, di, _, _ = A_in.download()
    assert np.array_equal(qi[0].astype(np.float64) * np.repeat(di[0], ae.BLK[at]), x)     # the input's quantisation is exact
    rows, labels = chain_rows(wt)
    yd = gpu.DevBuf(M * 4)
    for r in range(rows.shape[0]):
        dec = [_decompose(v, exps) for v in rows[r]]
        src = [where[(a, c)] for a, c, _ in dec]
        W = gpu.Weight(wt, K, M, selector_blocks(wt, K, src, [p for _, _, p in dec]))
        A_out = gpu.ActQ(wt, M, 1)
        assert gpu.lib().b200_mul_mat_vec_q_chain(W.h, A_in.h, yd.ptr, 0, A_out.h) == 1
        y = yd.download(F32, (M,))
        assert np.all(y == rows[r]), ("y is not the designed row", int(np.flatnonzero(y != rows[r])[0]))
        _check(at, A_out, _want(orc, at, y[None, :]), labels[r][None, :], "chain row %d" % r)


@gpu_mark
def test_chain_handover_gelu_real_width(gpu, orc):
    """ffn_up -> ffn_down at Falcon-40B width: GELU outputs on the fp16 grid contain half-way products and repeated magnitudes"""
    import ggllm_cpp_b200.ggcc as ggcc
    K, M, wt = 8192, 32768, po.Q4_K
    rng = np.random.default_rng(5)
    W = gpu.Weight(wt, K, M, ggcc.random_blocks(wt, M, K, rng))
    x = rng.standard_normal(K).astype(F32)
    A_in, A_out, yd = gpu.ActQ(wt, K, 1), gpu.ActQ(wt, M, 1), gpu.DevBuf(M * 4)
    xd = gpu.DevBuf(src=x)
    A_in.quantize(xd.ptr)
    assert gpu.lib().b200_mul_mat_vec_q_chain(W.h, A_in.h, yd.ptr, 1, A_out.h) == 1
    y = yd.download(F32, (M,))
    blocks = y.reshape(-1, 256)
    assert sum(ae.halfway(po.Q8_K, b).any() for b in blocks) >= 1         # the premise: the row has half-way products
    _check(po.Q8_K, A_out, _want(orc, po.Q8_K, y[None, :]), None, "chain gelu")


# ------------------------------------------------------------------------------------------------ attention hand-over
@gpu_mark
@pytest.mark.parametrize("tier", ATTN_TIERS)
@pytest.mark.parametrize("G,hkv,wt", ATTN)
def test_attention_handover_on_edge_rows(gpu, orc, monkeypatch, G, hkv, wt, tier):
    monkeypatch.setenv("B200_ATTN_LONG_FROM", "0" if tier == "long" else "1000000")      # long kernels above n_past + 1 > threshold
    at = po.VEC_DOT_TYPE[wt]
    n_head, hd, n_ctx = G * hkv, 64, 16
    rows, labels = attn_rows(G, hkv, wt, tier)
    rng = np.random.default_rng(G + hkv)
    for r in range(rows.shape[0]):
        v = rows[r]
        qkv = np.concatenate([rng.standard_normal((n_head + hkv) * hd).astype(F32), v])[None, :]
        kc = np.zeros((n_ctx, hkv, hd), F32)
        qd, kd, vd, od = gpu.DevBuf(src=qkv), gpu.DevBuf(src=kc), gpu.DevBuf(src=kc), gpu.DevBuf(n_head * hd * 4)
        A = gpu.ActQ(wt, n_head * hd, 1)
        long0 = gpu.lib().b200_attention_long_launches()
        assert gpu.lib().b200_attention_decode(qd.ptr, kd.ptr, vd.ptr, od.ptr, n_head, hkv, hd, 0, n_ctx, n_ctx, A.h) == 1
        assert (gpu.lib().b200_attention_long_launches() > long0) == (tier == "long")
        out = od.download(F32, (n_head * hd,))
        want_out = np.repeat(v.reshape(hkv, 1, hd), G, axis=1).reshape(-1)
        # split-KV kernel: the output is the V row, by value (0 + 1 * -0.0 accumulates to +0.0; either zero quantises to code 0).
        # The long-context kernel does not reproduce V bit for bit here, so its hand-over is checked against its own output row.
        if tier == "split":
            assert np.array_equal(out, want_out), ("output is not the V row", r, int(np.flatnonzero(out != want_out)[0]))
        # the edge label of each output block: it copies (part of) its kv head's V row
        blk = ae.BLK[at]
        e_out = np.arange(n_head * hd // blk) * blk
        e_v = e_out // hd // G * hd + (e_out % hd if blk < hd else 0)
        lab = labels[r][e_v // blk]
        _check(at, A, _want(orc, at, out[None, :]), lab[None, :], "attention %s G %d row %d" % (tier, G, r))
