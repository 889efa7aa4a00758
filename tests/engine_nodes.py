"""Node-by-node check of one Falcon eval from the engine's test tap (b200_falcon_tap).

The logit comparisons of test_falcon_gpu.py cannot see a defect whose effect stays under 2e-3 of the logit scale, because a 1e-7
summation-order difference flips int8 activation codes and the flips spread.  Checked from the engine's OWN input to each node that
noise is gone: the device quantisers are bit-exact with the CPU and the integer block dots are exact, so every node has a tight bound.

  (a) residual chain      inp[0] = embedding rows, inp[l+1] = (dn[l] + ao[l]) + inp[l] (fp32), the final residual likewise: bit-exact
  (b) LayerNorm + Q8      xa / xm / xf = quantize_act(layernorm(inp)): bit-exact; generic path: fp32 gen_na / gen_nm to 1e-6
  (c) mat-muls            qkv, ao, up, dn, logits from the engine's codes: N <= mmv_max_n mmv_exact.reference at the launch shape;
                          larger N the fp64 product of fp16(W) and the fp16 operand (tensor-core accumulation bound), the operand
                          planes bit-exact with actq_edges.f16_plane; up on the fp16 GELU grid (gelu_ok)
  (d) RoPE + KV append    cache V rows [n_past, n_past + N) = qkv's V part, K rows = RoPE of qkv's K part (see rope64), every other row
                          unchanged, the fp16 shadow = fp16 of the cache
  (e) attention           att against attn_exact.reference, kind of the tier the engine took
  (f) hand-overs          xatt = Q(att), xup = Q(up): bit-exact
  (g)                     the logits the eval returned = the tapped logits node

RoPE bound (rope64).  Pair i of a head at position p has theta = p * scale^i built by repeated fp32 products on the device and here
alike, so theta is the same fp32 value on both sides; the device then forms x0 c' - x1 s' and x0 s' + x1 c' with cosf / sinf within
2 ulp (c' = c (1 + e), |e| <= 2^-22) and every product and the sum rounded once.  Against the float64 rotation with exact cos / sin of
that theta the error of one output is at most (|x0 c| + |x1 s|) (2^-22 + gamma(2)) to first order; a 2^-20 relative margin covers the
second-order terms.  Where the attention kernels rotate Q themselves (qkv_rotated == 0) that per-element bound, plus the fp32 rounding
of the float64 rotation handed to attn_exact, is its q_err term.

A failing node raises NodeError naming the node and the layer (-1: the head).
"""
import numpy as np
import pyoracle as po
import actq_edges
import attn_exact
import mmv_exact

U = 2.0 ** -24
FLOATS = (po.F16, po.F32)


class NodeError(AssertionError):
    def __init__(self, node, layer, msg):
        super().__init__("layer %d node %s: %s" % (layer, node, msg))
        self.node, self.layer = node, layer


def need(ok, node, layer, msg):
    if not ok:
        raise NodeError(node, layer, msg)


class Model:
    """hp and the tensors dict ({name: (ggml type, ne, raw array)}) the engine was given"""

    def __init__(self, hp, tensors):
        self.hp, self.t = hp, tensors
        self.E, self.H, self.HKV = hp["n_embd"], hp["n_head"], hp["n_head_kv"]
        self.D = self.E // self.H
        self.QKV, self.FF, self.V = (self.H + 2 * self.HKV) * self.D, 4 * self.E, hp["n_vocab"]
        self.dual = hp["falcon_type"] == 40

    def name(self, l, what):
        p = "transformer.h.%d." % l
        return p + {"qkv": "self_attention.query_key_value.weight", "wo": "self_attention.dense.weight", "up": "mlp.dense_h_to_4h.weight",
                    "down": "mlp.dense_4h_to_h.weight"}[what]

    def ln(self, l, which):
        p = "transformer.h.%d." % l
        base = {"attn": "ln_attn", "mlp": "ln_mlp" if self.dual else "input_layernorm"}[which]
        return self.t[p + base + ".weight"][2], self.t[p + base + ".bias"][2]

    def wtype(self, name):
        return self.t[name][0]

    def raw(self, name):
        t, ne, a = self.t[name]
        return np.ascontiguousarray(a).reshape(ne[1], -1)

    def raw_rows(self, name, rows):
        """the stored rows `rows` of a matrix (a model built lazily overrides this to make only those rows)"""
        return self.raw(name)[rows]

    def rows(self, name, rows):
        """float32 dequantised rows of a matrix"""
        t, ne, _ = self.t[name]
        r = self.raw_rows(name, rows)
        if t == po.F32:
            return r.view(np.float32) if r.dtype == np.uint8 else r.astype(np.float32)
        if t == po.F16:
            return (r.view(np.float16) if r.dtype == np.uint8 else r).astype(np.float32)
        return po.orc().dequantize(t, r, ne[0])


class Eval:
    """what one eval was: tokens at n_past, the head's first row r0, the KV cache of every local layer before and after it
    (kv_* [l] = (K, V) float32 [n_ctx][n_head_kv * head_dim]), the fp16 shadow after it (shadow[l] = (k16, vt16) of rows [0, T) or
    None), the logits the call returned, RoPE's theta scale, the mat-vec launch shape per (type, K) (mmv_exact.depth's kernel tuple),
    the attention kind (attn_exact.KINDS) and, at real widths, a subset of mat-mul output rows (rows_subset)."""

    def __init__(self, tokens, n_past, r0, kv_before, kv_after, shadow, logits, theta_scale, kernel_of, attn_kind, mmv_max_n=8,
                 rows_subset=False):
        self.tokens = np.asarray(tokens, np.int32)
        self.N, self.n_past, self.r0 = self.tokens.size, n_past, r0
        self.kv_before, self.kv_after, self.shadow, self.logits = kv_before, kv_after, shadow, logits
        self.theta_scale, self.kernel_of, self.attn_kind, self.mmv_max_n = theta_scale, kernel_of, attn_kind, mmv_max_n
        self.rows_subset = rows_subset


def attention_kind(N, n_past, shadow, mmv_max_n=8, long_from=1024):
    """the kernel family launch_attention takes: split-KV decode (long-context tier above long_from keys), wgmma prompt attention
    where an fp16 shadow exists and N exceeds the mat-vec batch, the fp32 prefill otherwise"""
    if N == 1:
        return "long" if n_past + 1 > long_from else "fp32"
    return "ws" if shadow and N > mmv_max_n else "fp32"


def output_rows(M, subset):
    """all rows, or the first and last row of every 128-row tile and row M - 1"""
    if not subset:
        return np.arange(M)
    t = np.arange(0, M, 128)
    return np.unique(np.concatenate([t, np.minimum(t + 127, M - 1), [M - 1]]))


# ------------------------------------------------------------------------------------------------ RoPE
def thetas(positions, D, scale):
    """[len(positions)][D/2] float64 values of the fp32 angles both sides use"""
    th = np.empty((len(positions), D // 2))
    cur = np.asarray(positions, np.float32)
    sc = np.float32(scale)
    for i in range(D // 2):
        th[:, i] = cur
        cur = (cur * sc).astype(np.float32)
    return th


def rope64(x, positions, scale):
    """x [N][heads][D] -> (the float64 NeoX rotation with exact cos / sin of the fp32 angles, the device's error bound on it)"""
    x = np.asarray(x, np.float64)
    D = x.shape[-1]
    th = thetas(positions, D, scale)[:, None, :]
    c, s = np.cos(th), np.sin(th)
    x0, x1 = x[..., :D // 2], x[..., D // 2:]
    out = np.concatenate([x0 * c - x1 * s, x0 * s + x1 * c], -1)
    mag = np.concatenate([np.abs(x0 * c) + np.abs(x1 * s), np.abs(x0 * s) + np.abs(x1 * c)], -1)
    return out, mag * (2.0 ** -22 + mmv_exact.gamma(2)) * (1 + 2.0 ** -20)


# ------------------------------------------------------------------------------------------------ activations
def quantize(wtype, x, K):
    """orc.quantize_act of fp32 rows in the device's ActQ layout: (q, d, s or None, bs)"""
    at = po.VEC_DOT_TYPE[wtype]
    return actq_edges.parse(at, po.orc().quantize_act(wtype, np.asarray(x, np.float32).reshape(-1, K)), K)


def tapped_actq(nodes, name, wtype, K, N):
    at = po.VEC_DOT_TYPE[wtype]
    blk = actq_edges.BLK[at]
    q = nodes[name + ".q"].reshape(N, K)
    d = nodes[name + ".d"].reshape(N, K // blk)
    s = nodes[name + ".s"].reshape(N, K // 32) if at == po.Q8_1 else None
    bs = nodes[name + ".bs"].reshape(N, -1)
    return q, d, s, bs


def check_actq(got, want, node, layer):
    """bit-exact: codes, scales, Q8_1 sums (where the type has them) and block sums"""
    for part, a, b in zip(("codes", "scales", "sums", "block sums"), got, want):
        if b is None:
            continue
        a = np.ascontiguousarray(a)
        b = np.ascontiguousarray(b, a.dtype).reshape(a.shape)
        bad = np.argwhere(a.view(np.uint8).reshape(a.shape[0], -1, a.itemsize) != b.view(np.uint8).reshape(a.shape[0], -1, a.itemsize))
        need(bad.size == 0, node, layer, "%s differ, first (token, index) %s" % (part, bad[:1, :2].tolist()))


# ------------------------------------------------------------------------------------------------ mat-muls
GELU_SLOPE = 1.13            # max |d gelu / dx| (1.1289 at x = 1.53): an input error e moves the output by at most 1.13 e


def _half_f16_spacing(v):
    h = np.asarray(v, np.float64).astype(np.float16)
    with np.errstate(over="ignore", invalid="ignore"):
        return np.abs(np.nextafter(h, np.float16(np.inf)).astype(np.float64) - h.astype(np.float64)) / 2


def gelu_ok(got, y, b):
    """GELU outputs of pre-GELU values y known within b.  Where b stays within half an fp16 spacing of y and the fp32 formula's error
    within half an fp16 spacing of the output, mmv_exact.gelu_ok: GELU of f16(y) or of its neighbour across the nearest midpoint.
    Elsewhere several fp16 inputs or outputs are possible -- b spans several inputs (the tensor-core GEMM's budget at small |y|), or the
    output is an fp16 subnormal (large negative y, where 1 + tanhf(arg) cancels and tanhf's 2-ulp error, 0.5 |f| 8 u absolute, exceeds
    the output spacing) -- and the check is an interval: |got - gelu(y)| <= 1.13 (b + the input's fp16 rounding) + the formula's error
    + the output's fp16 rounding (1.13 = max |d gelu / dx|, at x = 1.53)."""
    y = np.asarray(y, np.float64)
    g = 0.5 * y * (1.0 + np.tanh(0.7978845608028654 * y * (1.0 + 0.044715 * y * y)))
    din = b + (np.abs(y) + b) * 2.0 ** -11 + 2.0 ** -25
    fm = np.abs(y) + din
    ferr = 0.5 * fm * 8 * U * (1 + 0.7978845608028654 * fm * (1 + 0.044715 * fm * fm)) + 8 * U * np.abs(g)
    dout = GELU_SLOPE * din + ferr
    tot = dout + (np.abs(g) + dout) * 2.0 ** -11 + 2.0 ** -25
    wide = (b > _half_f16_spacing(y)) | (ferr > _half_f16_spacing(g))
    return np.where(wide, np.abs(np.asarray(got, np.float64) - g) <= tot, mmv_exact.gelu_ok(got, y, b))


def matmul_reference(m, wname, act, N, ev, rows):
    """exact outputs [N][rows] and their bounds for the engine's input to matrix `wname`: act = (q, d, s, bs) codes for a quantised
    matrix, fp32 rows [N][K] for F16 / F32"""
    t = m.wtype(wname)
    K = m.t[wname][1][0]
    if t not in FLOATS:
        q, d, s, _ = act
        if N <= ev.mmv_max_n:
            y, b = np.zeros((N, len(rows))), np.zeros((N, len(rows)))
            s0 = s if s is not None else np.zeros((N, K // 32), np.float32)
            wq = m.raw_rows(wname, rows)
            for n in range(N):
                y[n], b[n], _, _ = mmv_exact.reference(t, wq, K, q[n], d[n], s0[n], ev.kernel_of(t, K))
            return y, b
        x = actq_edges.f16_plane(po.VEC_DOT_TYPE[t], q, d).astype(np.float64)
    elif t == po.F16 and N > ev.mmv_max_n:
        x = np.asarray(act, np.float32).astype(np.float16).astype(np.float64)
    else:
        w = m.rows(wname, rows)
        y, b = np.zeros((N, len(rows))), np.zeros((N, len(rows)))
        for n in range(N):
            y[n], b[n] = mmv_exact.f_reference(t, w, act[n])
        return y, b
    # tensor-core GEMM: the fp64 product of the fp16 operands is exact; the fp32 accumulation runs through K / 16 k16 MMA steps and the
    # tensor cores do not round to nearest -- each step may lose up to one ulp in its internal sum and one in the accumulator update,
    # and truncation does not cancel (same-signed terms at K = 32768 show it: a bias of 4e-5 of sum |x w|) -- plus two roundings for a
    # split-K partial's atomicAdd: (K / 8 + 2) 2^-23 sum_k |x_k w_k|
    w = m.rows(wname, rows).astype(np.float16).astype(np.float64)
    return x @ w.T, (K / 8 + 2) * 2.0 ** -23 * (np.abs(x) @ np.abs(w).T) + 1e-30


def check_matmul(node, layer, m, wname, got, act, ev, gelu=False, rope=None):
    """got [N][M] tapped fp32 output.  rope = positions: qkv was rotated in place, so its Q and K parts are compared with the rotation
    of the exact outputs (error: the rotated mat-mul bound plus rope64's bound)"""
    N, M = got.shape
    rows = output_rows(M, ev.rows_subset)
    D = m.D
    nqk = (m.H + m.HKV) * D
    if rope is not None:                           # a rotated output needs its partner 32 elements away: take whole heads
        heads = np.unique(rows[rows < nqk] // D)
        rows = np.unique(np.concatenate([rows, (heads[:, None] * D + np.arange(D)).ravel()]))
    y, b = matmul_reference(m, wname, act, N, ev, rows)
    g = got[:, rows].astype(np.float64)
    if rope is not None:
        sel = np.nonzero(rows < nqk)[0]
        yh, bh = y[:, sel].reshape(N, -1, D), b[:, sel].reshape(N, -1, D)
        ry, _ = rope64(yh, rope, ev.theta_scale)
        th = thetas(rope, D, ev.theta_scale)[:, None, :]
        c, s = np.abs(np.cos(th)), np.abs(np.sin(th))
        b0, b1 = bh[..., :D // 2], bh[..., D // 2:]
        _, rerr = rope64(np.abs(yh) + bh, rope, ev.theta_scale)           # the device rotates its own outputs, within bh of yh
        y[:, sel] = ry.reshape(N, -1)
        b[:, sel] = (np.concatenate([b0 * c + b1 * s, b0 * s + b1 * c], -1) + rerr).reshape(N, -1)
    ok = gelu_ok(g, y, b) if gelu else np.abs(g - y) <= b
    bad = np.argwhere(~ok)
    need(bad.size == 0, node, layer, "%d of %d outputs outside the bound, first (token, row) %s: got %r want %r bound %r" % (
        len(bad), ok.size, bad[:1].tolist(), *([float(g[tuple(bad[0])]), float(y[tuple(bad[0])]), float(b[tuple(bad[0])])] if bad.size else [0, 0, 0])))


# ------------------------------------------------------------------------------------------------ one eval
def check_residuals(m, ev, residuals, head):
    """(a) alone over every layer: residuals[l] = {"inp", "ao", "dn"} of layer l = 0 .. n_layer - 1 (a tap of those three nodes is
    enough), head: the nodes after the head.  Raises NodeError at the first residual that is not exact."""
    N, E = ev.N, m.E
    want = m.rows("transformer.word_embeddings.weight", ev.tokens)
    for l, nd in enumerate(list(residuals) + [head]):
        got = nd["inp"].reshape(N, E)
        need(np.array_equal(got.view(np.uint32), want.view(np.uint32)), "inp", l if l < len(residuals) else -1,
             "not the embedding rows of the tokens" if l == 0 else "not (dn + ao) + inp of the layer before")
        if l < len(residuals):
            want = (nd["dn"].reshape(N, E) + nd["ao"].reshape(N, E)) + got


def check_eval(m, ev, layers, head, rotated, layer_ids=None):
    """layers[i]: {node: array} of local layer layer_ids[i] (default 0, 1, ...), head: the nodes after the head (None on a rank without
    it), rotated[i]: the tap's qkv_rotated.  The residual check (a) links layer_ids[i] to layer_ids[i - 1] only where they are
    consecutive, and the final residual to the last layer only where it is checked.  Raises NodeError at the first node that fails."""
    orc = po.orc()
    N, E, D, H, HKV = ev.N, m.E, m.D, m.H, m.HKV
    layer_ids = list(range(len(layers))) if layer_ids is None else layer_ids
    pos = ev.n_past + np.arange(N)
    T = ev.n_past + N
    prev, prev_l = None, None
    for i, (l, nd) in enumerate(zip(layer_ids, layers)):
        inp = nd["inp"].reshape(N, E)
        generic = "gen_nm" in nd
        # (a): linked to the layer before only where layer_ids holds it
        if prev_l is not None and l != prev_l + 1:
            prev = None
        if prev is None:
            if l == 0:
                want = m.rows("transformer.word_embeddings.weight", ev.tokens)
                need(np.array_equal(inp.view(np.uint32), want.view(np.uint32)), "inp", l, "not the embedding rows of the tokens")
        else:
            want = (prev["dn"].reshape(N, E) + prev["ao"].reshape(N, E)) + prev["inp"].reshape(N, E)
            need(np.array_equal(inp.view(np.uint32), want.view(np.uint32)), "inp", l, "not (dn + ao) + inp of the layer before")
        prev_l = l
        # (b)
        wq_name, wo_name, up_name, dn_name = (m.name(l, k) for k in ("qkv", "wo", "up", "down"))
        ln_m = orc.layernorm(inp, *m.ln(l, "mlp"))
        ln_a = orc.layernorm(inp, *m.ln(l, "attn")) if m.dual else ln_m
        if generic:
            need(np.allclose(nd["gen_nm"].reshape(N, E), ln_m, rtol=0, atol=1e-6), "gen_nm", l, "LayerNorm output")
            if m.dual:
                need(np.allclose(nd["gen_na"].reshape(N, E), ln_a, rtol=0, atol=1e-6), "gen_na", l, "LayerNorm output")
            x_qkv = nd["gen_na" if m.dual else "gen_nm"].reshape(N, E)
            x_up = nd["gen_nm"].reshape(N, E)

            def act_of(wname, x):
                t = m.wtype(wname)
                return np.asarray(x, np.float32) if t in FLOATS else quantize(t, x, m.t[wname][1][0])
            a_qkv, a_up = act_of(wq_name, x_qkv), act_of(up_name, x_up)
        else:
            wt = m.wtype(wq_name)
            a_up = tapped_actq(nd, "xm", wt, E, N)
            check_actq(a_up, quantize(wt, ln_m, E), "xm", l)
            if m.dual:
                a_qkv = tapped_actq(nd, "xa", wt, E, N)
                check_actq(a_qkv, quantize(wt, ln_a, E), "xa", l)
            else:
                a_qkv = a_up
        gemm = N > ev.mmv_max_n
        if gemm and not generic:
            want = actq_edges.f16_plane(po.VEC_DOT_TYPE[wt], a_up[0], a_up[1])
            need(np.array_equal(nd["xh_m"].reshape(N, E).view(np.uint16), want.view(np.uint16)), "xh_m", l, "not fp16(d q) of xm")
        # (c) qkv, (d) RoPE + KV append
        qkv = nd["qkv"].reshape(N, m.QKV)
        rot = bool(rotated[i])
        check_matmul("qkv", l, m, wq_name, qkv, a_qkv, ev, rope=pos if rot else None)
        q3 = qkv.reshape(N, H + 2 * HKV, D)
        Kb, Vb = ev.kv_before[i]
        Ka, Va = ev.kv_after[i]
        outside = np.ones(Ka.shape[0], bool)
        outside[ev.n_past:T] = False
        need(np.array_equal(Ka[outside].view(np.uint32), Kb[outside].view(np.uint32)), "k_cache", l, "rows outside the new positions changed")
        need(np.array_equal(Va[outside].view(np.uint32), Vb[outside].view(np.uint32)), "v_cache", l, "rows outside the new positions changed")
        need(np.array_equal(Va[ev.n_past:T].view(np.uint32), q3[:, H + HKV:].reshape(N, -1).view(np.uint32)), "v_cache", l,
             "new V rows are not qkv's V part")
        k_new = Ka[ev.n_past:T].reshape(N, HKV, D)
        if rot:
            need(np.array_equal(k_new.view(np.uint32), q3[:, H:H + HKV].view(np.uint32)), "k_cache", l, "new K rows are not qkv's rotated K part")
            q_rot, q_err = q3[:, :H], None
        else:
            kr, kerr = rope64(q3[:, H:H + HKV], pos, ev.theta_scale)
            need(np.all(np.abs(k_new - kr) <= kerr), "k_cache", l, "new K rows are not RoPE of qkv's K part (max excess %g)" % float(
                (np.abs(k_new - kr) - kerr).max()))
            q64, q_err = rope64(q3[:, :H], pos, ev.theta_scale)
            q_rot = q64.astype(np.float32)
            q_err = q_err + U * np.abs(q64)
        if ev.shadow is not None and ev.shadow[i] is not None:
            k16, vt16 = ev.shadow[i]
            need(np.array_equal(k16.reshape(T, -1), Ka[:T].astype(np.float16).view(np.uint16)), "k16", l, "shadow is not fp16 of the K cache")
            need(np.array_equal(vt16.reshape(HKV * D, T), Va[:T].astype(np.float16).view(np.uint16).T), "vt16", l,
                 "shadow is not fp16 of the V cache")
        # (e)
        att = nd["att"].reshape(N, H, D)
        out, bound = attn_exact.reference(q_rot, Ka[:T].reshape(T, HKV, D), Va[:T].reshape(T, HKV, D), ev.n_past, ev.attn_kind, q_err=q_err)
        bad = np.argwhere(np.abs(att - out) > bound)
        need(bad.size == 0, "att", l, "%d outputs outside the %s bound, first (token, head, i) %s" % (len(bad), ev.attn_kind, bad[:1].tolist()))
        # (f) + (c) wo
        att2 = nd["att"].reshape(N, E)
        if generic:
            a_wo = act_of(wo_name, att2)
        else:
            a_wo = tapped_actq(nd, "xatt", wt, E, N)
            check_actq(a_wo, quantize(wt, att2, E), "xatt", l)
            if gemm:
                want = actq_edges.f16_plane(po.VEC_DOT_TYPE[wt], a_wo[0], a_wo[1])
                need(np.array_equal(nd["xh_a"].reshape(N, E).view(np.uint16), want.view(np.uint16)), "xh_a", l, "not fp16(d q) of xatt")
        check_matmul("ao", l, m, wo_name, nd["ao"].reshape(N, E), a_wo, ev)
        # (c) up + GELU, (f) xup, (c) dn
        up = nd["up"].reshape(N, m.FF)
        check_matmul("up", l, m, up_name, up, a_up, ev, gelu=True)
        if generic:
            a_dn = act_of(dn_name, up)
        else:
            a_dn = tapped_actq(nd, "xup", wt, m.FF, N)
            check_actq(a_dn, quantize(wt, up, m.FF), "xup", l)
            if gemm:
                want = actq_edges.f16_plane(po.VEC_DOT_TYPE[wt], a_dn[0], a_dn[1])
                need(np.array_equal(nd["xh_b"].reshape(N, m.FF).view(np.uint16), want.view(np.uint16)), "xh_b", l, "not fp16(d q) of xup")
        check_matmul("dn", l, m, dn_name, nd["dn"].reshape(N, E), a_dn, ev)
        prev = nd
    if head is None:
        return
    # the head: (a) final residual (when the last layer was checked), (b) LayerNorm, (c) lm_head, (g) returned logits
    nr = N - ev.r0
    fin = head["inp"].reshape(N, E)
    if prev is not None and prev_l == m.hp["n_layer"] - 1:
        want = (prev["dn"].reshape(N, E) + prev["ao"].reshape(N, E)) + prev["inp"].reshape(N, E)
        need(np.array_equal(fin.view(np.uint32), want.view(np.uint32)), "inp", -1, "final residual is not (dn + ao) + inp of the last layer")
    ln = orc.layernorm(fin[ev.r0:], m.t["transformer.ln_f.weight"][2], m.t["transformer.ln_f.bias"][2])
    lm = "lm_head.weight"
    t = m.wtype(lm)
    if "gen_na" in head:
        x = head["gen_na"].reshape(nr, E)
        need(np.allclose(x, ln, rtol=0, atol=1e-6), "gen_na", -1, "final LayerNorm output")
        act = x if t in FLOATS else quantize(t, x, E)
    else:
        act = tapped_actq(head, "xf", t, E, nr)
        check_actq(act, quantize(t, ln, E), "xf", -1)
    logits = head["logits"].reshape(nr, m.V)
    check_matmul("logits", -1, m, lm, logits, act, ev)
    if ev.logits is not None:
        need(np.array_equal(np.asarray(ev.logits, np.float32).reshape(-1, m.V).view(np.uint32), logits[-len(ev.logits):].view(np.uint32)),
             "returned", -1, "the logits the eval returned are not the tapped logits")
