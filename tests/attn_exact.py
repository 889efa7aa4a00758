"""Exact-arithmetic restatement of the attention kernels (numpy, float64) and a per-element error bound.

Each kernel family's header comment promises a sequence of roundings; this module applies exactly those roundings and computes
everything else in float64, so the only differences left between a kernel and `reference()` are the ones the bound accounts for.

  "fp32"  attention.cu (split-KV decode), attention_prefill.cu:
            s = fp32(q . k) * 0.125,  x = f16(fp32(s - max)),  e = f16(exp(x)),  sum in double,  out = sum_k v_k * (e_k * fp32(1 / sum))
  "long"  attention_long.cu (long-context split-KV decode): the "fp32" contract, but both products run on the tensor cores with every
            fp32 operand split into fp16 hi + lo terms (22 significant bits, absolute 2^-25 below 0.125, attention_long.cu:23-29)
  "ws"    attention_ws.cu (wgmma prompt attention): q, k, v rounded to fp16 first; x = f16(fma(s, 0.125, -max * 0.125)) -- the same
            value as fp32(s - max) -- e = f16(exp(x)) through ex2.approx, an fp32 sum of the fp16 e, and 1 / sum applied after P V

Bound, per output element (derivation next to each term in `reference`):
  acc    fp32 accumulation of the P V product (and of the ws row sum), at most one rounding per term: c * sum_k p_k |v_k|
  flip   a key whose x lies within the kernel's score error of an fp16 rounding midpoint may land on another fp16 value, and
         a key whose exp(x) lies within the kernel's exp error of a midpoint may round to the neighbouring e: that key's e moves by
         |de| and the output by |de| |v_k - out| / sum <= |de| (|v_k| + |out|) / sum
  long   the hi / lo split of V: sum_k p_k (2^-22 |v_k| + 2^-25)
"""
import numpy as np

U24 = 2.0 ** -24                 # fp32 unit roundoff (round to nearest)
U23 = 2.0 ** -23                 # one fp32 ulp: tensor-core accumulation is not guaranteed to round to nearest
KINDS = ("fp32", "long", "ws")


def f32(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


def f16(x):
    return np.asarray(x, np.float64).astype(np.float16).astype(np.float64)


def _nearest_midpoint(x):
    """x: float64 values. -> (distance from x to the nearest fp16 rounding midpoint, the fp16 value on the other side of it)"""
    h = np.asarray(x, np.float64).astype(np.float16)
    with np.errstate(over="ignore", invalid="ignore"):
        up, dn = np.nextafter(h, np.float16(np.inf)), np.nextafter(h, np.float16(-np.inf))
        h64, up64, dn64 = h.astype(np.float64), up.astype(np.float64), dn.astype(np.float64)
        du, dd = (h64 + up64) / 2 - x, x - (h64 + dn64) / 2
    use_up = du < dd
    return np.where(use_up, du, dd), np.where(use_up, up64, dn64)


def reference(q, K, V, n_past, kind, vis_offset=0, drop_key=None, v_swap_key=None, q_err=None):
    """q: [n_tok][n_head][64] rotated query rows (float32), K, V: [>= T][n_head_kv][64] cache rows with the new tokens' rows appended,
    T = n_past + n_tok; query token t sees keys [0, n_past + t + 1).  -> (out, bound), float64 [n_tok][n_head][64].
    q_err: [n_tok][n_head][64] bound on |kernel's q - q| per element, for kernels that rotate Q themselves; it moves each score by at
    most 0.125 sum_i q_err_i |k_i|, which joins the score error ds (and so the flip windows).
    Mutations that the sensitivity tests use to show the bound can fail: vis_offset widens every causal limit, drop_key hides one key
    from every row, v_swap_key takes that key's V row from the next KV head."""
    assert kind in KINDS
    q = np.asarray(q, np.float32)
    n_tok, n_head, D = q.shape
    T = n_past + n_tok
    HKV = K.shape[1]
    G = n_head // HKV
    out = np.zeros((n_tok, n_head, D))
    bound = np.zeros_like(out)
    keys = np.arange(T)
    for g in range(HKV):
        Kg = np.asarray(K[:T, g], np.float64)
        Vg = np.array(V[:T, g], np.float64)
        if v_swap_key is not None:
            Vg[v_swap_key] = V[v_swap_key, (g + 1) % HKV]
        Qg = q[:, g * G:(g + 1) * G].reshape(n_tok * G, D).astype(np.float64)      # row = token * G + head in group
        Eg = None if q_err is None else np.asarray(q_err, np.float64)[:, g * G:(g + 1) * G].reshape(n_tok * G, D)
        if kind == "ws":
            Qg, Kg, Vg = f16(Qg), f16(Kg), f16(Vg)
        absV = np.abs(Vg)
        og, bg = np.zeros((n_tok * G, D)), np.zeros((n_tok * G, D))
        for r0 in range(0, n_tok * G, 1024):
            Qr = Qg[r0:r0 + 1024]
            tok = (r0 + np.arange(Qr.shape[0])) // G
            vis = np.minimum(n_past + tok + 1 + vis_offset, T)
            mask = keys[None, :] < vis[:, None]
            if drop_key is not None:
                mask[:, drop_key] = False
            n_vis = mask.sum(1)
            s = f32(Qr @ Kg.T) * 0.125                              # fp16 operand products are exact in fp64 (ws)
            sabs = np.abs(Qr) @ np.abs(Kg).T
            # score error of the kernel against fp32(q . k) * 0.125: fp32 (or tensor-core) accumulation of 64 products
            if kind == "fp32":
                ds = 0.125 * (D + 1) * U24 * sabs
            elif kind == "ws":
                ds = 0.125 * D * U23 * sabs
            else:   # hi x lo + lo x hi + hi x hi: the dropped lo x lo term and the split's own error 2^-22 |x| (or 2^-25 below 0.125)
                ds = 0.125 * ((3 * 2.0 ** -22 + 16 * U23) * sabs
                              + 2.0 ** -25 * (np.abs(Qr).sum(1)[:, None] + np.abs(Kg).sum(1)[None, :]))
            if Eg is not None:
                ds = ds + 0.125 * (Eg[r0:r0 + 1024] @ np.abs(Kg).T)
            s = np.where(mask, s, -np.inf)
            m = s.max(1, keepdims=True)
            ds_m = np.take_along_axis(ds, s.argmax(1)[:, None], 1)
            with np.errstate(invalid="ignore"):
                xf = f32(s - m)                                     # fp32 subtraction (one rounding), then the fp16 LUT index
            x16 = np.where(mask, f16(xf), -np.inf)
            y = np.exp(x16)
            e = np.where(mask, f16(y), 0.0)
            ssum = e.sum(1, keepdims=True)
            inv = f32(1.0 / ssum)
            o = (e @ Vg) * inv
            spv = (e / ssum) @ absV
            # flip terms.  x: device and reference scores differ by <= ds each (the maximum's too), and fp32(s - max) adds 2^-24 |x|
            # on each side.  A key within that window of an fp16 midpoint of x may take another LUT index: any one in
            # [f16(x - win), f16(x + win)] -- near the maximum (|x| << 1) the fp16 spacing of x is finer than the window, so that is
            # several indices, not just the neighbouring one; e is monotonic in x, so the ends of the range bound the change.
            xs = np.where(mask, xf, 0.0)
            dist, _ = _nearest_midpoint(xs)
            win = ds + ds_m + 2 * U24 * np.abs(xs)
            e_lo, e_hi = f16(np.exp(f16(xs - win))), f16(np.exp(f16(np.minimum(xs + win, 0.0))))
            de_x = np.where(mask & (dist <= win), np.maximum(np.abs(e_lo - e), np.abs(e_hi - e)), 0.0)
            # e: expf is within 2 ulp (2^-22 relative); ex2.approx.ftz within 2 ulp of 2^(x * log2 e), whose argument carries the fp32
            # rounding of that product (|x| 2^-24 relative in the result) -- a key within that of an fp16 midpoint of e may round the
            # other way
            rel = 2.0 ** -22 if kind != "ws" else 2.0 ** -21 + np.abs(xs) * U23
            ys = np.where(mask, y, 1.0)
            dist_e, alt_e = _nearest_midpoint(ys)
            de_e = np.where(mask & (dist_e <= rel * ys), np.abs(alt_e - e), 0.0)
            dE = de_x + de_e
            flip = (dE @ absV + dE.sum(1, keepdims=True) * np.abs(o)) / ssum
            # accumulation: p V in fp32 with <= one rounding per key (u for CUDA-core fp32, one ulp for the tensor cores) plus
            # fp32(1 / sum) and the final product; ws also sums the fp16 e in fp32 (the same relative error lands on out)
            nv = n_vis[:, None].astype(np.float64)
            if kind == "ws":
                c = (nv + 8) * U23 + (nv + 4) * U24
            elif kind == "long":
                c = (nv + 4) * U23 + 2.0 ** -22
            else:
                c = (nv + 4) * U24
            b = c * spv + flip + (2.0 ** -25 if kind == "long" else 0.0) + 1e-30
            og[r0:r0 + Qr.shape[0]], bg[r0:r0 + Qr.shape[0]] = o, b
        out[:, g * G:(g + 1) * G] = og.reshape(n_tok, G, D)
        bound[:, g * G:(g + 1) * G] = bg.reshape(n_tok, G, D)
    return out, bound
