"""An exact restatement of falcon_main's sampling chain (the reference's llama_sample_* calls in the order of oracle/ref_sample_chain.cpp),
stage by stage, with the float transcendentals passed in, and the stage checker the sampler tests use.

Two sets of transcendentals:
- GLIBC: this host's expf / logf / log2f / powf through ctypes, the functions the live reference resolves.
- CR: correctly rounded float(f(double(x))), what sampling.cu evaluates (ref_expf, ref_logf, ...).
glibc's float functions are not correctly rounded (logf differs from CR on about 0.7 % of probabilities), so twin(GLIBC) is held to
the reference and twin(CR) to the device, each bit for bit at every stage; where the two twins differ, a divergence between the device
and the reference is explained rather than tolerated.

Arithmetic is the reference's: every fp32 sum is sequential from 0.0f (np.add.accumulate on float32 is a sequential loop), elementwise
fp32 operations round once, mirostat's three fused multiply-adds round once (computed exactly with fractions), equal logits are
ordered by ascending id and equal typical scores by position (the device's order; the reference's std::sort leaves them unspecified,
which compare_ref allows for), and the draw is libstdc++'s discrete_distribution over std::mt19937.

Stages (the candidate list after each step, as refh_sample_chain_stages and b200_sampler_tap report them): row (logits after bias and
penalties, id order), order (after top-k / the whole-row sort; mirostat: after the temperature), tfs, typical, top_p, temp, final.
Each is {"n", "ids", "logits", "p"}; the reference's p after top-k and the device's p after order / temp are not compared."""
import ctypes as C
from fractions import Fraction
import numpy as np

f32 = np.float32
STAGES = ("row", "order", "tfs", "typical", "top_p", "temp", "final")


class _Glibc:
    name = "glibc"

    def __init__(self):
        m = C.CDLL("libm.so.6")
        self._f = {}
        for fn in ("expf", "logf", "log2f"):
            f = getattr(m, fn)
            f.restype, f.argtypes = C.c_float, [C.c_float]
            self._f[fn] = f
        self._pow = m.powf
        self._pow.restype, self._pow.argtypes = C.c_float, [C.c_float, C.c_float]

    def _v(self, fn, x):
        f = self._f[fn]
        return np.fromiter((f(v) for v in np.atleast_1d(np.asarray(x, f32)).tolist()), f32, count=np.size(x))

    def exp(self, x): return self._v("expf", x)
    def log(self, x): return self._v("logf", x)
    def log2(self, x): return self._v("log2f", x)
    def pow(self, x, y): return f32(self._pow(float(x), float(y)))


class _CR:
    name = "cr"

    def _v(self, f, x):
        with np.errstate(all="ignore"):
            return f(np.atleast_1d(np.asarray(x, f32)).astype(np.float64)).astype(f32)

    def exp(self, x): return self._v(np.exp, x)
    def log(self, x): return self._v(np.log, x)
    def log2(self, x): return self._v(np.log2, x)

    def pow(self, x, y):
        with np.errstate(all="ignore"):
            return f32(np.power(np.float64(x), np.float64(y)))


GLIBC, CR = _Glibc(), _CR()


class MT19937:
    """std::mt19937 seeded like std::mt19937(seed)"""

    def __init__(self, seed):
        mt = [seed & 0xffffffff]
        for i in range(1, 624):
            mt.append((1812433253 * (mt[-1] ^ (mt[-1] >> 30)) + i) & 0xffffffff)
        self.mt, self.i = mt, 624

    def next(self):
        mt = self.mt
        if self.i >= 624:
            for i in range(624):
                y = (mt[i] & 0x80000000) | (mt[(i + 1) % 624] & 0x7fffffff)
                mt[i] = mt[(i + 397) % 624] ^ (y >> 1) ^ (0x9908b0df if y & 1 else 0)
            self.i = 0
        y = mt[self.i]
        self.i += 1
        y ^= y >> 11
        y ^= (y << 7) & 0x9d2c5680
        y ^= (y << 15) & 0xefc60000
        y ^= y >> 18
        return y


def fsum(x):
    """float s = 0.0f; for (...) s += x[i];"""
    return np.add.accumulate(np.concatenate(([f32(0)], np.asarray(x, f32))))[-1]


def round_f32(q):
    """the float nearest to the rational q (ties to even): one rounding, as a fused multiply-add does"""
    c = f32(float(q))                                   # within one float ulp of q
    best = None
    for v in (np.nextafter(c, f32(-np.inf)), c, np.nextafter(c, f32(np.inf))):
        if not np.isfinite(v):
            continue
        d = abs(Fraction(float(v)) - q)
        if best is None or d < best[0] or (d == best[0] and int(v.view(np.uint32)) % 2 == 0):
            best = (d, v)
    return best[1]


def fma32(a, b, c):
    if not (np.isfinite(a) and np.isfinite(b) and np.isfinite(c)):
        return f32(np.float64(a) * np.float64(b) + np.float64(c))      # inf / NaN propagate the same way
    return round_f32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def x86_int(x):
    """int(float) as cvttss2si computes it: NaN and anything outside int32 give INT_MIN"""
    x = f32(x)
    return int(x) if (x > f32(-2147483904.0) and x < f32(2147483648.0)) else -2 ** 31


def canonical(mt):
    """generate_canonical<double, 53>(mt19937): two outputs, (x0 + x1 2^32) / 2^64 in double"""
    x0 = mt.next()
    x1 = mt.next()
    u = (float(x0) + float(x1) * 4294967296.0) / 18446744073709551616.0
    return u if u < 1.0 else float(np.nextafter(1.0, 0.0))


def discrete_table(p, force_last=True):
    """libstdc++'s discrete_distribution: probabilities as double, divided by their sequential sum, partial sums, last entry 1.0"""
    d = np.asarray(p, f32).astype(np.float64)
    s = np.add.accumulate(np.concatenate(([0.0], d)))[-1]
    cp = np.add.accumulate(d / s)
    if force_last:
        cp[-1] = 1.0
    return cp


def draw(p, mt, force_last=True):
    """-> (position, u); fewer than two entries draw nothing (libstdc++'s empty table)"""
    if len(p) < 2:
        return 0, -1.0
    u = canonical(mt)
    cp = discrete_table(p, force_last)
    return int(min(np.searchsorted(cp, u, side="left"), len(p) - 1)), u


def softmax(l, fn):
    """llama_sample_softmax over l in the order held: p = expf(l - l[0]) / sequential sum"""
    with np.errstate(all="ignore"):                              # an all -inf list gives NaN, as in the reference
        e = fn.exp((np.asarray(l, f32) - l[0]).astype(f32))
        return (e / fsum(e)).astype(f32)


def _lst(ids, l, p=None):
    return dict(n=len(ids), ids=np.asarray(ids, np.int32), logits=np.asarray(l, f32), p=None if p is None else np.asarray(p, f32))


def penalised_row(row, win, c, defects=()):
    """logit bias, llama_sample_repetition_penalty, llama_sample_frequency_and_presence_penalties (candidates in id order)"""
    r = np.array(row, f32)
    V = r.size
    for i, v in (c.get("logit_bias") or {}).items():
        r[i] = f32(r[i] + f32(v))
    w = [int(t) for t in win]
    if not w:
        return r
    ids, counts = np.unique(np.array(w, np.int64), return_counts=True)
    per_occurrence = "penalty_per_occurrence" in defects
    for i, n in zip(ids.tolist(), counts.tolist()):
        if not 0 <= i < V:
            continue
        l = r[i]
        for _ in range(n if per_occurrence else 1):
            if c["repeat_penalty"] != 1.0:
                pen = f32(c["repeat_penalty"])
                l = f32(l * pen) if l <= 0 else f32(l / pen)
        if c["frequency_penalty"] != 0.0 or c["presence_penalty"] != 0.0:
            l = f32(l - f32(f32(f32(n) * f32(c["frequency_penalty"])) + f32(f32(1.0) * f32(c["presence_penalty"]))))
        r[i] = l
    return r


def run(row, win, c, mt, mu, n_ctx_vocab, fn, defects=()):
    """one step of the chain.  row: the logits; win: the penalty window (oldest first); c: chain parameters (sampling_chain_cases keys);
    mt: MT19937 (advanced in place); mu: mirostat's state; n_ctx_vocab: mirostat 1's N; fn: GLIBC or CR.
    defects: names of seeded defects (tests only).  -> (id, mu after the step, stages); stages that did not run have n = -1."""
    st = {s: dict(n=-1) for s in STAGES}
    r = penalised_row(row, win, c, defects)
    V = r.size
    st["row"] = dict(n=V, ids=np.arange(V, dtype=np.int32), logits=r.copy())
    temp = f32(c["temp"])
    if temp <= 0:                                                # llama_sample_token_greedy: the first maximum
        i = int(np.argmax(r))
        st["order"] = _lst([i], [r[i]])
        st["final"] = dict(_lst([i], [r[i]], [1.0]), pick=0, u=-1.0, id=i, k=-1, mu=f32(mu))
        return i, f32(mu), st
    mir = c["mirostat"]
    if mir:
        r = (r / temp).astype(f32)
        st["temp_row"] = dict(n=V, ids=np.arange(V, dtype=np.int32), logits=r.copy())
    order = np.argsort(-r, kind="stable")                        # descending, equal logits by ascending id
    if "duplicate_neg_inf" in defects and not mir and 1 <= c["top_k"] <= 1024:
        order = order.copy()                                     # seeded defect: taken entries marked -inf win again (lowest id)
        order[np.isneginf(r[order])] = 0
    k = V if (mir or c["top_k"] <= 0) else min(max(int(c["top_k"]), 1), V)
    ids, l, p = order[:k].astype(np.int32), r[order[:k]], None
    st["order"] = _lst(ids, l)
    kk = -1
    if mir == 1:
        p = softmax(l, fn)
        s_bi, s_sq = f32(0), f32(0)
        for i in range(min(99, len(ids) - 1)):
            t_i = fn.log(f32(f32(i + 2) / f32(i + 1)))[0]
            with np.errstate(all="ignore"):
                b_i = fn.log(f32(p[i] / p[i + 1]))[0]
            s_bi, s_sq = fma32(t_i, b_i, s_bi), fma32(t_i, t_i, s_sq)
        with np.errstate(all="ignore"):
            s_hat = f32(s_bi / s_sq)
            eps = f32(s_hat - f32(1))
            kf = fn.pow(f32(f32(eps * fn.pow(f32(2), f32(mu))) / f32(f32(1) - fn.pow(f32(n_ctx_vocab), -eps))), f32(f32(1) / s_hat))
        kk = min(max(x86_int(kf), 1), len(ids))
        ids, l = ids[:kk], l[:kk]
    elif mir == 2:
        p = softmax(l, fn)
        cut = len(ids)
        for i in range(len(ids)):
            if -fn.log2(p[i:i + 1])[0] > f32(mu):
                cut = i
                break
        ids, l = ids[:max(cut, 1)], l[:max(cut, 1)]
    else:
        if c["tfs_z"] < 1.0 and len(ids) > 2:
            p = softmax(l, fn)
            d1 = (p[:-1] - p[1:]).astype(f32)
            d2 = np.abs((d1[:-1] - d1[1:]).astype(f32))
            with np.errstate(all="ignore"):                          # a flat row sums to 0: NaN, no cut, as in the reference
                cum = np.add.accumulate(np.concatenate(([f32(0)], (d2 / fsum(d2)).astype(f32))))[1:]
            last = len(ids)
            for i in np.nonzero(cum > f32(c["tfs_z"]))[0].tolist():
                if i >= 1:
                    last = i + 1 if "tfs_last_plus_one" in defects else i
                    break
            ids, l, p = ids[:last], l[:last], p[:last]
            st["tfs"] = _lst(ids, l, p)
        if c["typical_p"] < 1.0:
            p = softmax(l, fn)
            with np.errstate(all="ignore"):
                lp = fn.log(p)
                ent = fsum((-p * lp).astype(f32))
                score = np.abs((-lp - ent).astype(f32))
            perm = np.argsort(score, kind="stable")
            if "typical_ties_reversed" in defects:                   # equal scores by descending position
                perm = (len(score) - 1 - np.argsort(score[::-1], kind="stable"))
            cum = np.add.accumulate(np.concatenate(([f32(0)], p[perm])))[1:]
            hit = np.nonzero(cum > f32(c["typical_p"]))[0]
            last = int(hit[0]) + 1 if hit.size else len(ids)
            perm = perm[:last]
            ids, l, p = ids[perm], l[perm], p[perm]
            st["typical"] = dict(_lst(ids, l, p), entropy=ent)
        if c["top_p"] < 1.0:
            p = softmax(l, fn)
            cum = np.add.accumulate(np.concatenate(([f32(0)], p)))[1:]
            last = len(ids)
            op = np.greater_equal if "top_p_ge" in defects else np.greater
            for i in np.nonzero(op(cum, f32(c["top_p"])))[0].tolist():
                if i >= 1:
                    last = i
                    break
            ids, l, p = ids[:last], l[:last], p[:last]
            st["top_p"] = _lst(ids, l, p)
        l = (l / temp).astype(f32)
        st["temp"] = _lst(ids, l)
    p = softmax(l, fn) if len(ids) >= 2 else np.ones(1, f32)
    pick, u = draw(p, mt, force_last="table_last_not_forced" not in defects)
    if mir:
        e = f32(-fn.log2(p[pick:pick + 1])[0] - f32(c["mirostat_tau"]))
        mu = fma32(f32(-f32(c["mirostat_eta"])), e, f32(mu))
    st["final"] = dict(_lst(ids, l, p), pick=pick, u=u, id=int(ids[pick]), k=kk, mu=f32(mu))
    return int(ids[pick]), f32(mu), st


# ------------------------------------------------------------------------------------------------------------------ checking

def _bits_equal(a, b):
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


FIELDS = {"row": ("logits",), "order": ("ids", "logits"), "tfs": ("ids", "logits", "p"), "typical": ("ids", "logits", "p"),
          "top_p": ("ids", "logits", "p"), "temp": ("ids", "logits"), "final": ("ids", "logits", "p")}


def compare_device(dev, twin):
    """the device tap against twin(CR): every stage, every field, bit for bit.  -> first difference as a string, or None"""
    for s in STAGES:
        a, b = dev[s], twin[s]
        if a["n"] != b["n"]:
            return "%s: n %d != %d" % (s, a["n"], b["n"])
        if a["n"] < 0:
            continue
        for f in FIELDS[s]:
            x, y = np.asarray(a[f]), np.asarray(b[f])
            ok = (x == y) if f == "ids" else _bits_equal(x, y)
            if not ok.all():
                i = int(np.argmin(ok))
                return "%s.%s[%d]: %r != %r" % (s, f, i, x[i], y[i])
    if twin["typical"]["n"] >= 0 and not _bits_equal([dev["typical"]["entropy"]], [twin["typical"]["entropy"]]).all():
        return "typical.entropy: %r != %r" % (dev["typical"]["entropy"], twin["typical"]["entropy"])
    fd, ft = dev["final"], twin["final"]
    for k in ("pick", "id", "k"):
        if fd[k] != ft[k]:
            return "final.%s: %r != %r" % (k, fd[k], ft[k])
    if fd["u"] != ft["u"]:
        return "final.u: %r != %r" % (fd["u"], ft["u"])
    if not _bits_equal([fd["mu"]], [ft["mu"]]).all():
        return "final.mu: %r != %r" % (fd["mu"], ft["mu"])
    return None


def ref_view(twin, c):
    """the candidates array after each call of refh_sample_chain_stages, from a twin's stages (a stage that did not run leaves the
    array as it was)"""
    if c["temp"] <= 0:
        return {"row": twin["row"]}
    if c["mirostat"]:
        return {"row": twin["row"], "temp": twin["temp_row"], "final": twin["final"]}
    v, prev = {"row": twin["row"], "order": twin["order"]}, twin["order"]
    for s in ("tfs", "typical", "top_p", "temp", "final"):
        if twin[s]["n"] >= 0:
            prev = dict(twin[s], p=twin[s].get("p", prev.get("p")))
        v[s] = prev
    return v


def _runs(l):
    """run index of each entry: maximal runs of equal values (-0 == +0) in the order held"""
    l = np.asarray(l, f32)
    brk = np.ones(l.size, bool)
    brk[1:] = ~(l[1:] == l[:-1])
    return np.cumsum(brk) - 1


def compare_ref(ref, twin, c):
    """the reference's stages against twin(GLIBC).  Equal logits (-0 == +0) sit in an unspecified order in the reference (std::sort /
    std::partial_sort), so within each run of equal logits the ids compare as sets and the logits and p as multisets of bit patterns;
    a run that a cut divides (the last run of the list) may hold any of the tied ids.  -> the first difference, or None"""
    for s, b in ref_view(twin, c).items():
        if s not in ref:
            return "%s: missing in the reference" % s
        a = ref[s]
        if a["n"] != b["n"]:
            return "%s: n %d != %d" % (s, a["n"], b["n"])
        fields = [f for f in ("logits", "p") if b.get(f) is not None and (f == "logits" or s in ("tfs", "typical", "top_p", "temp", "final"))]
        if s == "row" or (s == "temp" and c["mirostat"]):             # id order
            for f in fields:
                ok = _bits_equal(a[f], b[f])
                if not ok.all():
                    i = int(np.argmin(ok))
                    return "%s.%s[%d]: %r != %r" % (s, f, i, a[f][i], b[f][i])
            continue
        run = _runs(b["logits"])
        row = (twin["temp_row"] if c["mirostat"] else twin["row"])["logits"]
        single = (np.bincount(run)[run] == 1) & (run != run[-1])    # most runs hold one candidate: compare those in place
        if not (np.asarray(a["ids"])[single] == np.asarray(b["ids"])[single]).all():
            i = int(np.nonzero(single & (np.asarray(a["ids"]) != np.asarray(b["ids"])))[0][0])
            return "%s.ids[%d]: %d != %d" % (s, i, a["ids"][i], b["ids"][i])
        for f in fields:
            ok = _bits_equal(np.asarray(a[f])[single], np.asarray(b[f])[single])
            if not ok.all():
                return "%s.%s: a single candidate differs" % (s, f)
        for ri in np.unique(run[~single]).tolist():
            sel = run == ri
            for f in fields:
                x, y = np.sort(np.asarray(a[f], f32)[sel].view(np.uint32)), np.sort(np.asarray(b[f], f32)[sel].view(np.uint32))
                if not ((x == y) | (np.isnan(x.view(f32)) & np.isnan(y.view(f32)))).all():
                    return "%s.%s: the run at %d differs" % (s, f, int(np.argmax(sel)))
            x, y = set(np.asarray(a["ids"])[sel].tolist()), set(np.asarray(b["ids"])[sel].tolist())
            if x == y:
                continue
            allowed = set(np.nonzero(np.isin(row, row[sorted(y)]))[0].tolist()) if ri == run[-1] else set()
            if not (x <= allowed and len(x) == len(y)):
                return "%s: ids of the run at %d differ: %s != %s" % (s, int(np.argmax(sel)), sorted(x)[:8], sorted(y)[:8])
    return None
