"""The whole-chain sampling cases (b200_sampling_chain) shared by tests/golden/make_sampling_chain.py, which records the reference's
ids for them in tests/golden/sampling_chain.json, and tests/test_sampling_chain*.py, which replay them; plus numpy restatements of the
device's exact fp32 arithmetic that the CPU tests check.

Rows.  The reference orders candidates with std::sort / std::partial_sort, which leave equal logits in an unspecified order; the device
orders them by ascending id.  Random N(0, 3) rows of 65,024 floats do contain equal values, so a golden row is only used when the row
the sorts see -- after the logit bias, the penalties and (mirostat) the temperature -- has pairwise distinct values: row(case, step,
attempt) is redrawn with the next attempt number until it does, and the attempt used is stored with the ids.
"""
import os
import numpy as np

N_VOCAB, STEPS, SEED = 65024, 48, 4242
BIAS = {11: float("-inf"), 500: 4.0, 4000: -2.5}       # id 11 is boosted in every row, so -inf (falcon_main's --ignore-eos) matters

_BASE = dict(top_k=40, top_p=0.95, tfs_z=1.0, typical_p=1.0, temp=0.8, repeat_penalty=1.1, frequency_penalty=0.0, presence_penalty=0.0,
             repeat_last_n=64, mirostat=0, mirostat_tau=5.0, mirostat_eta=0.1, logit_bias=None)


def _case(**kw):
    c = dict(_BASE)
    c.update(kw)
    return c


CASES = {
    "bias": _case(logit_bias=BIAS),
    "freq_pres": _case(repeat_penalty=1.0, frequency_penalty=0.5, presence_penalty=0.7),
    "freq_pres_rep": _case(repeat_penalty=1.1, frequency_penalty=0.3, presence_penalty=0.4, repeat_last_n=128),
    "tfs": _case(tfs_z=0.95),
    "typical": _case(typical_p=0.9),
    "tfs_typical_top_p": _case(top_k=100, tfs_z=0.97, typical_p=0.95, top_p=0.9),
    "top_k0_top_p": _case(top_k=0, top_p=0.95),
    "top_k5000": _case(top_k=5000, top_p=1.0),
    "mirostat1_5_0.1": _case(mirostat=1, mirostat_tau=5.0, mirostat_eta=0.1),
    "mirostat1_3_0.5": _case(mirostat=1, mirostat_tau=3.0, mirostat_eta=0.5),
    "mirostat2_5_0.1": _case(mirostat=2, mirostat_tau=5.0, mirostat_eta=0.1),
    "mirostat2_3_0.5": _case(mirostat=2, mirostat_tau=3.0, mirostat_eta=0.5),
    "greedy_penalties_bias": _case(temp=0.0, repeat_penalty=1.2, frequency_penalty=0.2, presence_penalty=0.3, logit_bias=BIAS),
}


def case_seed(name):
    return sorted(CASES).index(name) + 1


def history(name):
    return [int(t) for t in np.random.default_rng(case_seed(name)).integers(0, N_VOCAB, size=100)]


def window0(name):
    n = CASES[name]["repeat_last_n"]
    return history(name)[-n:] if n > 0 else []


def row(name, step, attempt, win):
    """one logits row: N(0, 3)-shaped values, five dominant candidates, the last window id and id 11 made attractive.
    The values are sorted float64 samples spread apart by 1e-5 per rank before the fp32 cast (more than two fp32 ulps for |x| < 40),
    so they are pairwise distinct with wide gaps, and then dealt out in random order."""
    rng = np.random.default_rng([case_seed(name), step, attempt])
    v = np.sort(rng.standard_normal(N_VOCAB) * 3.0) + np.arange(N_VOCAB) * 1e-5
    r = v.astype(np.float32)[rng.permutation(N_VOCAB)]
    r[rng.integers(0, N_VOCAB, size=5)] += 6.0
    r[11] += 10.0
    if win:
        r[win[-1]] += 5.0
    return r


def effective_row(c, r, win):
    """the row the reference sorts: bias, repetition penalty, frequency / presence penalties, and mirostat's temperature (fp32)"""
    r = r.copy()
    for i, v in (c["logit_bias"] or {}).items():
        r[i] = np.float32(r[i] + np.float32(v))
    ids, counts = np.unique(np.array(win, np.int64), return_counts=True) if win else ([], [])
    for i, n in zip(ids, counts):
        l = r[i]
        if c["repeat_penalty"] != 1.0:
            pen = np.float32(c["repeat_penalty"])
            l = l * pen if l <= 0 else l / pen
        if c["frequency_penalty"] != 0.0 or c["presence_penalty"] != 0.0:
            l = np.float32(l - (np.float32(n) * np.float32(c["frequency_penalty"]) + np.float32(1.0) * np.float32(c["presence_penalty"])))
        r[i] = l
    if c["mirostat"] and c["temp"] > 0:
        r = (r / np.float32(c["temp"])).astype(np.float32)
    return r


def distinct(r):
    return np.unique(r).size == r.size


def seq_sum(x):
    """the fp32 sum x[0] + x[1] + ... in index order (the reference's softmax / accumulate loops)"""
    s = np.float32(0)
    for v in np.asarray(x, np.float32):
        s = np.float32(s + v)
    return s


def seq_sum_desc(x):
    """restatement of sampling.cu's seq_sum_desc: the same sequential sum, stopped at the first term below ulp(S)/4"""
    s = np.float32(0)
    for v in np.asarray(x, np.float32):
        if s > 0:
            ulp = np.float32(2.0 ** (np.frexp(s)[1] - 1)) * np.float32(2.0 ** -23)
            if v < ulp * np.float32(0.25):
                break
        s = np.float32(s + v)
    return s


def x86_float_to_int(x):
    """int(float) as x86's cvttss2si computes it (sampling.cu's x86_float_to_int): NaN and anything outside int32 give INT_MIN"""
    x = np.float32(x)
    if x > np.float32(-2147483904.0) and x < np.float32(2147483648.0):
        return int(x)
    return -2 ** 31


# ---- stage-by-stage cases (tests/test_sampler_stages*.py): chains at every row width where the sampler's code paths branch
WIDTHS = (2, 3, 40, 512, 1024, 1025, 4096, 4097, 65024)     # top-k rounds vs radix sort at 1024 / 1025, draw table at 4096 / 4097


def wrow(W, seed, step=0):
    """a width-W row shaped like row(): pairwise distinct values, a few dominant candidates"""
    rng = np.random.default_rng([W, seed, step])
    v = np.sort(rng.standard_normal(W) * 3.0) + np.arange(W) * 1e-5
    r = v.astype(np.float32)[rng.permutation(W)]
    r[rng.integers(0, W, size=min(5, W))] += 6.0
    return r


def _edges(W):
    """one parameter at a time at its edges, the rest at falcon_main's defaults"""
    out = []
    for k in sorted({1, 2, 1023, 1024, 1025, 5000, W - 1, W, W + 7, 0, -3}):
        out.append(("top_k=%d" % k, _case(top_k=k)))
    for key in ("top_p", "tfs_z", "typical_p"):
        for v in (0.0, 0.5, 0.95):
            out.append(("%s=%g" % (key, v), _case(top_k=0 if W <= 4097 else 200, **{key: v})))
    for t in (1e-3, 1.0, 7.0):
        out.append(("temp=%g" % t, _case(temp=t, tfs_z=0.97, typical_p=0.95)))
    for m in (1, 2):
        for tau in (0.5, 12.0):
            for eta in (0.1, 1.0):
                out.append(("mirostat%d_%g_%g" % (m, tau, eta), _case(mirostat=m, mirostat_tau=tau, mirostat_eta=eta)))
    return out


def _random_chain(rng, W):
    c = _case(top_k=int(rng.choice([1, 2, 7, 40, 1023, 1024, 1025, 0, -1, W, W + 3])),
              top_p=float(rng.choice([1.0, 0.0, 0.5, 0.9, 0.95])), tfs_z=float(rng.choice([1.0, 0.0, 0.5, 0.95])),
              typical_p=float(rng.choice([1.0, 0.0, 0.5, 0.95])), temp=float(rng.choice([0.0, 1e-3, 0.5, 0.8, 1.5, 7.0])),
              repeat_penalty=float(rng.choice([1.0, 1.1, 1.5])), frequency_penalty=float(rng.choice([0.0, 0.3])),
              presence_penalty=float(rng.choice([0.0, 0.4])), repeat_last_n=int(rng.choice([0, 8, 64])),
              mirostat=int(rng.choice([0, 0, 0, 1, 2])), mirostat_tau=float(rng.choice([0.5, 3.0, 12.0])),
              mirostat_eta=float(rng.choice([0.1, 1.0])))
    if rng.random() < 0.3:
        c["logit_bias"] = {int(i): float(rng.choice([-np.inf, 2.0, -1.5])) for i in rng.choice(W, size=min(3, W), replace=False)}
        if c["typical_p"] < 1.0:                                 # p = 0 under typical: the excluded region (typical_nan_cases)
            c["logit_bias"] = {i: (v if v != -np.inf else -3.0) for i, v in c["logit_bias"].items()}
    return c


def distinct_cases(W, n_random):
    """(name, chain, steps): the whole-chain cases, the one-at-a-time edges and a seeded sample of combinations; multi-step, the
    window following the drawn ids"""
    out = [("case:" + n, dict(CASES[n], logit_bias={i: v for i, v in (CASES[n]["logit_bias"] or {}).items() if i < W} or None), 3)
           for n in sorted(CASES)]
    out += [("edge:" + n, c, 2) for n, c in _edges(W)]
    rng = np.random.default_rng(W)
    out += [("random:%d" % i, _random_chain(rng, W), 2) for i in range(n_random)]
    return out


def special_cases(W):
    """(name, chain, row, window): single-step rows for ties, -inf, windows and probabilities below expf's range"""
    rng = np.random.default_rng([W, 99])
    out = []
    q = (np.round(rng.standard_normal(W) * 3.0 * 8) / 8).astype(np.float32)              # logits quantised to 1/8: many ties
    # no typical here: groups of different logits can round to the same typical score, and the reference's unstable sort then
    # mixes them before its cut (an unspecified order); the all-equal rows below tie typical's scores within one group
    for k in (1, 5, 40, 0):
        out.append(("ties_eighths_k%d" % k, _case(top_k=k, repeat_penalty=1.0, tfs_z=0.95, top_p=0.9), q, []))
    s = np.full(W, -1.0, np.float32)                                                     # a tie run straddling the top-k boundary
    s[: min(3, W)] = [3.0, 2.0, 1.0][: min(3, W)]
    for k in (2, 4, 40):
        out.append(("ties_straddle_k%d" % k, _case(top_k=k, repeat_penalty=1.0, top_p=1.0), s, []))
    z = np.zeros(W, np.float32)
    for key in ("top_p", "tfs_z", "typical_p"):
        out.append(("all_equal_%s" % key, _case(top_k=0, repeat_penalty=1.0, **{key: 0.5}), z, []))
    for g in (2, 4, 8, 16):                                                              # 2^g equal candidates, p = 2^-g exactly
        if g <= W:
            r = np.full(W, -200.0, np.float32)                                           # expf(-200) = 0: p = 0 for the rest
            r[rng.choice(W, size=g, replace=False)] = 1.0
            for key in ("top_p", "tfs_z"):
                out.append(("pow2_%d_%s" % (g, key), _case(top_k=0, repeat_penalty=1.0, **{key: 0.5}), r, []))
    d = wrow(W, 7)
    bias = {int(i): -np.inf for i in rng.choice(W, size=min(max(1, W // 3), 64), replace=False)}   # W <= 192: fewer finite than W
    for k in (W, 1024, 40):
        out.append(("neg_inf_bias_k%d" % k, _case(top_k=k, logit_bias=bias), d, []))
    m = np.full(W, -np.inf, np.float32)                                                  # masked row: two finite values
    m[rng.choice(W, size=min(2, W), replace=False)] = [1.0, 0.5][: min(2, W)]
    for name, c in (("masked_top_k40", _case(top_k=40, top_p=1.0)), ("masked_top_k0", _case(top_k=0, top_p=0.95, tfs_z=0.95)),
                    ("masked_greedy", _case(temp=0.0)), ("masked_mirostat2", _case(mirostat=2, mirostat_tau=3.0))):
        out.append((name, c, m, []))
    win = [int(t) for t in rng.integers(0, W + 50, size=40)] + [1, 1, 1, 0, 0, W, W + 3]   # repeated ids, ids >= W
    pz = wrow(W, 8)
    pz[: min(2, W)] = [0.0, -0.0][: min(2, W)]                                            # +-0.0 under the repetition penalty
    out.append(("window_rep_pm0", _case(repeat_penalty=1.3, top_k=0 if W <= 4097 else 40), pz, win))
    out.append(("window_freq_counts", _case(repeat_penalty=1.2, frequency_penalty=0.6, presence_penalty=0.3), pz, win))
    sp = (-np.arange(W, dtype=np.float64) * (400.0 / max(W - 1, 1))).astype(np.float32)[rng.permutation(W)]   # p = 0 below expf's range
    for key in ("tfs_z", "top_p"):
        out.append(("spread_%s" % key, _case(top_k=0, temp=1.0, repeat_penalty=1.0, **{key: 0.95}), sp, []))
    return out


def typical_nan_cases(W):
    """typical over zero probabilities: the reference's entropy is NaN and it sorts NaN keys, so no order is defined.  Only a valid
    id is asked for here."""
    r = np.full(W, -200.0, np.float32)
    r[: min(3, W)] = [1.0, 0.5, 0.25][: min(3, W)]
    return [("typical_zero_p", _case(top_k=0, typical_p=0.9, repeat_penalty=1.0), r, [])]


_REF = {}


def ref_context(W):
    """a reference context whose n_vocab is W (mirostat 1 reads its N there): a tiny synthetic GGCC model; None if it refuses W"""
    if W not in _REF:
        import tempfile
        import refchain
        import pyoracle as po
        import ggllm_cpp_b200.ggcc as ggcc
        from helpers import synth_model, TINY_40B
        hp = dict(TINY_40B, n_vocab=W, n_layer=1)
        path = os.path.join(tempfile.mkdtemp(), "w%d.ggcc" % W)
        ggcc.write_ggcc(path, hp, synth_model(hp, po.Q4_K, seed=W), ftype=15)
        try:
            _REF[W] = refchain.RefChain(path)
        except RuntimeError:
            _REF[W] = None
        os.remove(path)
    return _REF[W]
