"""The whole-chain sampling cases (b200_sampling_chain) shared by tests/golden/make_sampling_chain.py, which records the reference's
ids for them in tests/golden/sampling_chain.json, and tests/test_sampling_chain*.py, which replay them; plus numpy restatements of the
device's exact fp32 arithmetic that the CPU tests check.

Rows.  The reference orders candidates with std::sort / std::partial_sort, which leave equal logits in an unspecified order; the device
orders them by ascending id.  Random N(0, 3) rows of 65,024 floats do contain equal values, so a golden row is only used when the row
the sorts see -- after the logit bias, the penalties and (mirostat) the temperature -- has pairwise distinct values: row(case, step,
attempt) is redrawn with the next attempt number until it does, and the attempt used is stored with the ids.
"""
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
