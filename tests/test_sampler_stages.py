"""CPU checks of the sampling chain's exact twin (tests/sampler_twin.py) against the reference, stage by stage.

- twin(glibc) -- the chain restated with this host's expf / logf / log2f / powf -- reproduces every id and mirostat mu recorded in
  golden/sampling_chain.json and golden/sampling.json, bit for bit.
- Where oracle/_ref/libfalcon_chain.so is built: refh_sample_chain_stages (the candidates array after each llama_sample_* call) draws
  what refh_sample_chain draws, and twin(glibc) equals it at every stage on the case groups of sampling_chain_cases at every width.
  The reference cannot load a 2- or 3-token model (its loader crashes), so those widths run in the 40-token context, without
  mirostat 1, whose N is the context's vocabulary.
- The MT19937 restatement gives std::mt19937's 10000th output; the draw follows libstdc++'s discrete_distribution.
- The checker finds defects seeded into otherwise correct stage dumps, each at its own stage."""
import json
import os
import zlib
import numpy as np
import pytest
import sampler_twin as tw
import sampling_chain_cases as sc

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# crc32 of glibc's expf / logf / log2f over a fixed set of arguments, for the glibc the goldens were recorded with (2.39, x86-64 with FMA)
GLIBC_PRINT = 0x8f61d8d3


def _glibc_print():
    x = np.linspace(-30, 0, 4001, dtype=np.float32)
    p = np.linspace(1e-6, 1, 4001, dtype=np.float32)
    return zlib.crc32(tw.GLIBC.exp(x).tobytes() + tw.GLIBC.log(p).tobytes() + tw.GLIBC.log2(p).tobytes())


def _skip_if_other_glibc(ok):
    """a mismatch is a failure on the goldens' glibc, and a skip on a glibc that rounds differently"""
    if not ok and _glibc_print() != GLIBC_PRINT:
        pytest.skip("this host's glibc float functions round differently from the one the goldens were recorded with (fingerprint %08x)"
                    % _glibc_print())


def test_mt19937_anchor():
    m = tw.MT19937(5489)
    for _ in range(9999):
        m.next()
    assert m.next() == 4123659995


def test_discrete_table_forces_last_entry():
    p = np.array([0.1, 0.2, 0.3, 0.4], np.float32)
    cp = tw.discrete_table(p)
    assert cp[-1] == 1.0 and (np.diff(cp) >= 0).all()
    assert [tw.draw(p, _FixedU(u))[0] for u in (0.0, 0.05, 0.2, 0.45, 0.7, 0.99)] == [0, 0, 1, 2, 3, 3]


class _FixedU:
    """an MT19937 stand-in whose two outputs make generate_canonical return u (u a multiple of 2^-64 up to rounding)"""

    def __init__(self, u):
        v = int(u * 2.0 ** 64)
        self.out = [v & 0xffffffff, v >> 32]

    def next(self):
        return self.out.pop(0)


def _golden_chain(name, fn):
    g = json.load(open(os.path.join(GOLD, "sampling_chain.json")))[name]
    c = sc.CASES[name]
    win, mt, mu = sc.window0(name), tw.MT19937(sc.SEED), np.float32(2 * c["mirostat_tau"])
    for s in range(sc.STEPS):
        i, mu, _ = tw.run(sc.row(name, s, g["attempts"][s], win), win, c, mt, mu, sc.N_VOCAB, fn)
        if i != g["ids"][s] or ("mu" in g and mu != np.float32(g["mu"][s])):
            return s, i, g["ids"][s], mu
        if c["repeat_last_n"] > 0:
            win = (win + [i])[-c["repeat_last_n"]:]
    return None


@pytest.mark.parametrize("name", sorted(sc.CASES))
def test_twin_glibc_reproduces_golden_chain(name):
    bad = _golden_chain(name, tw.GLIBC)
    _skip_if_other_glibc(bad is None)
    assert bad is None, bad


@pytest.mark.parametrize("top_k,top_p,temp,penalty,last_n", [(40, 0.95, 0.8, 1.1, 64), (1, 1.0, 0.8, 1.0, 0), (200, 0.5, 1.3, 1.3, 16),
                                                             (40, 1.0, 0.0, 1.2, 64), (7, 0.9, 0.7, 1.0, 0), (1000, 0.999, 2.0, 1.05, 200)])
def test_twin_glibc_reproduces_golden_default_chain(top_k, top_p, temp, penalty, last_n):
    ref_ids = json.load(open(os.path.join(GOLD, "sampling.json")))["%d/%g/%g/%g/%d" % (top_k, top_p, temp, penalty, last_n)]
    n_vocab = 65024
    rng = np.random.default_rng(top_k + last_n)
    history = [int(t) for t in rng.integers(0, n_vocab, size=100)]
    c = sc._case(top_k=top_k, top_p=top_p, temp=temp, repeat_penalty=penalty, repeat_last_n=last_n)
    win, mt, got = history[-last_n:] if last_n > 0 else [], tw.MT19937(4242), []
    for s in range(48):
        logits = (rng.standard_normal(n_vocab) * 3.0).astype(np.float32)
        logits[rng.integers(0, n_vocab, size=5)] += 6.0
        if win:
            logits[win[-1]] += 5.0
        i, _, _ = tw.run(logits, win, c, mt, 0.0, n_vocab, tw.GLIBC)
        got.append(i)
        if last_n > 0:
            win = (win + [ref_ids[s]])[-last_n:]
    _skip_if_other_glibc(got == ref_ids)
    assert got == ref_ids


# ---------------------------------------------------------------------------------------------------- against the live reference

def _ref(W):
    import refchain
    if not refchain.have_chain():
        pytest.skip("oracle/_ref/libfalcon_chain.so is not built here (needs the reference sources)")
    if not refchain.have_stages():
        pytest.skip("oracle/_ref/libfalcon_chain.so was built from an older ref_sample_chain.cpp and the reference sources to rebuild it are absent")
    return sc.ref_context(max(W, 40))


def _ref_step(ref, row, win, c, mu):
    return ref.sample_chain_stages(row, win, mu, **{k: c[k] for k in ("top_k", "top_p", "tfs_z", "typical_p", "temp", "repeat_penalty",
                                                                       "frequency_penalty", "presence_penalty", "mirostat", "mirostat_tau",
                                                                       "mirostat_eta", "logit_bias")})


def check_twin_against_reference(ref, W, c, rows_and_windows, seed, fresh=False):
    """twin(glibc) against refh_sample_chain_stages, step by step; the window follows the reference's ids.  -> None or the difference"""
    ref.set_seed(seed)
    mt, mu = tw.MT19937(seed), np.float32(2 * c["mirostat_tau"])
    for s, (row, win) in enumerate(rows_and_windows):
        if fresh:
            ref.set_seed(seed)
            mt, mu = tw.MT19937(seed), np.float32(2 * c["mirostat_tau"])
        rid, rmu, rst = _ref_step(ref, row, win, c, float(mu))
        tid, tmu, tst = tw.run(row, win, c, mt, mu, ref.n_vocab, tw.GLIBC)
        d = tw.compare_ref(rst, tst, c)
        if d is None and rid != tid:
            pen = (tst["temp_row"] if c["mirostat"] else tst["row"])["logits"]
            if not (pen[rid] == pen[tid]):
                d = "id %d != %d" % (rid, tid)
        if d is None and c["mirostat"] and np.float32(rmu).view(np.uint32) != np.float32(tmu).view(np.uint32):
            d = "mu %r != %r" % (rmu, tmu)
        if d:
            return "step %d: %s" % (s, d)
        mu = np.float32(rmu)
    return None


def _window0(W, c, seed):
    return [int(t) for t in np.random.default_rng([W, seed]).integers(0, W, size=c["repeat_last_n"])] if c["repeat_last_n"] else []


@pytest.mark.parametrize("W", sc.WIDTHS)
def test_reference_stages_draw_what_the_chain_draws(W):
    ref = _ref(W)
    for n, c, _ in sc.distinct_cases(W, 6)[:: 3]:
        if c["mirostat"] == 1 and W < 40:
            continue
        row = sc.wrow(W, 3)
        args = {k: c[k] for k in ("top_k", "top_p", "tfs_z", "typical_p", "temp", "repeat_penalty", "frequency_penalty",
                                  "presence_penalty", "mirostat", "mirostat_tau", "mirostat_eta", "logit_bias")}
        ref.set_seed(11)
        a = ref.sample_chain(row, [0, 1], 4.0, **args)
        ref.set_seed(11)
        b = _ref_step(ref, row, [0, 1], c, 4.0)[:2]
        assert a[0] == b[0] and np.float32(a[1]) == np.float32(b[1]), n


def _distinct_ids(W):
    n_random = {65024: 4, 4096: 12, 4097: 12}.get(W, 40)
    return [(n, c, steps) for n, c, steps in sc.distinct_cases(W, n_random) if not (W < 40 and c["mirostat"] == 1)]


@pytest.mark.parametrize("W", sc.WIDTHS)
def test_twin_equals_reference_on_distinct_rows(W):
    ref = _ref(W)
    bad = []
    for k, (name, c, steps) in enumerate(_distinct_ids(W)):
        seed = 1000 + k
        win = _window0(W, c, seed)
        ref.set_seed(seed)
        mt, mu = tw.MT19937(seed), np.float32(2 * c["mirostat_tau"])
        for s in range(steps):
            row = sc.wrow(W, seed, s)
            rid, rmu, rst = _ref_step(ref, row, win, c, float(mu))
            tid, tmu, tst = tw.run(row, win, c, mt, mu, ref.n_vocab, tw.GLIBC)
            d = tw.compare_ref(rst, tst, c)
            if d is None and rid != tid:
                d = "id %d != %d" % (rid, tid)
            if d is None and c["mirostat"] and np.float32(rmu).view(np.uint32) != tmu.view(np.uint32):
                d = "mu %r != %r" % (rmu, tmu)
            if d:
                bad.append((name, s, d))
                break
            mu = np.float32(rmu)
            if c["repeat_last_n"] > 0:
                win = (win + [rid])[-c["repeat_last_n"]:]
    assert not bad, bad[:5]


@pytest.mark.parametrize("W", sc.WIDTHS)
def test_twin_equals_reference_on_ties_inf_windows_and_spread(W):
    ref = _ref(W)
    bad = []
    for k, (name, c, row, win) in enumerate(sc.special_cases(W)):
        if W < 40 and c["mirostat"] == 1:
            continue
        d = check_twin_against_reference(ref, W, c, [(row, win)], 500 + k, fresh=True)
        if d:
            bad.append((name, d))
    assert not bad, bad[:5]


@pytest.mark.parametrize("W", (40, 1024))
def test_typical_over_zero_probabilities_gives_a_valid_id(W):
    """the excluded region: the reference's entropy is NaN there and it sorts NaN keys; only a valid id is defined"""
    ref = _ref(W)
    for name, c, row, win in sc.typical_nan_cases(W):
        ref.set_seed(3)
        rid = _ref_step(ref, row, win, c, 10.0)[0]
        tid = tw.run(row, win, c, tw.MT19937(3), np.float32(10.0), W, tw.GLIBC)[0]
        assert 0 <= rid < W and 0 <= tid < W


# ------------------------------------------------------------------------------------------------------------ seeded defects

def _defect_case(defect):
    """(chain, row, window, W, the stage the defect must be found at)"""
    W = 1024
    if defect == "top_p_ge":                                    # four candidates of p = 1/4 exactly: the running sum meets 0.5
        r = np.full(W, -200.0, np.float32)
        r[[3, 9, 500, 700]] = 1.0
        return sc._case(top_k=0, top_p=0.5, repeat_penalty=1.0), r, [], W, "top_p"
    if defect == "tfs_last_plus_one":
        return sc._case(top_k=100, tfs_z=0.95), sc.wrow(W, 1), [], W, "tfs"
    if defect == "typical_ties_reversed":                       # all equal: every score ties
        return sc._case(top_k=0, typical_p=0.5, repeat_penalty=1.0), np.zeros(W, np.float32), [], W, "typical"
    if defect == "penalty_per_occurrence":
        return sc._case(repeat_penalty=1.3), sc.wrow(W, 2), [5, 5, 7], W, "row"
    if defect == "table_last_not_forced":                       # a draw that falls past the last partial sum (about 1 - 2^-53)
        return sc._case(top_k=3, top_p=1.0, repeat_penalty=1.0, temp=1.0), np.array([0.0, -1.0, -2.0] + [-9.0] * (W - 3), np.float32), [], W, "final"
    if defect == "duplicate_neg_inf":                            # fewer finite values than top_k
        r = sc.wrow(W, 4)
        r[50:] = -np.inf
        return sc._case(top_k=1024, top_p=1.0, repeat_penalty=1.0), r, [], W, "order"
    raise KeyError(defect)


DEFECTS = ("top_p_ge", "tfs_last_plus_one", "typical_ties_reversed", "penalty_per_occurrence", "table_last_not_forced",
           "duplicate_neg_inf")
# An early stop of the softmax sum at ulp(S)/2 instead of ulp(S)/4 changes a sum only through a term of exactly half an ulp, i.e. an
# expf result that is a power of two; no float argument near -k ln 2 (k = 24..39) gives one, so no chain row can show that defect.
# test_sampling_chain.py's half-ulp rows check the sum itself.


def first_difference_stage(a, b):
    d = tw.compare_device(a, b)
    return None if d is None else d.split(":")[0].split(".")[0]


@pytest.mark.parametrize("defect", DEFECTS)
def test_checker_finds_seeded_defect_at_its_stage(defect):
    c, row, win, W, stage = _defect_case(defect)
    if defect == "table_last_not_forced":
        # the unforced table's last partial sum falls short of 1 by rounding on some rows; a variate above it then runs off the table
        # (position n), where the forced table draws the last candidate
        rng = np.random.default_rng(1)
        for _ in range(200):
            p = tw.softmax(rng.standard_normal(W).astype(np.float32), tw.CR)
            if tw.discrete_table(p, force_last=False)[-1] < 1.0:
                break
        u = float(np.nextafter(1.0, 0.0))
        assert int(np.searchsorted(tw.discrete_table(p), u, side="left")) == W - 1
        assert int(np.searchsorted(tw.discrete_table(p, force_last=False), u, side="left")) == W
        return
    good = tw.run(row, win, c, tw.MT19937(7), np.float32(10.0), W, tw.CR)[2]
    bad = tw.run(row, win, c, tw.MT19937(7), np.float32(10.0), W, tw.CR, defects=(defect,))[2]
    assert tw.compare_device(good, good) is None
    assert first_difference_stage(bad, good) == stage, tw.compare_device(bad, good)
