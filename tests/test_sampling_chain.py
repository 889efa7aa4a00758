"""CPU checks of the whole-chain sampler's exact arithmetic (sampling.cu) and of its golden data.

- seq_sum_desc: the device stops a softmax sum at the first term below ulp(S)/4 (every later term then rounds away).  Its numpy
  restatement must equal the sequential fp32 loop bit for bit: on seeded softmax rows, on rows built so that terms land exactly on
  half an ulp of the running sum (ties to even), and on rows where the early stop cuts most of the row.
- x86_float_to_int: mirostat 1's int(k) is cvttss2si, which gives INT_MIN for NaN, +-inf and 2^31.
- Where oracle/_ref/libfalcon_chain.so is built: the whole-chain harness with every extra off draws the ids the default-chain
  harness (refh_sample) draws.
- tests/golden/sampling_chain.json has an entry for every case the GPU test replays."""
import json
import os
import numpy as np
import pytest
import sampling_chain_cases as sc

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _softmax_terms(rng, n, scale):
    l = np.sort((rng.standard_normal(n) * scale).astype(np.float32))[::-1]
    return np.exp((l - l[0]).astype(np.float64)).astype(np.float32)     # any fp32 values in descending order


@pytest.mark.parametrize("seed", range(24))
def test_early_stop_sum_equals_sequential_loop(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(2, 20000))
    e = _softmax_terms(rng, n, float(rng.choice([0.5, 3.0, 8.0, 30.0])))
    assert sc.seq_sum_desc(e).view(np.uint32) == sc.seq_sum(e).view(np.uint32)


@pytest.mark.parametrize("s0", [1.0, 1.5, 3.0, 7.75])
def test_early_stop_sum_on_half_ulp_ties(s0):
    """terms of exactly ulp(S)/2 (round to even: they change S when its last bit is odd) and just below and above it"""
    s = np.float32(s0)
    ulp = np.float32(2.0 ** (np.frexp(s)[1] - 1)) * np.float32(2.0 ** -23)
    half = ulp / np.float32(2)
    for tail in ([half] * 7, [half * np.float32(1.5), half, half, half], [np.nextafter(half, np.float32(1)), half, np.nextafter(half, np.float32(0))],
                 [half, ulp / np.float32(4), ulp / np.float32(8)], [ulp, half, half, ulp / np.float32(4)]):
        e = np.array([s] + tail, np.float32)
        assert sc.seq_sum_desc(e).view(np.uint32) == sc.seq_sum(e).view(np.uint32), (s0, tail)


def test_early_stop_really_stops():
    e = _softmax_terms(np.random.default_rng(5), 65024, 3.0)
    s = np.float32(0)
    for i, v in enumerate(e):                                          # where the device loop stops
        if s > 0 and v < np.float32(2.0 ** (np.frexp(s)[1] - 1)) * np.float32(2.0 ** -25):
            break
        s = np.float32(s + v)
    assert i < 65024 and sc.seq_sum_desc(e) == sc.seq_sum(e)


def test_x86_int_conversion():
    INT_MIN = -2 ** 31
    assert sc.x86_float_to_int(float("nan")) == INT_MIN
    assert sc.x86_float_to_int(float("inf")) == INT_MIN
    assert sc.x86_float_to_int(float("-inf")) == INT_MIN
    assert sc.x86_float_to_int(2.0 ** 31) == INT_MIN
    assert sc.x86_float_to_int(-2.0 ** 31) == INT_MIN
    assert sc.x86_float_to_int(2147483520.0) == 2147483520            # the largest fp32 below 2^31
    assert sc.x86_float_to_int(-3.7) == -3 and sc.x86_float_to_int(41.99) == 41


def test_golden_has_every_case():
    g = json.load(open(os.path.join(GOLD, "sampling_chain.json")))
    assert sorted(g) == sorted(sc.CASES)
    for name, v in g.items():
        assert len(v["ids"]) == len(v["attempts"]) == sc.STEPS
        assert all(0 <= t < sc.N_VOCAB for t in v["ids"])
        assert ("mu" in v) == bool(sc.CASES[name]["mirostat"])


def test_golden_rows_are_distinct_after_bias_and_penalties():
    g = json.load(open(os.path.join(GOLD, "sampling_chain.json")))
    for name in ("bias", "mirostat1_5_0.1"):
        c, win = sc.CASES[name], sc.window0(name)
        for s in range(3):
            assert sc.distinct(sc.effective_row(c, sc.row(name, s, g[name]["attempts"][s], win), win))
            win = (win + [g[name]["ids"][s]])[-c["repeat_last_n"]:]


def test_reference_chain_with_extras_off_equals_default_chain():
    import refchain
    if not refchain.have_chain():
        pytest.skip("oracle/_ref/libfalcon_chain.so is not built here (needs the reference sources)")
    import tempfile
    from helpers import po, ggcc, synth_model, TINY_40B
    hp = dict(TINY_40B)
    path = os.path.join(tempfile.mkdtemp(), "chain.ggcc")
    ggcc.write_ggcc(path, hp, synth_model(hp, po.Q4_K, seed=1234), ftype=15)
    ref = refchain.RefChain(path)
    rng = np.random.default_rng(1)
    for top_k, top_p, temp, pen in [(40, 0.95, 0.8, 1.1), (200, 0.5, 1.3, 1.3), (40, 1.0, 0.0, 1.2), (1000, 0.999, 2.0, 1.05)]:
        rows = [(rng.standard_normal(4096) * 3.0).astype(np.float32) for _ in range(8)]
        win = [int(t) for t in rng.integers(0, 4096, size=32)]
        ref.set_seed(77)
        a = [ref.sample(r, win, top_k, top_p, temp, pen) for r in rows]
        ref.set_seed(77)
        b = [ref.sample_chain(r, win, 10.0, top_k=top_k, top_p=top_p, temp=temp, repeat_penalty=pen)[0] for r in rows]
        assert a == b
    ref.close()
    os.remove(path)
