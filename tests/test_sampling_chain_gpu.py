"""-m gpu: the whole device sampling chain (b200_sampler_create_chain, b200_falcon_generate_chain; sampling.cu) against the REFERENCE's
own llama_sample_* functions in falcon_main's order (oracle/ref_sample_chain.cpp; the ids, row attempts and mirostat mu trajectories
are stored in tests/golden/sampling_chain.json by tests/golden/make_sampling_chain.py over the rows of tests/sampling_chain_cases.py).

Divergence model: every cut, sort and sum is restated bit for bit, so an id can only differ when the device's expf / logf / log2f /
powf and glibc's differ by an ulp AND that ulp moves a value across a boundary: the uniform variate within ~1e-7 of a table entry,
a running sum within ~1e-7 of top_p / tfs_z / typical_p, -log2f(p) within an ulp of mu, or mirostat 1's k within an ulp of an
integer.  The rows have pairwise distinct values after bias, penalties and temperature (see sampling_chain_cases), so the
reference's unstable sorts cannot order ties differently.  The fixed sequences below do not hit a boundary: a failing id is a real
divergence, and the tests stop at the first one (the windows would differ afterwards).

mirostat's mu is held bit for bit to the exact twin of the chain over correctly rounded transcendentals (tests/sampler_twin.py), which
is what the device evaluates; the recorded mu comes from glibc's log2f / logf / powf and may differ from it in the last bits (the CPU
test test_sampler_stages.py holds the recorded values to the twin over glibc's functions)."""
import json
import os
import numpy as np
import pytest
import pyoracle as po
import sampling_chain_cases as sc
import sampler_twin as tw
from helpers import TINY_40B, synth_model

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CHAIN_KEYS = ("top_k", "top_p", "tfs_z", "typical_p", "temp", "repeat_penalty", "frequency_penalty", "presence_penalty", "repeat_last_n",
              "mirostat", "mirostat_tau", "mirostat_eta", "logit_bias")


def chain(gpu, c, seed):
    return gpu.SamplingChain(seed=seed, **{k: c[k] for k in CHAIN_KEYS})


@pytest.mark.parametrize("name", sorted(sc.CASES))
def test_chain_matches_reference(gpu, name):
    gold = json.load(open(os.path.join(GOLD, "sampling_chain.json")))[name]
    c = sc.CASES[name]
    win = sc.window0(name)
    dev = gpu.Sampler(chain(gpu, c, sc.SEED), sc.history(name))
    mt, twin_mu = tw.MT19937(sc.SEED), np.float32(2.0 * c["mirostat_tau"])
    if c["mirostat"]:
        assert dev.mirostat_mu() == np.float32(2.0 * c["mirostat_tau"])
    for s in range(sc.STEPS):
        r = sc.row(name, s, gold["attempts"][s], win)
        d = gpu.DevBuf(src=r)
        g = dev.sample(d.ptr, sc.N_VOCAB)
        w = gold["ids"][s]
        assert g == w, (name, s, g, w)
        if c["mirostat"]:
            twin_id, twin_mu, _ = tw.run(r, win, c, mt, twin_mu, sc.N_VOCAB, tw.CR)
            mu = np.float32(dev.mirostat_mu())
            assert twin_id == g and mu.view(np.uint32) == twin_mu.view(np.uint32), (name, s, mu, twin_mu, gold["mu"][s])
        if c["repeat_last_n"] > 0:
            win = (win + [w])[-c["repeat_last_n"]:]


SAMPLING_CASES = [(40, 0.95, 0.8, 1.1, 64), (1, 1.0, 0.8, 1.0, 0), (200, 0.5, 1.3, 1.3, 16), (40, 1.0, 0.0, 1.2, 64), (7, 0.9, 0.7, 1.0, 0),
                  (1000, 0.999, 2.0, 1.05, 200)]


def _old_logits(rng, n_vocab, win):                                    # the row stream of tests/test_sampling_gpu.py
    logits = (rng.standard_normal(n_vocab) * 3.0).astype(np.float32)
    logits[rng.integers(0, n_vocab, size=5)] += 6.0
    if win:
        logits[win[-1]] += 5.0
    return logits


@pytest.mark.parametrize("top_k,top_p,temp,penalty,last_n", SAMPLING_CASES)
def test_chain_with_extras_off_matches_default_chain_golden(gpu, top_k, top_p, temp, penalty, last_n):
    ref_ids = json.load(open(os.path.join(GOLD, "sampling.json")))["%d/%g/%g/%g/%d" % (top_k, top_p, temp, penalty, last_n)]
    n_vocab = 65024
    rng = np.random.default_rng(top_k + last_n)
    history = list(rng.integers(0, n_vocab, size=100))
    dev = gpu.Sampler(gpu.SamplingChain(top_k=top_k, top_p=top_p, temp=temp, repeat_penalty=penalty, repeat_last_n=last_n, seed=4242), history)
    win = history[-last_n:] if last_n > 0 else []
    for s in range(48):
        d = gpu.DevBuf(src=_old_logits(rng, n_vocab, win))
        g = dev.sample(d.ptr, n_vocab)
        assert g == ref_ids[s], (s, g, ref_ids[s])
        if last_n > 0:
            win = (win + [ref_ids[s]])[-last_n:]


def test_mirostat1_flat_row_takes_x86_int_conversion(gpu):
    """a flat row makes s_hat 0, so k = powf(x, 1/0) = inf; x86's int(inf) is INT_MIN, which top_k clamps to 1: the first candidate
    (id 0 under ties by id), every step.  A saturating conversion would give the whole vocabulary and random ids."""
    dev = gpu.Sampler(gpu.SamplingChain(mirostat=1, mirostat_tau=10.0, repeat_penalty=1.0, repeat_last_n=0, seed=3))
    d = gpu.DevBuf(src=np.zeros(4096, np.float32))
    assert [dev.sample(d.ptr, 4096) for _ in range(8)] == [0] * 8


@pytest.mark.parametrize("kw", [dict(mirostat=3), dict(mirostat=-1), dict(repeat_last_n=257), dict(repeat_last_n=-1), dict(top_p=float("nan")),
                                dict(temp=float("nan")), dict(mirostat_tau=float("nan")), dict(logit_bias={-1: 1.0}),
                                dict(logit_bias={i: 1.0 for i in range(65)}), dict(logit_bias={5: float("nan")})])
def test_chain_rejects_bad_parameters(gpu, kw):
    with pytest.raises(ValueError):
        gpu.Sampler(gpu.SamplingChain(**kw))


def test_chain_rejects_duplicate_and_out_of_range_bias_ids(gpu):
    import ctypes as C
    c = gpu.SamplingChain()
    ids, vals = np.array([7, 7], np.int32), np.array([1.0, 2.0], np.float32)
    c.n_logit_bias, c.logit_bias_ids, c.logit_bias_values = 2, ids.ctypes.data, vals.ctypes.data
    assert not gpu.lib().b200_sampler_create_chain(C.byref(c), None, 0)
    s = gpu.Sampler(gpu.SamplingChain(logit_bias={600: 1.0}))
    d = gpu.DevBuf(src=np.zeros(512, np.float32))
    assert s.sample(d.ptr, 512) == -1                                  # id 600 is outside a 512-wide row: refused, nothing written


def test_generate_chain_equals_host_loop(gpu):
    """b200_falcon_generate_chain (sampler inside the step graph) == b200_falcon_eval + a stand-alone chain sampler over the same rows,
    on TINY_40B (n_vocab 512: the whole-vocabulary path): mu and the penalty window persist across the graph replays."""
    hp = dict(TINY_40B)
    tensors = synth_model(hp, po.Q4_K, seed=1234)
    a, b = gpu.Falcon(hp, n_ctx=64, n_batch=8), gpu.Falcon(hp, n_ctx=64, n_batch=8)
    a.set_tensors(tensors); b.set_tensors(tensors)
    prompt = np.array([11, 100, 101, 102, 103], np.int32)
    steps = 24
    chains = [dict(mirostat=2, mirostat_tau=3.0, mirostat_eta=0.5, temp=1.2, frequency_penalty=0.2, seed=9),
              dict(top_k=0, tfs_z=0.97, typical_p=0.95, top_p=0.95, temp=1.5, presence_penalty=0.3, logit_bias={7: -3.0}, seed=5)]
    for kw in chains:
        a.eval(prompt, 0); b.eval(prompt, 0)
        first = 42
        win = prompt.tolist() + [first]
        dev = a.generate_chain(gpu.SamplingChain(**kw), win, first, len(prompt), steps)
        s, host, tok = gpu.Sampler(gpu.SamplingChain(**kw), win), [], first
        for i in range(steps):
            lg = b.eval(np.array([tok], np.int32), len(prompt) + i)
            d = gpu.DevBuf(src=np.ascontiguousarray(lg[0]))
            tok = s.sample(d.ptr, hp["n_vocab"])
            host.append(tok)
        assert dev.tolist() == host, kw
    # the greedy and default-chain generations still work afterwards (the step graph is rebuilt around their kernels)
    g1 = a.generate_greedy(first, len(prompt), 4)
    g2 = a.generate(gpu.SamplingParams(top_k=1, top_p=1.0, temp=0.0, repeat_penalty=1.0, repeat_last_n=0, seed=1), [], first, len(prompt), 4)
    assert g1.tolist() == g2.tolist()
    with pytest.raises(RuntimeError):
        a.generate_chain(gpu.SamplingChain(mirostat=5), [], first, len(prompt), 2)
    with pytest.raises(RuntimeError):
        a.generate_chain(gpu.SamplingChain(logit_bias={512: 1.0}), [], first, len(prompt), 2)
    a.free(); b.free()
