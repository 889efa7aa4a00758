"""-m gpu: the device sampler (b200_sampler_*, b200_falcon_generate; sampling.cu) against the REFERENCE's own sampling functions
(llama_sample_repetition_penalty / top_k / top_p / temperature / token, called in falcon_main's order by oracle/ref_harness.cpp; the ids
they drew, with the logits rows they drew from, are stored in tests/golden/sampling.json and generate.npz by tests/golden/make_golden.py): the same seed must sample the same
token ids -- the MT19937 stream, libstdc++'s
discrete_distribution table and every cut are restated bit for bit.  A draw can differ only when device expf and glibc expf differ by an
ulp AND the uniform variate lands within ~1e-7 of a table boundary; the sequences below are fixed and short enough that this does
not occur (a failing id would be a real divergence)."""
import json
import os
import numpy as np
import pytest
import pyoracle as po
from helpers import TINY_40B, synth_model

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _logits(rng, n_vocab, win):
    logits = (rng.standard_normal(n_vocab) * 3.0).astype(np.float32)
    logits[rng.integers(0, n_vocab, size=5)] += 6.0                          # a few dominant candidates, like real logits
    if win:
        logits[win[-1]] += 5.0                                              # make the penalty matter: the last id stays attractive
    return logits


@pytest.mark.parametrize("top_k,top_p,temp,penalty,last_n", [(40, 0.95, 0.8, 1.1, 64), (1, 1.0, 0.8, 1.0, 0), (200, 0.5, 1.3, 1.3, 16),
                                                              (40, 1.0, 0.0, 1.2, 64), (7, 0.9, 0.7, 1.0, 0), (1000, 0.999, 2.0, 1.05, 200)])
def test_sampler_matches_reference_chain(gpu, top_k, top_p, temp, penalty, last_n):
    ref_ids = json.load(open(os.path.join(GOLD, "sampling.json")))["%d/%g/%g/%g/%d" % (top_k, top_p, temp, penalty, last_n)]
    n_vocab, steps, seed = 65024, 48, 4242
    rng = np.random.default_rng(top_k + last_n)
    history = list(rng.integers(0, n_vocab, size=100))
    sp = gpu.SamplingParams(top_k=top_k, top_p=top_p, temp=temp, repeat_penalty=penalty, repeat_last_n=last_n, seed=seed)
    dev = gpu.Sampler(sp, history)
    want, got = [], []
    win = history[-last_n:] if last_n > 0 else []
    for s in range(steps):
        logits = _logits(rng, n_vocab, win)
        w = ref_ids[s]
        d = gpu.DevBuf(src=logits)
        g = dev.sample(d.ptr, n_vocab)
        want.append(w); got.append(g)
        if last_n > 0:
            win = (win + [w])[-last_n:]
        assert g == w, (s, got, want)                                       # stop at the first divergence: the windows would differ afterwards
    assert got == want


def test_generate_with_sampler_equals_host_loop_with_reference_sampler(gpu):
    """(1) the device sampler, fed the logits rows of falcon_main's loop (eval -> sampling chain -> eval), draws the ids the reference's
    chain drew from the same rows (golden/generate.npz); (2) b200_falcon_generate (sampler inside the step graph, ids never leave the GPU)
    == the same loop on the host with this library's logits and the device sampler"""
    g = np.load(os.path.join(GOLD, "generate.npz"))
    prompt, seed, steps = g["prompt"], int(g["seed"]), len(g["ids"])
    n_vocab = g["logits"].shape[1]
    sp = gpu.SamplingParams(top_k=40, top_p=0.95, temp=0.8, repeat_penalty=1.1, repeat_last_n=64, seed=seed)

    def draw(sampler, row):
        d = gpu.DevBuf(src=np.ascontiguousarray(row, np.float32))
        return sampler.sample(d.ptr, n_vocab)

    first = draw(gpu.Sampler(sp, prompt.tolist()), g["logits"][0])          # the stream starts at the seed for the first id and again after it
    assert first == int(g["first"])
    s = gpu.Sampler(sp, prompt.tolist() + [first])
    assert [draw(s, row) for row in g["logits"][1:]] == g["ids"].tolist()

    hp = dict(TINY_40B)
    tensors = synth_model(hp, po.Q4_K, seed=1234)
    a, b = gpu.Falcon(hp, n_ctx=64, n_batch=8), gpu.Falcon(hp, n_ctx=64, n_batch=8)
    a.set_tensors(tensors); b.set_tensors(tensors)
    a.eval(prompt, 0); lg = b.eval(prompt, 0)
    first = draw(gpu.Sampler(sp, prompt.tolist()), lg[0])
    win = prompt.tolist() + [first]
    dev = a.generate(sp, win, first, len(prompt), steps)
    s, host, tok = gpu.Sampler(sp, win), [], first
    for i in range(steps):
        lg = b.eval(np.array([tok], np.int32), len(prompt) + i)
        tok = draw(s, lg[0])
        host.append(tok)
    assert dev.tolist() == host
    # greedy generation still works afterwards (the step graph is rebuilt around the arg-max kernel)
    g1 = a.generate_greedy(first, len(prompt), 4)
    sp0 = gpu.SamplingParams(top_k=1, top_p=1.0, temp=0.0, repeat_penalty=1.0, repeat_last_n=0, seed=1)
    g2 = a.generate(sp0, [], first, len(prompt), 4)
    assert g1.tolist() == g2.tolist()
    with pytest.raises(RuntimeError):
        a.generate(gpu.SamplingParams(top_k=0), [], first, len(prompt), 2)      # "whole vocabulary" is not supported on the device
    a.free(); b.free()
