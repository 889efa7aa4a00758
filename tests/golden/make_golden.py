"""Generate the committed golden vectors from the UNMODIFIED reference (oracle/_ref, built by `make -C oracle ref` from the
reference sources).

Run where oracle/_ref is built:   python tests/golden/make_golden.py
Outputs (small, committed):
  codecs.npz          for every weight type: the reference's own test vector x[i] = 0.1 + 2 cos(i) (test-quantize-fns.cpp:26-30),
                      the reference's quantised bytes, its dequantised values, its Q8 activation bytes and vec_dot result
  tiny40b_q4_K.npz    logits of falcon_eval (CPU build) for the synthetic model recipe tests/helpers.synth_model
  tiny7b_q4_0.npz
  codecs_random.json  SHA-256 of the reference's quantised bytes, dequantised values and Q8 activation bytes of seeded random rows
                      (the bit-exact comparison of tests/test_oracle.py, stored as digests to stay small)
  tiny40b_q3_K_live.npz  all logits of a 5-token prompt through falcon_eval (CPU build) for the Q3_K synthetic model
  sampling.json       the ids the reference's sampling chain (falcon_main's order) draws for seeded logits rows, per parameter set
  generate.npz        the logits rows of a 20-token generation (oracle falcon_eval) and the ids the reference's chain drew from them
The tests compare against these files; they do not need the reference.
"""
import hashlib
import json
import os
import sys
import tempfile
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from helpers import po, ggcc, synth_model, TINY_40B, TINY_7B  # noqa: E402


def codecs():
    r = po.ref()
    out = {}
    x = po.synth_vector(4096).reshape(4, 1024)
    a = po.synth_vector(4096, offset=1.0).reshape(4, 1024)
    out["x"], out["a"] = x, a
    for t in po.WEIGHT_TYPES:
        n = po.TYPE_NAMES[t]
        q = r.quantize(t, x)
        out[n + "_q"] = q
        out[n + "_deq"] = r.dequantize(t, q, 1024)
        aq = r.quantize_act(t, a)
        out[n + "_aq"] = aq
        out[n + "_dot"] = np.array([r.vec_dot(t, 1024, q[i], aq[i]) for i in range(4)], np.float32)
    np.savez_compressed(os.path.join(HERE, "codecs.npz"), **out)


def model(name, hp, wt, seed, n_ctx=64):
    tensors = synth_model(hp, wt, seed)
    path = os.path.join(tempfile.gettempdir(), name + ".ggcc")
    ggcc.write_ggcc(path, hp, tensors, ftype=ggcc.FTYPE_OF_TYPE[wt])
    ref = po.RefFalcon(path, n_ctx=n_ctx, n_batch=8, logits_all=True)
    prompt = np.array([11, 100, 101, 102, 103, 104, 105], np.int32)
    pl = ref.eval(prompt, 0, n_threads=4)
    dec = np.array([200, 17, 333, 42], np.int32)
    dl = np.concatenate([ref.eval(dec[i:i + 1], len(prompt) + i, n_threads=4) for i in range(len(dec))])
    ref.close()
    os.remove(path)
    np.savez_compressed(os.path.join(HERE, name + ".npz"), prompt=prompt, prompt_logits=pl, decode_tokens=dec, decode_logits=dl,
                        wtype=wt, seed=seed, n_ctx=n_ctx, **{"hp_" + k: v for k, v in hp.items()})


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def random_rows(t, scale):
    """the inputs of tests/test_oracle.py::test_codecs_bit_exact_vs_reference_random"""
    rng = np.random.default_rng(t)
    xs = []
    for s in (1.0, 0.02, 30.0):
        x = (rng.standard_normal((8, 2048)) * s).astype(np.float32)
        x[0, :300] = 0
        xs.append(x)
    return xs[(1.0, 0.02, 30.0).index(scale)]


def codecs_random():
    r = po.ref()
    out = {}
    for t in po.WEIGHT_TYPES + [po.Q8_K]:
        for scale in (1.0, 0.02, 30.0):
            x = random_rows(t, scale)
            q = r.quantize(t, x)
            key = "%s/%g" % (po.TYPE_NAMES[t], scale)
            if t == po.Q8_K:
                out[key] = {"q": sha(q.reshape(8, -1, 292)[:, 1:])}
                continue
            out[key] = {"q": sha(q), "deq": sha(r.dequantize(t, q, 2048).view(np.uint32)), "aq": sha(r.quantize_act(t, x)[..., :260])}
    json.dump(out, open(os.path.join(HERE, "codecs_random.json"), "w"), indent=1, sort_keys=True)


def live_eval():
    hp = dict(TINY_40B)
    tensors = synth_model(hp, po.Q3_K, seed=31)
    path = os.path.join(tempfile.gettempdir(), "live_q3k.ggcc")
    ggcc.write_ggcc(path, hp, tensors, ftype=12)
    ref = po.RefFalcon(path, n_ctx=64, n_batch=8, logits_all=True)
    toks = np.array([11, 70, 71, 72, 73], np.int32)
    logits = ref.eval(toks, 0, n_threads=2)
    ref.close()
    os.remove(path)
    np.savez_compressed(os.path.join(HERE, "tiny40b_q3_K_live.npz"), tokens=toks, logits=logits)


SAMPLING_CASES = [(40, 0.95, 0.8, 1.1, 64), (1, 1.0, 0.8, 1.0, 0), (200, 0.5, 1.3, 1.3, 16), (40, 1.0, 0.0, 1.2, 64), (7, 0.9, 0.7, 1.0, 0),
                  (1000, 0.999, 2.0, 1.05, 200)]


def sampling_logits(rng, n_vocab, win):
    """one row of the seeded logits stream of tests/test_sampling_gpu.py"""
    logits = (rng.standard_normal(n_vocab) * 3.0).astype(np.float32)
    logits[rng.integers(0, n_vocab, size=5)] += 6.0
    if win:
        logits[win[-1]] += 5.0
    return logits


def _ref_model():
    hp = dict(TINY_40B)
    tensors = synth_model(hp, po.Q4_K, seed=1234)
    path = os.path.join(tempfile.gettempdir(), "samp.ggcc")
    ggcc.write_ggcc(path, hp, tensors, ftype=15)
    return po.RefFalcon(path, n_ctx=64, n_batch=8), hp, tensors, path


def sampling():
    ref, _, _, path = _ref_model()
    out = {}
    n_vocab, steps, seed = 65024, 48, 4242
    for top_k, top_p, temp, penalty, last_n in SAMPLING_CASES:
        rng = np.random.default_rng(top_k + last_n)
        history = list(rng.integers(0, n_vocab, size=100))
        ref.set_seed(seed)
        win, ids = history[-last_n:] if last_n > 0 else [], []
        for _ in range(steps):
            w = ref.sample(sampling_logits(rng, n_vocab, win), win, top_k, top_p, temp, penalty)
            ids.append(w)
            if last_n > 0:
                win = (win + [w])[-last_n:]
        out["%d/%g/%g/%g/%d" % (top_k, top_p, temp, penalty, last_n)] = ids
    ref.close()
    os.remove(path)
    json.dump(out, open(os.path.join(HERE, "sampling.json"), "w"))


def generate():
    """falcon_main's loop: eval -> the reference's sampling chain on the host -> eval, with the logits of the oracle's falcon_eval.
    Stores every logits row the chain sampled from with the ids it drew, so that the device sampler can be replayed on the same rows."""
    ref, hp, tensors, path = _ref_model()
    o = po.OrcFalcon(hp, tensors, n_ctx=64)
    prompt = np.array([11, 100, 101, 102, 103], np.int32)
    rows = [o.eval(prompt, 0)[0]]
    seed, steps = 77, 20
    ref.set_seed(seed)
    win = [int(t) for t in prompt]
    first = ref.sample(rows[0], win, 40, 0.95, 0.8, 1.1)
    ref.set_seed(seed)
    win.append(first)
    ids, tok = [], first
    for i in range(steps):
        rows.append(o.eval(np.array([tok], np.int32), len(prompt) + i)[0])
        tok = ref.sample(rows[-1], win[-64:], 40, 0.95, 0.8, 1.1)
        win.append(tok); ids.append(tok)
    ref.close()
    os.remove(path)
    np.savez_compressed(os.path.join(HERE, "generate.npz"), prompt=prompt, logits=np.array(rows, np.float32), first=first, ids=np.array(ids, np.int32),
                        seed=seed)


if __name__ == "__main__":
    codecs_random()
    generate()
    live_eval()
    sampling()
    codecs()
    model("tiny40b_q4_K", TINY_40B, po.Q4_K, 1234)
    model("tiny7b_q4_0", TINY_7B, po.Q4_0, 1234)
    print("golden vectors written to", HERE)
