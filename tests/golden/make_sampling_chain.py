"""Generate tests/golden/sampling_chain.json from the UNMODIFIED reference: falcon_main's whole sampling chain (oracle/ref_sample_chain.cpp,
built into oracle/_ref/libfalcon_chain.so by `make -C oracle -f sample_chain.mk` after `make -C oracle ref`) over the rows of
tests/sampling_chain_cases.py.

Run where oracle/_ref is built:   python tests/golden/make_sampling_chain.py

Mirostat 1 takes N from the context's n_vocab, so the reference context is a tiny model (n_embd 256, 2 layers) with n_vocab 65,024,
written to a temporary GGCC file that is removed afterwards.  Per case the file stores the ids drawn, the row attempt used at every
step (see sampling_chain_cases.row) and, for mirostat, mu after every step.
"""
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from helpers import po, ggcc, synth_model, TINY_40B  # noqa: E402
import refchain  # noqa: E402
import sampling_chain_cases as sc  # noqa: E402


def reference_context():
    hp = dict(TINY_40B, n_vocab=sc.N_VOCAB)
    path = os.path.join(tempfile.gettempdir(), "chain_v65024.ggcc")
    ggcc.write_ggcc(path, hp, synth_model(hp, po.Q4_0, seed=7), ftype=ggcc.FTYPE_OF_TYPE[po.Q4_0])
    return refchain.RefChain(path, n_ctx=64), path


def run_case(ref, name):
    c = sc.CASES[name]
    args = {k: c[k] for k in ("top_k", "top_p", "tfs_z", "typical_p", "temp", "repeat_penalty", "frequency_penalty", "presence_penalty",
                              "mirostat", "mirostat_tau", "mirostat_eta", "logit_bias")}
    ref.set_seed(sc.SEED)
    mu = 2.0 * c["mirostat_tau"]
    win, ids, attempts, mus = sc.window0(name), [], [], []
    for s in range(sc.STEPS):
        a = 0
        while not sc.distinct(sc.effective_row(c, sc.row(name, s, a, win), win)):
            a += 1
        tok, mu = ref.sample_chain(sc.row(name, s, a, win), win, mu, **args)
        ids.append(tok); attempts.append(a); mus.append(mu)
        if c["repeat_last_n"] > 0:
            win = (win + [tok])[-c["repeat_last_n"]:]
    out = {"ids": ids, "attempts": attempts}
    if c["mirostat"]:
        out["mu"] = mus
    return out


def main():
    ref, path = reference_context()
    assert ref.n_vocab == sc.N_VOCAB
    out = {name: run_case(ref, name) for name in sorted(sc.CASES)}
    ref.close()
    os.remove(path)
    json.dump(out, open(os.path.join(HERE, "sampling_chain.json"), "w"))
    print("wrote", os.path.join(HERE, "sampling_chain.json"))


if __name__ == "__main__":
    main()
