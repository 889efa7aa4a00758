"""The oracle's final LayerNorm row (embedding_ref.orc_embedding) against the unmodified reference's falcon_get_embeddings (CPU build,
context loaded with embedding = true), eval by eval: DESIGN §2's loose bound on every eval, the tight one on at least half of them."""
import os
import numpy as np
import pytest
import pyoracle as po
from helpers import TINY_40B, TINY_7B, synth_model, ggcc
from embedding_ref import EMB_CPU, RefEmbedding, loose_and_tight, orc_embedding

N_CTX = 64
PROMPT = np.array([11, 100, 101, 102, 103, 104], np.int32)
# a prompt at 0, decode steps, a 12-token batch, one more step
SEQUENCE = [(PROMPT, 0)] + [(np.array([200 + i], np.int32), 6 + i) for i in range(3)] + \
           [(np.arange(120, 132, dtype=np.int32), 9), (np.array([300], np.int32), 21)]


@pytest.mark.skipif(not os.path.exists(EMB_CPU), reason="oracle/_ref/libfalcon_emb.so not present (built by oracle/embedding.mk from the reference sources)")
@pytest.mark.parametrize("hp,wt,ftype", [(TINY_40B, po.Q4_K, 15), (TINY_7B, po.Q4_0, 2)], ids=["40b-q4_K", "7b-q4_0"])
def test_oracle_row_is_the_reference_row(tmp_path, hp, wt, ftype):
    tensors = synth_model(hp, wt, seed=1234)
    path = str(tmp_path / "m.ggcc")
    ggcc.write_ggcc(path, hp, tensors, ftype=ftype)
    ref = RefEmbedding(path, n_ctx=N_CTX, n_batch=16)
    o = po.OrcFalcon(hp, tensors, n_ctx=N_CTX)
    try:
        tight = 0
        for toks, n_past in SEQUENCE:
            ref.eval(toks, n_past, n_threads=2)
            got = ref.embeddings()
            assert got.shape == (hp["n_embd"],) and np.all(np.isfinite(got))
            tight += loose_and_tight(orc_embedding(o, tensors, toks, n_past), got)
        assert 2 * tight >= len(SEQUENCE), tight
    finally:
        ref.close()
