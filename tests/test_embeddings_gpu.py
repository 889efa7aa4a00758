"""-m gpu: falcon_get_embeddings from the device.  b200_falcon_set_embeddings(f, 1) makes every b200_falcon_eval also return the last
token's row of the final LayerNorm ("result_norm", libfalcon.cpp:2409-2435, 2551-2557); behind the operator hook that row fills
"result_norm" of a taken-over eval.
  (a) exact: the row is orc.layernorm of the tapped head "inp" last row with ln_f, bit for bit, for the fused head (the fp32 values its
      LayerNorm kernel quantises), and the tapped "gen_na" last row for the generic head (an F16 lm_head, an F16 model); over prompts on
      the GEMM and the mat-vec path, decode steps through the captured graph, each with all_logits 0 and 1, and an fp16 KV cache;
  (b) every LayerNorm kernel that gained the output, at the real widths: the cluster kernel (decode at 8192 and 4544 columns, the
      latter with idle lanes), reg<., 2> (14848), reg<., 1> (prompt rows; decode with B200_LN_NOCLUSTER), the shared-memory kernel
      (B200_LN_SMEM; decode with B200_LN_NOCLUSTER too, the cluster kernel being chosen first);
  (c) off changes nothing: logits and launch counts bit-identical off / on / off, and a decode row after a mid-sequence switch equals
      the row of an engine that had embeddings on from its first eval;
  (d) the row within DESIGN §2's bounds of the oracle's;
  (e) behind the hook (the unmodified reference loaded with embedding = true and logits_all): falcon_get_embeddings is the standalone
      engine's row bit for bit after every taken-over eval, within the loose bound of the per-node path's, and in a saved session;
  (f) b200_falcon_embeddings is NULL before any eval, after score and decode_dev, and once switched off."""
import os
import numpy as np
import pytest
import pyoracle as po
from helpers import TINY_40B, TINY_7B, synth_model, ggcc
from embedding_ref import EMB_HOOK, RefEmbedding, loose_and_tight, orc_embedding, session_embedding
from test_real_geometry_gpu import GEOM, MODEL_SEED, random_model

pytestmark = pytest.mark.gpu
N_CTX = 64
PROMPT = np.array([11] + list(range(100, 111)), np.int32)             # 12 tokens: the GEMM with n_batch 16
BATCH = np.array([400, 401, 402, 403, 404], np.int32)                  # the mat-vec
# (tokens, n_past, all_logits)
SEQ = [(PROMPT, 0, al) for al in (False, True)] + [(BATCH, 12, al) for al in (False, True)] + \
      [(np.array([300 + i], np.int32), 17 + i, i % 2 == 1) for i in range(4)]


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def check_row(f, tensors, N, all_logits):
    """the row of the most recent eval against the tapped head: orc.layernorm of "inp" (fused head) or "gen_na" (generic head)"""
    E = f.hp["n_embd"]
    row = f.embeddings()
    assert row is not None and row.shape == (E,)
    try:
        want = f.tap_read(-1, "gen_na", np.float32, (N if all_logits else 1, E))[-1]
    except KeyError:
        inp = f.tap_read(-1, "inp", np.float32, (N, E))
        want = po.orc().layernorm(inp[-1:], tensors["transformer.ln_f.weight"][2], tensors["transformer.ln_f.bias"][2])[0]
    d = np.flatnonzero(bits(row) != bits(want))
    assert d.size == 0, "N %d all_logits %d: %d values differ, first %d: %r vs %r" % (N, all_logits, d.size, d[0], row[d[0]], want[d[0]])


def run_exact(f, tensors, seq):
    f.set_embeddings(True)
    f.tap(True)
    try:
        for toks, n_past, al in seq:
            f.eval(toks, n_past, N_CTX, all_logits=al)
            check_row(f, tensors, toks.size, al)
    finally:
        f.tap(False)


@pytest.mark.parametrize("hp,wt,overrides,kv_f16", [(TINY_40B, po.Q4_K, None, False), (TINY_7B, po.Q4_0, None, False),
                                                    (TINY_40B, po.Q4_K, {"lm_head": po.F16}, False), (TINY_40B, po.F16, None, False),
                                                    (TINY_40B, po.Q4_K, None, True)],
                         ids=["40b-q4_K", "7b-q4_0", "40b-q4_K-f16-head", "40b-f16", "40b-q4_K-kv16"])
def test_row_is_the_heads_layernorm(gpu, hp, wt, overrides, kv_f16):
    tensors = synth_model(hp, wt, seed=1234, overrides=overrides)
    f = gpu.Falcon(hp, n_ctx=N_CTX, n_batch=16, kv_f16=kv_f16)
    f.set_tensors(tensors)
    try:
        run_exact(f, tensors, SEQ)
    finally:
        f.free()


# (geometry, weights, environment, evals): which LayerNorm kernel each head row goes through is in the comment
REAL = [("40b", po.Q4_K, {}, [(12, 0, True), (5, 12, False), (1, 17, False)]),          # reg<., 1>; cluster (one head row); cluster
        ("40b", po.Q4_K, {"B200_LN_NOCLUSTER": "1"}, [(1, 0, False), (1, 1, True)]),     # reg<., 1>
        ("40b", po.Q4_K, {"B200_LN_SMEM": "1"}, [(12, 0, True)]),                         # shared memory
        ("40b", po.Q4_K, {"B200_LN_SMEM": "1", "B200_LN_NOCLUSTER": "1"}, [(1, 0, False), (1, 1, False)]),   # shared memory
        ("7b", po.Q4_0, {}, [(3, 0, True), (1, 3, False), (1, 4, False)]),                # reg<., 1>; cluster with idle lanes
        ("180b", po.Q4_K, {}, [(1, 0, False), (1, 1, False), (4, 2, True)])]              # reg<., 2>


@pytest.mark.parametrize("geom,wt,env,evals", REAL, ids=["40b", "40b-nocluster", "40b-smem", "40b-smem-nocluster", "7b", "180b"])
def test_every_layernorm_kernel_at_real_widths(gpu, monkeypatch, geom, wt, env, evals):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    hp = dict(GEOM[geom], n_layer=1)                       # the head's kernel depends on n_embd only
    tensors = random_model(hp, wt, seed=MODEL_SEED[geom] + wt)
    f = gpu.Falcon(hp, n_ctx=N_CTX, n_batch=16)
    f.set_tensors(tensors)
    try:
        rng = np.random.default_rng(5)
        run_exact(f, tensors, [(rng.integers(0, hp["n_vocab"], n).astype(np.int32), n_past, al) for n, n_past, al in evals])
    finally:
        f.free()


def test_off_changes_nothing(gpu):
    hp, tensors = TINY_40B, synth_model(TINY_40B, po.Q4_K, seed=1234)
    engines = []
    for _ in range(2):
        f = gpu.Falcon(hp, n_ctx=N_CTX, n_batch=16)
        f.set_tensors(tensors)
        engines.append(f)
    f, g = engines
    try:
        runs = []
        for on in (False, True, False):
            f.set_embeddings(on)
            out = []
            for toks, n_past, al in SEQ:
                lg = f.eval(toks, n_past, N_CTX, all_logits=al)
                out.append((lg, f.last_launches()))
                assert (f.embeddings() is not None) == on
            runs.append(out)
        for other in runs[1:]:
            for i, ((a, la), (b, lb)) in enumerate(zip(runs[0], other)):
                assert np.array_equal(bits(a), bits(b)) and la == lb, i
        # switched on between decode steps (the captured graphs are rebuilt) vs on from the first eval
        g.set_embeddings(True)
        f.set_embeddings(False)
        for k, (toks, n_past, al) in enumerate(SEQ):
            if k == 6:
                f.set_embeddings(True)
            lf, lg = f.eval(toks, n_past, N_CTX, all_logits=al), g.eval(toks, n_past, N_CTX, all_logits=al)
            assert np.array_equal(bits(lf), bits(lg)), k
            if k >= 6:
                assert np.array_equal(bits(f.embeddings()), bits(g.embeddings())), k
    finally:
        f.free()
        g.free()


ORACLE_SEQ = [(PROMPT[:6], 0)] + [(np.array([200 + i], np.int32), 6 + i) for i in range(3)] + \
             [(np.arange(120, 132, dtype=np.int32), 9), (np.array([300], np.int32), 21)]


@pytest.mark.parametrize("hp,wt", [(TINY_40B, po.Q4_K), (TINY_7B, po.Q4_0)], ids=["40b-q4_K", "7b-q4_0"])
def test_row_against_the_oracle(gpu, hp, wt):
    tensors = synth_model(hp, wt, seed=1234)
    f = gpu.Falcon(hp, n_ctx=N_CTX, n_batch=16)
    f.set_tensors(tensors)
    f.set_embeddings(True)
    o = po.OrcFalcon(hp, tensors, n_ctx=N_CTX)
    try:
        tight = 0
        for k, (toks, n_past) in enumerate(ORACLE_SEQ):
            f.eval(toks, n_past, N_CTX)
            # from the 12-token batch on, rows and KV come from the prompt GEMM's fp16 operands: DESIGN §2's bound for that path
            tight += loose_and_tight(f.embeddings(), orc_embedding(o, tensors, toks, n_past), gemm=k >= 4)
        assert 2 * tight >= len(ORACLE_SEQ), tight
    finally:
        f.free()


# test_surface_nodes_gpu.py's takeover sequence: a 6-token prompt at 0 (the learning eval), 4 decode steps, a 12-token batch at 10,
# 3 more steps
HOOK_MODELS = [(TINY_40B, po.Q4_K, 15, None), (TINY_7B, po.Q4_0, 2, None), (TINY_40B, po.Q4_K, 15, {"lm_head": po.F16})]
HOOK_SEQ = [(PROMPT[:6], 0)] + [(np.array([200 + i], np.int32), 6 + i) for i in range(4)] + [(PROMPT, 10)] + \
           [(np.array([300 + i], np.int32), 22 + i) for i in range(3)]


def hook_rows(path, tmp_path, eng=None):
    """HOOK_SEQ behind the hook -> (falcon_get_embeddings after each eval, takeover counter advanced per eval, session row)"""
    import ggllm_cpp_b200.binding as b
    ref = RefEmbedding(path, n_ctx=N_CTX, n_batch=16, logits_all=True, hook=True, n_gpu_layers=99)
    rows, taken = [], []
    try:
        for toks, n_past in HOOK_SEQ:
            t0 = b.lib().b200_surface_takeover_evals()
            ref.eval(toks, n_past, n_threads=2)
            taken.append(b.lib().b200_surface_takeover_evals() == t0 + 1)
            rows.append(ref.embeddings())
            if eng is not None:
                eng.eval(toks, n_past, N_CTX, all_logits=True)
                if taken[-1]:
                    d = np.flatnonzero(bits(rows[-1]) != bits(eng.embeddings()))
                    assert d.size == 0, "eval at n_past %d: %d values differ" % (n_past, d.size)
        sess = str(tmp_path / "s.bin")
        ref.save_session(sess, np.concatenate([t for t, _ in HOOK_SEQ]))
        return rows, taken, session_embedding(sess)
    finally:
        ref.close()


@pytest.mark.skipif(not os.path.exists(EMB_HOOK), reason="oracle/_ref/libfalcon_hook_emb.so not present (built by oracle/embedding.mk from the reference sources)")
@pytest.mark.parametrize("hp,wt,ftype,overrides", HOOK_MODELS, ids=["40b-q4_K", "7b-q4_0", "40b-q4_K-f16-head"])
def test_hook_fills_result_norm(gpu, tmp_path, monkeypatch, hp, wt, ftype, overrides):
    path = str(tmp_path / "m.ggcc")
    ggcc.write_ggcc(path, hp, synth_model(hp, wt, seed=1234, overrides=overrides), ftype=ftype)
    monkeypatch.delenv("B200_NO_TAKEOVER", raising=False)
    eng = gpu.Falcon(gpu.Falcon.read_hparams(path), n_ctx=N_CTX, n_batch=512)
    eng.load_ggcc(path)
    eng.set_embeddings(True)
    try:
        rows, taken, sess_row = hook_rows(path, tmp_path, eng)
    finally:
        eng.free()
    assert taken == [False] + [True] * (len(HOOK_SEQ) - 1)
    assert np.array_equal(bits(sess_row), bits(rows[-1]))
    monkeypatch.setenv("B200_NO_TAKEOVER", "1")
    cpu_rows, cpu_taken, cpu_sess = hook_rows(path, tmp_path)
    assert not any(cpu_taken) and np.array_equal(bits(cpu_sess), bits(cpu_rows[-1]))
    for got, want in zip(rows, cpu_rows):
        loose_and_tight(got, want, gemm=True)          # the per-node path's rows after the 12-token batch hold its fp16-operand GEMM


def test_null_when_not_produced(gpu):
    hp, tensors = TINY_40B, synth_model(TINY_40B, po.Q4_K, seed=1234)
    f = gpu.Falcon(hp, n_ctx=N_CTX, n_batch=16)
    f.set_tensors(tensors)
    tok = gpu.DevBuf(src=np.array([7], np.int32))
    try:
        f.set_embeddings(True)
        assert f.embeddings() is None
        f.eval(PROMPT, 0, N_CTX)
        assert f.embeddings() is not None
        f.score(BATCH, 12, np.array([401, 402, 403, 404, -1], np.int32), N_CTX)
        assert f.embeddings() is None
        f.eval(BATCH[:1], 12, N_CTX)
        assert f.embeddings() is not None
        f.decode_dev(tok.ptr, 13, N_CTX)
        assert f.embeddings() is None
        f.eval(BATCH[1:2], 13, N_CTX)
        assert f.embeddings() is not None
        f.set_embeddings(False)
        assert f.embeddings() is None
    finally:
        tok.free()
        f.free()
