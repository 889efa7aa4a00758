"""CPU: the node checker of tests/engine_nodes.py passes a tap built from the oracle and fails, at the named node, on each seeded defect.

The synthetic tap is what a correct engine would record: every node computed from the previous nodes with the oracle's LayerNorm and
quantiser, the exact block dots / fp16 GEMM products / exact-softmax attention of mmv_exact and attn_exact rounded once to fp32, and
GELU on its fp16 grid.  One tap per eval kind the engine has: a decode step (RoPE inside the attention kernels), a mat-vec batch and a
GEMM batch (wgmma prompt attention over the fp16 shadow).  The defects are the wiring mistakes the logit tests cannot see."""
import copy
import numpy as np
import pytest
import pyoracle as po
import actq_edges
import attn_exact
import engine_nodes as en
import mmv_exact
from helpers import TINY_40B, TINY_7B, synth_model

N_CTX = 32
KINDS = {"decode": (1, 5), "batch": (4, 3), "gemm": (12, 2)}          # (N, n_past)


def _put_actq(nd, name, a):
    for part, v in zip(("q", "d", "s", "bs"), a):
        if v is not None:
            nd[name + "." + part] = np.ascontiguousarray(v)


def simulate(hp, wt, kind, seed=5):
    """-> (model, layers, head, rotated, ev, aux): the tap of one correct eval of kind `kind` (all logits returned)"""
    orc = po.orc()
    tensors = synth_model(hp, wt, seed=seed)
    m = en.Model(hp, tensors)
    N, n_past = KINDS[kind]
    E, D, H, HKV = m.E, m.D, m.H, m.HKV
    T = n_past + N
    rng = np.random.default_rng(seed)
    tokens = rng.integers(0, hp["n_vocab"], N).astype(np.int32)
    kv_before, kv_after, shadow = [], [], [] if kind == "gemm" else None
    ev = en.Eval(tokens, n_past, 0, kv_before, kv_after, shadow, None, orc.theta_scale(D, N_CTX), lambda t, K: ("generic",),
                 en.attention_kind(N, n_past, kind == "gemm"))
    pos = n_past + np.arange(N)
    f32 = np.float32

    def mm(wname, act):
        y, _ = en.matmul_reference(m, wname, act, N, ev, np.arange(m.t[wname][1][1]))
        return y

    inp = m.rows("transformer.word_embeddings.weight", tokens)
    layers, rotated, aux = [], [], {"q_rot": [], "up_pre": []}
    for l in range(hp["n_layer"]):
        nd = {"inp": inp}
        xm = en.quantize(wt, orc.layernorm(inp, *m.ln(l, "mlp")), E)
        xa = en.quantize(wt, orc.layernorm(inp, *m.ln(l, "attn")), E) if m.dual else xm
        _put_actq(nd, "xm", xm)
        _put_actq(nd, "xa", xa)
        q3 = mm(m.name(l, "qkv"), xa).astype(f32).reshape(N, H + 2 * HKV, D)
        rot = kind != "decode"
        qr, _ = en.rope64(q3[:, :H], pos, ev.theta_scale)
        kr, _ = en.rope64(q3[:, H:H + HKV], pos, ev.theta_scale)
        if rot:
            q3[:, :H], q3[:, H:H + HKV] = qr, kr
        nd["qkv"] = q3.reshape(N, -1)
        Kb = rng.standard_normal((N_CTX, HKV * D)).astype(f32)
        Vb = rng.standard_normal((N_CTX, HKV * D)).astype(f32)
        Kb[T + 3:] = Vb[T + 3:] = 0
        Ka, Va = Kb.copy(), Vb.copy()
        Ka[n_past:T] = kr.astype(f32).reshape(N, -1)
        Va[n_past:T] = q3[:, H + HKV:].reshape(N, -1)
        kv_before.append((Kb, Vb)); kv_after.append((Ka, Va))
        if shadow is not None:
            shadow.append((Ka[:T].astype(np.float16).view(np.uint16), Va[:T].astype(np.float16).view(np.uint16).T.copy()))
        q_rot = qr.astype(f32)
        att, _ = attn_exact.reference(q_rot, Ka[:T].reshape(T, HKV, D), Va[:T].reshape(T, HKV, D), n_past, ev.attn_kind)
        nd["att"] = att.astype(f32).reshape(N, E)
        xatt = en.quantize(wt, nd["att"], E)
        _put_actq(nd, "xatt", xatt)
        nd["ao"] = mm(m.name(l, "wo"), xatt).astype(f32)
        up_pre = mm(m.name(l, "up"), xm)
        nd["up"] = mmv_exact._gelu_outputs(up_pre.astype(np.float16).astype(np.float64))[0].astype(f32)
        xup = en.quantize(wt, nd["up"], m.FF)
        _put_actq(nd, "xup", xup)
        nd["dn"] = mm(m.name(l, "down"), xup).astype(f32)
        if kind == "gemm":
            at = po.VEC_DOT_TYPE[wt]
            nd["xh_m"], nd["xh_b"], nd["xh_a"] = (actq_edges.f16_plane(at, a[0], a[1]) for a in (xm, xup, xatt))
        layers.append(nd); rotated.append(int(rot))
        aux["q_rot"].append(q_rot); aux["up_pre"].append(up_pre)
        inp = (nd["dn"] + nd["ao"]) + inp
    head = {"inp": inp}
    lm = "lm_head.weight"
    xf = en.quantize(m.wtype(lm), orc.layernorm(inp, m.t["transformer.ln_f.weight"][2], m.t["transformer.ln_f.bias"][2]), E)
    _put_actq(head, "xf", xf)
    head["logits"] = mm(lm, xf).astype(f32)
    ev.logits = head["logits"].copy()
    return m, layers, head, rotated, ev, aux


_cache = {}


def tap_of(hp, wt, kind):
    key = (hp["falcon_type"], wt, kind)
    if key not in _cache:
        _cache[key] = simulate(hp, wt, kind)
    return copy.deepcopy(_cache[key])


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("hp,wt", [(TINY_40B, po.Q4_K), (TINY_7B, po.Q4_0)])
def test_checker_passes_a_correct_tap(hp, wt, kind):
    m, layers, head, rotated, ev, _ = tap_of(hp, wt, kind)
    en.check_eval(m, ev, layers, head, rotated)


def _code(m, layers, head, ev, aux):
    q = layers[0]["xm.q"]
    q[0, 5] = q[0, 5] + 1 if q[0, 5] < 127 else q[0, 5] - 1


def _qkv_row(m, layers, head, ev, aux):
    layers[1]["qkv"][0] = layers[1]["qkv"][1]


def _k_at_next(m, layers, head, ev, aux):
    Kb, _ = ev.kv_before[0]
    Ka, _ = ev.kv_after[0]
    Ka[ev.n_past + 1:ev.n_past + ev.N + 1] = Ka[ev.n_past:ev.n_past + ev.N].copy()
    Ka[ev.n_past] = Kb[ev.n_past]


def _v_heads(m, layers, head, ev, aux):
    _, Va = ev.kv_after[1]
    D = m.D
    new = Va[ev.n_past:ev.n_past + ev.N]
    new[:, :D], new[:, D:2 * D] = new[:, D:2 * D].copy(), new[:, :D].copy()


def _kv_group(m, layers, head, ev, aux):
    l, T, D, HKV = 1, ev.n_past + ev.N, m.D, m.HKV
    Ka, Va = ev.kv_after[l]
    K, V = Ka[:T].reshape(T, HKV, D), Va[:T].reshape(T, HKV, D)
    wrong, _ = attn_exact.reference(aux["q_rot"][l], np.roll(K, 1, 1), np.roll(V, 1, 1), ev.n_past, ev.attn_kind)
    layers[l]["att"].reshape(ev.N, m.H, D)[:, 0] = wrong[:, 0]


def _rb_missing(m, layers, head, ev, aux):
    layers[1]["inp"] = layers[0]["dn"] + layers[0]["inp"]


def _gelu_skipped(m, layers, head, ev, aux):
    layers[0]["up"][:, 256:512] = aux["up_pre"][0][:, 256:512]


def _logits_row(m, layers, head, ev, aux):
    ev.logits[ev.N - 1] = ev.logits[ev.N - 2]


DEFECTS = {"activation code +-1": (_code, "batch", "xm", 0),
           "qkv row of token t taken from t+1": (_qkv_row, "batch", "qkv", 1),
           "K appended at n_past + 1": (_k_at_next, "decode", "k_cache", 0),
           "K appended at n_past + 1 (batch)": (_k_at_next, "batch", "k_cache", 0),
           "two V heads swapped": (_v_heads, "batch", "v_cache", 1),
           "query head reads the wrong KV group": (_kv_group, "batch", "att", 1),
           "query head reads the wrong KV group (decode)": (_kv_group, "decode", "att", 1),
           "rb missing from the residual add": (_rb_missing, "batch", "inp", 1),
           "GELU skipped on one 256-value chunk": (_gelu_skipped, "batch", "up", 0),
           "GELU skipped on one 256-value chunk (GEMM)": (_gelu_skipped, "gemm", "up", 0),
           "logits row of token N-2 returned for N-1": (_logits_row, "batch", "returned", -1)}


@pytest.mark.parametrize("defect", list(DEFECTS))
def test_checker_reports_each_seeded_defect_at_its_node(defect):
    fn, kind, node, layer = DEFECTS[defect]
    m, layers, head, rotated, ev, aux = tap_of(TINY_40B, po.Q4_K, kind)
    fn(m, layers, head, ev, aux)
    with pytest.raises(en.NodeError) as e:
        en.check_eval(m, ev, layers, head, rotated)
    assert (e.value.node, e.value.layer) == (node, layer), str(e.value)
