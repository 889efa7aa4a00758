"""-m gpu: the models bench.py times, node by node at full depth and width, on the data the device makes for them.

bench.py builds every model with Falcon.set_random (weights hashed straight into the planar layout on the device, LayerNorm vectors
from fill_kernel) and pre-fills config 5's 8000 KV positions with kv_fill_random.  tests/device_random.py makes the same bytes on the
host, so engine_nodes.check_eval can hold each node of those models to its exact bound.  Geometry, weight type, n_ctx, first position
and RoPE context come from bench.py's own tables; each engine is built through bench.Ctx.make_model and driven through the prefix of
bench.decode_leg / prompt_leg (BOS eval or kv_fill_random, decode_dev steps with token 1234, three eval steps; the prompt's warm-up
chunk, then its chunks).

At each checked step:
  * the rows the step writes are saved for every layer, the step runs with the tap off (logits, KV rows of the checked layers kept),
    the rows are restored and the step runs again with the tap on the checked layers; a graph replay reruns the step before it too,
    so the tapped step is a replay as well;
  * (h) logits and the checked layers' KV rows are bit-identical between the two runs;
  * full nodes (a)-(g) on the layer windows {0, 1}, {NL/2 - 1, NL/2}, {NL - 2, NL - 1} and the head (mat-mul outputs: the first and
    last row of every 128-row tile and the last row);
  * at one token per step, the residual chain (a) over all NL layers, from a tap of every layer (at n_batch 512 in groups of layers,
    each group from its own rerun, each rerun held to (h)).

| config   | model                   | checked                                                                                     |
| headline | 40B Q4_K, n_ctx 2048, n_batch 512 | BOS eval at 0, the first decode_dev graph at 1, a replay at 31; greedy generation of 8 |
| 3        | the same model and engine shape   | prompt chunk 0, and chunk 3 (n_past 1536) on {NL-2, NL-1}: GEMMs, wgmma prompt attention, fp16 shadow |
| 2        | 7B Q4_0                 | decode_dev at 1 (capture) and 127 (replay)                                                  |
| 4        | 40B Q3_K                | decode_dev at 1, two-stream per-node path                                                   |
| 5        | 40B Q4_K, n_ctx 8192    | decode_dev at 8000 and eval at 8003 over the kv_fill_random rows (long-context tier)        |

Sensitivity (headline): a twin with one nibble of layer NL - 1's wo flipped fails at that layer's ao; a twin whose layer-0 qkv takes
the neighbouring tensor's seed fails at qkv, and one of model seed + 1 at layer 0's input rows.

Each configuration prints the largest |residual| per checked layer, the logit scale, the share of attention rows whose top probability
exceeds 0.99, the wall time and the device memory in use at its peak; only their finiteness is asserted.
"""
import inspect
import subprocess
import time
import types

import numpy as np
import pytest
import pyoracle as po

import bench
import device_random as dr
import engine_nodes as en
from helpers import ggcc
from test_engine_nodes_gpu import _kernel_of, read_tap

pytestmark = pytest.mark.gpu

MODEL_SEED = inspect.signature(bench.Ctx.make_model).parameters["seed"].default
KV_SEED = 77            # bench.decode_leg: kv_fill_random(0, pos0, seed=77)
DEV_TOKEN = 1234        # bench.decode_leg: the token decode_dev feeds every step
BOS = 11                # bench.decode_leg: the BOS warm-up eval
WARMUP = 3              # bench.main: warmup = max(--warmup, 3)


def device_used_mb():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=memory.used", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout
        return float(out.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return float("nan")


# ------------------------------------------------------------------------------------------------ the twin as an engine_nodes.Model
class _Tensors(dict):
    """{name: (type, ne, data)}: 1-D LayerNorm vectors made on first use, matrices as (type, ne, None) -- their rows come from
    TwinModel.raw_rows"""

    def __init__(self, shapes, wtype, seeds):
        super().__init__()
        self.shapes, self.wtype, self.seeds = shapes, wtype, seeds

    def __missing__(self, name):
        ne = self.shapes[name]
        v = (po.F32, ne, dr.layernorm_vector(name, ne[0], self.seeds[name])) if len(ne) == 1 else (self.wtype, ne, None)
        self[name] = v
        return v


class TwinModel(en.Model):
    """the model Falcon.set_random(falcon_shapes(hp), wtype, seed) makes, built lazily: only the rows a check asks for.
    seed_delta {name: d}: that tensor takes seed + d (sensitivity); patch {name: fn(rows, blocks)} edits the rows made"""

    def __init__(self, hp, wtype, seed, seed_delta=None, patch=None):
        shapes = ggcc.falcon_shapes(hp)
        self.seeds = dr.tensor_seeds(shapes, seed)
        for n, d in (seed_delta or {}).items():
            self.seeds[n] += d
        super().__init__(hp, _Tensors(shapes, wtype, self.seeds))
        self.patch, self.cache = patch or {}, {}

    def raw_rows(self, name, rows):
        rows = np.atleast_1d(np.asarray(rows, np.int64))
        key = (name, rows.tobytes())
        if key not in self.cache:
            t, ne, _ = self.t[name]
            blocks = dr.weight_rows(t, ne[0], rows, self.seeds[name])
            if name in self.patch:
                self.patch[name](rows, blocks)
            self.cache[key] = blocks
        return self.cache[key]


# ------------------------------------------------------------------------------------------------ driving an engine like bench.py
def make_engine(gpu, hp, wtype, n_ctx, n_batch):
    cx = types.SimpleNamespace(world=1, rank=0, b=gpu)
    return bench.Ctx.make_model(cx, hp, wtype, n_ctx, n_batch)


def windows(NL):
    return [0, 1, NL // 2 - 1, NL // 2, NL - 2, NL - 1]


class Driver:
    """runs steps ("eval" | "dev", token(s), n_past) on one engine with bench.py's RoPE context, and checks chosen steps"""

    def __init__(self, gpu, f, hp, wtype, n_ctx, n_batch, rope, name):
        self.gpu, self.f, self.hp, self.wtype = gpu, f, hp, wtype
        self.n_ctx, self.n_batch, self.rope, self.name = n_ctx, n_batch, rope, name
        self.NL = hp["n_layer"]
        self.m = TwinModel(hp, wtype, MODEL_SEED)
        self.L = gpu.lib()
        self.tok = gpu.DevBuf(src=np.array([DEV_TOKEN], np.int32))
        self.windows_at = {}                                # {n_past: the checked layers of that step}, default windows(NL)
        self.stats = {"max_residual": {}, "logit_scale": [], "top_p_over_0.99": [], "device_used_mb": device_used_mb()}
        self.t0 = time.time()

    def run(self, step):
        """-> (logits [rows][n_vocab], r0) of one step"""
        kind, toks, n_past = step
        f = self.f
        if kind == "eval":
            toks = np.atleast_1d(np.asarray(toks, np.int32))
            return f.eval(toks, n_past, self.rope), toks.size - 1
        buf = self.tok if toks == DEV_TOKEN else self.gpu.DevBuf(src=np.array([toks], np.int32))
        f.decode_dev(buf.ptr, n_past, self.rope)
        self.L.b200_stream_synchronize(f.stream())
        out = np.empty((1, f.n_vocab), np.float32)
        self.L.b200_memcpy_d2h(out.ctypes.data, f.logits_dev(), out.nbytes)
        return out, 0

    def kv(self, layers, pos=0, n=None):
        return [self.f.kv_read(l, pos, self.n_ctx if n is None else n) for l in layers]

    def restore(self, saved, pos):
        for l, (k, v) in enumerate(saved):
            self.f.kv_write(l, pos, k, v)

    def check(self, steps, sens=None):
        """steps: the step before the checked one (a replay) and the checked one, or the checked one alone.  sens: called with
        (model, Eval, layers, head, rotated) of the window {NL-2, NL-1} and {0, 1} after they passed"""
        f, NL, m = self.f, self.NL, self.m
        kind, toks, n_past = steps[-1]
        toks = np.atleast_1d(np.asarray(toks, np.int32))
        N, T = toks.size, n_past + toks.size
        print("[bench model check] %s: %s at n_past %d, %d token(s), %.0f s" % (self.name, kind, n_past, N, time.time() - self.t0), flush=True)
        p0 = steps[0][2]
        win = self.windows_at.get(n_past, windows(NL))
        saved = self.kv(range(NL), p0, T - p0)
        for s in steps[:-1]:
            self.run(s)
        before = self.kv(win)
        logits_off, r0 = self.run(steps[-1])
        kv_off = self.kv(win)
        shadow = self.n_batch > 8 and m.D == 64

        def tapped_run(layers):
            self.restore(saved, p0)
            f.tap_layers(layers)
            for s in steps[:-1]:
                self.run(s)
            logits, _ = self.run(steps[-1])
            assert np.array_equal(logits.view(np.uint32), logits_off.view(np.uint32)), \
                "%s n_past %d: logits differ with the tap on layers %s" % (self.name, n_past, list(layers)[:3])
            return logits

        try:
            logits = tapped_run(win)
            after = self.kv(win)
            for l, (a, b) in zip(win, zip(after, kv_off)):
                assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32)), \
                    "%s n_past %d: layer %d KV differs with the tap on" % (self.name, n_past, l)
            self.stats["device_used_mb"] = max(self.stats["device_used_mb"], device_used_mb())
            layers, head, rotated = read_tap(f, m, N, N - r0, layer_ids=win)
            sh = [f.kv_shadow_read(l, 0, T) for l in win] if shadow else None
            theta = po.orc().theta_scale(m.D, self.rope or self.n_ctx)
            ev = en.Eval(toks, n_past, r0, before, after, sh, logits, theta, _kernel_of,
                         en.attention_kind(N, n_past, shadow), rows_subset=True)
            last = len(win) // 2 - 1
            for w in range(last + 1):
                sel = slice(2 * w, 2 * w + 2)
                ev_w = en.Eval(toks, n_past, r0, before[sel], after[sel], sh[sel] if sh else None, logits, theta, _kernel_of,
                               ev.attn_kind, rows_subset=True)
                en.check_eval(m, ev_w, layers[sel], head if w == last else None, rotated[sel], layer_ids=win[sel])
                if sens is not None:
                    sens(w, ev_w, layers[sel], head if w == last else None, rotated[sel], win[sel])
            self.data_stats(ev, layers, head, rotated, win)
            if N == 1:                                        # (a) over every layer
                group = NL if self.n_batch == 1 else 15
                res = []
                for g0 in range(0, NL, group):
                    ids = list(range(g0, min(NL, g0 + group)))
                    tapped_run(ids)
                    self.stats["device_used_mb"] = max(self.stats["device_used_mb"], device_used_mb())
                    for l in ids:
                        res.append({k: f.tap_read(l, k, np.float32, (N, m.E)) for k in ("inp", "ao", "dn")})
                    if g0 + group >= NL:
                        hd = {"inp": f.tap_read(-1, "inp", np.float32, (N, m.E))}
                en.check_residuals(m, ev, res, hd)
        finally:
            f.tap(False)
        return ev, layers, head, rotated

    def data_stats(self, ev, layers, head, rotated, win):
        m = self.m
        N, H, HKV, D = ev.N, m.H, m.HKV, m.D
        pos = ev.n_past + np.arange(N)
        T = ev.n_past + N
        top = []
        for i, (l, nd) in enumerate(zip(win, layers)):
            self.stats["max_residual"][l] = max(self.stats["max_residual"].get(l, 0.0), float(np.abs(nd["inp"]).max()))
            q3 = nd["qkv"].reshape(N, H + 2 * HKV, D)
            q = q3[:, :H] if rotated[i] else en.rope64(q3[:, :H], pos, ev.theta_scale)[0].astype(np.float32)
            K = ev.kv_after[i][0][:T].reshape(T, HKV, D)
            for g in range(HKV):
                s = np.einsum("nhd,td->nht", q[:, g * (H // HKV):(g + 1) * (H // HKV)], K[:, g]) / np.float32(np.sqrt(D))
                s = np.where(np.arange(T)[None, None, :] <= pos[:, None, None], s, -np.inf)
                s = s - s.max(-1, keepdims=True)
                p = np.exp(s)
                top.append((p.max(-1) / p.sum(-1)).ravel())
        top = np.concatenate(top)
        self.stats["top_p_over_0.99"].append(float((top > 0.99).mean()))
        self.stats["logit_scale"].append(float(np.abs(head["logits"]).max()))

    def report(self):
        st = self.stats
        st["seconds"] = round(time.time() - self.t0, 1)
        print("\n[bench model data] %s: %s" % (self.name, st))
        vals = list(st["max_residual"].values()) + st["logit_scale"] + st["top_p_over_0.99"]
        assert vals and np.all(np.isfinite(vals)), st


def prefix(first, last, evals_at=(), start_with_bos=True):
    """bench.decode_leg's order: BOS eval at 0 (or nothing: kv_fill_random), decode_dev steps, eval steps at `evals_at`"""
    steps = [("eval", [BOS], 0)] if start_with_bos else []
    for p in range(first, last + 1):
        steps.append(("eval", [100 + p % 1000], p) if p in evals_at else ("dev", DEV_TOKEN, p))
    return steps


def drive(d, steps, checked, sens=None):
    """run `steps`; at a position in `checked` (value: replay or not) check it instead of just running it.  sens: {position: the
    sensitivity callback of that step's check}"""
    for i, s in enumerate(steps):
        if s[2] in checked:
            d.check(steps[i - 1:i + 1] if checked[s[2]] else [s], (sens or {}).get(s[2]))
        elif not (i + 1 < len(steps) and checked.get(steps[i + 1][2])):
            d.run(s)                                       # the step before a checked replay runs inside check


def config(key):
    model, wtype, n_ctx, pos0, _ = bench.decode_config(key, 1)
    hp = dict(bench.MODELS[model])
    return hp, wtype, n_ctx, pos0, 129 if pos0 == 0 else n_ctx


# ------------------------------------------------------------------------------------------------ sensitivity
def _flip_nibble(m, layer, nd):
    """a patch for layer `layer`'s Q4_K wo: in row 0, the element with the largest activation code among those whose 6-bit sub-scale
    is not zero gets its 4-bit code XOR 8"""
    K, name = m.E, m.name(layer, "wo")
    q = np.abs(nd["xatt.q"].reshape(-1, K)[0].astype(np.int32))
    planes = dr.weight_planes(m.wtype(name), K, [0], m.seeds[name])
    sc = planes[1].reshape(K // 256, 4, 4)[:, :, :2].reshape(K // 256, 8)               # expanded {sc0, sc1, m0, m1} x 4 per block
    usable = sc[np.arange(K) // 256, (np.arange(K) % 256) // 32] != 0
    e = int(np.argmax(np.where(usable, q, -1)))
    b, i = e // 256, e % 256
    sub, l = i // 32, i % 32
    off = b * 144 + 16 + (sub // 2) * 32 + l                                             # block_q4_K: d, dmin, scales[12], qs[128]

    def patch(rows, blocks):
        blocks[rows == 0, off] ^= np.uint8(0x08 << (4 * (sub & 1)))
    return patch


def headline_sensitivity(hp, wtype):
    """-> (the check callback, {case: (layer, node) where the mutated twin failed})"""
    NL, hit = hp["n_layer"], {}
    qkv0 = "transformer.h.0.self_attention.query_key_value.weight"

    def sens(w, ev, layers, head, rotated, ids):
        cases = []
        if w == 2:
            m = TwinModel(hp, wtype, MODEL_SEED)
            m.patch = {m.name(NL - 1, "wo"): _flip_nibble(m, NL - 1, layers[1])}
            cases = [("flip", m, head)]
        if w == 0:
            cases = [("tensor_seed", TwinModel(hp, wtype, MODEL_SEED, seed_delta={qkv0: 1}), None),
                     ("model_seed", TwinModel(hp, wtype, MODEL_SEED + 1), None)]
        for what, m, hd in cases:
            with pytest.raises(en.NodeError) as e:
                en.check_eval(m, ev, layers, hd, rotated, layer_ids=ids)
            hit[what] = (e.value.layer, e.value.node)
    return sens, hit


# ------------------------------------------------------------------------------------------------ the configurations
def test_headline(gpu):
    """the headline engine (bench.py builds it with n_batch 512 so that config 3's prompt can run on it): BOS eval, the first
    decode_dev graph, a replay 30 positions later; the sensitivity cases; greedy generation against a host arg-max loop"""
    hp, wtype, n_ctx, pos0, rope = config("headline")
    f = make_engine(gpu, hp, wtype, n_ctx, 512)
    try:
        d = Driver(gpu, f, hp, wtype, n_ctx, 512, rope, "headline")
        sens, hit = headline_sensitivity(hp, wtype)
        drive(d, prefix(1, 34, evals_at=(32, 33, 34)), {0: False, 1: False, 31: True}, sens={31: sens})
        # the checks fail at depth: mutated twins against the replayed step's tap (the true twin passed it)
        assert hit == {"flip": (hp["n_layer"] - 1, "ao"), "tensor_seed": (0, "qkv"), "model_seed": (0, "inp")}, hit
        # greedy generation (on one GPU the step graph of bench's N > 1 value path) against teacher-forced decode_dev steps
        P = 35
        saved = d.kv(range(d.NL), P, 8)
        got = f.generate_greedy(DEV_TOKEN, P, 8, rope)
        d.restore(saved, P)
        want, tok = [], DEV_TOKEN
        for i in range(8):
            tok = int(np.argmax(d.run(("dev", tok, P + i))[0][0]))
            want.append(tok)
        assert got.tolist() == want, (got.tolist(), want)
        d.report()
    finally:
        f.free()


def test_prompt_config3(gpu):
    """config 3 on an engine built like the headline one (n_batch 512): bench.prompt_leg's warm-up chunk, then chunks 0 .. 3 of its
    2048 tokens at RoPE context 0, chunk 0 checked on every window, chunk 3 (n_past 1536) on {NL - 2, NL - 1} and the head: wgmma
    GEMMs, wgmma prompt attention, fp16 shadow"""
    hp, wtype, n_ctx, _, _ = config("headline")
    f = make_engine(gpu, hp, wtype, n_ctx, 512)
    try:
        toks = np.random.default_rng(7).integers(12, hp["n_vocab"], size=2048).astype(np.int32)      # bench.prompt_leg's tokens
        d = Driver(gpu, f, hp, wtype, n_ctx, 512, 0, "config 3 prompt")
        d.windows_at[1536] = [d.NL - 2, d.NL - 1]                 # the exact attention reference over 2048 keys is the slow part
        d.run(("eval", toks[:512], 0))
        drive(d, [("eval", toks[512 * c:512 * (c + 1)], 512 * c) for c in range(4)], {0: False, 1536: False})
        d.report()
    finally:
        f.free()


@pytest.mark.parametrize("key", ["2", "4", "5"])
def test_decode_config(gpu, key):
    hp, wtype, n_ctx, pos0, rope = config(key)
    f = make_engine(gpu, hp, wtype, n_ctx, 1)
    try:
        d = Driver(gpu, f, hp, wtype, n_ctx, 1, rope, "config " + key)
        long0 = gpu.lib().b200_attention_long_launches()
        if key == "2":
            drive(d, prefix(1, 127, evals_at=(WARMUP + 1, WARMUP + 2, WARMUP + 3)), {1: False, 127: True})
        elif key == "4":
            drive(d, prefix(1, 1), {1: False})
        else:
            f.kv_fill_random(0, pos0, seed=KV_SEED)
            w = hp["n_head_kv"] * (hp["n_embd"] // hp["n_head"])
            for l in windows(d.NL):
                k, v = f.kv_read(l, 0, pos0)
                kt, vt = dr.kv_rows(l, 0, pos0, w, KV_SEED)
                assert np.array_equal(k.view(np.uint32), kt.view(np.uint32)) and np.array_equal(v.view(np.uint32), vt.view(np.uint32)), l
            steps = prefix(pos0, pos0 + 2 * WARMUP - 1, evals_at=range(pos0 + WARMUP, pos0 + 2 * WARMUP), start_with_bos=False)
            drive(d, steps, {pos0: False, pos0 + WARMUP: False})
            assert gpu.lib().b200_attention_long_launches() > long0
        d.report()
    finally:
        f.free()
