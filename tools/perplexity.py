"""falcon_perplexity on the device (b200_falcon_perplexity): prints the reference program's line "[1]x.xxxx,[2]x.xxxx,..." and the rate.

usage: python tools/perplexity.py MODEL.ggcc --tokens ids.npy --ctx N [--batch B] [--kv f16]
       python tools/perplexity.py --synthetic 40b|7b [--synthetic ...] [--ctx 2048] [--chunks 2] [--reps 3] [--kv f16]

MODEL.ggcc is a GGCC v10 file, ids.npy the token ids of the text (the tokenizer is not part of this library).  n_batch is
min(--batch, --ctx) as in the reference (default 512), the rope context is --ctx.  --synthetic runs bench.py's model shapes with
random weights (Falcon-40B Q4_K, Falcon-7B Q4_0) on random tokens and, with several models given, alternates them in one process.  Per
model it times the same batches three ways:
  perplexity   b200_falcon_perplexity: the head over every batch with a scored row, the scoring kernel, only the terms come back
  all_logits   b200_falcon_eval(all_logits = 1) and the copied logits scored on the host (numpy, the same arithmetic): what the
               reference's program does on this library
  prompt       b200_falcon_eval(all_logits = 0): plain prompt processing, the head over the last row of each batch
and reports tokens/s of each, the device time of one batch each way, and b200_token_nll's own time (CUDA events) on n_batch rows."""
import argparse
import json
import math
import os
import subprocess
import sys
import time
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import ggllm_cpp_b200.binding as b  # noqa: E402
import ggllm_cpp_b200.ggcc as ggcc  # noqa: E402

SYNTH = {"40b": (dict(n_vocab=65024, n_embd=8192, n_head=128, n_head_kv=8, n_layer=60, falcon_type=40), 12),     # Q4_K
         "7b": (dict(n_vocab=65024, n_embd=4544, n_head=71, n_head_kv=1, n_layer=32, falcon_type=7), 2)}         # Q4_0


def ppl_line(ppl):
    return "".join("[%d]%.4f," % (c + 1, p) for c, p in enumerate(ppl))


def host_terms(logits, targets):
    """falcon_perplexity's softmax + -log over rows of copied logits (float32 [n][V]), vectorised over the rows"""
    l = np.asarray(logits, np.float32)
    e = np.exp((l - l.max(axis=1, keepdims=True)).astype(np.float64)).astype(np.float32)
    S = np.add.accumulate(e.astype(np.float64), axis=1)[:, -1]                # sequential in id order, row by row
    p = (e[np.arange(len(targets)), targets].astype(np.float64) / S).astype(np.float32)
    with np.errstate(divide="ignore"):
        return -np.log(p.astype(np.float64)).astype(np.float32)


def all_logits_path(f, toks, n_ctx, n_batch):
    """the reference's loop on this library: every batch's logits to the host, scored there -> ppl after each chunk"""
    nll, count, ppl = 0.0, 0, []
    first = min(512, n_ctx // 2)
    for start in range(0, toks.size - n_ctx + 1, n_ctx):
        rows = [f.eval(toks[start + p0:start + min(p0 + n_batch, n_ctx)], p0, n_ctx, all_logits=True) for p0 in range(0, n_ctx, n_batch)]
        logits = np.concatenate(rows)
        t = host_terms(logits[first:n_ctx - 1], toks[start + first + 1:start + n_ctx])
        for x in t:
            nll += float(x)
            count += 1
        ppl.append(math.exp(nll / count))
    return np.array(ppl)


def prompt_path(f, toks, n_ctx, n_batch):
    for start in range(0, toks.size - n_ctx + 1, n_ctx):
        for p0 in range(0, n_ctx, n_batch):
            f.eval(toks[start + p0:start + min(p0 + n_batch, n_ctx)], p0, n_ctx)


def batch_device_ms(f, toks, n_ctx, n_batch, reps=5):
    """device time (the eval's own CUDA events) of one full batch at n_past n_batch: all_logits 0 / 1"""
    t = toks[n_batch:2 * n_batch]
    out = {}
    for key, al in (("prompt", False), ("all_logits", True)):
        ms = []
        for _ in range(reps):
            f.eval(t, n_batch, n_ctx, all_logits=al)
            ms.append(f.last_ms())
        out[key] = float(np.median(ms))
    return out


def token_nll_ms(f, n_rows, V, reps=20):
    """b200_token_nll alone over n_rows rows of the engine's logits buffer, CUDA events on the eval stream"""
    L, st = b.lib(), f.stream()
    tg = b.DevBuf(src=np.random.default_rng(3).integers(0, V, n_rows).astype(np.int32))
    out = b.DevBuf(n_rows * 4)
    e0, e1 = L.b200_event_create(), L.b200_event_create()
    b.token_nll(f.logits_dev(), V, n_rows, tg.ptr, out.ptr, stream=st)
    L.b200_event_record(e0, st)
    for _ in range(reps):
        b.token_nll(f.logits_dev(), V, n_rows, tg.ptr, out.ptr, stream=st)
    L.b200_event_record(e1, st)
    L.b200_event_synchronize(e1)
    ms = L.b200_event_elapsed_ms(e0, e1) / reps
    L.b200_event_destroy(e0)
    L.b200_event_destroy(e1)
    return ms


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def synthetic(args):
    engines = {}
    n_ctx = args.ctx
    n_batch = min(args.batch, n_ctx)
    for m in args.synthetic:
        hp, wt = SYNTH[m]
        f = b.Falcon(hp, n_ctx=n_ctx, n_batch=n_batch, kv_f16=args.kv == "f16")
        f.set_random(ggcc.falcon_shapes(hp), wt, seed=1234)
        toks = np.random.default_rng(7).integers(12, hp["n_vocab"], size=args.chunks * n_ctx).astype(np.int32)
        f.perplexity(toks[:n_ctx], n_ctx)                                  # warm-up: every batch shape, the decode graphs, the scratch
        f.eval(toks[:n_batch], 0, n_ctx, all_logits=True)
        engines[m] = (f, toks, {"perplexity": [], "all_logits": [], "prompt": []})
    n_tok = args.chunks * n_ctx
    for _ in range(args.reps):
        for m, (f, toks, t) in engines.items():
            t0 = time.perf_counter()
            ppl, _ = f.perplexity(toks, n_ctx)
            t["perplexity"].append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            ppl_host = all_logits_path(f, toks, n_ctx, n_batch)
            t["all_logits"].append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            prompt_path(f, toks, n_ctx, n_batch)
            t["prompt"].append(time.perf_counter() - t0)
            t.setdefault("ppl", ppl_line(ppl))
            t.setdefault("same_ppl", bool(np.array_equal(ppl, ppl_host)))
    gpu = card()
    for m, (f, toks, t) in engines.items():
        hp, wt = SYNTH[m]
        rate = {k: round(n_tok / float(np.median(t[k])), 1) for k in ("perplexity", "all_logits", "prompt")}
        dev = batch_device_ms(f, toks, n_ctx, n_batch)
        res = dict(model="falcon" + m, weights=ggcc.TYPE_NAME[wt], kv=args.kv, n_ctx=n_ctx,
                   n_batch=n_batch, tokens=n_tok, reps=args.reps, tok_s=rate,
                   perplexity_overhead_vs_prompt_pct=round(100.0 * (rate["prompt"] / rate["perplexity"] - 1.0), 2),
                   batch_device_ms=dict((k, round(v, 3)) for k, v in dev.items()),
                   head_all_rows_ms_per_batch=round(dev["all_logits"] - dev["prompt"], 3),
                   token_nll_ms_per_batch=round(token_nll_ms(f, n_batch, hp["n_vocab"]), 3),
                   ppl=t["ppl"], ppl_equal_to_host_scoring=t["same_ppl"], gpu=gpu)
        print(json.dumps(res))
        f.free()


def from_file(args):
    hp = b.Falcon.read_hparams(args.model)
    toks = np.load(args.tokens).astype(np.int32).ravel()
    n_batch = min(args.batch, args.ctx)
    f = b.Falcon(hp, n_ctx=args.ctx, n_batch=n_batch, kv_f16=args.kv == "f16")
    f.load_ggcc(args.model)
    t0 = time.perf_counter()
    ppl, _ = f.perplexity(toks, args.ctx)
    dt = time.perf_counter() - t0
    print(ppl_line(ppl))
    n = ppl.size * args.ctx
    print("%d chunks of %d tokens, n_batch %d: %.2f s, %.1f tokens/s (%s)" % (ppl.size, args.ctx, n_batch, dt, n / dt if dt > 0 else 0.0, card()),
          file=sys.stderr)
    f.free()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("model", nargs="?")
    ap.add_argument("--tokens")
    ap.add_argument("--ctx", type=int, default=2048)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--kv", choices=("f32", "f16"), default="f32")
    ap.add_argument("--synthetic", action="append", choices=sorted(SYNTH))
    ap.add_argument("--chunks", type=int, default=2, help="synthetic: chunks of --ctx tokens per timed pass")
    ap.add_argument("--reps", type=int, default=3, help="synthetic: timed passes per model (models alternate)")
    args = ap.parse_args()
    if not args.synthetic and not (args.model and args.tokens):
        ap.error("give MODEL.ggcc --tokens ids.npy, or --synthetic 40b|7b")
    b.init(0)
    synthetic(args) if args.synthetic else from_file(args)


if __name__ == "__main__":
    main()
