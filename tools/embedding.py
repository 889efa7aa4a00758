"""falcon_get_embeddings on the device (b200_falcon_set_embeddings / b200_falcon_embeddings): the last token's row of the final LayerNorm.

usage: python tools/embedding.py MODEL.ggcc --tokens ids.npy [--ctx N] [--batch B]
       python tools/embedding.py --synthetic 40b|7b [--synthetic ...] --bench [--steps 64] [--reps 5]

MODEL.ggcc is a GGCC v10 file, ids.npy the token ids of the text (the tokenizer is not part of this library).  The ids are evaluated in
chunks of n_batch (default 512) from position 0 and the row of the last one is printed as the reference's embedding example prints it:
n_embd values, "%f " each, then a newline.
--bench times decode steps (b200_falcon_eval of one token, the captured graph with its logits copy) with embeddings off and on on
bench.py's model shapes with random weights (Falcon-40B Q4_K, Falcon-7B Q4_0).  Off and on alternate in one process, --reps times each;
every switch rebuilds the decode graph, which the untimed warm-up steps after it absorb.  Prints one JSON line per model."""
import argparse
import json
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
PROMPT = 32                                     # decode steps start after a prompt of this many tokens
WARMUP = 4                                      # untimed steps after every switch


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def decode_steps(f, toks, n_ctx):
    """one b200_falcon_eval per token at positions PROMPT.. -> seconds for all of them (each eval ends in a stream synchronise)"""
    t0 = time.perf_counter()
    for i, t in enumerate(toks):
        f.eval(toks[i:i + 1], PROMPT + i, n_ctx)
    return time.perf_counter() - t0


def bench(args):
    engines = {}
    n_ctx = PROMPT + WARMUP + args.steps
    for m in args.synthetic:
        hp, wt = SYNTH[m]
        f = b.Falcon(hp, n_ctx=n_ctx, n_batch=PROMPT)
        f.set_random(ggcc.falcon_shapes(hp), wt, seed=1234)
        toks = np.random.default_rng(7).integers(12, hp["n_vocab"], size=PROMPT + WARMUP + args.steps).astype(np.int32)
        f.eval(toks[:PROMPT], 0, n_ctx)
        engines[m] = (f, toks, {"off": [], "on": []}, {})
    for _ in range(args.reps):
        for m, (f, toks, t, launches) in engines.items():
            for mode in ("off", "on"):
                f.set_embeddings(mode == "on")
                decode_steps(f, toks[PROMPT:PROMPT + WARMUP], n_ctx)            # rebuilds the decode graph
                t[mode].append(decode_steps(f, toks[PROMPT + WARMUP:], n_ctx))
                launches[mode] = f.last_launches()
                assert (f.embeddings() is not None) == (mode == "on")
    gpu = card()
    for m, (f, toks, t, launches) in engines.items():
        hp, wt = SYNTH[m]
        rate = {k: [round(args.steps / s, 2) for s in v] for k, v in t.items()}
        med = {k: round(float(np.median(v)), 2) for k, v in rate.items()}
        print(json.dumps(dict(model="falcon" + m, weights=ggcc.TYPE_NAME[wt], steps=args.steps, reps=args.reps, decode_tok_s=rate,
                              median_tok_s=med, on_vs_off_pct=round(100.0 * (med["on"] / med["off"] - 1.0), 2),
                              launches_per_step=launches, embedding_bytes=hp["n_embd"] * 4, gpu=gpu)))
        f.free()


def from_file(args):
    hp = b.Falcon.read_hparams(args.model)
    toks = np.load(args.tokens).astype(np.int32).ravel()
    if toks.size == 0 or toks.size > args.ctx:
        sys.exit("embedding: %d tokens for a context of %d" % (toks.size, args.ctx))
    n_batch = min(args.batch, args.ctx)
    f = b.Falcon(hp, n_ctx=args.ctx, n_batch=n_batch)
    f.load_ggcc(args.model)
    f.set_embeddings(True)
    for p0 in range(0, toks.size, n_batch):
        f.eval(toks[p0:p0 + n_batch], p0, args.ctx)
    print("".join("%f " % v for v in f.embeddings()))
    f.free()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("model", nargs="?")
    ap.add_argument("--tokens")
    ap.add_argument("--ctx", type=int, default=512)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--synthetic", action="append", choices=sorted(SYNTH))
    ap.add_argument("--bench", action="store_true")
    ap.add_argument("--steps", type=int, default=64, help="bench: timed decode steps per pass")
    ap.add_argument("--reps", type=int, default=5, help="bench: timed passes per mode (off and on alternate)")
    args = ap.parse_args()
    if args.synthetic and not args.bench:
        ap.error("--synthetic goes with --bench")
    if not args.synthetic and not (args.model and args.tokens):
        ap.error("give MODEL.ggcc --tokens ids.npy, or --synthetic 40b|7b --bench")
    b.init(0)
    bench(args) if args.synthetic else from_file(args)


if __name__ == "__main__":
    main()
