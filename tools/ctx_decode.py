"""Decode tok/s as a function of the context position (run on the GPU box).
usage: python tools/ctx_decode.py <n_ctx> [40b|7b] [--kv f32|f16|both]
--kv both builds an f32-cache and an fp16-cache engine in one process and alternates them at every position.  Each line also gives the
KV bytes one decode step reads (n_past + 1 rows of K and V, every layer) and the card and power limit it was measured on."""
import sys, os, json, subprocess
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ggllm_cpp_b200.binding as b
import ggllm_cpp_b200.ggcc as ggcc

args = [a for a in sys.argv[1:] if not a.startswith("--")]
kv = "f32"
if "--kv" in sys.argv:
    kv = sys.argv[sys.argv.index("--kv") + 1]
    args.remove(kv)
assert kv in ("f32", "f16", "both"), kv
n_ctx = int(args[0]) if len(args) > 0 else 2048
model = args[1] if len(args) > 1 else "40b"
b.init(0); L = b.lib()
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
hp = dict(n_vocab=65024, n_embd=8192, n_head=128, n_head_kv=8, n_layer=60, falcon_type=40) if model == "40b" else \
     dict(n_vocab=65024, n_embd=4544, n_head=71, n_head_kv=1, n_layer=32, falcon_type=7)
hd = hp["n_embd"] // hp["n_head"]
engines = {}
for t in (("f32", "f16") if kv == "both" else (kv,)):
    f = engines[t] = b.Falcon(hp, n_ctx=n_ctx, n_batch=1, kv_f16=(t == "f16"))
    f.set_random(ggcc.falcon_shapes(hp), 12 if model == "40b" else 2, seed=1234)
tok = b.DevBuf(src=np.array([1234], np.int32))
e0, e1 = L.b200_event_create(), L.b200_event_create()
for f in engines.values():
    for p in range(8): f.decode_dev(tok.ptr, p, 0)
for start in [8, 128, 512, 1024, 2040, 4088, 8184, 16376, 32760]:
    if start + 8 > n_ctx: break
    for t, f in engines.items():
        f.decode_dev(tok.ptr, start, 0)                             # (builds the decode graph of this tier outside the timed region)
        L.b200_stream_synchronize(f.stream())
        L.b200_event_record(e0, f.stream())
        for i in range(8): f.decode_dev(tok.ptr, start + i, 0)      # (the KV slots in between hold zeros: timing only)
        L.b200_event_record(e1, f.stream()); L.b200_event_synchronize(e1)
        ms = L.b200_event_elapsed_ms(e0, e1) / 8
        kv_bytes = (start + 4) * 2 * hp["n_head_kv"] * hd * (2 if t == "f16" else 4) * hp["n_layer"]
        print(json.dumps(dict(model=model, kv=t, n_past=start, ms_per_tok=round(ms, 3), tok_s=round(1e3 / ms, 1),
                              kv_bytes_per_step=kv_bytes, card=card)), flush=True)
for f in engines.values():
    f.free()
