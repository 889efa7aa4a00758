"""Decode tok/s of a random-init Falcon model of a given shape / weight type (needs an H100).
usage: python tools/decode_any.py 7b|40b <ggml type id> [steps]"""
import sys, os, json
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ggllm_cpp_b200.binding as b
import ggllm_cpp_b200.ggcc as ggcc
from bench import peaks

SHAPES = {"7b": dict(n_vocab=65024, n_embd=4544, n_head=71, n_head_kv=1, n_layer=32, falcon_type=7),
          "40b": dict(n_vocab=65024, n_embd=8192, n_head=128, n_head_kv=8, n_layer=60, falcon_type=40),
          "180b10": dict(n_vocab=65024, n_embd=14848, n_head=232, n_head_kv=8, n_layer=10, falcon_type=40)}      # one 8-GPU stage of Falcon-180B
hp = dict(SHAPES[sys.argv[1]]); t = int(sys.argv[2]); steps = int(sys.argv[3]) if len(sys.argv) > 3 else 128
b.init(0); L = b.lib()
n_ctx = int(os.environ.get("N_CTX", "2048")); start = int(os.environ.get("N_PAST", "8"))
f = b.Falcon(hp, n_ctx=n_ctx, n_batch=1)
f.set_random(ggcc.falcon_shapes(hp), t, seed=1234)
tok = b.DevBuf(src=np.array([1234], np.int32))
e0, e1 = L.b200_event_create(), L.b200_event_create()
for p in range(8): f.decode_dev(tok.ptr, p, 0)
f.decode_dev(tok.ptr, start, 0)           # builds the decode graph of this context length's tier outside the timed region
L.b200_stream_synchronize(f.stream())
L.b200_event_record(e0, f.stream())
for i in range(steps): f.decode_dev(tok.ptr, start + i, 0)
L.b200_event_record(e1, f.stream()); L.b200_event_synchronize(e1)
ms = L.b200_event_elapsed_ms(e0, e1) / steps
wb = f.weight_bytes()
print(json.dumps(dict(model=sys.argv[1], type=t, n_past=start, ms_per_tok=round(ms, 4), tok_s=round(1e3 / ms, 1), weight_GB=round(wb / 1e9, 3),
                      roofline_tok_s=round(peaks()[0] * 1e9 / wb, 1), frac=round(wb / (ms / 1e3) / (peaks()[0] * 1e9), 3), launches=f.last_launches())))
