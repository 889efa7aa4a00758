"""Streamed layers on one H100 (b200_falcon_create_streamed): decode and prompt rates against the PCIe copy bound.

usage: python tools/stream_bench.py [--steps 128] [--steps-180b 32] [--out FILE]

1. pinned host -> device bandwidth: a 1 GB b200_memcpy_h2d from b200_host_malloc memory into b200_malloc memory, host clock around the
   synchronous copy, best of several runs.  This is the bound a streamed layer's copy runs against.
2. Falcon-40B Q4_K (random weights) with 0, 10, 20 and 30 of its last layers streamed: decode (decode_dev, --steps tokens) and a
   2048-token prompt in chunks of 512.
3. Falcon-180B Q4_K decode at n_ctx 2048, then at n_ctx 8192 with the KV cache pre-filled to 8000 (BASELINE config 5): the resident
   layer count comes from the device's free memory (plan_resident_layers), the last layers are streamed.

Prints one JSON document: the card, its power limit and SM clock, the bandwidth, and per run tok/s, copy bytes per eval, the achieved copy
rate over the measured bandwidth, and the device and pinned bytes.  The planning arithmetic below is plain Python, checked on the CPU.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FALCON_40B = dict(n_vocab=65024, n_embd=8192, n_head=128, n_head_kv=8, n_layer=60, falcon_type=40)
FALCON_180B = dict(n_vocab=65024, n_embd=14848, n_head=232, n_head_kv=8, n_layer=80, falcon_type=40)
F16, Q4_0, Q8_0, Q3_K, Q4_K, Q6_K = 1, 2, 8, 11, 12, 14
# ggml type -> (elements per block, bytes per block of each device plane) -- formats.cuh's TypeSpec
PLANES = {F16: (1, (2,)), Q4_0: (32, (16, 2)), Q8_0: (32, (32, 2)), Q3_K: (256, (64, 32, 16, 2)), Q4_K: (256, (128, 16, 4)),
          Q6_K: (256, (128, 64, 16, 2))}
GIB = 1 << 30
MARGIN = 2 * GIB            # CUDA context growth, the prompt attention scratch, allocator rounding


def round_up(v, a):
    return (v + a - 1) // a * a


def matrix_image_bytes(wtype, K, M):
    """device bytes of one [M][K] matrix in the planar layout (wplanes_layout): each plane's rows padded to 16 B, each plane to 256 B"""
    blk, planes = PLANES[wtype]
    nb = K // blk
    return sum(round_up(round_up(nb * b, 16) * M, 256) for b in planes)


def layer_shapes(hp):
    """(K, M) of a layer's wqkv, wo, ffn_up, ffn_down"""
    E, H, HKV = hp["n_embd"], hp["n_head"], hp["n_head_kv"]
    qkv = (H + 2 * HKV) * (E // H)
    return [(E, qkv), (E, E), (E, 4 * E), (4 * E, E)]


def layer_image_bytes(hp, wtype):
    """one layer's four matrices: its pinned image, what one eval copies for it, and the size of a device slot"""
    return sum(matrix_image_bytes(wtype, K, M) for K, M in layer_shapes(hp))


def kv_cache_bytes(hp, n_ctx, n_batch=1):
    """the f32 KV cache of every layer, plus the fp16 K and V^T planes the prompt kernel reads when n_batch > 8 (head_dim 64)"""
    row = hp["n_head_kv"] * (hp["n_embd"] // hp["n_head"])
    b = 2 * hp["n_layer"] * n_ctx * row * 4
    if n_batch > 8 and hp["n_embd"] // hp["n_head"] == 64:
        b += 2 * hp["n_layer"] * hp["n_head_kv"] * 64 * round_up(n_ctx, 64) * 2
    return b


def activation_bytes(hp, n_batch=1):
    """the engine's activation rows for n_batch tokens: residual, qkv, attention, branch outputs, ffn_up, logits (f32)"""
    E, H, HKV, V = hp["n_embd"], hp["n_head"], hp["n_head_kv"], hp["n_vocab"]
    return 4 * n_batch * (5 * E + (H + 2 * HKV) * (E // H) + 4 * E + V)


def plan_resident_layers(hp, wtype, free_bytes, n_ctx, n_batch=1):
    """-> how many layers stay resident when `free_bytes` of device memory are free: the embedding table, lm_head, the KV cache, the
    activations, the two slots and MARGIN come first; each resident layer then takes one layer image.  The rest are streamed."""
    E, V = hp["n_embd"], hp["n_vocab"]
    lay = layer_image_bytes(hp, wtype)
    fixed = 2 * matrix_image_bytes(wtype, E, V) + kv_cache_bytes(hp, n_ctx, n_batch) + activation_bytes(hp, n_batch) + 2 * lay + MARGIN
    return max(0, min(hp["n_layer"], (free_bytes - fixed) // lay))


# ------------------------------------------------------------------------------------------------ GPU part
def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().split("\n")[0]
    name, power, sm, sm_max = [s.strip() for s in q.split(",")]
    return dict(name=name, power_limit=power, sm_clock=sm, sm_clock_max=sm_max)


def h2d_bandwidth(b, nbytes=1 << 30, runs=5):
    """best of `runs` synchronous 1 GB pinned host -> device copies, bytes/s"""
    L = b.lib()
    h, d = L.b200_host_malloc(nbytes), L.b200_malloc(nbytes)
    L.b200_memset(d, 0, nbytes)
    best = 0.0
    for _ in range(runs):
        t0 = time.perf_counter()
        L.b200_memcpy_h2d(d, h, nbytes)
        best = max(best, nbytes / (time.perf_counter() - t0))
    L.b200_free(d)
    L.b200_host_free(h)
    return best


def device_used():
    import torch
    free, total = torch.cuda.mem_get_info()
    return total - free


def run_one(b, np, ggcc, hp, wtype, n_stream, n_ctx, bw, steps, prompt, prefill=0):
    """one engine with its last n_stream layers streamed -> dict of its decode (and prompt) rates"""
    L = b.lib()
    used0 = device_used()
    nl = hp["n_layer"]
    streamed = list(range(nl - n_stream, nl))
    n_batch = 512 if prompt else 1
    f = b.Falcon(hp, n_ctx=n_ctx, n_batch=n_batch, streamed=streamed)
    f.set_random(ggcc.falcon_shapes(hp), wtype, seed=1234)
    if prefill:
        f.kv_fill_random(0, prefill, seed=7)
    info = f.stream_info()
    r = dict(layers=nl, streamed=n_stream, n_ctx=n_ctx, first_pos=prefill, copy_bytes_per_eval=info["copy_bytes"],
             pinned_bytes=info["host_bytes"], slot_bytes=info["slot_bytes"])
    tok = b.DevBuf(src=np.array([1234], np.int32))
    e0, e1 = L.b200_event_create(), L.b200_event_create()
    for p in range(3):
        f.decode_dev(tok.ptr, prefill + p, 0)                    # builds the step graph, warms the copies
    L.b200_stream_synchronize(f.stream())
    L.b200_event_record(e0, f.stream())
    for i in range(steps):
        f.decode_dev(tok.ptr, prefill + i, 0)
    L.b200_event_record(e1, f.stream())
    L.b200_event_synchronize(e1)
    s = L.b200_event_elapsed_ms(e0, e1) / 1e3 / steps
    r.update(decode_tok_s=round(1.0 / s, 3), decode_ms_per_tok=round(s * 1e3, 2), decode_steps=steps,
             decode_copy_frac=round(info["copy_bytes"] / s / bw, 3) if n_stream else None)
    if prompt:
        toks = (np.arange(2048, dtype=np.int32) * 7919) % hp["n_vocab"]
        f.eval(toks[:512], 0)                                    # warm-up
        t0 = time.perf_counter()
        for c in range(0, 2048, 512):
            f.eval(toks[c:c + 512], c)                           # synchronous: logits of the chunk's last row come back
        s = (time.perf_counter() - t0) / 4
        r.update(prompt_tok_s=round(512 / s, 1), prompt_ms_per_chunk=round(s * 1e3, 1),
                 prompt_copy_frac=round(info["copy_bytes"] / s / bw, 3) if n_stream else None)
    r["device_bytes"] = device_used() - used0
    L.b200_event_destroy(e0)
    L.b200_event_destroy(e1)
    f.free()
    return r


def host_available():
    for line in open("/proc/meminfo"):
        if line.startswith("MemAvailable:"):
            return int(line.split()[1]) * 1024
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--steps-180b", type=int, default=32)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    import ggllm_cpp_b200.binding as b
    import ggllm_cpp_b200.ggcc as ggcc
    b.init(0)
    torch.cuda.init()
    out = dict(card=card())
    bw = h2d_bandwidth(b)
    out["h2d_bytes_per_s"] = round(bw)
    out["falcon40b_q4_k"] = []
    for n in (0, 10, 20, 30):
        out["falcon40b_q4_k"].append(run_one(b, np, ggcc, FALCON_40B, Q4_K, n, 2048, bw, a.steps, prompt=True))
        print(json.dumps(out["falcon40b_q4_k"][-1]), file=sys.stderr, flush=True)
    out["falcon180b_q4_k"] = []
    lay = layer_image_bytes(FALCON_180B, Q4_K)
    for n_ctx, prefill in ((2048, 0), (8192, 8000)):
        free, _ = torch.cuda.mem_get_info()
        n_res = plan_resident_layers(FALCON_180B, Q4_K, free, n_ctx)
        n_stream = FALCON_180B["n_layer"] - n_res
        need_host = n_stream * lay
        if need_host + 8 * GIB > host_available():
            out["falcon180b_q4_k"].append(dict(n_ctx=n_ctx, streamed=n_stream, device_free=free,
                                               not_measured="the host has %.1f GB available, %.1f GB of pinned images needed"
                                               % (host_available() / 1e9, need_host / 1e9)))
            continue
        r = run_one(b, np, ggcc, FALCON_180B, Q4_K, n_stream, n_ctx, bw, a.steps_180b, prompt=False, prefill=prefill)
        r["device_free_at_plan"] = free
        out["falcon180b_q4_k"].append(r)
        print(json.dumps(r), file=sys.stderr, flush=True)
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as fp:
            fp.write(s + "\n")


if __name__ == "__main__":
    main()
