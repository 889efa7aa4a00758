"""falcon_quantize on the device (b200_quantize_ggcc):

    python tools/quantize.py [--allow-requantize] [--leave-output-tensor] IN OUT TYPE [nthread]

TYPE by name or number as examples/falcon_quantize/quantize.cpp takes it (Q4_0 Q4_1 Q5_0 Q5_1 Q2_K Q3_K Q4_K Q5_K Q6_K Q8_0 F16 F32,
or 2 3 8 9 10 12 15 17 18 7 1 0).  nthread only decides the chunk plan, as the reference's does (default: the host's CPU count).
Prints the reference's closing lines: model size, quant size and the total histogram.

    python tools/quantize.py --bench [--layers N] [--dir DIR] [--type Q4_K]

writes a synthetic F16 GGCC file at Falcon-40B widths (n_embd 8192, 128 + 2 * 8 heads, vocabulary 65024) with N layers
(default 2), quantises it with the device and with the reference's falcon_model_quantize from oracle/_ref (nthread = the host's
CPU count) in this one call, checks that the two files are byte-identical, and prints input GB/s for both with the card's name and
power limit.
"""
import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]

# examples/falcon_quantize/quantize.cpp:17-114, in its order
QUANT_OPTIONS = [("Q4_0", 2), ("Q4_1", 3), ("Q5_0", 8), ("Q5_1", 9), ("Q2_K", 10), ("Q3_K", 12), ("Q4_K", 15), ("Q5_K", 17),
                 ("Q6_K", 18), ("Q8_0", 7), ("F16", 1), ("F32", 0)]


def parse_ftype(s):
    """try_parse_ftype: the name (any case), or the number of a listed option -> (ftype, name), or None"""
    for name, ft in QUANT_OPTIONS:
        if name == s.upper():
            return ft, name
    try:
        v = int(s)
    except ValueError:
        return None
    for name, ft in QUANT_OPTIONS:
        if ft == v:
            return ft, name
    return None


def report_lines(rep):
    mb = 1024.0 * 1024.0
    lines = ["falcon_model_quantize_internal: model size  = %8.2f MB" % (rep.size_org / mb),
             "falcon_model_quantize_internal: quant size  = %8.2f MB" % (rep.size_new / mb)]
    total = sum(rep.hist)
    if total > 0:
        lines.append("falcon_model_quantize_internal: hist: " + "".join("%5.3f " % (h / total) for h in rep.hist))
    return lines


def bench(args):
    import numpy as np
    import ggllm_cpp_b200.binding as b
    import ggllm_cpp_b200.ggcc as ggcc
    import pyoracle as po
    import quantize_file_twin as tw          # the reference's falcon_model_quantize through ctypes
    b.init(0)
    hp = dict(n_vocab=65024, n_embd=8192, n_head=128, n_head_kv=8, n_layer=args.layers, falcon_type=40)
    d = args.dir
    os.makedirs(d, exist_ok=True)
    src, dev, ref = os.path.join(d, "bench_f16.bin"), os.path.join(d, "bench_dev.bin"), os.path.join(d, "bench_ref.bin")
    rng = np.random.default_rng(1)
    tensors = {}
    for name, ne in ggcc.falcon_shapes(hp).items():
        if len(ne) == 1:
            tensors[name] = (po.F32, ne, np.ones(ne[0], np.float32))
        else:             # i.i.d. fp16 noise from a pool of rows (cheap to make, no repeated 256-blocks within a chunk)
            pool = (0.02 * rng.standard_normal((97, ne[0]))).astype(np.float16)
            idx = (np.arange(ne[1]) * 31) % 97
            tensors[name] = (po.F16, ne, pool[idx])
    ggcc.write_ggcc(src, hp, tensors, ftype=1)
    in_bytes = os.path.getsize(src)
    ftype = parse_ftype(args.type)[0]
    ncpu = os.cpu_count()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    b.quantize_ggcc(src, dev, ftype, ncpu)                  # warm-up: module load, page cache
    t0 = time.perf_counter()
    rc, rep = b.quantize_ggcc(src, dev, ftype, ncpu)
    t_dev = time.perf_counter() - t0
    assert rc == 0
    t0 = time.perf_counter()
    assert tw.ref_quantize_file(src, ref, ftype, ncpu) == 0
    t_ref = time.perf_counter() - t0
    same = open(dev, "rb").read() == open(ref, "rb").read()
    print("card: %s" % gpu)
    print("input %.2f GB F16, %d layers at Falcon-40B widths -> %s, host threads %d" % (in_bytes / 1e9, args.layers, args.type, ncpu))
    print("device    : %.2f s  %.2f GB/s input (report %.2f s, %.2f GB device memory)" % (t_dev, in_bytes / 1e9 / t_dev, rep.seconds, rep.device_bytes / 1e9))
    print("reference : %.2f s  %.2f GB/s input" % (t_ref, in_bytes / 1e9 / t_ref))
    print("byte-identical: %s" % same)
    for p in (src, dev, ref):
        os.remove(p)
    return 0 if same else 1


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--allow-requantize", action="store_true")
    ap.add_argument("--leave-output-tensor", action="store_true")
    ap.add_argument("--bench", action="store_true")
    ap.add_argument("--layers", type=int, default=2)
    ap.add_argument("--type", default="Q4_K")
    ap.add_argument("--dir", default=os.environ.get("TMPDIR", "/tmp"))
    ap.add_argument("args", nargs="*")
    a = ap.parse_args()
    if a.bench:
        return bench(a)
    if len(a.args) not in (3, 4):
        ap.error("IN OUT TYPE [nthread]")
    ft = parse_ftype(a.args[2])
    if ft is None:
        ap.error("invalid ftype '%s'" % a.args[2])
    nthread = int(a.args[3]) if len(a.args) == 4 else 0
    import ggllm_cpp_b200.binding as b
    b.init(0)
    rc, rep = b.quantize_ggcc(a.args[0], a.args[1], ft[0], nthread, a.allow_requantize, not a.leave_output_tensor)
    if rc != 0:
        print("failed to quantize model from '%s' (%d)" % (a.args[0], rc), file=sys.stderr)
        return 1
    print("\n".join(report_lines(rep)))
    print("quantized %d of %d tensors as %s in %.2f s" % (rep.n_quantized, rep.n_tensors, ft[1], rep.seconds))
    return 0


if __name__ == "__main__":
    sys.exit(main())
