"""Device time of b200_quantize_weights_rows on one Falcon-40B ffn_up-sized matrix (32768 rows of 8192) per type (needs an H100).
Prints one JSON line per type: milliseconds per call, the median of 3 after a warm-up, from CUDA events on the backend stream.

On an H100 80GB HBM3 at its 700 W limit: Q4_0 1.13 ms, Q2_K 3.98, Q3_K 4.09, Q4_K 5.52, Q5_K 5.76, Q6_K 5.76.  Q2_K / Q4_K /
Q5_K run one thread per row so that each row's blocks see the codes of the block before; with one thread per block (which
got rows with repeating blocks wrong) they took 2.70, 4.58 and 4.98 ms, timed on the host around a synchronised call."""
import sys, os, json
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ggllm_cpp_b200.binding as b

BLOCK = {2: (32, 18), 10: (256, 84), 11: (256, 110), 12: (256, 144), 13: (256, 176), 14: (256, 210)}


def main():
    b.init(0)
    L = b.lib()
    rows, K = 32768, 8192
    types = [int(t) for t in sys.argv[1].split(",")] if len(sys.argv) > 1 else [12, 2, 10, 11, 13, 14]
    x = np.random.default_rng(0).standard_normal((rows, K), dtype=np.float32)
    xd = b.DevBuf(src=x)
    e0, e1 = L.b200_event_create(), L.b200_event_create()
    for t in types:
        qk, bb = BLOCK[t]
        out = b.DevBuf(rows * K // qk * bb)
        ms = []
        for _ in range(4):
            L.b200_event_record(e0, None)
            assert L.b200_quantize_weights_rows(t, xd.ptr, out.ptr, rows * K, K) == 1
            L.b200_event_record(e1, None)
            L.b200_synchronize()
            ms.append(L.b200_event_elapsed_ms(e0, e1))
        out.free()
        print(json.dumps({"type": t, "rows": rows, "K": K, "ms": round(float(np.median(ms[1:])), 2)}))
    L.b200_event_destroy(e0), L.b200_event_destroy(e1)


if __name__ == "__main__":
    main()
