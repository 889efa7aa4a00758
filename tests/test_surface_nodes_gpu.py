"""-m gpu: the ggml_cuda_* operator surface (csrc/ggml_surface.cu) node by node, called exactly as ggml.c calls it, and the surface's
whole-graph takeover held to the engine it drives, bit for bit.

Nodes.  ggml_init_cublas(false) first; weights uploaded with ggml_cuda_transform_tensor and released with ggml_cuda_free_data; every
node run through ggml_cuda_compute_forward (ADD / MUL also through ggml_cuda_mul).  A device-resident result is read back through a
SCALE by 1.0 into a host tensor (an exact copy); every host destination sits inside a guard array whose canaries must survive.
  MUL_MAT   (a) bit-identical to b200_mul_mat on the same weights and rows (the same quantise -> mat-vec / GEMM path);
            (b) inside the exact bound: N <= 8 mmv_exact.reference for the launched kernel, N > 8 the fp64 product of fp16(W) and the
                fp16 operand planes of the oracle's codes (engine_nodes.matmul_reference; the CUDA-core GEMM that takes K = 32 mod 64
                adds its K products one after another: gamma(K) sum |x w|), F16 / F32 weights mmv_exact.f_reference;
            (c) dst->meta.cuda_perf_mal_mul_type 1 for N <= 8, 16 above.
            N crosses the GEMM's 512-token chunks; src1 / dst host (staged), src1 device-resident, dst device-resident.
  ADD / MUL / SCALE   bit-identical to numpy float32, broadcasts b[i % nb] included.
  GELU      every finite fp16 input and every fp32 midpoint between neighbours: orc.gelu, or one fp16 step away where tanhf's error
            reaches that step's midpoint (mmv_exact.gelu_ok).
  NORM      bit-identical to orc.norm, except a row whose fp32 mean or variance lies within the double-summation-order error of an
            fp32 midpoint: that row must be ggml's formula with the neighbouring value.
Protocol: ith != 0, INIT and FINALIZE claim the node and write nothing; OP_NONE is claimed; a node without a device operand and a node
with cuda_op_directive 0 are not; ggml_cuda_can_mul_mat's precedence; VIEW / RESHAPE / PERMUTE / TRANSPOSE and in-place results alias
their source, with the scratch ring and without.

Takeover (needs oracle/_ref/libfalcon_hook.so, as test_dropin_gpu.py): the unmodified reference behind the hook and a b200_falcon loaded
from the same file run the same evals; every eval after the first ("learning") one must return identical logits.
"""
import math
import os
import types
import numpy as np
import pytest
import pyoracle as po
import actq_edges
import engine_nodes as en
import ggllm_cpp_b200.binding as binding
import ggml_abi as ga
import mmv_exact as mx
from helpers import TINY_40B, TINY_7B, synth_model, ggcc

pytestmark = pytest.mark.gpu
HOOK = os.path.join(po.HERE, "_ref", "libfalcon_hook.so")
CANARY = np.uint32(0x7FC0DEAD)
PAD = 64


@pytest.fixture(scope="module")
def L(gpu):
    L = ga.surface(gpu.lib())
    assert L.ggml_init_cublas(False)
    return L


class Mem:
    """device residency made through the surface, released at teardown (only what owns its memory: uploads and no-scratch nodes)"""

    def __init__(self, L):
        self.L, self.owned = L, []

    def upload(self, nd):
        nd.s.backend = ga.BACKEND_GPU
        self.L.ggml_cuda_transform_tensor(nd.s.data, nd.ptr)
        assert nd.s.extra
        self.owned.append(nd)
        return nd

    def assign(self, nd, scratch=False, owns=True):
        (self.L.ggml_cuda_assign_buffers if scratch else self.L.ggml_cuda_assign_buffers_no_scratch)(nd.ptr)
        assert nd.on_device() and nd.s.extra
        if owns and not scratch:
            self.owned.append(nd)
        return nd

    def free(self):
        for nd in reversed(self.owned):
            self.L.ggml_cuda_free_data(nd.ptr)
            assert not nd.s.extra
        self.owned = []


@pytest.fixture
def mem(L):
    m = Mem(L)
    yield m
    m.free()


class Out:
    """a host destination inside a guard array of NaN canaries"""

    def __init__(self, shape):
        n = int(np.prod(shape))
        self.full = np.full(n + 2 * PAD, CANARY, np.uint32).view(np.float32)
        self.arr = self.full[PAD:PAD + n].reshape(shape)

    def intact(self):
        u = self.full.view(np.uint32)
        return bool(np.all(u[:PAD] == CANARY) and np.all(u[-PAD:] == CANARY))

    def poisoned(self):
        return bool(np.all(self.full.view(np.uint32) == CANARY))


def bits(a):
    """the float32 bit patterns of a, flattened"""
    return np.ascontiguousarray(a, np.float32).reshape(-1).view(np.uint32)


def to_device(L, mem, x, name="x_dev"):
    """a device-resident F32 node (no-scratch buffer) holding x: SCALE by 1.0 of a host tensor into it"""
    d = ga.node(ga.OP_SCALE, ga.f32(np.ascontiguousarray(x, np.float32), name + "_h"), ga.scalar(1.0), name=name)
    mem.assign(d)
    assert ga.forward(L, d)
    return d


def readback(L, dev, shape=None):
    """the device node's values (flat unless shape is given), through SCALE by 1.0 into a guarded host tensor"""
    out = Out(shape or [dev.n])
    rb = ga.node(ga.OP_SCALE, dev, ga.scalar(1.0), name="readback", out=out.arr)
    assert ga.forward(L, rb)
    assert out.intact()
    return out.arr


# ================================================================================================ MUL_MAT
FULL_N = (1, 8, 9, 64, 65, 257, 512, 513, 1030)
LAYOUTS = ("host", "src1_dev", "dst_dev")
FLOATS = (po.F16, po.F32)


def _ks(t):
    return (8192,) if po.BLOCK_ELEMS[t] == 256 else (4544, 8192) if t in FLOATS else (4544, 8192, 4576)


def _cases():
    out = []
    for t in (po.Q4_K, po.Q4_0, po.Q3_K, po.F16):                   # the whole N sweep
        for i, N in enumerate(FULL_N):
            out.append((t, _ks(t)[i % len(_ks(t))], (300, 1000)[(i // 2) % 2], N, LAYOUTS[(i + i // 3) % 3]))
    for t in po.WEIGHT_TYPES + [po.F32]:
        if t in (po.Q4_K, po.Q4_0, po.Q3_K):
            continue
        for i, N in enumerate((1, 9, 513)):
            out.append((t, _ks(t)[i % len(_ks(t))], 300, N, LAYOUTS[(i + t) % 3]))
    out.append((po.Q4_K, 8192, 1000, 1030, "host"))                   # the largest reference: 8.4e9 fp64 multiply-adds
    return out


def _cid(c):
    return "%s-K%d-M%d-N%d-%s" % (po.TYPE_NAMES[c[0]], c[1], c[2], c[3], c[4])


def _inputs(t, K, M, N, seed):
    """weights (mmv_exact.swept_weights, ggcc.random_blocks for F16 / F32) and fp32 rows, every third one from actq_edges.edge_rows
    (E6's huge blocks only where no fp16 operand is built from them: the GEMM's fp16 planes overflow there, on the device too)"""
    rng = np.random.default_rng(seed)
    wq = ggcc.random_blocks(t, M, K, rng) if t in FLOATS else mx.swept_weights(t, M, K, rng)
    x = rng.standard_normal((N, K)).astype(np.float32)
    if t not in FLOATS:
        edge, _ = actq_edges.edge_rows(po.VEC_DOT_TYPE[t], K, only=None if N <= 8 else (lambda fam, label, b: fam != "E6"))
        idx = np.arange(1, N, 3)[:edge.shape[0]]
        x[idx] = edge[:idx.size]
    return wq, x


def _surface_mul_mat(L, mem, w, x, layout):
    """MUL_MAT of the uploaded weight node w and rows x through compute_forward in one of the three operand layouts -> (y, tag)"""
    N, M = x.shape[0], w.s.ne[1]
    out = Out((N, M))
    if layout == "host":
        mm = ga.node(ga.OP_MUL_MAT, w, ga.f32(x, "x"), name="mm", out=out.arr)
        assert ga.forward(L, mm)
    elif layout == "src1_dev":
        mm = ga.node(ga.OP_MUL_MAT, w, to_device(L, mem, x), name="mm", out=out.arr)
        assert ga.forward(L, mm)
    else:
        mm = ga.node(ga.OP_MUL_MAT, w, ga.f32(x, "x"), name="mm")
        mem.assign(mm)
        assert ga.forward(L, mm)
        rb = ga.node(ga.OP_SCALE, mm, ga.scalar(1.0), name="readback", out=out.arr)
        assert ga.forward(L, rb)
    assert out.intact()
    return out.arr.copy(), mm.s.meta.cuda_perf_mal_mul_type


def _b200_mul_mat(gpu, t, K, M, wq, x):
    W = gpu.Weight(t, K, M, wq)
    xd, yd = gpu.DevBuf(src=x), gpu.DevBuf(x.shape[0] * M * 4)
    gpu.lib().b200_mul_mat(W.h, xd.ptr, K, x.shape[0], yd.ptr, M)
    y = yd.download(np.float32, (x.shape[0], M))
    W.free()
    return y


def _check_rows(N):
    """activation rows whose bound is evaluated for F16 / F32 weights (one mat-vec reference per row): all of a small batch, else
    both ends and both sides of every 256-token boundary"""
    if N <= 16:
        return np.arange(N)
    r = [0, 1, 2, 255, 256, 511, 512, 513, 767, 768, 1023, 1024, 1025, N - 2, N - 1]
    return np.unique([v for v in r if v < N])


def _within_bound(t, K, M, wq, x, got, rows=None):
    """(b) -> (the (token, row) indices of outputs outside the bound, largest error / bound)"""
    N = x.shape[0]
    rows = np.arange(M) if rows is None else rows
    if t in FLOATS:
        w = wq.astype(np.float32)[rows]
        act_rows = _check_rows(N)
        y, b = np.zeros((act_rows.size, rows.size)), np.zeros((act_rows.size, rows.size))
        for i, n in enumerate(act_rows):
            y[i], b[i] = mx.f_reference(t, w, x[n])
        g = got[act_rows][:, rows]
    else:
        m = en.Model(dict(n_embd=K, n_head=1, n_head_kv=1, n_vocab=M, falcon_type=7), {"w": (t, (K, M), wq)})
        shape = binding.mmv_launch_shape(t, K)
        ev = types.SimpleNamespace(mmv_max_n=binding.lib().b200_mmv_max_n(),
                                   kernel_of=lambda tt, kk: ("generic",) if shape is None else ("fast", shape[0], shape[1]))
        y, b = en.matmul_reference(m, "w", en.quantize(t, x, K), N, ev, rows)
        if N > ev.mmv_max_n and K % 64:
            # the CUDA-core GEMM (gemm_simt.cu) adds the K exact fp16 x fp16 products one after another
            b = (b - 1e-30) / ((K / 8 + 2) * 2.0 ** -23) * mx.gamma(K) + 1e-30
        g = got[:, rows]
    err = np.abs(g.astype(np.float64) - y)
    bad = np.argwhere(~(err <= b))
    return bad, float((err / b).max())


def _mul_mat_failures(gpu, t, K, M, wq, x, got, tag, what, rows=None):
    """checks (a), (b) and (c) of one MUL_MAT node, all of them evaluated -> the list of those that fail"""
    N = x.shape[0]
    out = []
    diff = np.flatnonzero(bits(got) != bits(_b200_mul_mat(gpu, t, K, M, wq, x)))
    if diff.size:
        out.append("%s: (a) %d outputs differ from b200_mul_mat, first (token, row) %s" % (what, diff.size, divmod(int(diff[0]), M)))
    bad, ratio = _within_bound(t, K, M, wq, x, got, rows)
    if bad.size:
        out.append("%s: (b) %d outputs outside the exact bound, first %s, largest error / bound %.3g" % (what, len(bad), bad[:1].tolist(), ratio))
    if tag != (1 if N <= 8 else 16):
        out.append("%s: (c) cuda_perf_mal_mul_type %d" % (what, tag))
    return out


def _mul_mat_case(L, mem, gpu, t, K, M, N, layout, seed, rows=None):
    wq, x = _inputs(t, K, M, N, seed)
    w = mem.upload(ga.weight(t, K, M, wq, name="w"))
    got, tag = _surface_mul_mat(L, mem, w, x, layout)
    fails = _mul_mat_failures(gpu, t, K, M, wq, x, got, tag, "%s K %d M %d N %d %s" % (po.TYPE_NAMES[t], K, M, N, layout), rows)
    assert not fails, fails


def test_mul_mat_buffers_grow_and_shrink(L, mem, gpu):
    """N = 1030 -> 1 -> 513 -> 9 on one weight, at a K no other test reaches (the staging and activation buffers grow on the first
    step and are reused by the smaller ones); every step in a different operand layout"""
    t, K, M = po.Q4_K, 14848, 300
    rng = np.random.default_rng(14848)
    wq = mx.swept_weights(t, M, K, rng)
    w = mem.upload(ga.weight(t, K, M, wq, name="w"))
    fails = []
    for i, N in enumerate((1030, 1, 513, 9)):
        x = rng.standard_normal((N, K)).astype(np.float32)
        got, tag = _surface_mul_mat(L, mem, w, x, LAYOUTS[i % 3])
        fails += _mul_mat_failures(gpu, t, K, M, wq, x, got, tag, "step %d N %d %s" % (i, N, LAYOUTS[i % 3]))
    assert not fails, fails


@pytest.mark.parametrize("case", _cases(), ids=_cid)
def test_mul_mat_node(L, mem, gpu, case):
    t, K, M, N, layout = case
    _mul_mat_case(L, mem, gpu, t, K, M, N, layout, seed=K + M + N + t)


def test_mul_mat_node_at_real_width(L, mem, gpu):
    """Falcon-40B's lm_head shape (8192 -> 65024) at N = 3: all outputs bit-identical to b200_mul_mat, a row subset (both ends of
    every 128-row tile) inside the bound"""
    _mul_mat_case(L, mem, gpu, po.Q4_K, 8192, 65024, 3, "host", seed=65024, rows=en.output_rows(65024, True))


# ================================================================================================ elementwise
# (ne0, N, a divisor of n other than n and ne0): 4544 x N and odd totals
EW_SHAPES = [(4544, 1, 71), (4544, 7, 448), (4544, 513, 13632), (1, 1, 1), (4545, 3, 909)]


def _ew_data(rng, n):
    v = (rng.standard_normal(n) * np.exp2(rng.integers(-20, 20, n))).astype(np.float32)
    v[::97] = (rng.standard_normal(v[::97].size) * 2.0 ** -140).astype(np.float32)       # subnormals
    v[5::101] = -0.0
    return v


@pytest.mark.parametrize("entry", ["ADD", "MUL", "ggml_cuda_mul"])
@pytest.mark.parametrize("where", ["src0_dev", "src1_kind1", "dst_dev"])
def test_add_mul_broadcast_bit_exact(L, mem, entry, where):
    """dst = src0 op src1[i % nb] for same-shape operands, row broadcasts (nb = ne0) and other divisors of n; src1 host with a device
    src0 or dst, or src1 a 1-D f32 uploaded with ggml_cuda_transform_tensor (kind 1: Falcon-7B's input_layernorm.weight)"""
    rng = np.random.default_rng(len(entry) * 7 + len(where))
    op = ga.OP_ADD if entry == "ADD" else ga.OP_MUL
    for ne0, N, div in EW_SHAPES:
        n = ne0 * N
        for nb in sorted({n, ne0, div}):
            a = _ew_data(rng, n).reshape(N, ne0)
            b = _ew_data(rng, nb)
            want = (a.reshape(-1) + np.tile(b, n // nb)) if op == ga.OP_ADD else (a.reshape(-1) * np.tile(b, n // nb))
            src1 = ga.f32(b.reshape(N, ne0) if nb == n else b, "b")
            if where == "src1_kind1":
                if nb == n and N > 1:
                    continue                                             # kind 1 is a 1-D vector
                mem.upload(src1)
            src0 = to_device(L, mem, a) if where == "src0_dev" else ga.f32(a, "a")
            out = Out((N, ne0))
            if where == "dst_dev":
                dst = ga.node(op, src0, src1, name="y")
                mem.assign(dst)
            else:
                dst = ga.node(op, src0, src1, name="y", out=out.arr)
            if entry == "ggml_cuda_mul":
                L.ggml_cuda_mul(src0.ptr, src1.ptr, dst.ptr)
            else:
                assert ga.forward(L, dst)
            got = readback(L, dst) if where == "dst_dev" else out.arr
            assert out.intact() or where == "dst_dev"
            d = np.flatnonzero(bits(got) != bits(want))
            assert d.size == 0, (entry, where, ne0, N, nb, d[:4].tolist())


@pytest.mark.parametrize("s", [0.125, 3.0, -0.0])
def test_scale_bit_exact(L, mem, s):
    """the factor is read from src1->data on the host; subnormal and signed-zero inputs; device src0 -> host dst and host src0 ->
    device dst"""
    rng = np.random.default_rng(int(s * 8) + 5)
    for ne0, N, _ in EW_SHAPES:
        x = _ew_data(rng, ne0 * N).reshape(N, ne0)
        want = x * np.float32(s)
        out = Out((N, ne0))
        assert ga.forward(L, ga.node(ga.OP_SCALE, to_device(L, mem, x), ga.scalar(s), name="y", out=out.arr))
        assert out.intact() and np.array_equal(bits(out.arr), bits(want)), (s, ne0, N)
        y = ga.node(ga.OP_SCALE, ga.f32(x, "x"), ga.scalar(s), name="y")
        mem.assign(y)
        assert ga.forward(L, y)
        assert np.array_equal(bits(readback(L, y)), bits(want)), (s, ne0, N)


def test_gelu_every_fp16_input_and_midpoint(L, mem):
    h = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(np.float16)
    fin = np.unique(h[np.isfinite(h)].astype(np.float64))                 # -0 and +0 merge here; both are fed below
    mids = (fin[:-1] + fin[1:]) / 2                                       # 12 significant bits: exact in fp32
    assert np.array_equal(mids.astype(np.float32).astype(np.float64), mids)
    x = np.concatenate([h[np.isfinite(h)].astype(np.float32), mids.astype(np.float32)])
    want = po.orc().gelu(x)
    out = Out(x.shape)
    assert ga.forward(L, ga.node(ga.OP_GELU, to_device(L, mem, x), name="g", out=out.arr))
    got = out.arr
    assert out.intact()
    same = bits(got) == bits(want)
    g16, w16 = got.astype(np.float16), want.astype(np.float16)
    with np.errstate(over="ignore"):
        step = (np.nextafter(w16, np.float16(np.inf)) == g16) | (np.nextafter(w16, np.float16(-np.inf)) == g16)
    flip = ~same & step & mx.gelu_ok(got, x.astype(np.float64), np.full(x.shape, -1.0))   # bound -1: the fp16 input is exactly f16(x)
    bad = np.flatnonzero(~(same | flip))
    assert bad.size == 0, (bad.size, x[bad[:4]].tolist(), got[bad[:4]].tolist(), want[bad[:4]].tolist())


def _f32_either(v, err):
    """the fp32 values a double within err of v may round to"""
    return sorted({float(np.float32(v - err)), float(np.float32(v)), float(np.float32(v + err))})


def _norm_rows(x):
    """-> (ggml's norm of the row for every (mean, variance) an fp64 sum in any order may give, ambiguous?)"""
    n = x.size
    x64 = x.astype(np.float64)
    S = math.fsum(x64)
    outs = []
    for mu in _f32_either(S / n, (n * 2.0 ** -53 * float(np.abs(x64).sum()) + 2.0 ** -52 * abs(S)) / n):
        v = x - np.float32(mu)
        S2 = math.fsum((v * v).astype(np.float64))
        for var in _f32_either(S2 / n, (n * 2.0 ** -53 + 2.0 ** -52) * S2 / n):
            scale = np.float32(1.0) / np.sqrt(np.float32(var) + np.float32(1e-5))
            outs.append(v * scale)
    return outs, len(outs) > 1


@pytest.mark.parametrize("n", [4544, 8192, 14848])
def test_norm_rows_bit_exact(L, mem, n):
    rng = np.random.default_rng(n)
    offs = np.array([0.0, 3.0, -250.0, 1e4, -3e5, 7e6])
    scales = np.array([1.0, 1e-3, 10.0, 1.0, 0.5, 1e3])
    x = (offs[:, None] + scales[:, None] * rng.standard_normal((offs.size, n))).astype(np.float32)
    want = po.orc().norm(x)
    y = ga.node(ga.OP_NORM, ga.f32(x, "x"), name="y")
    mem.assign(y)
    assert ga.forward(L, y)
    got = readback(L, y, x.shape)
    for r in range(x.shape[0]):
        cands, ambiguous = _norm_rows(x[r])
        if not ambiguous:
            assert np.array_equal(bits(cands[0]), bits(want[r])), r        # the restatement above is ggml's formula
        ok = np.array_equal(bits(got[r]), bits(want[r])) or (ambiguous and any(np.array_equal(bits(got[r]), bits(c)) for c in cands))
        assert ok, (n, r, ambiguous, int((bits(got[r]) != bits(want[r])).sum()))


# ================================================================================================ protocol
def _weight_node(mem, t=po.Q4_0, K=256, M=64, upload=True, seed=3):
    wq = mx.swept_weights(t, M, K, np.random.default_rng(seed))
    w = ga.weight(t, K, M, wq, name="w")
    return mem.upload(w) if upload else w


@pytest.mark.parametrize("ith,task", [(1, ga.TASK_COMPUTE), (3, ga.TASK_COMPUTE), (0, ga.TASK_INIT), (0, ga.TASK_FINALIZE)])
def test_other_threads_and_phases_claim_and_write_nothing(L, mem, ith, task):
    x = np.random.default_rng(1).standard_normal((3, 256)).astype(np.float32)
    nodes = [ga.node(ga.OP_MUL_MAT, _weight_node(mem), ga.f32(x, "x"), name="mm")]
    b = mem.upload(ga.f32(np.ones(256, np.float32), "b"))
    nodes.append(ga.node(ga.OP_ADD, ga.f32(x, "x"), b, name="add"))
    nodes.append(ga.node(ga.OP_GELU, to_device(L, mem, x), name="gelu"))
    for nd in nodes:
        out = Out(list(nd.s.ne)[::-1][2:])
        nd.s.data = out.arr.ctypes.data
        nd.keep.append(out)
        assert ga.forward(L, nd, ith=ith, task=task, nth=4) is True
        assert out.poisoned(), nd.s.name


def test_declined_and_trivial_nodes(L, mem):
    x = np.ones((2, 256), np.float32)
    out = Out((2, 256))
    assert ga.forward(L, ga.node(ga.OP_ADD, ga.f32(x, "a"), ga.f32(x, "b"), name="y", out=out.arr)) is False     # nothing on the device
    assert out.poisoned()
    none = ga.f32(np.zeros(4, np.float32), "leaf")
    assert ga.forward(L, none) is True                                  # OP_NONE
    w = _weight_node(mem)
    out = Out((2, 64))
    mm = ga.node(ga.OP_MUL_MAT, w, ga.f32(x, "x"), name="mm", out=out.arr)
    mm.s.meta.cuda_op_directive = 0                                     # libfalcon's KQ / KQV: CUDA forbidden
    assert ga.forward(L, mm) is False and out.poisoned()
    mm.s.meta.cuda_op_directive = 1
    assert ga.forward(L, mm) is True and out.intact() and not out.poisoned()


def test_can_mul_mat_precedence(L, mem):
    """dst's directive decides, then src0's, then src1's; without one: a device-resident weight and F32 src1 / dst"""
    wg, wc = _weight_node(mem), _weight_node(mem, upload=False)
    x, x16 = ga.f32(np.ones((2, 256), np.float32), "x"), ga.Node(po.F16, [256, 2], [2, 512, 1024, 1024], np.ones((2, 256), np.float16), name="x16")
    dst = ga.f32(np.zeros((2, 64), np.float32), "y")

    def can(w, s1, d=-1, d0=-1, d1=-1):
        dst.s.meta.cuda_op_directive, w.s.meta.cuda_op_directive, s1.s.meta.cuda_op_directive = d, d0, d1
        return L.ggml_cuda_can_mul_mat(w.ptr, s1.ptr, dst.ptr)

    assert can(wg, x) and not can(wc, x) and not can(wg, x16)
    assert not can(wg, x, d=0, d0=1, d1=1) and can(wc, x, d=1, d0=0, d1=0)
    assert not can(wg, x, d0=0, d1=1) and can(wc, x, d0=1, d1=0)
    assert not can(wg, x, d1=0) and can(wc, x, d1=1)
    can(wg, x)                                                          # directives back to -1


@pytest.mark.parametrize("scratch", [True, False], ids=["scratch", "no_scratch"])
def test_views_and_in_place_alias_their_source(L, mem, scratch):
    """assign_buffers places a VIEW at a non-zero offset (its offset read from opt[0]), a RESHAPE, a PERMUTE and a TRANSPOSE of a device
    node, and an in-place node, on their source's device memory; the surface reads every device operand as contiguous, so the
    PERMUTE / TRANSPOSE checks are of the aliasing only"""
    rng = np.random.default_rng(7)
    x = rng.standard_normal((4, 1024)).astype(np.float32)
    b = rng.standard_normal(1024).astype(np.float32)
    L.ggml_cuda_set_scratch_size(1 << 22 if scratch else 0)
    try:
        src = ga.node(ga.OP_SCALE, ga.f32(x, "x"), ga.scalar(1.0), name="src")
        mem.assign(src, scratch=scratch)
        assert ga.forward(L, src)
        v = ga.view(src, [1024, 2], 1024 * 4 * 1, name="rows12")                                  # rows 1, 2
        y = ga.node(ga.OP_ADD, v, ga.f32(b, "b"), name="y")
        mem.assign(y, scratch=scratch)                                  # places the view too (it is still on the CPU)
        assert v.on_device()
        assert ga.forward(L, v) and ga.forward(L, y)
        assert np.array_equal(bits(readback(L, y)), bits(x[1:3] + b))
        b2 = rng.standard_normal(2048).astype(np.float32)
        r = ga.alias(src, ga.OP_RESHAPE, [2048, 2], [4, 8192, 16384, 16384], name="reshape")
        y2 = ga.node(ga.OP_ADD, r, ga.f32(b2, "b2"), name="y2")
        mem.assign(y2, scratch=scratch)
        assert ga.forward(L, r) and ga.forward(L, y2)
        assert np.array_equal(bits(readback(L, y2)), bits(x.reshape(2, 2048) + b2))
        for op, ne, nb in ((ga.OP_PERMUTE, [4, 1024], [4096, 4, 16384, 16384]), (ga.OP_TRANSPOSE, [4, 1024], [4096, 4, 16384, 16384])):
            p = ga.alias(src, op, ne, nb, name="perm")
            mem.assign(p, scratch=scratch, owns=False)
            assert ga.forward(L, p)
            assert np.array_equal(bits(readback(L, p, [4096])), bits(x.reshape(-1)))          # the source's bytes, in its order
        ip = ga.node(ga.OP_ADD, src, ga.f32(b, "b"), name="inplace")
        ip.s.data = src.s.data
        mem.assign(ip, scratch=scratch, owns=False)
        assert ga.forward(L, ip)
        assert np.array_equal(bits(readback(L, src)), bits(x + b))                              # written where src lives
    finally:
        L.ggml_cuda_set_scratch_size(0)
        L.ggml_cuda_free_scratch()


def test_scratch_ring_wraps(L, mem):
    """a scratch arena of three buffers: the fourth node of a chain is placed where the first one was, after the first was consumed"""
    n = 4096
    rng = np.random.default_rng(11)
    x, b, c = (rng.standard_normal(n).astype(np.float32) for _ in range(3))
    L.ggml_cuda_set_scratch_size(3 * n * 4)
    try:
        s1 = ga.node(ga.OP_SCALE, ga.f32(x, "x"), ga.scalar(2.0), name="s1")
        s2 = ga.node(ga.OP_ADD, s1, ga.f32(b, "b"), name="s2")
        s3 = ga.node(ga.OP_MUL, s2, ga.f32(c, "c"), name="s3")
        s4 = ga.node(ga.OP_ADD, s3, ga.f32(b, "b"), name="s4")
        for nd in (s1, s2, s3, s4):
            mem.assign(nd, scratch=True)
        for nd in (s1, s2, s3, s4):
            assert ga.forward(L, nd)
        want = (x * np.float32(2) + b) * c + b
        assert np.array_equal(bits(readback(L, s4)), bits(want))
        assert np.array_equal(bits(readback(L, s1)), bits(want))        # s4 took s1's place in the ring
        assert np.array_equal(bits(readback(L, s3)), bits((x * np.float32(2) + b) * c))
    finally:
        L.ggml_cuda_set_scratch_size(0)
        L.ggml_cuda_free_scratch()


# ================================================================================================ takeover
MODELS = [(TINY_40B, po.Q4_K, 15, None), (TINY_7B, po.Q4_0, 2, None), (TINY_40B, po.Q4_K, 15, {"lm_head": po.F16})]
N_CTX = 64
SHORT = np.array([11, 100, 101, 102, 103, 104], np.int32)
PROMPT = np.array([11] + list(range(100, 111)), np.int32)
# a 6-token prompt at 0 (the first eval of a model is the learning one), 4 decode steps, a 12-token batch (the GEMM) at 10, 3 more steps
SEQUENCE = [(SHORT, 0)] + [(np.array([200 + i], np.int32), 6 + i) for i in range(4)] + [(PROMPT, 10)] + \
           [(np.array([300 + i], np.int32), 22 + i) for i in range(3)]


def _model_file(tmp_path, hp, wt, ftype, overrides, name):
    path = str(tmp_path / name)
    ggcc.write_ggcc(path, hp, synth_model(hp, wt, seed=1234, overrides=overrides), ftype=ftype)
    return path


def _pair(gpu, path):
    """the reference behind the hook, and a b200_falcon loaded from the same file with the hook engine's n_ctx / n_batch"""
    ref = po.RefFalcon(path, n_ctx=N_CTX, n_batch=16, logits_all=True, hook=True, n_gpu_layers=99)
    eng = gpu.Falcon(gpu.Falcon.read_hparams(path), n_ctx=N_CTX, n_batch=512)
    eng.load_ggcc(path)
    return ref, eng


def _run(gpu, ref, eng, n_max_real_ctx, learning):
    """SEQUENCE on both sides; the engine gets the rope context the reference's ROPE nodes carry (libfalcon.cpp:2229-2230:
    n_max_real_ctx, or the context's n_ctx when that is 0).  -> number of evals compared"""
    lib = gpu.lib()
    compared = 0
    for i, (toks, n_past) in enumerate(SEQUENCE):
        taken = lib.b200_surface_takeover_evals()
        got = ref.eval(toks, n_past, n_threads=2, n_max_real_ctx=n_max_real_ctx)
        want = eng.eval(toks, n_past, n_ctx_rope=n_max_real_ctx or N_CTX, all_logits=True)
        if learning and i == 0:
            assert lib.b200_surface_takeover_evals() == taken                # the per-node path computed it
            continue
        assert lib.b200_surface_takeover_evals() == taken + 1, (i, n_past)
        d = np.flatnonzero(bits(got) != bits(want))
        assert d.size == 0, "rope ctx %d, eval %d (N %d at n_past %d): %d logits differ, first (token, id) %s" % (
            n_max_real_ctx, i, toks.size, n_past, d.size, divmod(int(d[0]), want.shape[1]))
        compared += 1
    return compared


@pytest.mark.skipif(not os.path.exists(HOOK), reason="oracle/_ref/libfalcon_hook.so not present (built by make -C oracle ref from the reference sources)")
@pytest.mark.parametrize("hp,wt,ftype,overrides", MODELS, ids=["40b-q4_K", "7b-q4_0", "40b-q4_K-f16-head"])
def test_takeover_is_the_engine_bit_for_bit(gpu, tmp_path, monkeypatch, hp, wt, ftype, overrides):
    """the sequence with the context's own rope context, then again from n_past 0 with n_max_real_ctx 4096 (another theta scale)"""
    monkeypatch.delenv("B200_NO_TAKEOVER", raising=False)
    ref, eng = _pair(gpu, _model_file(tmp_path, hp, wt, ftype, overrides, "m.ggcc"))
    try:
        t0 = gpu.lib().b200_surface_takeover_evals()
        n = _run(gpu, ref, eng, 0, learning=True) + _run(gpu, ref, eng, 4096, learning=False)
        assert n == 2 * len(SEQUENCE) - 1 and gpu.lib().b200_surface_takeover_evals() - t0 == n
    finally:
        ref.close()
        eng.free()


@pytest.mark.skipif(not os.path.exists(HOOK), reason="oracle/_ref/libfalcon_hook.so not present (built by make -C oracle ref from the reference sources)")
def test_takeover_rebuilds_after_a_model_reload(gpu, tmp_path, monkeypatch):
    """a 40B file, closed, then a 7B file in the same process: the new model's learning eval rebuilds the engine behind the hook"""
    monkeypatch.delenv("B200_NO_TAKEOVER", raising=False)
    for k, (hp, wt, ftype, overrides) in enumerate(MODELS[:2]):
        ref, eng = _pair(gpu, _model_file(tmp_path, hp, wt, ftype, overrides, "m%d.ggcc" % k))
        try:
            assert _run(gpu, ref, eng, 0, learning=True) == len(SEQUENCE) - 1
        finally:
            ref.close()
            eng.free()
