"""ctypes mirror of the reference structs the ggml_cuda_* operator surface receives (csrc/ggml_abi_mirror.h, itself checked against
the reference headers by oracle/abi_check.cpp), and helpers that build tensors and graph nodes the way ggml.c does.

Crafted graphs must never look like a Falcon eval to the surface's whole-graph takeover: no tensor here is named "transformer.*",
"lm_head.weight" or "result_lm_head", and no GET_ROWS of an embedding is ever built.
"""
import ctypes as C
import numpy as np
import pyoracle as po

MAX_DIMS, MAX_OPT, MAX_NAME = 4, 4, 64
BACKEND_CPU, BACKEND_GPU, BACKEND_GPU_SPLIT = 0, 10, 20
TASK_INIT, TASK_COMPUTE, TASK_FINALIZE = 0, 1, 2
OPS = dict(OP_NONE=0, OP_ADD=2, OP_MUL=6, OP_REPEAT=14, OP_GELU=23, OP_SILU=25, OP_NORM=27, OP_RMS_NORM=28, OP_MUL_MAT=30,
           OP_SCALE=32, OP_SET=33, OP_CPY=34, OP_CONT=35, OP_RESHAPE=36, OP_VIEW=37, OP_PERMUTE=38, OP_TRANSPOSE=39,
           OP_GET_ROWS=40, OP_DIAG_MASK_INF=43, OP_SOFT_MAX=45, OP_ROPE=47)
globals().update(OPS)
I32 = 18                                   # GGML_TYPE_I32 (ggml.h:241-262)


class TensorMeta(C.Structure):
    _fields_ = [("layer_id", C.c_int8), ("short_name", C.c_char * MAX_NAME), ("cuda_op_directive", C.c_int8),
                ("cuda_info_op_on_device", C.c_int8), ("cuda_perf_mal_mul_type", C.c_uint8), ("f_custom", C.c_float * 4),
                ("i_custom", C.c_int * 4), ("debug_flag", C.c_uint8), ("padding", C.c_char * 15)]


class Tensor(C.Structure):
    pass


Tensor._fields_ = [("type", C.c_int), ("backend", C.c_int), ("n_dims", C.c_int), ("ne", C.c_int64 * MAX_DIMS),
                   ("nb", C.c_size_t * MAX_DIMS), ("op", C.c_int), ("is_param", C.c_bool), ("grad", C.POINTER(Tensor)),
                   ("src0", C.POINTER(Tensor)), ("src1", C.POINTER(Tensor)), ("opt", C.POINTER(Tensor) * MAX_OPT),
                   ("n_tasks", C.c_int), ("perf_runs", C.c_int), ("perf_cycles", C.c_int64), ("perf_time_us", C.c_int64),
                   ("data", C.c_void_p), ("name", C.c_char * MAX_NAME), ("extra", C.c_void_p), ("meta", TensorMeta),
                   ("padding", C.c_char * 4)]


class ComputeParams(C.Structure):
    _fields_ = [("type", C.c_int), ("ith", C.c_int), ("nth", C.c_int), ("wsize", C.c_size_t), ("wdata", C.c_void_p)]


P = C.POINTER(Tensor)
SURFACE = {
    "ggml_init_cublas": (C.c_bool, [C.c_bool]),
    "ggml_cuda_transform_tensor": (None, [C.c_void_p, P]),
    "ggml_cuda_free_data": (None, [P]),
    "ggml_cuda_assign_buffers": (None, [P]),
    "ggml_cuda_assign_buffers_no_scratch": (None, [P]),
    "ggml_cuda_set_scratch_size": (None, [C.c_size_t]),
    "ggml_cuda_free_scratch": (None, []),
    "ggml_cuda_can_mul_mat": (C.c_bool, [P, P, P]),
    "ggml_cuda_mul": (None, [P, P, P]),
    "ggml_cuda_compute_forward": (C.c_bool, [C.POINTER(ComputeParams), P]),
}


def surface(L):
    """give the surface symbols of libggml_b200.so (the CDLL `L`) their signatures; returns L"""
    for name, (res, args) in SURFACE.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    return L


class Node:
    """one ggml_tensor in Python-owned memory; keeps every array and tensor it points to alive"""

    def __init__(self, typ, ne, nb, data=None, op=OP_NONE, src0=None, src1=None, name=""):
        assert not name.startswith("transformer.") and name not in ("lm_head.weight", "result_lm_head")
        self.s = Tensor()
        s = self.s
        s.type, s.backend, s.op = typ, BACKEND_CPU, op
        ne = list(ne) + [1] * (MAX_DIMS - len(ne))
        s.n_dims = max(1, max(i + 1 for i in range(MAX_DIMS) if ne[i] != 1) if any(v != 1 for v in ne) else 1)
        for i in range(MAX_DIMS):
            s.ne[i], s.nb[i] = ne[i], nb[i]
        s.name = name.encode()
        s.meta.cuda_op_directive = -1
        self.keep = [data]
        s.data = data.ctypes.data if isinstance(data, np.ndarray) else data
        if src0 is not None:
            s.src0 = C.pointer(src0.s)
        if src1 is not None:
            s.src1 = C.pointer(src1.s)
        self.src0, self.src1 = src0, src1

    @property
    def ptr(self):
        return C.pointer(self.s)

    @property
    def n(self):
        return int(np.prod(list(self.s.ne)))

    def on_device(self):
        return self.s.backend in (BACKEND_GPU, BACKEND_GPU_SPLIT)


def _contig_nb(ne, elem_bytes, blk=1):
    nb = [elem_bytes, elem_bytes * ne[0] // blk]
    for i in range(2, MAX_DIMS):
        nb.append(nb[-1] * (ne[i - 1] if i - 1 < len(ne) else 1))
    return nb


def f32(arr, name="", op=OP_NONE, src0=None, src1=None):
    """a contiguous host F32 tensor around the float32 array `arr` (ne0 = its last axis)"""
    assert arr.dtype == np.float32 and arr.flags.c_contiguous
    ne = list(arr.shape[::-1]) or [1]
    return Node(po.F32, ne, _contig_nb(ne, 4), arr, op, src0, src1, name)


def scalar(v, name="s"):
    """the one-element host tensor SCALE reads its factor from"""
    return f32(np.array([v], np.float32), name)


def weight(t, K, M, raw, name="w"):
    """a 2-D weight of ggml type t, M rows of K values, around its raw rows (uint8 blocks, or float16 / float32 values)"""
    raw = np.ascontiguousarray(raw)
    be, bb = po.BLOCK_ELEMS[t], po.BLOCK_BYTES[t]
    assert raw.nbytes == M * (K // be) * bb
    n = Node(t, [K, M], [bb, K // be * bb, M * K // be * bb, M * K // be * bb], raw, name=name)
    return n


def view(src, ne, offset, name="view"):
    """ggml_view_*d as ggml.c builds it: data = src->data + offset, opt[0] an I32 tensor whose data holds the size_t byte offset"""
    off = np.zeros(2, np.int32)
    off.view(np.uint64)[0] = offset
    offs = Node(I32, [2], [4, 8, 8, 8], off, name=name + ".offs")
    v = Node(src.s.type, ne, _contig_nb(ne, 4), (src.s.data or 0) + offset, OP_VIEW, src0=src, name=name)
    v.s.opt[0] = C.pointer(offs.s)
    v.keep.append(offs)
    return v


def alias(src, op, ne, nb, name=""):
    """RESHAPE / PERMUTE / TRANSPOSE: same data as src, new ne / nb"""
    return Node(src.s.type, ne, nb, src.s.data, op, src0=src, name=name)


def node(op, src0, src1=None, name="node", out=None):
    """a graph node: op(src0, src1) with its own host destination `out` (default: a float32 array shaped like src0, or the
    MUL_MAT result [N][M])"""
    if out is None:
        if op == OP_MUL_MAT:
            out = np.zeros((src1.s.ne[1], src0.s.ne[1]), np.float32)
        else:
            out = np.zeros(list(src0.s.ne)[::-1], np.float32)
    return f32(out, name, op, src0, src1)


def forward(L, nd, ith=0, task=TASK_COMPUTE, nth=1):
    p = ComputeParams(task, ith, nth, 0, None)
    return bool(L.ggml_cuda_compute_forward(C.byref(p), nd.ptr))
