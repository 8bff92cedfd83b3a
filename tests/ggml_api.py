"""ctypes driver for the ggml C API -- the SAME script drives the reference (oracle/_ref/libggml_ref.so,
CPU) and our drop-in (fastllama_b200/lib/libggml_b200.so, H100), which is the point of boundary B1.

Struct layouts: reference include/ggml.h:267-342 (mirrored in include/fl_ggml.h).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

MAX_NODES = 4096
F32, F16, Q4_0, Q4_1, I32 = 0, 1, 2, 3, 9
TYPE_SIZE = {0: 4, 1: 2, 2: 20, 3: 24, 6: 40, 7: 1, 8: 2, 9: 4}
BLCK = {0: 1, 1: 1, 2: 32, 3: 32, 6: 32, 7: 1, 8: 1, 9: 1}
OP_NAMES = ["NONE", "DUP", "ADD", "SUB", "MUL", "DIV", "SQR", "SQRT", "SUM", "MEAN", "REPEAT", "ABS", "SGN", "NEG", "STEP",
            "RELU", "GELU", "SILU", "NORM", "RMS_NORM", "MUL_MAT", "SCALE", "CPY", "CONT", "RESHAPE", "VIEW", "PERMUTE",
            "TRANSPOSE", "GET_ROWS", "DIAG_MASK_INF", "SOFT_MAX", "ROPE"]


class Tensor(C.Structure):
    pass


TP = C.POINTER(Tensor)
Tensor._fields_ = [
    ("type", C.c_int), ("n_dims", C.c_int), ("ne", C.c_int64 * 4), ("nb", C.c_size_t * 4), ("op", C.c_int),
    ("is_param", C.c_bool), ("grad", TP), ("src0", TP), ("src1", TP), ("opt", TP * 4), ("n_tasks", C.c_int),
    ("perf_runs", C.c_int), ("perf_cycles", C.c_int64), ("perf_time_us", C.c_int64), ("data", C.c_void_p),
    ("padding", C.c_char * 8),
]
assert C.sizeof(Tensor) == 176


class CGraph(C.Structure):
    _fields_ = [
        ("n_nodes", C.c_int), ("n_leafs", C.c_int), ("n_threads", C.c_int), ("work_size", C.c_size_t), ("work", TP),
        ("nodes", TP * MAX_NODES), ("grads", TP * MAX_NODES), ("leafs", TP * MAX_NODES), ("perf_runs", C.c_int),
        ("perf_cycles", C.c_int64), ("perf_time_us", C.c_int64),
    ]


assert C.sizeof(CGraph) == 98360


class InitParams(C.Structure):
    _fields_ = [("mem_size", C.c_size_t), ("mem_buffer", C.c_void_p), ("no_alloc", C.c_bool)]


class Scratch(C.Structure):
    _fields_ = [("offs", C.c_size_t), ("size", C.c_size_t), ("data", C.c_void_p)]


CTX = C.c_void_p
_SIGS = {
    "ggml_init": (CTX, [InitParams]),
    "ggml_free": (None, [CTX]),
    "ggml_used_mem": (C.c_size_t, [CTX]),
    "ggml_set_scratch": (C.c_size_t, [CTX, Scratch]),
    "ggml_new_tensor_1d": (TP, [CTX, C.c_int, C.c_int64]),
    "ggml_new_tensor_2d": (TP, [CTX, C.c_int, C.c_int64, C.c_int64]),
    "ggml_new_tensor_3d": (TP, [CTX, C.c_int, C.c_int64, C.c_int64, C.c_int64]),
    "ggml_new_f32": (TP, [CTX, C.c_float]),
    "ggml_nbytes": (C.c_size_t, [TP]),
    "ggml_nelements": (C.c_int64, [TP]),
    "ggml_add": (TP, [CTX, TP, TP]),
    "ggml_add_inplace": (TP, [CTX, TP, TP]),
    "ggml_mul": (TP, [CTX, TP, TP]),
    "ggml_repeat": (TP, [CTX, TP, TP]),
    "ggml_silu": (TP, [CTX, TP]),
    "ggml_rms_norm": (TP, [CTX, TP]),
    "ggml_mul_mat": (TP, [CTX, TP, TP]),
    "ggml_scale": (TP, [CTX, TP, TP]),
    "ggml_cpy": (TP, [CTX, TP, TP]),
    "ggml_reshape_2d": (TP, [CTX, TP, C.c_int64, C.c_int64]),
    "ggml_reshape_3d": (TP, [CTX, TP, C.c_int64, C.c_int64, C.c_int64]),
    "ggml_view_1d": (TP, [CTX, TP, C.c_int64, C.c_size_t]),
    "ggml_view_2d": (TP, [CTX, TP, C.c_int64, C.c_int64, C.c_size_t, C.c_size_t]),
    "ggml_view_3d": (TP, [CTX, TP, C.c_int64, C.c_int64, C.c_int64, C.c_size_t, C.c_size_t, C.c_size_t]),
    "ggml_permute": (TP, [CTX, TP, C.c_int, C.c_int, C.c_int, C.c_int]),
    "ggml_transpose": (TP, [CTX, TP]),
    "ggml_get_rows": (TP, [CTX, TP, TP]),
    "ggml_diag_mask_inf": (TP, [CTX, TP, C.c_int]),
    "ggml_soft_max": (TP, [CTX, TP]),
    "ggml_rope": (TP, [CTX, TP, C.c_int, C.c_int, C.c_int]),
    "ggml_build_forward_expand": (None, [C.POINTER(CGraph), TP]),
    "ggml_graph_compute": (None, [CTX, C.POINTER(CGraph)]),
    "ggml_fp16_to_fp32": (C.c_float, [C.c_uint16]),
    "ggml_fp32_to_fp16": (C.c_uint16, [C.c_float]),
    "ggml_type_size": (C.c_size_t, [C.c_int]),
    "ggml_blck_size": (C.c_int, [C.c_int]),
    "ggml_is_quantized": (C.c_bool, [C.c_int]),
    "ggml_element_size": (C.c_size_t, [TP]),
}


class Ggml:
    def __init__(self, path: str):
        self.lib = C.CDLL(path)
        for name, (res, args) in _SIGS.items():
            fn = getattr(self.lib, name)
            fn.restype, fn.argtypes = res, args
            setattr(self, name[5:], fn)            # g.new_tensor_1d(...), g.mul_mat(...)

    def context(self, mem_size: int) -> "Arena":
        return Arena(self, mem_size)


class Arena:
    """A ggml context over a numpy buffer we own (like Model::buf_compute)."""

    def __init__(self, g: Ggml, mem_size: int):
        self.g = g
        self.buf = np.zeros(mem_size + 64, dtype=np.uint8)
        base = self.buf.ctypes.data
        self.base = (base + 15) & ~15
        self.ctx = g.init(InitParams(mem_size, self.base, False))
        assert self.ctx

    def free(self):
        if self.ctx:
            self.g.free(self.ctx)
            self.ctx = None

    def offset(self, t) -> int:
        """data offset relative to the arena base (comparable across libraries)."""
        return t.contents.data - self.base

    def numpy(self, t) -> np.ndarray:
        """Contiguous tensor contents as numpy (host memory)."""
        tt = t.contents
        n = int(np.prod([tt.ne[i] for i in range(4)]))
        nbytes = n * TYPE_SIZE[tt.type] // BLCK[tt.type]
        raw = (C.c_uint8 * nbytes).from_address(tt.data)
        a = np.frombuffer(raw, dtype=np.uint8)
        if tt.type == F32:
            return a.view(np.float32).reshape([tt.ne[i] for i in (3, 2, 1, 0)])
        if tt.type == I32:
            return a.view(np.int32)
        return a

    def set(self, t, values: np.ndarray):
        tt = t.contents
        v = np.ascontiguousarray(values)
        n = int(np.prod([tt.ne[i] for i in range(4)]))
        nbytes = n * TYPE_SIZE[tt.type] // BLCK[tt.type]
        assert v.nbytes == nbytes, (v.nbytes, nbytes)
        C.memmove(tt.data, v.ctypes.data, nbytes)


def new_graph(n_threads: int = 4) -> CGraph:
    g = CGraph()
    g.n_threads = n_threads
    return g


def is_contiguous(tt) -> bool:
    ts, bs = TYPE_SIZE[tt.type], BLCK[tt.type]
    return (tt.nb[0] == ts and tt.nb[1] == tt.nb[0] * tt.ne[0] // bs and tt.nb[2] == tt.nb[1] * tt.ne[1]
            and tt.nb[3] == tt.nb[2] * tt.ne[2])
