"""ctypes bindings of include/fl_cuda.h -- the thin extern-"C" CUDA layer (libfl_cuda.so).

Host-buffer entry points take/return numpy arrays; they are the drop-in replacements of the row
functions the reference hands out through ``ggml_internal_get_quantize_fn`` (reference
include/ggml.h:841-862).  There is no fallback: if the library or a CUDA device is missing these
raise.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .build import lib_path

Q4_0, Q4_1, Q8_0 = 2, 3, 6
BLOCK_BYTES = {Q4_0: 20, Q4_1: 24, Q8_0: 40}
QK = 32


class FlView(C.Structure):
    _fields_ = [("data", C.c_void_p), ("ne", C.c_int64 * 4), ("nb", C.c_int64 * 4)]


class FlCudaError(RuntimeError):
    pass


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if isinstance(a, np.ndarray) else C.c_void_p(a)


_VP = C.POINTER(FlView)

PRO_PLAIN, PRO_RMSNORM, PRO_SILUMUL = 0, 1, 2
EPI_STORE, EPI_RESADD, EPI_QKV = 0, 1, 2


class FlMvArgs(C.Structure):          # struct fl_mv_args, include/fl_cuda.h
    _fields_ = [("type", C.c_int), ("K", C.c_int), ("nseg", C.c_int), ("seg_w", C.c_void_p * 3), ("seg_rows", C.c_int * 3),
                ("seg_dst", C.c_void_p * 3), ("pro", C.c_int), ("x", C.c_void_p), ("gamma", C.c_void_p), ("b", C.c_void_p),
                ("normed_out", C.c_void_p), ("xadd", C.c_void_p), ("sum_out", C.c_void_p), ("row_stride_bytes", C.c_size_t),
                ("silu_tab", C.c_void_p), ("epi", C.c_int), ("res", C.c_void_p), ("n_past", C.c_void_p),
                ("n_ctx", C.c_int), ("n_embd", C.c_int), ("head_dim", C.c_int), ("rope_cs", C.c_void_p), ("kcache", C.c_void_p),
                ("vcache", C.c_void_p), ("dst_peer", C.c_void_p * 7), ("n_dst_peer", C.c_int), ("x_ll", C.c_int), ("x_seq", C.c_int), ("out_ll", C.c_int),
                ("out_seq", C.c_int), ("res_ll", C.c_int), ("swiglu", C.c_int)]


class FlTokenStep(C.Structure):       # struct fl_token_step, include/fl_cuda.h
    _fields_ = [("kind", C.c_int), ("mv", FlMvArgs), ("q", C.c_void_p), ("kcache", C.c_void_p), ("vcache", C.c_void_p),
                ("out", C.c_void_p), ("n_past", C.c_void_p), ("k_row_stride", C.c_int), ("n_head", C.c_int), ("head_dim", C.c_int),
                ("n_ctx", C.c_int), ("scale", C.c_float), ("out_ll", C.c_int), ("out_seq", C.c_int), ("n_out_peer", C.c_int), ("out_peer", C.c_void_p * 7)]


SIGNATURES = {
    "fl_init": (C.c_int, [C.c_int]),
    "fl_shutdown": (None, []),
    "fl_is_initialized": (C.c_int, []),
    "fl_last_error": (C.c_char_p, []),
    "fl_device_props": (C.c_int, [C.c_char_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_size_t), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "fl_stream": (C.c_void_p, []),
    "fl_quantize_row_q8_0": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int]),
    "fl_quantize_rows_q8_0": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int]),
    "fl_quantize_rows_q4": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int]),
    "fl_dequantize_rows_q4": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int]),
    "fl_vec_dot_q4_q8": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "fl_mul_mat_q_f32": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "fl_get_rows_q": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "fl_dev_malloc": (C.c_void_p, [C.c_size_t]),
    "fl_dev_free": (C.c_int, [C.c_void_p]),
    "fl_dev_memset": (C.c_int, [C.c_void_p, C.c_int, C.c_size_t]),
    "fl_h2d": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "fl_d2h": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "fl_d2d": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "fl_d2d_2d": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t]),
    "fl_sync": (C.c_int, []),
    "fl_host_alloc_pinned": (C.c_void_p, [C.c_size_t]),
    "fl_host_free_pinned": (C.c_int, [C.c_void_p]),
    "fl_dev_quantize_q8_0": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_int, C.c_int]),
    "fl_dev_mul_mat_q": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_int]),
    "fl_dev_dequantize_rows": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]),
    "fl_dev_quantize_q4": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int]),
    "fl_quantize_rows_q4_simd": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int]),
    "fl_dev_quantize_q4_simd": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int]),
    "fl_dev_add_q_f32": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]),
    "fl_dev_mul_mat_f32_ref": (C.c_int, [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_size_t]),
    "fl_dev_time_mul_mat_q": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_size_t, C.POINTER(C.c_float)]),
    "fl_dev_time_mul_mat_q_rot": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_size_t, C.c_size_t, C.c_int, C.POINTER(C.c_float)]),
    "fl_dev_rms_norm": (C.c_int, [_VP, _VP]),
    "fl_dev_add": (C.c_int, [_VP, _VP, _VP]),
    "fl_dev_mul": (C.c_int, [_VP, _VP, _VP]),
    "fl_dev_repeat": (C.c_int, [_VP, _VP]),
    "fl_dev_scale": (C.c_int, [_VP, C.c_float]),
    "fl_dev_silu": (C.c_int, [_VP, _VP]),
    "fl_dev_diag_mask_inf": (C.c_int, [_VP, C.c_int]),
    "fl_dev_soft_max": (C.c_int, [_VP]),
    "fl_dev_rope": (C.c_int, [_VP, C.c_int, C.c_int, C.c_int]),
    "fl_dev_cpy_f32": (C.c_int, [_VP, _VP]),
    "fl_dev_mul_mat_f32": (C.c_int, [_VP, _VP, _VP]),
    "fl_dev_mv_fused_supported": (C.c_int, [C.c_int, C.c_int, C.c_int]),
    "fl_dev_mv_fused": (C.c_int, [C.POINTER(FlMvArgs)]),
    "fl_token_plan_create": (C.c_int, [C.POINTER(FlTokenStep), C.c_int, C.POINTER(C.c_void_p)]),
    "fl_token_plan_create_ll": (C.c_int, [C.POINTER(FlTokenStep), C.c_int, C.c_void_p, C.POINTER(C.c_void_p)]),
    "fl_token_plan_launch": (C.c_int, [C.c_void_p]),
    "fl_token_plan_destroy": (C.c_int, [C.c_void_p]),
    "fl_token_plan_error": (C.c_int, [C.c_void_p]),
    "fl_comm_shared_alloc": (C.c_int, [C.c_size_t, C.POINTER(C.c_void_p)]),
    "fl_token_plan_profile": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_int)]),
    "fl_token_plan_profile2": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "fl_dev_attn_decode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float]),
    "fl_comm_unique_id": (C.c_int, [C.c_void_p]),
    "fl_comm_init": (C.c_int, [C.c_int, C.c_int, C.c_void_p]),
    "fl_comm_rank": (C.c_int, []),
    "fl_comm_world": (C.c_int, []),
    "fl_comm_allreduce_f32": (C.c_int, [C.c_void_p, C.c_size_t]),
    "fl_comm_allgather_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "fl_dev_pack_cols": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_size_t]),
    "fl_dev_rope_table": (C.c_int, [C.c_int, C.c_int]),
    "fl_graph_begin_capture": (C.c_int, []),
    "fl_graph_end_capture": (C.c_int, [C.POINTER(C.c_void_p)]),
    "fl_graph_launch": (C.c_int, [C.c_void_p]),
    "fl_graph_destroy": (C.c_int, [C.c_void_p]),
    "fl_dev_fill_normal": (C.c_int, [C.c_void_p, C.c_size_t, C.c_uint64, C.c_float]),
    "fl_event_create": (C.c_void_p, []),
    "fl_event_destroy": (C.c_int, [C.c_void_p]),
    "fl_event_record": (C.c_int, [C.c_void_p]),
    "fl_event_sync": (C.c_int, [C.c_void_p]),
    "fl_event_elapsed_ms": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_float)]),
    "fl_launch_count": (C.c_uint64, []),
}

# Bound on first use (FlCuda.fn) rather than at load, so that a stand-in library without them still loads for
# everything else.  libfl_cuda.so exports them like every function of include/fl_cuda.h.
LAZY_SIGNATURES = {
    # type, src_type (0 f32, 1 f16, 2 f32 rounded to f16 and widened back), x, y, k, nrows, hist
    "fl_dev_quantize_q4_file": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    # type, src_type (also 3: f16 data of an f32 file), x, delta_type (-1 none, 0 f32, 1 f16), delta, y, k, nrows, hist
    "fl_dev_quantize_q4_file_lora": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                              C.c_void_p]),
    "fl_dev_tp_unshard": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "fl_dev_tp_unshard_v": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_void_p,
                                      C.c_void_p]),
    "fl_dev_add_q_f16": (C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]),
    "fl_dev_scale_f16": (C.c_int, [_VP, C.c_float]),
}


class FlCuda:
    """Loaded libfl_cuda.so.  ``FlCuda(init=True)`` needs an H100."""

    def __init__(self, path: str | None = None, init: bool = True, device: int = -1):
        path = path or lib_path("libfl_cuda.so")
        if not os.path.exists(path):
            raise FlCudaError(f"{path} is missing: run __graft_entry__.build() first (no CPU fallback exists)")
        self.lib = C.CDLL(path)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(self.lib, name)       # AttributeError here == header/library mismatch
            fn.restype, fn.argtypes = res, args
        if init:
            self.check(self.lib.fl_init(device))

    # ---- helpers ---------------------------------------------------------------------------
    def fn(self, name: str):
        """An entry point of LAZY_SIGNATURES, typed; raises FlCudaError when the library lacks it."""
        f = getattr(self.lib, name, None)
        if f is None:
            raise FlCudaError(f"{self.lib._name} does not export {name}")
        f.restype, f.argtypes = LAZY_SIGNATURES[name]
        return f

    def check(self, rc: int) -> None:
        if rc != 0:
            raise FlCudaError(f"libfl_cuda rc={rc}: {self.lib.fl_last_error().decode(errors='replace')}")

    def device_props(self):
        name = C.create_string_buffer(256)
        sm, hbm, maj, mnr = C.c_int(), C.c_size_t(), C.c_int(), C.c_int()
        self.check(self.lib.fl_device_props(name, 256, C.byref(sm), C.byref(hbm), C.byref(maj), C.byref(mnr)))
        return {"name": name.value.decode(), "sm_count": sm.value, "hbm_bytes": hbm.value, "cc": (maj.value, mnr.value)}

    # ---- host-buffer row functions (quantize_fns_t replacements) ------------------------------
    def quantize_q8_0(self, x: np.ndarray) -> np.ndarray:
        x = np.ascontiguousarray(x, dtype=np.float32)
        k = x.shape[-1]
        rows = x.reshape(-1, k)
        out = np.empty((rows.shape[0], k // QK * 40), dtype=np.uint8)
        self.check(self.lib.fl_quantize_rows_q8_0(_p(rows), _p(out), k, rows.shape[0]))
        return out.reshape(x.shape[:-1] + (k // QK * 40,))

    def quantize_q4(self, x: np.ndarray, t: int) -> np.ndarray:
        x = np.ascontiguousarray(x, dtype=np.float32)
        k = x.shape[-1]
        rows = x.reshape(-1, k)
        out = np.empty((rows.shape[0], k // QK * BLOCK_BYTES[t]), dtype=np.uint8)
        self.check(self.lib.fl_quantize_rows_q4(t, _p(rows), _p(out), k, rows.shape[0]))
        return out.reshape(x.shape[:-1] + (k // QK * BLOCK_BYTES[t],))

    def dequantize_q4(self, w: np.ndarray, t: int, k: int) -> np.ndarray:
        w = np.ascontiguousarray(w, dtype=np.uint8).reshape(-1, k // QK * BLOCK_BYTES[t])
        out = np.empty((w.shape[0], k), dtype=np.float32)
        self.check(self.lib.fl_dequantize_rows_q4(t, _p(w), _p(out), k, w.shape[0]))
        return out

    def vec_dot(self, wrow: np.ndarray, q8row: np.ndarray, t: int, k: int) -> np.float32:
        s = np.zeros(1, dtype=np.float32)
        self.check(self.lib.fl_vec_dot_q4_q8(t, k, _p(s), _p(np.ascontiguousarray(wrow)), _p(np.ascontiguousarray(q8row))))
        return s[0]

    def mul_mat_q(self, w: np.ndarray, x: np.ndarray, t: int) -> np.ndarray:
        """w [M, K/32*bb] u8, x [N, K] f32 -> [N, M] f32; ggml_compute_forward_mul_mat_q_f32."""
        w = np.ascontiguousarray(w, dtype=np.uint8)
        x = np.ascontiguousarray(x, dtype=np.float32)
        m, (n, k) = w.shape[0], x.shape
        dst = np.empty((n, m), dtype=np.float32)
        self.check(self.lib.fl_mul_mat_q_f32(t, m, k, n, _p(w), _p(x), _p(dst)))
        return dst

    def get_rows_q(self, w: np.ndarray, ids: np.ndarray, t: int, k: int) -> np.ndarray:
        w = np.ascontiguousarray(w, dtype=np.uint8)
        ids = np.ascontiguousarray(ids, dtype=np.int32)
        dst = np.empty((ids.size, k), dtype=np.float32)
        self.check(self.lib.fl_get_rows_q(t, k, ids.size, _p(w), w.shape[0], _p(ids), _p(dst)))
        return dst

    # ---- device memory ---------------------------------------------------------------------------
    def to_device(self, a: np.ndarray) -> int:
        a = np.ascontiguousarray(a)
        d = self.alloc(max(a.nbytes, 16))
        self.check(self.lib.fl_h2d(d, _p(a), a.nbytes))
        self.check(self.lib.fl_sync())
        return d

    def alloc(self, nbytes: int) -> int:
        d = self.lib.fl_dev_malloc(nbytes)
        if not d:
            raise FlCudaError(self.lib.fl_last_error().decode())
        return d

    def to_host(self, d: int, shape, dtype) -> np.ndarray:
        out = np.empty(shape, dtype=dtype)
        self.check(self.lib.fl_d2h(_p(out), d, out.nbytes))
        self.check(self.lib.fl_sync())
        return out

    def free(self, d: int) -> None:
        self.check(self.lib.fl_dev_free(d))

    @staticmethod
    def view(d: int, shape_ne, itemsize=4, nb=None) -> FlView:
        """ggml-style view: shape_ne = (ne0, ne1, ...) fastest first."""
        ne = list(shape_ne) + [1] * (4 - len(shape_ne))
        if nb is None:
            nb = [itemsize]
            for i in range(1, 4):
                nb.append(nb[-1] * ne[i - 1])
        v = FlView()
        v.data = d
        v.ne = (C.c_int64 * 4)(*ne)
        v.nb = (C.c_int64 * 4)(*nb)
        return v
