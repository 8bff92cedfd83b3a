"""Test-only builds for cached f16 LoRA adapters on the CPU:

  * mock_dir(): the CPU stand-in of the device layer (tests/mock/mock_fl_cuda.c) with the f16 LoRA entry points of
    tests/mock/mock_lora_f16.c (and, for tensor parallelism, fl_dev_tp_unshard), linked into one libfl_cuda.so in a temporary
    directory next to copies of the host libraries, whose $ORIGIN rpath then resolves to it -- as tests/test_tp_ingest.py does;
  * F16Oracle: the C restatement of add_q_f16 / scale_f16 (oracle/lora_f16_oracle.c over oracle/q4_oracle.c) through ctypes."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "fastllama_b200", "lib")
MOCK_SRC = os.path.join(ROOT, "tests", "mock")
ORACLE = os.path.join(ROOT, "oracle")
CFLAGS = ["-O2", "-mavx2", "-mfma", "-mf16c", "-msse3", "-ffp-contract=off", "-fPIC", "-shared", "-w"]
HAVE_LIBS = all(os.path.exists(os.path.join(LIB, n)) for n in ("libggml_b200.so", "pyfastllama.so"))


def _gcc(out, sources):
    subprocess.run(["/usr/bin/gcc", *CFLAGS, "-I" + os.path.join(ROOT, "include"), "-o", out, *sources, "-lm", "-lrt"], check=True,
                   capture_output=True, timeout=300)


def mock_dir(tp=False) -> str:
    """A new temporary directory holding libfl_cuda.so (CPU stand-in with the f16 LoRA ops), libggml_b200.so and pyfastllama.so.
    The caller removes it (shutil.rmtree)."""
    d = tempfile.mkdtemp(prefix="fl_mock_lora_f16_")
    srcs = [os.path.join(MOCK_SRC, "mock_fl_cuda.c"), os.path.join(MOCK_SRC, "mock_lora_f16.c"),
            os.path.join(ORACLE, "lora_f16_oracle.c"), os.path.join(ORACLE, "q4_oracle.c")]
    if tp:
        srcs.append(os.path.join(MOCK_SRC, "mock_tp_unshard.c"))
    _gcc(os.path.join(d, "libfl_cuda.so"), srcs)
    for n in ("libggml_b200.so", "pyfastllama.so"):
        shutil.copy(os.path.join(LIB, n), d)
    return d


def _fptr(a):
    return a.ctypes.data_as(C.c_void_p)


class F16Oracle:
    """orc_add_q_f16 / orc_scale_f16 (oracle/lora_f16_oracle.c), compiled into a temporary library."""

    def __init__(self):
        self.dir = tempfile.mkdtemp(prefix="fl_lora_f16_oracle_")
        path = os.path.join(self.dir, "liblora_f16_oracle.so")
        _gcc(path, [os.path.join(ORACLE, "lora_f16_oracle.c"), os.path.join(ORACLE, "q4_oracle.c")])
        self.lib = C.CDLL(path)
        self.lib.orc_add_q_f16.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        self.lib.orc_add_q_f16.restype = C.c_int
        self.lib.orc_scale_f16.argtypes = [C.c_void_p, C.c_long, C.c_float]
        self.lib.orc_scale_f16.restype = None

    def add_q_f16(self, w: np.ndarray, x: np.ndarray, ggml_type: int) -> np.ndarray:
        """ggml_compute_forward_add_q_f16 (lib/ggml.c:12372-12483): dequantise, add the f16 delta widened exactly, re-quantise with
        the SIMD quantiser."""
        x = np.ascontiguousarray(x, dtype=np.float16)
        rows, k = x.shape
        w = np.ascontiguousarray(w, dtype=np.uint8).reshape(rows, -1)
        out = np.empty_like(w)
        assert self.lib.orc_add_q_f16(ggml_type, rows, k, _fptr(w), _fptr(x), _fptr(out)) == 0
        return out

    def scale_f16(self, x: np.ndarray, v: float) -> np.ndarray:
        """ggml_compute_forward_scale_f16 (lib/ggml.c:12485-12524) on a copy of x."""
        out = np.array(x, dtype=np.float16, order="C", copy=True)
        self.lib.orc_scale_f16(_fptr(out), out.size, v)
        return out

    def close(self):
        shutil.rmtree(self.dir, ignore_errors=True)
