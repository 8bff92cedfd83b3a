"""fastllama_b200 -- H100-native (sm_90a) backend for fastLLaMa's q4_0/q4_1 matmul hot path.

The package holds only what the path needs:
  csrc/      CUDA kernels + the extern-"C" layer (libfl_cuda.so) and the ggml-compatible host
             library (libggml_b200.so)
  cuda_abi   ctypes bindings of include/fl_cuda.h (host-buffer row functions, device entry points)
  model      ctypes mirror of the reference's fastllama.Model over the drop-in pyfastllama.so
  ggjt       synthetic GGJT model-file writer (bench/test tooling)
There is no CPU compute path: importing works anywhere, using it needs an H100.
"""
from .build import LIB_DIR, build_all, lib_path  # noqa: F401
