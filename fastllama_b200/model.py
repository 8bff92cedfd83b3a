"""Host-side mirror of the reference's Python API (reference interfaces/python/fastllama.py:194-479)
over the same C ABI (reference interfaces/c/fastllama.h), so a user of ``fastllama.Model`` can switch by
changing the import.  By default it loads the drop-in ``pyfastllama.so`` of this repository (the
reference's unchanged bridge over the H100 backend); ``library_path`` may point at any library that
exports the same 17 ``llama_*`` symbols -- the tests pass the reference build to get the CPU oracle.

Same names, argument meaning and error behaviour as the reference: ``bool`` returns, RuntimeError when
the model cannot be loaded, ``None``/empty results on an invalid context.
"""
from __future__ import annotations

import ctypes as C
import multiprocessing
from typing import Callable, List, Optional

from .build import lib_path

LOGGER_FUNC = C.CFUNCTYPE(None, C.c_char_p, C.c_int, C.c_char_p, C.c_int)
LOGGER_RESET_FUNC = C.CFUNCTYPE(None)
LOGGER_PROGRESS_FUNC = C.CFUNCTYPE(None, C.c_uint8, C.c_size_t, C.c_size_t)
STREAM_FUNC = C.CFUNCTYPE(None, C.c_char_p, C.c_int)


class Logger:
    """Override any of these to receive the bridge's log callbacks (reference fastllama.py:59-105)."""

    def log_info(self, func_name: str, message: str) -> None:
        print(f"[Info]: Func('{func_name}') {message}", end="", flush=True)

    def log_err(self, func_name: str, message: str) -> None:
        print(f"[Error]: Func('{func_name}') {message}", end="", flush=True)

    def log_warn(self, func_name: str, message: str) -> None:
        print(f"[Warn]: Func('{func_name}') {message}", end="", flush=True)

    def progress(self, tag: int, done_size: int, total_size: int) -> None:
        pass

    def reset(self) -> None:
        pass


class QuietLogger(Logger):
    def log_info(self, func_name, message):
        pass

    def log_warn(self, func_name, message):
        pass


class _CLogger(C.Structure):          # struct llama_logger, reference interfaces/c/fastllama.h:30-36
    _fields_ = [("log", LOGGER_FUNC), ("log_err", LOGGER_FUNC), ("log_warn", LOGGER_FUNC),
                ("reset", LOGGER_RESET_FUNC), ("progress", LOGGER_PROGRESS_FUNC)]


class _ArrayViewF(C.Structure):       # struct llama_array_view_f, fastllama.h:39-42
    _fields_ = [("data", C.POINTER(C.c_float)), ("size", C.c_size_t)]


class _ContextArgs(C.Structure):      # struct llama_model_context_args, fastllama.h:46-61
    _fields_ = [("embedding_eval_enabled", C.c_bool), ("should_get_all_logits", C.c_bool), ("use_mmap", C.c_bool),
                ("use_mlock", C.c_bool), ("load_parallel", C.c_bool), ("seed", C.c_int), ("n_keep", C.c_int),
                ("n_ctx", C.c_int), ("n_threads", C.c_int), ("n_batch", C.c_int), ("n_load_parallel_blocks", C.c_uint32),
                ("last_n_tokens", C.c_size_t), ("allocate_extra_mem", C.c_size_t), ("logger", _CLogger)]


_CTX = C.c_void_p


class Model:
    def __init__(self, path: str, num_threads: int = multiprocessing.cpu_count(), n_ctx: int = 512, last_n_size: int = 64,
                 seed: int = 0, tokens_to_keep: int = 200, n_batch: int = 16, use_mmap: bool = False, use_mlock: bool = False,
                 should_get_all_logits: bool = False, embedding_eval_enabled: bool = False, allocate_extra_mem: int = 0,
                 logger: Optional[Logger] = None, load_parallel: bool = False, n_load_parallel_blocks: int = 1,
                 library_path: Optional[str] = None):
        self.lib = C.CDLL(library_path or lib_path("pyfastllama.so"))
        L = self.lib
        L.llama_create_default_context_args.restype = _ContextArgs
        L.llama_create_context.restype, L.llama_create_context.argtypes = _CTX, [_ContextArgs]
        for name in ("llama_load_model", "llama_ingest", "llama_ingest_system_prompt", "llama_save_state", "llama_load_state",
                     "llama_attach_lora"):
            getattr(L, name).restype, getattr(L, name).argtypes = C.c_bool, [_CTX, C.c_char_p]
        for name in ("llama_detach_lora", "llama_reset_model"):
            getattr(L, name).restype, getattr(L, name).argtypes = C.c_bool, [_CTX]
        L.llama_generate.restype = C.c_bool
        L.llama_generate.argtypes = [_CTX, STREAM_FUNC, C.c_size_t, C.c_float, C.c_float, C.c_float, C.c_float]
        L.llama_perplexity.restype, L.llama_perplexity.argtypes = C.c_float, [_CTX, C.c_char_p]
        L.llama_get_logits.restype, L.llama_get_logits.argtypes = _ArrayViewF, [_CTX]
        L.llama_get_embeddings.restype, L.llama_get_embeddings.argtypes = _ArrayViewF, [_CTX]
        L.llama_free_context.restype, L.llama_free_context.argtypes = None, [_CTX]

        args = L.llama_create_default_context_args()
        args.seed, args.n_keep, args.n_ctx, args.n_threads, args.n_batch = seed, tokens_to_keep, n_ctx, num_threads, n_batch
        args.last_n_tokens = last_n_size
        args.embedding_eval_enabled, args.should_get_all_logits = embedding_eval_enabled, should_get_all_logits
        args.allocate_extra_mem, args.use_mmap, args.use_mlock = allocate_extra_mem, use_mmap, use_mlock
        args.load_parallel, args.n_load_parallel_blocks = load_parallel, n_load_parallel_blocks
        if logger is not None:
            def _txt(f):
                return LOGGER_FUNC(lambda fn, fl, msg, ml: f(C.string_at(fn, fl).decode("utf-8", "replace"), C.string_at(msg, ml).decode("utf-8", "replace")))
            self._logger = _CLogger(_txt(logger.log_info), _txt(logger.log_err), _txt(logger.log_warn), LOGGER_RESET_FUNC(logger.reset),
                                    LOGGER_PROGRESS_FUNC(lambda t, d, n: logger.progress(int(t), int(d), int(n))))
            args.logger = self._logger
        self.ctx = L.llama_create_context(args)
        if not self.ctx or not L.llama_load_model(self.ctx, path.encode("utf-8")):
            raise RuntimeError("Unable to load model")

    # ---- the reference's public methods ------------------------------------------------------------
    def ingest(self, prompt: str, is_system_prompt: bool = False) -> bool:
        fn = self.lib.llama_ingest_system_prompt if is_system_prompt else self.lib.llama_ingest
        return bool(fn(self.ctx, prompt.encode("utf-8")))

    def generate(self, streaming_fn: Callable[[str], None], num_tokens: int = 100, top_k: int = 40, top_p: float = 0.95,
                 temp: float = 0.8, repeat_penalty: float = 1.0, stop_words: List[str] = []) -> bool:
        arr = (C.c_char_p * len(stop_words))(*[s.encode("utf-8") for s in stop_words])
        self.lib.llama_set_stop_words.restype = C.c_bool
        self.lib.llama_set_stop_words.argtypes = [_CTX, type(arr), C.c_size_t]
        self.lib.llama_set_stop_words(self.ctx, arr, len(stop_words))
        cb = STREAM_FUNC(lambda tok, n: streaming_fn(C.string_at(tok, int(n)).decode("utf-8")))
        return bool(self.lib.llama_generate(self.ctx, cb, num_tokens, float(top_k), top_p, temp, repeat_penalty))

    def perplexity(self, prompt: str) -> Optional[float]:
        res = float(self.lib.llama_perplexity(self.ctx, prompt.encode("utf-8")))
        return None if res < 0 else res

    def get_logits(self) -> List[float]:
        v = self.lib.llama_get_logits(self.ctx)
        return [v.data[i] for i in range(v.size)]

    def get_logits_array(self):
        """numpy view copy of get_logits() (ours; the reference returns a Python list)."""
        import numpy as np

        v = self.lib.llama_get_logits(self.ctx)
        return np.ctypeslib.as_array(v.data, shape=(v.size,)).copy() if v.size else np.zeros(0, dtype=np.float32)

    def get_embeddings(self) -> List[float]:
        v = self.lib.llama_get_embeddings(self.ctx)
        return [v.data[i] for i in range(v.size)]

    def save_state(self, filepath: str) -> bool:
        return bool(self.lib.llama_save_state(self.ctx, filepath.encode("utf-8")))

    def load_state(self, filepath: str) -> bool:
        return bool(self.lib.llama_load_state(self.ctx, filepath.encode("utf-8")))

    def attach_lora(self, filepath: str) -> bool:
        return bool(self.lib.llama_attach_lora(self.ctx, filepath.encode("utf-8")))

    def detach_lora(self) -> bool:
        return bool(self.lib.llama_detach_lora(self.ctx))

    def reset(self) -> bool:
        return bool(self.lib.llama_reset_model(self.ctx))

    def close(self) -> None:
        if getattr(self, "ctx", None):
            self.lib.llama_free_context(self.ctx)
            self.ctx = None
            # The bridge has no hook for device memory, so the mirror of the reference API does it: the device allocations of this
            # context (weights / KV mirrors, decode state, its share of the workspaces) are released, and a later model can never see
            # its weights.  Other live contexts keep theirs.  (A library without the symbol -- the reference build the tests use as
            # CPU oracle -- has nothing to release.)
            try:
                release = self.lib.ggml_b200_release_unused
            except AttributeError:
                release = None
            if release is not None:
                release.restype, release.argtypes = None, []
                release()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
