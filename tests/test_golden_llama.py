"""Whole-graph golden vectors (tests/golden/llama_toy_*.npz, written by oracle/gen_golden.py from the reference LIBRARY):
a tiny LLaMA built through the ggml C API like Model::eval builds it, 5-token prompt + three decode steps.

  * CPU: the reference library still reproduces the fixture bit for bit (pins the fixture; needs oracle/_ref);
  * CPU: our host stack (arena mirrors, executor, decode plan as the token program) on the CPU stand-in of the device layer;
  * GPU: the real thing -- prompt through the tensor-core ingest kernel, decode steps as the persistent token kernel.
Bar for ours: the SAME BITS as the reference library, logits and embeddings, prompt eval and decode steps (every fp32 operation of the
path follows the reference's order, fl_exact.cuh; the 5-token prompt stays below the 16 columns from which the wgmma GEMM takes over)."""
import os

import numpy as np
import pytest

from oracle.gen_golden import LLAMA_TOY, LLAMA_TOY_SEED, LLAMA_TOY_STEPS
from oracle.pyoracle import REF_GGML_SO, Oracle
from tests import ggml_api as G
from tests.llama_graph import HParams, MiniLlama, make_weights
from tests.mockbuild import ensure_mock

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TYPES = [("q4_0", G.Q4_0), ("q4_1", G.Q4_1)]


def run_steps(lib_path, t):
    orc = Oracle()
    hp = HParams(**LLAMA_TOY)
    w = make_weights(hp, t, lambda x, tt: orc.quantize_q4(x, tt), seed=LLAMA_TOY_SEED)
    m = MiniLlama(G.Ggml(lib_path), hp, w, compute_mb=32)
    outs = []
    for tokens, n_past in LLAMA_TOY_STEPS:
        c, gf, named = m.eval(tokens, n_past)
        m.compute(c, gf)
        outs.append((c.numpy(named["logits"]).copy(), c.numpy(named["embeddings"]).copy()))
    return outs


def check_close(outs, gold):
    for i, (lg, emb) in enumerate(outs):
        rl, re = gold[f"logits{i}"], gold[f"emb{i}"]
        assert np.isfinite(lg).all()
        nd = int((rl.view(np.uint32) != lg.view(np.uint32)).sum()), int((re.view(np.uint32) != emb.view(np.uint32)).sum())
        assert nd == (0, 0), (i, nd, rl.size, float(np.abs(rl - lg).max()), float(np.abs(rl).max()))


@pytest.mark.parametrize("name,t", TYPES)
def test_reference_library_reproduces_the_fixture(name, t):
    if not os.path.exists(REF_GGML_SO):
        pytest.skip("oracle/_ref not built")
    gold = np.load(os.path.join(GOLDEN, f"llama_toy_{name}.npz"))
    for i, (lg, emb) in enumerate(run_steps(REF_GGML_SO, t)):
        assert np.array_equal(lg.view(np.uint32), gold[f"logits{i}"].view(np.uint32))
        assert np.array_equal(emb.view(np.uint32), gold[f"emb{i}"].view(np.uint32))


MOCK_RUN = r"""
import ctypes as C, os, sys, numpy as np
sys.path.insert(0, sys.argv[1])
from tests.test_golden_llama import GOLDEN, check_close, run_steps
lib, name, t = sys.argv[2], sys.argv[3], int(sys.argv[4])
check_close(run_steps(lib, t), np.load(os.path.join(GOLDEN, f"llama_toy_{name}.npz")))
assert C.CDLL(lib).ggml_b200_decode_mode() == 2          # the decode steps ran as the token program
"""


@pytest.mark.parametrize("name,t", TYPES)
def test_host_stack_on_cpu_mock_matches_the_fixture(name, t):
    """In a subprocess: the mock's libfl_cuda.so must not meet the real one (same soname) in one process."""
    import subprocess
    import sys

    lib = os.path.join(ensure_mock(), "libggml_b200.so")
    if not os.path.exists(lib):
        pytest.skip("tests/mock not built")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, "-c", MOCK_RUN, root, lib, name, str(t)], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stderr[-3000:]


@pytest.mark.gpu
@pytest.mark.parametrize("name,t", TYPES)
def test_b200_matches_the_fixture(name, t):
    import ctypes as C

    from fastllama_b200.build import lib_path

    lib = lib_path("libggml_b200.so")
    check_close(run_steps(lib, t), np.load(os.path.join(GOLDEN, f"llama_toy_{name}.npz")))
    assert C.CDLL(lib).ggml_b200_decode_mode() == 2          # persistent token kernel
