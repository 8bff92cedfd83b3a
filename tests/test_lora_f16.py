"""The ops of attaching / detaching a cached f16 LoRA adapter (convert-lora-to-ggml.py --dtype fp16), against the fixture
tests/golden/lora_f16_ops.npz = outputs of the reference LIBRARY (oracle/gen_golden_lora_f16.py):
    add_inplace(W_quantised, X_f16)                  attach: ggml_compute_forward_add_q_f16 (reference lib/ggml.c:12372-12483)
    add_inplace(W_quantised, scale(X_f16, -1))       detach: ggml_compute_forward_scale_f16 (:12485-12524) in place on X, then as above
and scale_f16 with a factor that rounds.  Every comparison is on the bytes, at zero tolerance.

  * CPU: the reference library still reproduces the fixture (pins the fixture; needs oracle/_ref);
  * CPU: the C oracle (oracle/lora_f16_oracle.c) matches it;
  * CPU: our host stack (f16 src1 of the quantised add, f16 scale) on the CPU stand-in of the device layer (tests/lora_mock.py);
  * GPU: the kernels of fastllama_b200/csrc/fl_lora_kernels.cu through libggml_b200."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from oracle.gen_golden_lora_f16 import LORA_F16_SCALE, LORA_F16_SHAPES
from oracle.pyoracle import REF_GGML_SO
from tests import ggml_api as G
from tests.lora_mock import HAVE_LIBS, F16Oracle, mock_dir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "lora_f16_ops.npz")
TYPES = [("q4_0", G.Q4_0), ("q4_1", G.Q4_1)]
SHAPES = [f"{k}x{m}" for k, m in LORA_F16_SHAPES]


def run_lora_f16_graphs(lib_path, name, t, shape):
    """-> (merged bytes, detached bytes, X scaled by LORA_F16_SCALE) computed by the library at lib_path."""
    gold = np.load(GOLDEN)
    g = G.Ggml(lib_path)
    k, m = (int(v) for v in shape.split("x"))
    x = gold[f"x_{shape}"]
    base = gold[f"{name}_base_{shape}"]
    # the weights live in their own (persistent) arena, the adapter in the graph's arena, as in the reference's loader
    wa = g.context(4 << 20)
    tw = g.new_tensor_2d(wa.ctx, t, k, m)
    wa.set(tw, base)
    sync = getattr(g.lib, "ggml_b200_sync_to_host", None)
    if sync is not None:
        sync.argtypes, sync.restype = [G.C.c_void_p, G.C.c_size_t], None

    def weights():
        if sync is not None:                       # ours: the merged weights are on the device; fetch them for the comparison
            sync(tw.contents.data, base.nbytes)
        return wa.numpy(tw).reshape(m, -1).copy()

    def compute(ar, node):
        gf = G.new_graph()
        g.build_forward_expand(gf, node)
        g.graph_compute(ar.ctx, gf)

    ar = g.context(16 << 20)
    tx = g.new_tensor_2d(ar.ctx, G.F16, k, m)
    ar.set(tx, x)
    compute(ar, g.add_inplace(ar.ctx, tw, tx))
    merged = weights()
    compute(ar, g.add_inplace(ar.ctx, tw, g.scale(ar.ctx, tx, g.new_f32(ar.ctx, -1.0))))
    detached = weights()
    ar.free()

    ar = g.context(16 << 20)
    tx = g.new_tensor_2d(ar.ctx, G.F16, k, m)
    ar.set(tx, x)
    sc = g.scale(ar.ctx, tx, g.new_f32(ar.ctx, LORA_F16_SCALE))
    compute(ar, sc)
    if sync is not None:
        sync(sc.contents.data, x.nbytes)
    scaled = ar.numpy(tx).view(np.float16).reshape(m, k).copy()
    ar.free()
    wa.free()
    return merged, detached, scaled


def check(outs, name, shape):
    gold = np.load(GOLDEN)
    merged, detached, scaled = outs
    assert np.array_equal(merged, gold[f"{name}_merged_{shape}"]), "merged weights differ from the reference's bytes"
    assert np.array_equal(detached, gold[f"{name}_detached_{shape}"]), "detached weights differ from the reference's bytes"
    assert np.array_equal(scaled.view(np.uint16), gold[f"x_scaled_{shape}"].view(np.uint16)), "scale_f16 differs from the reference's bits"
    assert not np.array_equal(merged, gold[f"{name}_base_{shape}"])


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("name,t", TYPES)
def test_reference_library_reproduces_the_fixture(name, t, shape):
    if not os.path.exists(REF_GGML_SO):
        pytest.skip("oracle/_ref not built")
    check(run_lora_f16_graphs(REF_GGML_SO, name, t, shape), name, shape)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("name,t", TYPES)
def test_oracle_matches_the_fixture(name, t, shape):
    orc = F16Oracle()
    try:
        gold = np.load(GOLDEN)
        x = gold[f"x_{shape}"]
        merged = orc.add_q_f16(gold[f"{name}_base_{shape}"], x, t)
        detached = orc.add_q_f16(merged, orc.scale_f16(x, -1.0), t)
        check((merged, detached, orc.scale_f16(x, LORA_F16_SCALE)), name, shape)
    finally:
        orc.close()


MOCK_RUN = r"""
import sys
sys.path.insert(0, sys.argv[1])
from tests.test_lora_f16 import check, run_lora_f16_graphs
lib, name, t, shape = sys.argv[2], sys.argv[3], int(sys.argv[4]), sys.argv[5]
check(run_lora_f16_graphs(lib, name, t, shape), name, shape)
print("OK")
"""


@pytest.fixture(scope="module")
def mock():
    if not HAVE_LIBS:
        pytest.skip("needs the built host libraries")
    d = mock_dir()
    yield d
    shutil.rmtree(d, ignore_errors=True)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("name,t", TYPES)
def test_host_stack_on_cpu_mock(mock, name, t, shape):
    lib = os.path.join(mock, "libggml_b200.so")
    res = subprocess.run([sys.executable, "-c", MOCK_RUN, ROOT, lib, name, str(t), shape], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0 and "OK" in res.stdout, res.stdout[-2000:] + res.stderr[-2000:]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("name,t", TYPES)
def test_lora_f16_ops_on_gpu(name, t, shape):
    from fastllama_b200.build import lib_path

    check(run_lora_f16_graphs(lib_path("libggml_b200.so"), name, t, shape), name, shape)
