"""On the H100, through the real library: the multi-context scenario of tests/test_multi_context.py (interleaved contexts, a context
closed while another is alive, two contexts over one mapped file, `m = Model(...)` rebinding, n_ctx 64 / 128, head dimensions 64 / 32,
save_state / load_state next to a live context) against the reference library's bits, for toy models and for a 2-layer 7B-shaped q4_0
model whose decode steps run as the persistent token kernel.  Every step runs as the token kernel (decode mode 2), switching contexts
builds and captures nothing, and after both contexts are closed the device memory in use is back to its level before the scenario."""
import os

import pytest

from tests.test_multi_context import STEPS, _models, check, run_scenario

pytestmark = pytest.mark.gpu
SLACK = 64 << 20


def _lib():
    from fastllama_b200.build import lib_path

    return lib_path("pyfastllama.so")


def _ref():
    from oracle.pyoracle import REF_PYFASTLLAMA_SO

    if not os.path.exists(REF_PYFASTLLAMA_SO):
        pytest.skip("oracle/_ref not built")
    return REF_PYFASTLLAMA_SO


def _check_gpu(ours, ref, use_mmap):
    check(ours, ref, use_mmap)
    modes = {s: int(ours[s + "_mode"]) for s in STEPS}
    assert all(v == 2 for v in modes.values()), modes
    before, after = int(ours["free_before"]), int(ours["free_after"])
    assert abs(before - after) <= SLACK, (before, after)


@pytest.mark.parametrize("use_mmap", [True, False])
def test_toy_contexts_interleave_with_the_reference_bits(tmp_path, use_mmap):
    paths = _models(tmp_path)
    ref = run_scenario(tmp_path, _ref(), paths, use_mmap, "ref")
    ours = run_scenario(tmp_path, _lib(), paths, use_mmap, "ours", env={"FL_TEST_MEMINFO": "1"})
    _check_gpu(ours, ref, use_mmap)


def test_7b_shaped_contexts_interleave_with_the_reference_bits(tmp_path):
    """Two 2-layer 7B-shaped q4_0 files (n_embd 4096, 32 heads, n_vocab 32000); the third model of the scenario is the first file again
    at n_ctx 128."""
    from fastllama_b200.ggjt import write_synthetic_gpu

    paths = []
    for seed in (0, 1):
        p = str(tmp_path / f"7b_2l_seed{seed}.bin")
        write_synthetic_gpu(p, size="7B", wtype=2, seed=seed, std=0.02, n_layer=2)
        paths.append(p)
    paths.append(paths[0])
    ref = run_scenario(tmp_path, _ref(), paths, True, "ref7")
    ours = run_scenario(tmp_path, _lib(), paths, True, "ours7", env={"FL_TEST_MEMINFO": "1"})
    _check_gpu(ours, ref, True)
