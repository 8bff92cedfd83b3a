"""On the H100, through the real library: the adapter-file scenario of tests/test_lora_files.py (every adapter form the reference's
converter writes, attached, detached and attached again between decode steps; the reference's refusals; an attach next to other live
contexts on the same mapped file) against the reference library's bits, for toy models and for a 2-layer 7B-shaped q4_0 model with
adapters on wq / wk / wv / wo / w1 / w2 / w3.  Every decode step runs as the token kernel (decode mode 2), and after the last context is
closed the device memory in use is back to its level before the scenario."""
import os

import pytest

from tests.lora_files import FORMS
from tests.test_lora_files import check, run_scenario, steps, toy_adapters, toy_model

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


def _check_gpu(ours, ref, adapters, use_mmap):
    check(ours, ref, adapters, use_mmap)
    modes = {s: int(ours[s + "_mode"]) for s in steps(ours)}
    assert all(v == 2 for v in modes.values()), modes
    before, after = int(ours["free_before"]), int(ours["free_after"])
    assert abs(before - after) <= SLACK, (before, after)


@pytest.mark.parametrize("use_mmap", [True, False])
@pytest.mark.parametrize("wtype", [2, 3], ids=["q4_0", "q4_1"])
def test_toy_adapter_files_with_the_reference_bits(tmp_path, wtype, use_mmap):
    path = toy_model(tmp_path, wtype)
    adapters = toy_adapters(tmp_path)
    ref = run_scenario(tmp_path, _ref(), path, adapters, use_mmap, "ref")
    ours = run_scenario(tmp_path, _lib(), path, adapters, use_mmap, "ours", env={"FL_TEST_MEMINFO": "1"})
    _check_gpu(ours, ref, adapters, use_mmap)


def test_7b_shaped_adapter_files_with_the_reference_bits(tmp_path):
    """2-layer 7B-shaped q4_0 file (n_embd 4096, n_ff 11008, 32 heads, n_vocab 32000); each form adapts the seven matrices of layer 1."""
    from fastllama_b200.ggjt import write_synthetic_gpu

    path = str(tmp_path / "7b_2l.bin")
    write_synthetic_gpu(path, size="7B", wtype=2, seed=3, std=0.02, n_layer=2)
    adapters = toy_adapters(tmp_path, forms=FORMS, layers=(1,), n_embd=4096, n_ff=11008, std=0.01)
    ref = run_scenario(tmp_path, _ref(), path, adapters, False, "ref7")
    ours = run_scenario(tmp_path, _lib(), path, adapters, False, "ours7", env={"FL_TEST_MEMINFO": "1"})
    _check_gpu(ours, ref, adapters, False)
