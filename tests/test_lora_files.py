"""Model.attach_lora / detach_lora end to end through the bridge, on the CPU stand-in of the device layer (tests/lora_mock.py), against the
reference library running the same script (the child-process pattern of tests/test_multi_context.py).

For toy q4_0 and q4_1 models, each adapter form the reference's converter writes (cached f32, uncached f32, cached f16) and use_mmap on
and off: ingest, generate 4, attach, generate 4, detach, generate 4, then attach / generate / detach once more.  Every step's tokens and
logits must be the reference's bits, and attach / detach must return what the reference returns, including its False for an uncached
f16 file, for an adapter whose shapes fit no weight, for a second attach and for a detach with nothing attached.  With use_mmap, a
second and third context on the same file show that an attach on one context leaves the others' logits untouched."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
from tests.lora_files import FORMS, write_adapter  # noqa: E402
from tests.lora_mock import HAVE_LIBS, mock_dir  # noqa: E402

WORKER = r'''
import ctypes as C, json, os, sys, numpy as np
sys.path.insert(0, sys.argv[1])
from fastllama_b200.model import Model, QuietLogger
lib, out, use_mmap, path, adapters = sys.argv[2], sys.argv[3], sys.argv[4] == "1", sys.argv[5], json.loads(sys.argv[6])
if "mock" in lib:
    C.CDLL(os.path.join(os.path.dirname(lib), "libfl_cuda.so"), mode=C.RTLD_GLOBAL)
greedy = dict(temp=0.0, top_k=1, top_p=1.0, repeat_penalty=1.0)
res = {}
q = C.CDLL(lib)
have_q = hasattr(q, "ggml_b200_decode_mode")
PROMPT = "An adapter changes the weights."
def model():
    return Model(path, num_threads=2, n_ctx=64, n_batch=4, use_mmap=use_mmap, logger=QuietLogger(), library_path=lib)
def run(tag, m, n=4):
    toks = []
    assert m.generate(lambda s: toks.append(s), num_tokens=n, **greedy)
    res[tag + "_tokens"] = np.array(toks)
    res[tag + "_logits"] = m.get_logits_array()
    if have_q:
        res[tag + "_mode"] = np.int64(q.ggml_b200_decode_mode())

# FL_TEST_MEMINFO=1 (GPU): device memory in use after a warm-up context and after the scenario
meminfo = os.environ.get("FL_TEST_MEMINFO") == "1"
if meminfo:
    import torch
    w = model(); assert w.ingest("Warm up."); assert w.generate(lambda s: None, num_tokens=4, **greedy); w.close(); del w
    res["free_before"] = np.int64(torch.cuda.mem_get_info()[0])
# what the reference refuses, on a model that then runs unchanged
m = model(); assert m.ingest(PROMPT)
for bad in ("uncached_f16", "mismatch"):
    if bad in adapters:
        res["ret_" + bad] = np.int64(m.attach_lora(adapters[bad]))
res["ret_detach_none"] = np.int64(m.detach_lora())
run("refused", m); m.close()
for form in (f for f in adapters if f not in ("uncached_f16", "mismatch")):
    m = model(); assert m.ingest(PROMPT)
    run(form + "_0", m)
    res[form + "_ret_attach"] = np.int64(m.attach_lora(adapters[form])); run(form + "_1", m)
    res[form + "_ret_attach_again"] = np.int64(m.attach_lora(adapters[form]))
    res[form + "_ret_detach"] = np.int64(m.detach_lora()); run(form + "_2", m)
    res[form + "_ret_reattach"] = np.int64(m.attach_lora(adapters[form])); run(form + "_3", m)
    res[form + "_ret_redetach"] = np.int64(m.detach_lora()); run(form + "_4", m)
    m.close()
# use_mmap: three contexts on one file; A attaches, B runs on next to it, C ran the same steps before anything was attached
if use_mmap and "cached_f16" in adapters:
    A, B, Cx = model(), model(), model()
    for x in (A, B, Cx):
        assert x.ingest(PROMPT)
    run("c1", Cx); run("c2", Cx); run("b1", B); run("a1", A)
    res["a_ret_attach"] = np.int64(A.attach_lora(adapters["cached_f16"])); run("a2", A)
    run("b2", B)
    res["a_ret_detach"] = np.int64(A.detach_lora()); run("a3", A)
    A.close(); B.close(); Cx.close()
if meminfo:
    res["free_after"] = np.int64(torch.cuda.mem_get_info()[0])
np.savez(out, **res)
'''


def toy_model(tmp_path, wtype, seed=21):
    from fastllama_b200.ggjt import write_synthetic_numpy
    from oracle.pyoracle import Oracle

    orc = Oracle()
    p = str(tmp_path / f"toy_{wtype}.bin")
    write_synthetic_numpy(p, wtype, n_vocab=512, n_embd=256, n_mult=256, n_head=4, n_layer=3, seed=seed, std=0.01,
                          quantize=lambda w, t: orc.quantize_q4(w, t))
    return p


def toy_adapters(tmp_path, forms=FORMS + ("uncached_f16", "mismatch"), layers=(0, 1, 2), n_embd=256, n_ff=768, std=0.02):
    paths = {}
    for i, form in enumerate(forms):
        p = str(tmp_path / f"lora_{form}.bin")
        write_adapter(p, form, n_embd, n_ff, layers, seed=100 + i, std=std)
        paths[form] = p
    return paths


def run_scenario(tmp_path, lib, path, adapters, use_mmap, tag, env=None):
    script = tmp_path / "lora_worker.py"
    script.write_text(WORKER)
    out = str(tmp_path / f"{tag}.npz")
    p = subprocess.run([sys.executable, str(script), ROOT, lib, out, "1" if use_mmap else "0", path, json.dumps(adapters)], capture_output=True,
                       text=True, timeout=2400, env=dict(os.environ, OMP_NUM_THREADS="2", **(env or {})))
    assert p.returncode == 0, p.stderr[-3000:]
    return np.load(out)


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def steps(res):
    return sorted(k[:-7] for k in res.files if k.endswith("_tokens"))


def check(ours, ref, adapters, use_mmap):
    assert steps(ours) == steps(ref)
    for s in steps(ref):
        assert list(ours[s + "_tokens"]) == list(ref[s + "_tokens"]), s
        assert same_bits(ours[s + "_logits"], ref[s + "_logits"]), s
    rets = sorted(k for k in ref.files if "ret_" in k)
    assert rets == sorted(k for k in ours.files if "ret_" in k)
    for k in rets:
        assert int(ours[k]) == int(ref[k]), k
    # what the reference does, so that the comparison above covers what it should
    assert int(ref["ret_detach_none"]) == 0
    for bad in ("uncached_f16", "mismatch"):
        if bad in adapters:
            assert int(ref["ret_" + bad]) == 0, bad
    forms = [f for f in adapters if f not in ("uncached_f16", "mismatch")]
    for f in forms:
        assert [int(ref[f + k]) for k in ("_ret_attach", "_ret_attach_again", "_ret_detach", "_ret_reattach", "_ret_redetach")] == [1, 0, 1, 1, 1]
        assert not same_bits(ref[f + "_1_logits"], ref[f + "_0_logits"]), f"{f}: the adapter must change the logits"
        assert same_bits(ref["refused_logits"], ref[f + "_0_logits"]), "a refused adapter must leave the weights alone"
    if use_mmap and "cached_f16" in adapters:
        assert int(ref["a_ret_attach"]) == 1 and int(ref["a_ret_detach"]) == 1
        assert not same_bits(ref["a2_logits"], ref["a1_logits"])
        for o in (ours, ref):
            assert same_bits(o["b1_logits"], o["c1_logits"]) and same_bits(o["b2_logits"], o["c2_logits"]), "an attach leaked into another context"


@pytest.fixture(scope="module")
def mock():
    import shutil

    d = mock_dir()
    yield d
    shutil.rmtree(d, ignore_errors=True)


@pytest.mark.skipif(not HAVE_LIBS, reason="needs the built host libraries and the drop-in pyfastllama.so")
@pytest.mark.parametrize("use_mmap", [True, False])
@pytest.mark.parametrize("wtype", [2, 3], ids=["q4_0", "q4_1"])
def test_adapter_files_attach_and_detach_with_the_reference_bits_on_cpu_mock(tmp_path, mock, wtype, use_mmap):
    from oracle.pyoracle import REF_PYFASTLLAMA_SO

    if not os.path.exists(REF_PYFASTLLAMA_SO):
        pytest.skip("oracle/_ref not built")
    path = toy_model(tmp_path, wtype)
    adapters = toy_adapters(tmp_path)
    ref = run_scenario(tmp_path, REF_PYFASTLLAMA_SO, path, adapters, use_mmap, "ref")
    ours = run_scenario(tmp_path, os.path.join(mock, "pyfastllama.so"), path, adapters, use_mmap, "ours")
    check(ours, ref, adapters, use_mmap)
    assert all(int(ours[s + "_mode"]) == 2 for s in steps(ours))       # the stand-in takes every plan as a token-kernel program
