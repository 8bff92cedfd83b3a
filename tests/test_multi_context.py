"""Several live model contexts in one process, on the CPU stand-in of the device layer (tests/mock) against the reference library running
the same script.

Each context keeps its own decode state (plan, token-kernel program, captured graph), keyed by its KV-cache arena, so switching back to a
context replays its graph; mmap'ed weight ranges are mirrored by file identity, so two contexts over one file share one device copy; and
Model.close() (ggml_b200_release_unused) frees only what belongs to the closed context.  The scenario interleaves contexts, closes one
while another is alive, opens a second context on a live context's file, rebinds `m = Model(...)` the way a web UI switches models,
mixes n_ctx 64 / 128 and head dimensions 64 / 32, and saves / loads the state of one context while another is alive.  Every step's tokens
and logits must be the reference's bits."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
from tests.mockbuild import ensure_mock  # noqa: E402

MOCK = ensure_mock()

WORKER = r'''
import ctypes as C, os, sys, numpy as np
sys.path.insert(0, sys.argv[1])
from fastllama_b200.model import Model, QuietLogger
lib, out, use_mmap, tmp = sys.argv[2], sys.argv[3], sys.argv[4] == "1", sys.argv[5]
path_a, path_b, path_h8 = sys.argv[6:9]
if "mock" in lib:
    C.CDLL(os.path.join(os.path.dirname(lib), "libfl_cuda.so"), mode=C.RTLD_GLOBAL)
greedy = dict(temp=0.0, top_k=1, top_p=1.0, repeat_penalty=1.0)
res = {}
q = C.CDLL(lib)
have_q = hasattr(q, "ggml_b200_get_contexts")
class Contexts(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("live_states", "plan_builds", "graph_captures", "external_copies", "external_mappings", "external_bytes")]
class Mem(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("weight_mirror_bytes", "shard_bytes", "mirror_bytes", "kv_gathers")]
def snap(tag):
    if not have_q:
        return
    c, m = Contexts(), Mem()
    q.ggml_b200_get_contexts(C.byref(c))
    q.ggml_b200_get_memory(C.byref(m))
    res[tag + "_ctx"] = np.array([getattr(c, n) for n, _ in Contexts._fields_], dtype=np.uint64)
    res[tag + "_mem"] = np.array([getattr(m, n) for n, _ in Mem._fields_], dtype=np.uint64)
    res[tag + "_mode"] = np.int64(q.ggml_b200_decode_mode())
def model(path, n_ctx):
    return Model(path, num_threads=2, n_ctx=n_ctx, n_batch=4, use_mmap=use_mmap, logger=QuietLogger(), library_path=lib)
def run(tag, m, n=4):
    toks = []
    assert m.generate(lambda s: toks.append(s), num_tokens=n, **greedy)
    res[tag + "_tokens"] = np.array(toks)
    res[tag + "_logits"] = m.get_logits_array()
    snap(tag)

# FL_TEST_MEMINFO=1 (GPU): device memory in use after a warm-up context (kernels loaded, tables built) and after the scenario
meminfo = os.environ.get("FL_TEST_MEMINFO") == "1"
if meminfo:
    import torch
    w = model(path_a, 64); assert w.ingest("Warm up."); run("warm", w); w.close(); del w
    res["free_before"] = np.int64(torch.cuda.mem_get_info()[0])
# A, B, A, B, B.close(), A
A = model(path_a, 64); assert A.ingest("Two contexts, one process."); run("a1", A)
B = model(path_b, 64); assert B.ingest("A second model joins."); run("b1", B)
run("a2", A); run("b2", B)
B.close(); snap("b_closed")
run("a3", A)
# C on A's file, interleaved with A; A.close(); C
Cx = model(path_a, 64); assert Cx.ingest("The same file, mapped again."); run("c1", Cx)
run("a4", A); run("c2", Cx)
A.close(); snap("a_closed")
run("c3", Cx)
# save_state / load_state of one context while another is alive (n_ctx 128 next to 64)
D = model(path_b, 128); assert D.ingest("A longer window next to a short one."); run("d1", D)
sd, sc = os.path.join(tmp, "d.state"), os.path.join(tmp, "c.state")
assert D.save_state(sd); run("d2", D); run("c4", Cx)
assert D.load_state(sd); run("d3", D)
assert Cx.save_state(sc); run("c5", Cx); run("d4", D)
assert Cx.load_state(sc); run("c6", Cx)
Cx.close(); D.close(); snap("cd_closed")
# m = Model(x); m = Model(y): the new model is built before the old one is dropped; head dimension 32 next to 64
m = model(path_a, 64); assert m.ingest("Switch models."); run("w1", m)
m = model(path_h8, 128); assert m.ingest("Switch models."); run("w2", m)
E = model(path_a, 64); assert E.ingest("Switch back."); run("e1", E)
run("w3", m); run("e2", E)
E.close(); m.close(); snap("end")
if meminfo:
    res["free_after"] = np.int64(torch.cuda.mem_get_info()[0])
np.savez(out, **res)
'''

STEPS = ["a1", "b1", "a2", "b2", "a3", "c1", "a4", "c2", "c3", "d1", "d2", "c4", "d3", "c5", "d4", "c6", "w1", "w2", "e1", "w3", "e2"]


def _models(tmp_path):
    from fastllama_b200.ggjt import Q4_0, write_synthetic_numpy
    from oracle.pyoracle import Oracle

    orc = Oracle()
    paths = []
    for seed, n_head in ((11, 4), (12, 4), (13, 8)):          # head dimensions 64, 64, 32
        p = str(tmp_path / f"toy{seed}.bin")
        write_synthetic_numpy(p, Q4_0, n_vocab=512, n_embd=256, n_mult=256, n_head=n_head, n_layer=3, seed=seed, std=0.01,
                              quantize=lambda w, t: orc.quantize_q4(w, t))
        paths.append(p)
    return paths


def run_scenario(tmp_path, lib, paths, use_mmap, tag, env=None):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    out = str(tmp_path / f"{tag}.npz")
    work = tmp_path / tag
    work.mkdir(exist_ok=True)
    p = subprocess.run([sys.executable, str(script), ROOT, lib, out, "1" if use_mmap else "0", str(work)] + paths, capture_output=True, text=True,
                       timeout=1200, env=dict(os.environ, OMP_NUM_THREADS="2", **(env or {})))
    assert p.returncode == 0, p.stderr[-3000:]
    return np.load(out)


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def check(ours, ref, use_mmap):
    for s in STEPS:
        assert list(ours[s + "_tokens"]) == list(ref[s + "_tokens"]), s
        assert same_bits(ours[s + "_logits"], ref[s + "_logits"]), s
    assert list(ref["a1_tokens"]) != list(ref["b1_tokens"]), "the toy models must behave differently"
    assert list(ref["d3_tokens"]) == list(ref["d2_tokens"]), "load_state must bring back the saved context"
    assert list(ref["c6_tokens"]) == list(ref["c5_tokens"])
    ctx = {k[:-4]: ours[k] for k in ours.files if k.endswith("_ctx")}
    mem = {k[:-4]: ours[k] for k in ours.files if k.endswith("_mem")}
    LIVE, BUILDS, CAPTURES, COPIES, MAPPINGS = 0, 1, 2, 3, 4
    WEIGHTS, MIRRORS = 0, 2
    # every context builds its plan once; switching back replays it
    for prev, cur in (("b1", "a2"), ("a2", "b2"), ("b2", "a3"), ("c1", "a4"), ("a4", "c2"), ("c2", "c3"), ("d1", "d2"), ("d2", "c4"),
                      ("c4", "d3"), ("d3", "c5"), ("c5", "d4"), ("d4", "c6"), ("e1", "w3"), ("w3", "e2")):
        assert ctx[cur][BUILDS] == ctx[prev][BUILDS], (prev, cur, ctx[prev], ctx[cur])
        assert ctx[cur][CAPTURES] == ctx[prev][CAPTURES], (prev, cur, ctx[prev], ctx[cur])
    assert ctx["b1"][LIVE] == 2 and ctx["b_closed"][LIVE] == 1 and ctx["c1"][LIVE] == 2 and ctx["a_closed"][LIVE] == 1
    assert int(ctx["b1"][CAPTURES]) - int(ctx["a1"][CAPTURES]) == 1 and int(ctx["c1"][CAPTURES]) - int(ctx["b1"][CAPTURES]) == 1
    # two contexts over one mapped file hold one device copy of its weights
    if use_mmap:
        assert int(ctx["c1"][MAPPINGS]) == 2 * int(ctx["c1"][COPIES]) > 0
        assert int(mem["c1"][WEIGHTS]) == int(mem["a1"][WEIGHTS]) > 0
    else:
        assert int(ctx["c1"][COPIES]) == 0
        assert int(mem["c1"][WEIGHTS]) == 2 * int(mem["a1"][WEIGHTS]) > 0
    for t in ("cd_closed", "end"):
        assert int(ctx[t][LIVE]) == 0 and int(mem[t][MIRRORS]) == 0 and int(ctx[t][COPIES]) == 0, (t, ctx[t], mem[t])


@pytest.mark.skipif(not os.path.exists(os.path.join(MOCK, "pyfastllama.so")), reason="tests/mock not built (needs the drop-in library)")
@pytest.mark.parametrize("use_mmap", [True, False])
def test_contexts_interleave_with_the_reference_bits_on_cpu_mock(tmp_path, use_mmap):
    from oracle.pyoracle import REF_PYFASTLLAMA_SO

    if not os.path.exists(REF_PYFASTLLAMA_SO):
        pytest.skip("oracle/_ref not built")
    paths = _models(tmp_path)
    ref = run_scenario(tmp_path, REF_PYFASTLLAMA_SO, paths, use_mmap, "ref")
    ours = run_scenario(tmp_path, os.path.join(MOCK, "pyfastllama.so"), paths, use_mmap, "ours")
    check(ours, ref, use_mmap)
    assert all(int(ours[s + "_mode"]) == 2 for s in STEPS)       # the stand-in takes every plan as a token-kernel program
