"""CPU, 2 and 4 ranks over gloo: the tensor-parallel prompt plan (ggml_b200.cpp run_prompt_plan) on the CPU stand-in of the device layer
(tests/mock/mock_fl_cuda.c, with fl_dev_tp_unshard from tests/mock/mock_tp_unshard.c), launched like tests/test_tp_gloo.py.  A multi-token eval runs on each rank's weight shards -- wq/wk/wv by heads, w1/w3 by
n_ff slices, wo, w2 and the output matrix by rows -- with the activations all-gathered, and must give the single-rank run's tokens and
logit bits, with no device copy of the model on any rank.  The prompts are longer than n_batch, so several chunks are evaluated with
n_past > 0, and the scenarios interleave them with sharded decode steps and a state file."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "fastllama_b200", "lib")
HAVE_MOCK = all(os.path.exists(os.path.join(LIB, n)) for n in ("libggml_b200.so", "pyfastllama.so"))

WORKER = r'''
import ctypes as C, os, sys, numpy as np
sys.path.insert(0, sys.argv[1])
import torch, torch.distributed as dist
from fastllama_b200.model import Model, QuietLogger
rank, world, mock, path, out, n_batch = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), sys.argv[2], sys.argv[3], sys.argv[4], int(sys.argv[5])
if world > 1:
    dist.init_process_group("gloo", rank=rank, world_size=world)
lib = C.CDLL(os.path.join(mock, "libfl_cuda.so"), mode=C.RTLD_GLOBAL)
CB = C.CFUNCTYPE(None, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t)
def coll(kind, send, recv, n):
    if kind == 0:
        t = torch.from_numpy(np.ctypeslib.as_array((C.c_float * n).from_address(send))); dist.all_reduce(t)
    else:
        s = torch.from_numpy(np.ctypeslib.as_array((C.c_float * n).from_address(send)).copy())
        r = np.ctypeslib.as_array((C.c_float * (n * world)).from_address(recv))
        parts = [torch.empty(n) for _ in range(world)]
        dist.all_gather(parts, s)
        r[:] = torch.cat(parts).numpy()
cb = CB(coll)
lib.fl_mock_set_collective(cb, rank, world)
g = C.CDLL(os.path.join(mock, "libggml_b200.so"))
class Mem(C.Structure):
    _fields_ = [("weight_mirror_bytes", C.c_uint64), ("shard_bytes", C.c_uint64), ("mirror_bytes", C.c_uint64), ("kv_gathers", C.c_uint64)]
def mem():
    m = Mem(); g.ggml_b200_get_memory(C.byref(m)); return np.array([m.weight_mirror_bytes, m.shard_bytes, m.mirror_bytes, m.kv_gathers], dtype=np.uint64)
P1 = "Tensor parallel prompt ingest on the weight shards of every rank."          # both prompts and the decode steps fit n_ctx 128
P2 = " A second prompt attends to all of it."
so = os.path.join(mock, "pyfastllama.so")
m = Model(path, num_threads=2, n_ctx=128, n_batch=n_batch, logger=QuietLogger(), library_path=so)
toks = []
gen = lambda n: m.generate(lambda s: toks.append(s), num_tokens=n, temp=0.0, top_k=1, top_p=1.0, repeat_penalty=1.0)
gathers, modes, logits = [], [], []
def step():
    gathers.append(int(mem()[3])); logits.append(m.get_logits_array())
assert m.ingest(P1); modes.append(g.ggml_b200_prompt_mode()); step()
gen(4); step()
assert m.ingest(P2); modes.append(g.ggml_b200_prompt_mode()); step()
gen(4); step()
assert m.save_state(out + f".rank{rank}.state"); step()
gen(3)
first = list(toks[-3:])
assert m.load_state(out + f".rank{rank}.state")
gen(3); step()
assert list(toks[-3:]) == first, (toks[-3:], first)
mem_kv = mem()
m.close()
# every column's logits, the embeddings and the perplexity
m = Model(path, num_threads=2, n_ctx=128, n_batch=n_batch, should_get_all_logits=True, embedding_eval_enabled=True, logger=QuietLogger(), library_path=so)
assert m.ingest(P1)
modes.append(g.ggml_b200_prompt_mode())
all_logits, emb = m.get_logits_array(), np.array(m.get_embeddings(), dtype=np.float32)
ppl = m.perplexity("The quick brown fox jumps over the lazy dog. " * 6)
mem_all = mem()
m.close()
np.savez(out + f".rank{rank}.npz", toks=np.array(toks), gathers=np.array(gathers), modes=np.array(modes), logits=np.stack(logits), mem_kv=mem_kv,
         all_logits=all_logits, emb=emb, ppl=np.float64(ppl), mem_all=mem_all)
'''

# toy shapes of tests/test_tp_gloo.py; n_mult 256 gives n_ff 768, which 4 ranks split into 32-row multiples as the decode plan needs
DIMS = dict(n_vocab=512, n_embd=256, n_mult=256, n_head=4, n_layer=3)


@pytest.fixture(scope="module")
def mock():
    """The CPU stand-in of the device layer plus its fl_dev_tp_unshard, built as one libfl_cuda.so in a temporary directory with the
    stand-in's flags, next to copies of the host libraries (their $ORIGIN runpath resolves libfl_cuda.so there)."""
    import shutil
    import tempfile

    d = tempfile.mkdtemp(prefix="fl_mock_tp_")
    src = os.path.join(ROOT, "tests", "mock")
    subprocess.run(["/usr/bin/gcc", "-O2", "-mavx2", "-mfma", "-mf16c", "-ffp-contract=off", "-fPIC", "-shared", "-w",
                    "-I" + os.path.join(ROOT, "include"), "-o", os.path.join(d, "libfl_cuda.so"), os.path.join(src, "mock_fl_cuda.c"),
                    os.path.join(src, "mock_tp_unshard.c"), os.path.join(ROOT, "oracle", "q4_oracle.c"), "-lm", "-lrt"],
                   check=True, capture_output=True, timeout=300)
    for n in ("libggml_b200.so", "pyfastllama.so"):
        shutil.copy(os.path.join(LIB, n), d)
    yield d
    shutil.rmtree(d, ignore_errors=True)


@pytest.fixture(scope="module")
def toy(tmp_path_factory, mock):
    from fastllama_b200.ggjt import Q4_0, write_synthetic_numpy
    from oracle.pyoracle import Oracle

    orc = Oracle()
    d = tmp_path_factory.mktemp("tp_ingest")
    path = str(d / "toy.bin")
    write_synthetic_numpy(path, Q4_0, seed=5, std=0.01, quantize=lambda w, t: orc.quantize_q4(w, t), **DIMS)
    script = d / "worker.py"
    script.write_text(WORKER)
    return d, path, script, {}, mock


def launch(toy, world, n_batch, env=None, tag=""):
    d, path, script, cache, mock = toy
    key = (world, n_batch, tag)
    if key in cache:
        return cache[key]
    out = str(d / f"w{world}_b{n_batch}{tag}")
    procs = []
    for r in range(world):
        e = dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT="29651", OMP_NUM_THREADS="2",
                 FL_MOCK_SESSION=f"{os.getpid()}_ingest_{world}_{n_batch}{tag}", **(env or {}))
        procs.append(subprocess.Popen([sys.executable, str(script), ROOT, mock, path, out, str(n_batch)], env=e, stdout=subprocess.DEVNULL,
                                      stderr=subprocess.PIPE))
    errs = [p.communicate(timeout=600)[1] for p in procs]
    for p, err in zip(procs, errs):
        assert p.returncode == 0, err.decode()[-3000:]
    cache[key] = [np.load(out + f".rank{r}.npz") for r in range(world)]
    return cache[key]


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def weight_bytes():
    """(matrix bytes, embedding table bytes, norm bytes) of the toy q4_0 model"""
    E, V, L = DIMS["n_embd"], DIMS["n_vocab"], DIMS["n_layer"]
    F = ((2 * (4 * E) // 3 + DIMS["n_mult"] - 1) // DIMS["n_mult"]) * DIMS["n_mult"]
    q4 = lambda n: n // 32 * 20
    return q4(L * (4 * E * E + 3 * E * F) + V * E), q4(V * E), (2 * L + 1) * E * 4


@pytest.mark.skipif(not HAVE_MOCK, reason="needs the built host libraries and the drop-in pyfastllama.so")
@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("n_batch", [4, 8, 32])
def test_prompt_plan_matches_single_rank(toy, n_batch, world):
    """Ingest, decode, ingest, decode, save_state, load_state: the one-rank tokens and logit bits after every step; every multi-token eval
    ran through the prompt plan; no rank mirrored a weight; the KV cache was gathered for the state file, never for an ingest."""
    single = launch(toy, 1, n_batch)[0]
    mats, table, norms = weight_bytes()
    for r in launch(toy, world, n_batch):
        assert list(r["toks"]) == list(single["toks"])
        assert len(r["logits"]) == len(single["logits"])
        for a, b in zip(r["logits"], single["logits"]):
            assert same_bits(a, b)
        assert list(r["modes"]) == [1, 1, 1]
        for mem in (r["mem_kv"], r["mem_all"]):
            assert int(mem[0]) == 0                                             # no device copy of any weight
            assert 0 < int(mem[1]) <= mats // world + table + norms            # this rank's rows, the table and the norms
        g = list(r["gathers"])                                                  # after: ingest, decode, ingest, decode, save_state
        assert g[0] == g[1] == g[2] == g[3] and g[4] == g[3] + 1, g


@pytest.mark.skipif(not HAVE_MOCK, reason="needs the built host libraries and the drop-in pyfastllama.so")
@pytest.mark.parametrize("world", [2, 4])
def test_prompt_plan_all_logits_embeddings_perplexity(toy, world):
    """should_get_all_logits: every column of a multi-token eval; embedding_eval_enabled: the embeddings; perplexity: the same float."""
    single = launch(toy, 1, 8)[0]
    for r in launch(toy, world, 8):
        assert same_bits(r["all_logits"], single["all_logits"]) and r["all_logits"].size == 8 * DIMS["n_vocab"]
        assert same_bits(r["emb"], single["emb"]) and r["emb"].size == DIMS["n_embd"]
        assert float(r["ppl"]) == float(single["ppl"]) and float(r["ppl"]) > 1.0


@pytest.mark.skipif(not HAVE_MOCK, reason="needs the built host libraries and the drop-in pyfastllama.so")
def test_replicated_switch_mirrors_the_weights_with_the_same_bits(toy):
    """FASTLLAMA_B200_TP_INGEST=replicated: the node-by-node executor on every rank (prompt mode 0), which mirrors the weights it reads;
    tokens and logit bits as with the prompt plan."""
    single = launch(toy, 1, 8)[0]
    for r in launch(toy, 2, 8, env={"FASTLLAMA_B200_TP_INGEST": "replicated"}, tag="_repl"):
        assert list(r["modes"]) == [0, 0, 0]
        assert int(r["mem_kv"][0]) > 0
        assert list(r["toks"]) == list(single["toks"])
        for a, b in zip(r["logits"], single["logits"]):
            assert same_bits(a, b)
        assert same_bits(r["all_logits"], single["all_logits"]) and same_bits(r["emb"], single["emb"])


@pytest.mark.skipif(not HAVE_MOCK, reason="needs the built host libraries and the drop-in pyfastllama.so")
def test_unshard_stand_in_against_numpy(mock):
    lib = C.CDLL(os.path.join(mock, "libfl_cuda.so"))
    fn = lib.fl_dev_tp_unshard
    fn.restype, fn.argtypes = C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    rng = np.random.default_rng(3)
    for world, N, nl in [(2, 5, 12), (4, 3, 7), (3, 1, 4)]:
        g = rng.standard_normal((world, N, nl)).astype(np.float32)
        res = rng.standard_normal((N, world * nl)).astype(np.float32)
        want = g.transpose(1, 0, 2).reshape(N, world * nl)
        for residual in (None, res):
            dst = np.empty((N, world * nl), dtype=np.float32)
            assert fn(g.ctypes.data, world, N, nl, None if residual is None else residual.ctypes.data, dst.ctypes.data) == 0
            ref = want if residual is None else (want + residual).astype(np.float32)
            assert np.array_equal(dst.view(np.uint32), ref.view(np.uint32))
