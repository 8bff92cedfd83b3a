"""CPU, 2 ranks over gloo: two live contexts under tensor parallelism on the CPU stand-in of the device layer, launched like
tests/test_tp_ingest.py.  Each context keeps its own record of its head-sharded KV cache, so interleaved prompt ingests and decode steps of
two contexts, then save_state of each, give the single-rank run's tokens, logit bits and state files."""
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
rank, world, mock, path_a, path_b, out = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), sys.argv[2], sys.argv[3], sys.argv[4], sys.argv[5]
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
so = os.path.join(mock, "pyfastllama.so")
A = Model(path_a, num_threads=2, n_ctx=128, n_batch=8, logger=QuietLogger(), library_path=so)
B = Model(path_b, num_threads=2, n_ctx=64, n_batch=8, logger=QuietLogger(), library_path=so)
toks, logits, modes = [], [], []
def gen(m, n):
    t = []
    assert m.generate(lambda s: t.append(s), num_tokens=n, temp=0.0, top_k=1, top_p=1.0, repeat_penalty=1.0)
    toks.extend(t); logits.append(m.get_logits_array())
def ingest(m, p):
    assert m.ingest(p); modes.append(g.ggml_b200_prompt_mode()); logits.append(m.get_logits_array())
ingest(A, "Tensor parallel ingest of the first context.")
ingest(B, "And of a second one, next to it.")
gen(A, 4); gen(B, 4)
ingest(A, " More for the first.")
gen(B, 3)
ingest(B, " More for the second.")
gen(A, 3); gen(B, 2)
assert A.save_state(out + f".rank{rank}.a.state")
assert B.save_state(out + f".rank{rank}.b.state")
gen(A, 2); gen(B, 2)
A.close(); B.close()
np.savez(out + f".rank{rank}.npz", toks=np.array(toks), logits=np.concatenate(logits), modes=np.array(modes))
'''

DIMS = dict(n_vocab=512, n_embd=256, n_mult=256, n_head=4, n_layer=3)


@pytest.fixture(scope="module")
def mock():
    """The CPU stand-in of the device layer plus its fl_dev_tp_unshard, built as one libfl_cuda.so in a temporary directory next to copies
    of the host libraries (as tests/test_tp_ingest.py does)."""
    import shutil
    import tempfile

    d = tempfile.mkdtemp(prefix="fl_mock_mc_tp_")
    src = os.path.join(ROOT, "tests", "mock")
    subprocess.run(["/usr/bin/gcc", "-O2", "-mavx2", "-mfma", "-mf16c", "-ffp-contract=off", "-fPIC", "-shared", "-w",
                    "-I" + os.path.join(ROOT, "include"), "-o", os.path.join(d, "libfl_cuda.so"), os.path.join(src, "mock_fl_cuda.c"),
                    os.path.join(src, "mock_tp_unshard.c"), os.path.join(ROOT, "oracle", "q4_oracle.c"), "-lm", "-lrt"],
                   check=True, capture_output=True, timeout=300)
    for n in ("libggml_b200.so", "pyfastllama.so"):
        shutil.copy(os.path.join(LIB, n), d)
    yield d
    shutil.rmtree(d, ignore_errors=True)


def launch(tmp_path, mock, paths, world):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    out = str(tmp_path / f"w{world}")
    procs = []
    for r in range(world):
        e = dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT="29657", OMP_NUM_THREADS="2",
                 FL_MOCK_SESSION=f"{os.getpid()}_multi_context_{world}")
        procs.append(subprocess.Popen([sys.executable, str(script), ROOT, mock] + paths + [out], env=e, stdout=subprocess.DEVNULL,
                                      stderr=subprocess.PIPE))
    errs = [p.communicate(timeout=900)[1] for p in procs]
    for p, err in zip(procs, errs):
        assert p.returncode == 0, err.decode()[-3000:]
    return [(np.load(out + f".rank{r}.npz"), open(out + f".rank{r}.a.state", "rb").read(), open(out + f".rank{r}.b.state", "rb").read())
            for r in range(world)]


@pytest.mark.skipif(not HAVE_MOCK, reason="needs the built host libraries and the drop-in pyfastllama.so")
def test_two_contexts_under_tensor_parallelism_match_single_rank(tmp_path, mock):
    from fastllama_b200.ggjt import Q4_0, write_synthetic_numpy
    from oracle.pyoracle import Oracle

    orc = Oracle()
    paths = []
    for seed in (5, 6):
        p = str(tmp_path / f"toy{seed}.bin")
        write_synthetic_numpy(p, Q4_0, seed=seed, std=0.01, quantize=lambda w, t: orc.quantize_q4(w, t), **DIMS)
        paths.append(p)
    (single, sa, sb), = launch(tmp_path, mock, paths, 1)
    for r, a, b in launch(tmp_path, mock, paths, 2):
        assert list(r["toks"]) == list(single["toks"])
        assert np.array_equal(r["logits"].view(np.uint32), single["logits"].view(np.uint32))
        assert list(r["modes"]) == [1, 1, 1, 1]
        assert a == sa and b == sb                 # each context's KV cache was gathered from its own shards
