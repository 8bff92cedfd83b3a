"""CPU, 2 ranks over gloo: attach_lora / detach_lora between decode steps under tensor parallelism, on the CPU stand-in of the device
layer, launched like tests/test_multi_context_tp.py.  A merge rewrites the whole weight on every rank, so the row shards cut from the old
weights must be cut again: every rank's tokens and logit bits must be the single-rank run's, for a cached f16 and an uncached f32
adapter attached, detached and attached again."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
from tests.lora_mock import HAVE_LIBS  # noqa: E402

WORKER = r'''
import ctypes as C, os, sys, numpy as np
sys.path.insert(0, sys.argv[1])
import torch, torch.distributed as dist
from fastllama_b200.model import Model, QuietLogger
rank, world, mock, path, lora_f16, lora_f32, out = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), *sys.argv[2:7]
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
    _fields_ = [(n, C.c_uint64) for n in ("weight_mirror_bytes", "shard_bytes", "mirror_bytes", "kv_gathers")]
mirrors = []
def weight_mirrors():
    x = Mem(); g.ggml_b200_get_memory(C.byref(x)); mirrors.append(x.weight_mirror_bytes)
so = os.path.join(mock, "pyfastllama.so")
m = Model(path, num_threads=2, n_ctx=64, n_batch=8, logger=QuietLogger(), library_path=so)
toks, logits, rets = [], [], []
def gen(n):
    t = []
    assert m.generate(lambda s: t.append(s), num_tokens=n, temp=0.0, top_k=1, top_p=1.0, repeat_penalty=1.0)
    toks.extend(t); logits.append(m.get_logits_array())
assert m.ingest("Adapters under tensor parallelism.")
gen(3); weight_mirrors()
rets.append(m.attach_lora(lora_f16)); gen(3); weight_mirrors()
rets.append(m.detach_lora()); gen(2)
rets.append(m.attach_lora(lora_f32)); gen(3)
rets.append(m.detach_lora()); gen(2)
m.close()
np.savez(out + f".rank{rank}.npz", toks=np.array(toks), logits=np.concatenate(logits), rets=np.array(rets), mirrors=np.array(mirrors))
'''

DIMS = dict(n_vocab=512, n_embd=256, n_mult=256, n_head=4, n_layer=3)


@pytest.fixture(scope="module")
def mock():
    """The CPU stand-in of the device layer with the f16 LoRA ops and fl_dev_tp_unshard (tests/lora_mock.py)."""
    import shutil

    from tests.lora_mock import mock_dir

    d = mock_dir(tp=True)
    yield d
    shutil.rmtree(d, ignore_errors=True)


def launch(tmp_path, mock, args, world):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    out = str(tmp_path / f"w{world}")
    procs = []
    for r in range(world):
        e = dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT="29671", OMP_NUM_THREADS="2",
                 FL_MOCK_SESSION=f"{os.getpid()}_lora_{world}")
        procs.append(subprocess.Popen([sys.executable, str(script), ROOT, mock] + args + [out], env=e, stdout=subprocess.DEVNULL,
                                      stderr=subprocess.PIPE))
    errs = [p.communicate(timeout=900)[1] for p in procs]
    for p, err in zip(procs, errs):
        assert p.returncode == 0, err.decode()[-3000:]
    return [np.load(out + f".rank{r}.npz") for r in range(world)]


@pytest.mark.skipif(not HAVE_LIBS, reason="needs the built host libraries and the drop-in pyfastllama.so")
def test_attach_and_detach_under_tensor_parallelism_match_single_rank(tmp_path, mock):
    from fastllama_b200.ggjt import Q4_0, write_synthetic_numpy
    from oracle.pyoracle import Oracle
    from tests.lora_files import write_adapter

    orc = Oracle()
    path = str(tmp_path / "toy.bin")
    write_synthetic_numpy(path, Q4_0, seed=8, std=0.01, quantize=lambda w, t: orc.quantize_q4(w, t), **DIMS)
    f16, f32 = str(tmp_path / "lora_f16.bin"), str(tmp_path / "lora_f32.bin")
    write_adapter(f16, "cached_f16", 256, 768, (0, 1, 2), seed=1)
    write_adapter(f32, "uncached_f32", 256, 768, (0, 2), seed=2)
    single, = launch(tmp_path, mock, [path, f16, f32], 1)
    assert list(single["rets"]) == [True] * 4
    n = len(single["logits"]) // 5
    parts = single["logits"].reshape(5, n)
    assert not np.array_equal(parts[0], parts[1]) and not np.array_equal(parts[2], parts[3]), "the adapters must change the logits"
    for r in launch(tmp_path, mock, [path, f16, f32], 2):
        assert list(r["rets"]) == list(single["rets"])
        assert list(r["toks"]) == list(single["toks"])
        assert np.array_equal(r["logits"].view(np.uint32), single["logits"].view(np.uint32))
        # the shards alone until the attach; the merge mirrors the weights it rewrites on every rank
        assert r["mirrors"][0] == 0 and r["mirrors"][1] > 0, r["mirrors"]
