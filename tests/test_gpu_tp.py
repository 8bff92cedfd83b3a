"""GPU (needs >= 2 GPUs on the box; skipped otherwise): tensor-parallel decode (row-split matrices, activation vectors gathered over
NVLink as dataflow vectors inside the token kernel) against the single-GPU run: the same tokens and the same logit BITS.
Launched like bench.py is: one process per GPU, rendezvous on 127.0.0.1."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import ctypes as C, os, sys, numpy as np
sys.path.insert(0, sys.argv[1])
rank, world, path, out = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), sys.argv[2], sys.argv[3]
os.environ["FASTLLAMA_DEVICE"] = str(rank)
from fastllama_b200.cuda_abi import FlCuda
from fastllama_b200.model import Model, QuietLogger
fl = FlCuda()
if world > 1:
    import torch, torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    idbuf = torch.zeros(128, dtype=torch.uint8, device="cuda")
    if rank == 0:
        raw = C.create_string_buffer(128); fl.check(fl.lib.fl_comm_unique_id(raw))
        idbuf = torch.tensor(list(raw.raw), dtype=torch.uint8, device="cuda")
    dist.broadcast(idbuf, 0)
    fl.check(fl.lib.fl_comm_init(rank, world, idbuf.cpu().numpy().tobytes()))
scenario = sys.argv[4] if len(sys.argv) > 4 else "decode"
m = Model(path, num_threads=2, n_ctx=64 if scenario == "decode" else 128, n_batch=8, logger=QuietLogger())
m.ingest("Tensor parallel decode over two ranks.")
toks = []
gen = lambda n: m.generate(lambda s: toks.append(s), num_tokens=n, temp=0.0, top_k=1, top_p=1.0, repeat_penalty=1.0)
if scenario == "reingest":       # sharded decode, then a replicated multi-token eval and a state file: both need the KV gather
    gen(5)
    m.ingest(" And a second prompt that attends to all of it.")
    gen(4)
    assert m.save_state(out + f".rank{rank}.state")
    gen(3)
    first = list(toks[-3:])
    assert m.load_state(out + f".rank{rank}.state")
    gen(3)
    assert list(toks[-3:]) == first, (toks[-3:], first)
else:
    gen(16)
np.savez(out + f".rank{rank}.npz", toks=np.array(toks), logits=m.get_logits_array())
m.close()
'''


def _n_gpus():
    try:
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True, timeout=20).stdout
        return sum(1 for ln in out.splitlines() if ln.startswith("GPU "))
    except Exception:
        return 0


@pytest.mark.skipif(_n_gpus() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("scenario", ["decode", "reingest"])
def test_tp2_matches_single_gpu(tmp_path, scenario):
    from fastllama_b200.ggjt import Q4_0, write_synthetic_numpy
    from oracle.pyoracle import Oracle

    orc = Oracle()
    path = str(tmp_path / "toy.bin")
    write_synthetic_numpy(path, Q4_0, n_vocab=512, n_embd=512, n_mult=64, n_head=4, n_layer=3, seed=5, std=0.01, quantize=lambda w, t: orc.quantize_q4(w, t))
    script = tmp_path / "worker.py"
    script.write_text(WORKER)

    def launch(world, tag):
        procs = []
        for r in range(world):
            env = dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), LOCAL_RANK=str(r), MASTER_ADDR="127.0.0.1", MASTER_PORT="29641")
            procs.append(subprocess.Popen([sys.executable, str(script), ROOT, path, str(tmp_path / tag), scenario], env=env, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE))
        for p in procs:
            _, err = p.communicate(timeout=300)
            assert p.returncode == 0, err.decode()[-2000:]
        return [np.load(str(tmp_path / tag) + f".rank{r}.npz") for r in range(world)]

    single = launch(1, "w1")[0]
    tp = launch(2, "w2")
    for r in tp:
        assert list(r["toks"]) == list(single["toks"])
        assert np.array_equal(r["logits"].view(np.uint32), single["logits"].view(np.uint32))
