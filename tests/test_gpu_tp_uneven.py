"""GPU: tensor parallelism at world sizes that do not divide the model's shapes, and an odd vocabulary on one GPU.

On one GPU: fl_dev_tp_unshard_v against numpy (worlds 2 to 8, uneven counts, residual on and off, the float4 and the scalar path), and a
2-layer 7B-shaped q4_0 file with a 32001-token vocabulary, which decodes through the token kernel (decode mode 2; its last LM-head row
runs as a row pair of its own) with the logit bits of the reference-order node-by-node executor (FASTLLAMA_B200_NO_FUSED=1) over 16
greedy steps.
With more GPUs (each test skipped when the box has fewer than it needs), launched like tests/test_gpu_tp.py: a toy model with 5 heads of
128 and a 515-token vocabulary at worlds 2 and 3, a 2-layer 7B-shaped model at world 3 and a 2-layer 30B-shaped model (52 heads) at world
8, each against the single-GPU run: the same tokens and logit bits, every decode step through the token program and every multi-token
eval through the prompt plan, with no device copy of the model."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _n_gpus():
    try:
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True, timeout=20).stdout
        return sum(1 for ln in out.splitlines() if ln.startswith("GPU "))
    except Exception:
        return 0


@pytest.fixture(scope="module")
def fl():
    from fastllama_b200.cuda_abi import FlCuda
    return FlCuda()


def _unshard_cases():
    rng = np.random.default_rng(42)
    for world in range(2, 9):
        for N in (1, 2, 7, 33, 129):
            for kind in ("vector", "mixed", "scalar"):
                if kind == "vector":          # every count and first a multiple of 4: float4 for every rank
                    counts = (rng.integers(1, 40, size=world) * 4).tolist()
                elif kind == "mixed":         # ranks a..b start or end off a float4 boundary (the scalar path), the others take float4
                    counts = (rng.integers(1, 40, size=world) * 4).tolist()
                    a, b = world // 2 - 1, world - 2
                    counts[a] += 1
                    counts[b] += 3
                else:
                    counts = rng.integers(1, 160, size=world).tolist()
                yield world, N, kind, counts


@pytest.mark.parametrize("world,N,kind,counts", list(_unshard_cases()), ids=lambda v: str(v) if not isinstance(v, list) else "c")
def test_unshard_v_against_numpy(fl, world, N, kind, counts):
    f = fl.fn("fl_dev_tp_unshard_v")
    rng = np.random.default_rng(world * 1000 + N)
    stride, n = max(counts), sum(counts)
    first = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int32).tolist()
    g = rng.standard_normal((world, N * stride)).astype(np.float32)
    want = np.concatenate([g[r, :N * c].reshape(N, c) for r, c in enumerate(counts)], axis=1)
    res = rng.standard_normal((N, n)).astype(np.float32)
    F, Cn = (C.c_int * world)(*first), (C.c_int * world)(*counts)
    # one float of offset on every buffer: no rank may take the float4 path
    off = 4 if kind == "scalar" else 0
    dG, dR, dD = fl.alloc(g.nbytes + 16), fl.alloc(res.nbytes + 16), fl.alloc(res.nbytes + 16)
    try:
        fl.check(fl.lib.fl_h2d(dG + off, g.ctypes.data, g.nbytes))
        fl.check(fl.lib.fl_h2d(dR + off, res.ctypes.data, res.nbytes))
        fl.check(fl.lib.fl_dev_memset(dD, 0xFF, res.nbytes + 16))
        fl.check(f(dG + off, world, N, stride, F, Cn, None, dD + off))
        got = np.empty_like(res)
        fl.check(fl.lib.fl_d2h(got.ctypes.data, dD + off, got.nbytes))
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
        fl.check(f(dG + off, world, N, stride, F, Cn, dR + off, dD + off))
        fl.check(fl.lib.fl_d2h(got.ctypes.data, dD + off, got.nbytes))
        assert np.array_equal(got.view(np.uint32), (want + res).view(np.uint32))
        fl.check(f(dG + off, world, N, stride, F, Cn, dR + off, dR + off))     # in place on the residual, as after wo / w2
        fl.check(fl.lib.fl_d2h(got.ctypes.data, dR + off, got.nbytes))
        assert np.array_equal(got.view(np.uint32), (want + res).view(np.uint32))
    finally:
        for d in (dG, dR, dD):
            fl.free(d)


WORKER = r'''
import ctypes as C, os, sys, numpy as np
sys.path.insert(0, sys.argv[1])
rank, world, path, out, scenario = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), sys.argv[2], sys.argv[3], sys.argv[4]
os.environ["FASTLLAMA_DEVICE"] = str(rank)
from fastllama_b200.build import lib_path
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
g = C.CDLL(lib_path("libggml_b200.so"))
class Mem(C.Structure):
    _fields_ = [("weight_mirror_bytes", C.c_uint64), ("shard_bytes", C.c_uint64), ("mirror_bytes", C.c_uint64), ("kv_gathers", C.c_uint64)]
def mem():
    m = Mem(); g.ggml_b200_get_memory(C.byref(m)); return np.array([m.weight_mirror_bytes, m.shard_bytes, m.mirror_bytes, m.kv_gathers], dtype=np.uint64)
greedy = dict(temp=0.0, top_k=1, top_p=1.0, repeat_penalty=1.0)
toks, logits, pmodes, dmodes, mems = [], [], [], [], []
def step():
    logits.append(m.get_logits_array()); pmodes.append(g.ggml_b200_prompt_mode()); dmodes.append(g.ggml_b200_decode_mode()); mems.append(mem())
def gen(n):
    for _ in range(n):
        assert m.generate(lambda s: toks.append(s), num_tokens=1, **greedy); step()
m = Model(path, num_threads=2, n_ctx=128, n_batch=8, logger=QuietLogger())
assert m.ingest("Tensor parallel decode at an uneven world size."); step()
if scenario == "decode":
    gen(16)
else:                    # sharded decode steps, a second prompt through the prompt plan, a state file from the gathered cache
    gen(5)
    assert m.ingest(" And a second prompt that attends to all of it."); step()
    gen(4)
    assert m.save_state(out + f".rank{rank}.state")
    gen(3)
    first = list(toks[-3:])
    assert m.load_state(out + f".rank{rank}.state")
    gen(3)
    assert list(toks[-3:]) == first, (toks[-3:], first)
m.close()
np.savez(out + f".rank{rank}.npz", toks=np.array(toks), logits=np.stack(logits), pmodes=np.array(pmodes), dmodes=np.array(dmodes),
         mems=np.array(mems, dtype=np.uint64).reshape(-1, 4))
'''


def _launch(tmp_path, path, world, tag, scenario, port, env=None):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    procs = []
    for r in range(world):
        e = dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), LOCAL_RANK=str(r), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), **(env or {}))
        procs.append(subprocess.Popen([sys.executable, str(script), ROOT, path, str(tmp_path / tag), scenario], env=e, stdout=subprocess.DEVNULL,
                                      stderr=subprocess.PIPE))
    errs = [p.communicate(timeout=1200)[1] for p in procs]
    for p, err in zip(procs, errs):
        assert p.returncode == 0, err.decode()[-3000:]
    return [np.load(str(tmp_path / tag) + f".rank{r}.npz") for r in range(world)]


def _same(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _check(single, tp, matrix_bytes, world):
    """tp: every rank's results against the single-GPU run's; matrix_bytes: the model's matrix bytes (each rank holds about 1 / world)"""
    for r, res in enumerate(tp):
        assert list(res["toks"]) == list(single["toks"])
        assert len(res["logits"]) == len(single["logits"])
        for i, (a, b) in enumerate(zip(res["logits"], single["logits"])):
            assert _same(a, b), (r, i)
        for i, d in enumerate(single["dmodes"]):
            if d == 2:
                assert res["dmodes"][i] == 2, (r, i, res["dmodes"])              # every decode step: the token program
            else:
                assert res["dmodes"][i] == 0 and res["pmodes"][i] == 1, (r, i, res["pmodes"])   # every multi-token eval: the prompt plan
        for m in res["mems"]:
            assert int(m[0]) == 0                                                # no device copy of any weight
            assert 0 < int(m[1]) <= matrix_bytes / world * 1.25 + int(single["table_and_norms"])


def _toy(tmp_path):
    from fastllama_b200.ggjt import Q4_0, write_synthetic_numpy
    from oracle.pyoracle import Oracle

    orc = Oracle()
    path = str(tmp_path / "toy.bin")
    write_synthetic_numpy(path, Q4_0, n_vocab=515, n_embd=640, n_mult=256, n_head=5, n_layer=2, seed=7, std=0.01,
                          quantize=lambda w, t: orc.quantize_q4(w, t))
    return path, _sizes(515, 640, 1792, 2)


def _sizes(n_vocab, n_embd, n_ff, n_layer):
    q4 = lambda n: n // 32 * 20
    return q4(n_layer * (4 * n_embd * n_embd + 3 * n_embd * n_ff) + n_vocab * n_embd), q4(n_vocab * n_embd) + (2 * n_layer + 1) * n_embd * 4


def _with_sizes(res, table_and_norms):
    d = dict(res)
    d["table_and_norms"] = np.int64(table_and_norms)
    return d


def test_odd_vocabulary_7b_decodes_through_the_token_kernel_with_the_reference_order_bits(tmp_path):
    from fastllama_b200.ggjt import Q4_0, write_synthetic_gpu

    path = str(tmp_path / "7b_32001.bin")
    write_synthetic_gpu(path, size="7B", wtype=Q4_0, seed=3, std=0.02, n_vocab=32001, n_layer=2)
    ours = _launch(tmp_path, path, 1, "fused", "decode", 29681)[0]
    ref = _launch(tmp_path, path, 1, "nodes", "decode", 29681, env={"FASTLLAMA_B200_NO_FUSED": "1"})[0]
    assert list(ours["dmodes"][2:]) == [2] * 15                                   # after the ingest and generate()'s first eval
    assert set(ref["dmodes"].tolist()) == {0}
    assert list(ours["toks"]) == list(ref["toks"]) and len(ours["toks"]) == 16
    for i, (a, b) in enumerate(zip(ours["logits"], ref["logits"])):
        assert _same(a, b) and a.size == 32001, i


@pytest.mark.skipif(_n_gpus() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("scenario", ["decode", "state"])
def test_tp2_uneven_toy_matches_single_gpu(tmp_path, scenario):
    path, (mats, rest) = _toy(tmp_path)
    single = _with_sizes(_launch(tmp_path, path, 1, "w1", scenario, 29682)[0], rest)
    _check(single, _launch(tmp_path, path, 2, "w2", scenario, 29682), mats, 2)


@pytest.mark.skipif(_n_gpus() < 3, reason="needs 3 GPUs")
@pytest.mark.parametrize("scenario", ["decode", "state"])
def test_tp3_uneven_toy_matches_single_gpu(tmp_path, scenario):
    path, (mats, rest) = _toy(tmp_path)
    single = _with_sizes(_launch(tmp_path, path, 1, "w1", scenario, 29683)[0], rest)
    _check(single, _launch(tmp_path, path, 3, "w3", scenario, 29683), mats, 3)


@pytest.mark.skipif(_n_gpus() < 3, reason="needs 3 GPUs")
def test_tp3_7b_shapes_match_single_gpu(tmp_path):
    from fastllama_b200.ggjt import Q4_0, write_synthetic_gpu

    path = str(tmp_path / "7b_2layer.bin")
    write_synthetic_gpu(path, size="7B", wtype=Q4_0, seed=0, std=0.02, n_layer=2)
    mats, rest = _sizes(32000, 4096, 11008, 2)
    single = _with_sizes(_launch(tmp_path, path, 1, "w1", "state", 29684)[0], rest)
    _check(single, _launch(tmp_path, path, 3, "w3", "state", 29684), mats, 3)


@pytest.mark.skipif(_n_gpus() < 8, reason="needs 8 GPUs")
def test_tp8_30b_shapes_match_single_gpu(tmp_path):
    """52 heads on 8 GPUs: 7, 7, 7, 7, 6, 6, 6, 6"""
    from fastllama_b200.ggjt import Q4_0, write_synthetic_gpu

    path = str(tmp_path / "30b_2layer.bin")
    write_synthetic_gpu(path, size="30B", wtype=Q4_0, seed=0, std=0.02, n_layer=2)
    mats, rest = _sizes(32000, 6656, 17920, 2)
    single = _with_sizes(_launch(tmp_path, path, 1, "w1", "state", 29685)[0], rest)
    _check(single, _launch(tmp_path, path, 8, "w8", "state", 29685), mats, 8)
