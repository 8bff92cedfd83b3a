"""GPU: the tensor-parallel prompt plan.

On one GPU: the premise of its bit equality -- a row slice of the quantised GEMM gives the same bits as those rows of the whole GEMM,
for the kernel the executor picks (impl 0: the reference-order kernel below 16 columns, the wgmma GEMM from 16 on, whose column tile
depends on M) and for the reference-order kernel at every N -- and fl_dev_tp_unshard against numpy.

With >= 2 GPUs (skipped otherwise, like tests/test_gpu_tp.py): the scenarios of tests/test_tp_ingest.py on the toy model, and a 2-layer
7B-shaped q4_0 file with the full matrices and a prompt of 2 x 128 + 1 tokens at n_batch = 128, so the wgmma GEMM runs on realistic tile
counts.  Tokens and logit bits of the single-GPU run, no weight mirror, and each rank holds its rows of the matrices plus the embedding
table and the norms."""
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


def _random_q4(rng, t, M, K):
    """M rows of K/32 random q4 blocks (fp32 scale [and min], 16 nibble bytes), as the old ggml layout stores them"""
    nb = K // 32
    qs = rng.integers(0, 256, size=(M, nb, 16), dtype=np.uint8)
    d = (rng.random((M, nb, 1), dtype=np.float32) * 0.02 + 1e-3).view(np.uint8).reshape(M, nb, 4)
    parts = [d] if t == 2 else [d, (rng.standard_normal((M, nb, 1), dtype=np.float32) * 0.05).view(np.uint8).reshape(M, nb, 4)]
    return np.ascontiguousarray(np.concatenate(parts + [qs], axis=2).reshape(M, -1))


@pytest.mark.parametrize("t", [2, 3], ids=["q4_0", "q4_1"])
@pytest.mark.parametrize("M,K", [(4096, 4096), (11008, 4096), (4096, 11008), (32000, 4096)])
def test_gemm_row_slices_carry_the_full_gemm_bits(fl, t, M, K):
    """Rows [r * M/p, (r + 1) * M/p) computed on their own, for p = 2, 4, 8, written with the full result's row stride (as the prompt
    plan writes them), equal the full GEMM bit for bit: impl 0 (what the executor passes) and impl 8 (reference order)."""
    rng = np.random.default_rng(M + K + t)
    w = _random_q4(rng, t, M, K)
    wrs = w.shape[1]
    dW = fl.to_device(w)
    Nmax = 129
    x = (rng.standard_normal((Nmax, K)) * 0.5).astype(np.float32)
    dX = fl.to_device(x)
    dY = fl.alloc(Nmax * (K // 32) * 40)
    dFull, dParts = fl.alloc(Nmax * M * 4), fl.alloc(Nmax * M * 4)
    try:
        for N in (1, 8, 15, 16, 48, 128, 129):
            fl.check(fl.lib.fl_dev_quantize_q8_0(dX, K * 4, dY, K, N))
            for impl in (0, 8):
                fl.check(fl.lib.fl_dev_mul_mat_q(t, dW, wrs, M, K, dY, N, dFull, M, impl))
                full = fl.to_host(dFull, (N, M), np.float32)
                assert np.isfinite(full).all()
                for p in (2, 4, 8):
                    ms = M // p
                    fl.check(fl.lib.fl_dev_memset(dParts, 0xFF, N * M * 4))
                    for r in range(p):
                        fl.check(fl.lib.fl_dev_mul_mat_q(t, dW + r * ms * wrs, wrs, ms, K, dY, N, dParts + r * ms * 4, M, impl))
                    parts = fl.to_host(dParts, (N, M), np.float32)
                    bad = np.flatnonzero(parts.view(np.uint32) != full.view(np.uint32))
                    assert bad.size == 0, (N, impl, p, bad.size, bad[:4])
    finally:
        for d in (dW, dX, dY, dFull, dParts):
            fl.free(d)


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("N,nl", [(1, 512), (7, 1376), (33, 6), (128, 4000), (129, 344)])
def test_unshard_against_numpy(fl, world, N, nl):
    rng = np.random.default_rng(world * 1000 + N)
    f = fl.fn("fl_dev_tp_unshard")
    g = rng.standard_normal((world, N, nl)).astype(np.float32)
    res = rng.standard_normal((N, world * nl)).astype(np.float32)
    want = g.transpose(1, 0, 2).reshape(N, world * nl)
    dG, dR, dD = fl.to_device(g), fl.to_device(res), fl.alloc(res.nbytes)
    try:
        fl.check(f(dG, world, N, nl, None, dD))
        assert np.array_equal(fl.to_host(dD, want.shape, np.float32).view(np.uint32), want.view(np.uint32))
        fl.check(f(dG, world, N, nl, dR, dD))
        assert np.array_equal(fl.to_host(dD, want.shape, np.float32).view(np.uint32), (want + res).view(np.uint32))
        fl.check(f(dG, world, N, nl, dR, dR))                                   # in place on the residual, as after wo / w2
        assert np.array_equal(fl.to_host(dR, want.shape, np.float32).view(np.uint32), (want + res).view(np.uint32))
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
toks, logits, modes, gathers = [], [], [], []
def text(n_chars):          # every character one token with the synthetic vocabulary, plus BOS and the bridge's leading space
    return ("tensor parallel prompt ingest on weight shards " * 20)[:n_chars]
if scenario == "toy":
    n_batch = 8
    m = Model(path, num_threads=2, n_ctx=128, n_batch=n_batch, logger=QuietLogger())
    gen = lambda n: m.generate(lambda s: toks.append(s), num_tokens=n, temp=0.0, top_k=1, top_p=1.0, repeat_penalty=1.0)
    def step():
        gathers.append(int(mem()[3])); logits.append(m.get_logits_array())
    assert m.ingest(text(41)); modes.append(g.ggml_b200_prompt_mode()); step()
    gen(4); step()
    assert m.ingest(text(23)); modes.append(g.ggml_b200_prompt_mode()); step()
    gen(4); step()
    assert m.save_state(out + f".rank{rank}.state"); step()
    gen(3)
    first = list(toks[-3:])
    assert m.load_state(out + f".rank{rank}.state")
    gen(3); step()
    assert list(toks[-3:]) == first, (toks[-3:], first)
    m.close()
    m = Model(path, num_threads=2, n_ctx=128, n_batch=n_batch, should_get_all_logits=True, embedding_eval_enabled=True, logger=QuietLogger())
    assert m.ingest(text(41)); modes.append(g.ggml_b200_prompt_mode())
    logits.append(m.get_logits_array()[-512:]); logits.append(m.get_logits_array()[:512])
    emb = np.array(m.get_embeddings(), dtype=np.float32)
    ppl = m.perplexity(text(60))
else:
    m = Model(path, num_threads=2, n_ctx=512, n_batch=128, embedding_eval_enabled=True, logger=QuietLogger())
    gen = lambda n: m.generate(lambda s: toks.append(s), num_tokens=n, temp=0.0, top_k=1, top_p=1.0, repeat_penalty=1.0)
    assert m.ingest(text(2 * 128 + 1 - 2)); modes.append(g.ggml_b200_prompt_mode())
    logits.append(m.get_logits_array()); gathers.append(int(mem()[3]))
    gen(6); logits.append(m.get_logits_array())
    emb = np.array(m.get_embeddings(), dtype=np.float32)
    ppl = 0.0
memory = mem()
m.close()
np.savez(out + f".rank{rank}.npz", toks=np.array(toks), logits=np.stack(logits), modes=np.array(modes), gathers=np.array(gathers), emb=emb,
         ppl=np.float64(ppl), mem=memory)
'''


def _launch(tmp_path, path, world, tag, scenario, port):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    procs = []
    for r in range(world):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), LOCAL_RANK=str(r), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        procs.append(subprocess.Popen([sys.executable, str(script), ROOT, path, str(tmp_path / tag), scenario], env=env, stdout=subprocess.DEVNULL,
                                      stderr=subprocess.PIPE))
    errs = [p.communicate(timeout=900)[1] for p in procs]
    for p, err in zip(procs, errs):
        assert p.returncode == 0, err.decode()[-3000:]
    return [np.load(str(tmp_path / tag) + f".rank{r}.npz") for r in range(world)]


def _q4_bytes(n_vocab, n_embd, n_ff, n_layer):
    """(matrix bytes, embedding table bytes, norm bytes) of a q4_0 model"""
    q4 = lambda n: n // 32 * 20
    return q4(n_layer * (4 * n_embd * n_embd + 3 * n_embd * n_ff) + n_vocab * n_embd), q4(n_vocab * n_embd), (2 * n_layer + 1) * n_embd * 4


def _check(single, tp, world, sizes):
    mats, table, norms = sizes
    for r in tp:
        assert list(r["toks"]) == list(single["toks"])
        assert len(r["logits"]) == len(single["logits"])
        for a, b in zip(r["logits"], single["logits"]):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
        assert np.array_equal(r["emb"].view(np.uint32), single["emb"].view(np.uint32))
        assert float(r["ppl"]) == float(single["ppl"])
        assert all(int(x) == 1 for x in r["modes"])
        assert int(r["mem"][0]) == 0                                            # no device copy of any weight
        assert 0 < int(r["mem"][1]) <= mats // world + table + norms


@pytest.mark.skipif(_n_gpus() < 2, reason="needs 2 GPUs")
def test_tp2_prompt_plan_toy_matches_single_gpu(tmp_path):
    from fastllama_b200.ggjt import Q4_0, n_ff, write_synthetic_numpy
    from oracle.pyoracle import Oracle

    orc = Oracle()
    path = str(tmp_path / "toy.bin")
    write_synthetic_numpy(path, Q4_0, n_vocab=512, n_embd=512, n_mult=64, n_head=4, n_layer=3, seed=5, std=0.01, quantize=lambda w, t: orc.quantize_q4(w, t))
    single = _launch(tmp_path, path, 1, "w1", "toy", 29661)[0]
    tp = _launch(tmp_path, path, 2, "w2", "toy", 29661)
    _check(single, tp, 2, _q4_bytes(512, 512, n_ff(512, 64), 3))
    for r in tp:
        g = list(r["gathers"])                                                 # after: ingest, decode, ingest, decode, save_state
        assert g[0] == g[1] == g[2] == g[3] and g[4] == g[3] + 1, g


@pytest.mark.skipif(_n_gpus() < 2, reason="needs 2 GPUs")
def test_tp2_prompt_plan_7b_shapes_matches_single_gpu(tmp_path):
    from fastllama_b200.ggjt import Q4_0, n_ff, write_synthetic_gpu

    path = str(tmp_path / "7b_2layer.bin")
    write_synthetic_gpu(path, size="7B", wtype=Q4_0, seed=0, std=0.02, n_layer=2)
    single = _launch(tmp_path, path, 1, "w1", "7b", 29662)[0]
    tp = _launch(tmp_path, path, 2, "w2", "7b", 29662)
    _check(single, tp, 2, _q4_bytes(32000, 4096, n_ff(4096, 256), 2))
    for r in tp:
        assert int(r["gathers"][0]) == 0
