"""tools/time_tp_ingest.py -- prompt-ingest throughput and device memory of tensor-parallel ranks (the prompt plan of ggml_b200.cpp).

Writes a synthetic LLaMA-7B q4_0 file (once, to a temporary directory unless --model is given), then for world = 1, 2, 4 and 8 (as
many as there are GPUs) and for the replicated executor at world = 2 (FASTLLAMA_B200_TP_INGEST=replicated) launches one process per
GPU.  Each rank ingests a warm-up prompt, resets, then ingests a prompt of 2 x 128 + 1 tokens at n_batch = 128 (two 128-token evals;
the last token is left to the first generate call) and reports:
  - prompt tokens/s from the library's CUDA-event counters (ggml_b200_get_stats: device time of the timed evals), and wall clock;
  - device memory in use on its GPU (cudaMemGetInfo, which includes the CUDA and NCCL contexts) and ggml_b200_get_memory.
Prints one JSON line per configuration.  Asserts nothing about speed.

    python tools/time_tp_ingest.py [--model PATH] [--worlds 1,2] [--evals 2]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


class _Stats(C.Structure):
    _fields_ = [("n_evals", C.c_uint64), ("last_eval_device_us", C.c_double), ("total_device_us", C.c_double), ("launches", C.c_uint64),
                ("graph_replays", C.c_uint64)]


class _Mem(C.Structure):
    _fields_ = [("weight_mirror_bytes", C.c_uint64), ("shard_bytes", C.c_uint64), ("mirror_bytes", C.c_uint64), ("kv_gathers", C.c_uint64)]


def _text(n_chars: int, salt: int = 0) -> str:
    """ASCII text; with the synthetic vocabulary every character is one token, plus BOS and the bridge's leading space"""
    words = "the tensor parallel prompt plan runs every multi token eval on the weight shards of its rank and gathers activations".split()
    out, i = [], salt
    while sum(len(w) + 1 for w in out) < n_chars + 1:
        out.append(words[i % len(words)])
        i += 1
    return " ".join(out)[:n_chars]


def worker(path: str, out: str, evals: int) -> None:
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    os.environ["FASTLLAMA_DEVICE"] = str(rank)
    import torch

    from fastllama_b200.build import lib_path
    from fastllama_b200.cuda_abi import FlCuda
    from fastllama_b200.model import Model, QuietLogger

    fl = FlCuda()
    torch.cuda.set_device(rank)
    dist = None
    if world > 1:
        import torch.distributed as dist

        dist.init_process_group("nccl", rank=rank, world_size=world)
        idbuf = torch.zeros(128, dtype=torch.uint8, device="cuda")
        if rank == 0:
            raw = C.create_string_buffer(128)
            fl.check(fl.lib.fl_comm_unique_id(raw))
            idbuf = torch.tensor(list(raw.raw), dtype=torch.uint8, device="cuda")
        dist.broadcast(idbuf, 0)
        fl.check(fl.lib.fl_comm_init(rank, world, idbuf.cpu().numpy().tobytes()))
    g = C.CDLL(lib_path("libggml_b200.so"))
    g.ggml_b200_get_stats.argtypes = [C.POINTER(_Stats)]
    g.ggml_b200_get_memory.argtypes = [C.POINTER(_Mem)]

    def stats():
        s = _Stats()
        g.ggml_b200_get_stats(C.byref(s))
        return s

    m = Model(path, num_threads=1, n_ctx=512, n_batch=128, logger=QuietLogger(), library_path=lib_path("pyfastllama.so"))
    assert m.ingest(_text(128 + 1 - 2))                      # shard / mirror uploads and first launches, untimed
    m.generate(lambda s: None, num_tokens=1, temp=0.0, top_k=1, top_p=1.0, repeat_penalty=1.0)
    assert m.reset()
    if dist:
        dist.barrier()
    fl.check(fl.lib.fl_sync())
    s0 = stats()
    t0 = time.perf_counter()
    assert m.ingest(_text(evals * 128 + 1 - 2, salt=3))
    fl.check(fl.lib.fl_sync())
    t1 = time.perf_counter()
    s1 = stats()
    mem = _Mem()
    g.ggml_b200_get_memory(C.byref(mem))
    free, total = torch.cuda.mem_get_info(rank)
    n_evals = int(s1.n_evals - s0.n_evals)
    dev_s = (s1.total_device_us - s0.total_device_us) * 1e-6
    res = {"rank": rank, "world": world, "prompt_mode": int(g.ggml_b200_prompt_mode()), "evals": n_evals, "tokens": n_evals * 128,
           "device_s": dev_s, "wall_s": t1 - t0, "tokens_per_s_device": n_evals * 128 / dev_s if dev_s else 0.0,
           "tokens_per_s_wall": n_evals * 128 / (t1 - t0), "device_used_bytes": int(total - free),
           "weight_mirror_bytes": int(mem.weight_mirror_bytes), "shard_bytes": int(mem.shard_bytes), "mirror_bytes": int(mem.mirror_bytes),
           "kv_gathers": int(mem.kv_gathers), "gpu": torch.cuda.get_device_name(rank)}
    m.close()
    with open(out, "w") as f:
        json.dump(res, f)
    if dist:
        dist.destroy_process_group()


def run(path: str, world: int, evals: int, env: dict, tmp: str, port: int) -> list:
    procs, outs = [], []
    for r in range(world):
        out = os.path.join(tmp, f"w{world}_r{r}_{port}.json")
        outs.append(out)
        e = dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), LOCAL_RANK=str(r), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), **env)
        procs.append(subprocess.Popen([sys.executable, os.path.abspath(__file__), "--_worker", path, out, str(evals)], env=e, stdout=sys.stderr))
    rcs = [p.wait(timeout=1800) for p in procs]
    if any(rcs):
        raise SystemExit(f"world {world} {env}: worker exit codes {rcs}")
    return [json.load(open(o)) for o in outs]


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "--_worker":
        worker(sys.argv[2], sys.argv[3], int(sys.argv[4]))
        return
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default=None, help="an existing LLaMA-7B-shaped q4_0 file (default: write a synthetic one to a temporary directory)")
    ap.add_argument("--worlds", default=None, help="comma-separated world sizes (default: 1, 2, 4, 8 up to the number of GPUs)")
    ap.add_argument("--evals", type=int, default=2, help="timed 128-token evals (the prompt is evals x 128 + 1 tokens, n_ctx 512)")
    args = ap.parse_args()
    import torch

    n_gpus = torch.cuda.device_count()
    worlds = [int(w) for w in args.worlds.split(",")] if args.worlds else [w for w in (1, 2, 4, 8) if w <= n_gpus]
    with tempfile.TemporaryDirectory() as tmp:
        path = args.model
        if not path:
            path = os.path.join(tmp, "synth_7B_q4_0.bin")
            t0 = time.time()
            code = ("import sys; sys.path.insert(0, %r); from fastllama_b200.ggjt import write_synthetic_gpu; "
                    "write_synthetic_gpu(%r, size='7B', wtype=2, seed=0, std=0.02)" % (ROOT, path))
            subprocess.run([sys.executable, "-c", code], check=True, stdout=sys.stderr)
            print(f"[time_tp_ingest] wrote {os.path.getsize(path) / 1e9:.2f} GB in {time.time() - t0:.0f} s", file=sys.stderr)
        configs = [(w, {}) for w in worlds]
        if 2 in worlds:
            configs.insert(worlds.index(2) + 1, (2, {"FASTLLAMA_B200_TP_INGEST": "replicated"}))
        for i, (world, env) in enumerate(configs):
            ranks = run(path, world, args.evals, env, tmp, 29700 + i)
            slowest = min(r["tokens_per_s_device"] for r in ranks)
            print(json.dumps({"world": world, "path": "replicated executor" if env else ("prompt plan" if world > 1 else "single GPU"),
                              "prompt_tokens_per_s": slowest, "ranks": ranks}), flush=True)


if __name__ == "__main__":
    main()
