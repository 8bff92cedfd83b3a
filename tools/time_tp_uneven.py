"""tools/time_tp_uneven.py -- decode and prompt-ingest throughput of tensor-parallel ranks at any world size (ggml_b200.cpp tp_partition).

Run under torchrun, one process per GPU:

    torchrun --standalone --nproc-per-node 8 tools/time_tp_uneven.py --size 30B [--layers 60]
    torchrun --standalone --nproc-per-node 3 tools/time_tp_uneven.py --size 7B [--vocab 32001]
    python tools/time_tp_uneven.py --size 7B --vocab 32001                      # one GPU

Rank 0 writes a synthetic q4_0 file (LLaMA 7B with a 32000- or 32001-token vocabulary, or 30B; --layers keeps the first L layers) to a
temporary directory, unless --model names one.  Every rank then ingests a warm-up prompt, resets, and reports:
  - prompt-ingest tokens/s of two 128-token evals (n_batch 128) and decode tokens/s of --tokens greedy steps, both from the library's
    CUDA-event counters (ggml_b200_get_stats: device time of the timed evals, as bench.py measures), and wall clock;
  - its partition (first row and row count of n_embd, n_ff and n_vocab, restated from the rule), ggml_b200_decode_mode(),
    ggml_b200_prompt_mode() and ggml_b200_get_memory;
  - the card's name and power limit (nvidia-smi, read only).
Rank 0 prints one JSON line with every rank's report.  Asserts nothing about speed.
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


def tp_split(total, unit, world, rank):
    """the library's partition rule (ggml_b200.cpp tp_split): whole units dealt out in order, the first (units % world) ranks taking one
    more, the rows after the last whole unit with the last rank"""
    base, extra = divmod(total // unit, world)
    u0, nu = rank * base + min(rank, extra), base + (1 if rank < extra else 0)
    first, end = u0 * unit, total if rank == world - 1 else (u0 + nu) * unit
    return [first, end - first]


def _text(n_chars: int, salt: int = 0) -> str:
    """ASCII text; with the synthetic vocabulary every character is one token, plus BOS and the bridge's leading space"""
    words = "tensor parallel decode and prompt ingest at a world size that does not divide the heads of the model".split()
    out, i = [], salt
    while sum(len(w) + 1 for w in out) < n_chars + 1:
        out.append(words[i % len(words)])
        i += 1
    return " ".join(out)[:n_chars]


def _card(dev: int) -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", str(dev)], capture_output=True,
                           text=True, timeout=30).stdout.strip().split(", ")
        return {"card": q[0], "power_limit_w": float(q[1])}
    except Exception as e:  # noqa: BLE001 -- the report says what is missing
        return {"card": None, "power_limit_w": None, "card_error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", default="7B", choices=["7B", "30B"])
    ap.add_argument("--vocab", type=int, default=32000)
    ap.add_argument("--layers", type=int, default=None, help="keep the first L layers (default: all)")
    ap.add_argument("--model", default=None, help="an existing q4_0 file of that shape instead of a synthetic one")
    ap.add_argument("--tokens", type=int, default=64, help="timed decode steps")
    args = ap.parse_args()
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", str(rank)))
    os.environ["FASTLLAMA_DEVICE"] = str(local)
    import torch

    from fastllama_b200.build import lib_path
    from fastllama_b200.cuda_abi import FlCuda
    from fastllama_b200.ggjt import LLAMA_SIZES, n_ff
    from fastllama_b200.model import Model, QuietLogger

    fl = FlCuda()
    torch.cuda.set_device(local)
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
    tmp = tempfile.mkdtemp(prefix="fl_tp_uneven_") if rank == 0 else None
    path = args.model
    if not path:
        # rank 0 writes the file; the others wait for its name (the ranks share one host)
        names = [os.path.join(tmp, f"synth_{args.size}_{args.vocab}_q4_0.bin") if rank == 0 else None]
        if rank == 0:
            t0 = time.time()
            code = ("import sys; sys.path.insert(0, %r); from fastllama_b200.ggjt import write_synthetic_gpu; "
                    "write_synthetic_gpu(%r, size=%r, wtype=2, seed=0, std=0.02, n_vocab=%d, n_layer=%r)"
                    % (ROOT, names[0], args.size, args.vocab, args.layers))
            subprocess.run([sys.executable, "-c", code], check=True, stdout=sys.stderr, env=dict(os.environ, WORLD_SIZE="1", RANK="0"))
            print(f"[time_tp_uneven] wrote {os.path.getsize(names[0]) / 1e9:.2f} GB in {time.time() - t0:.0f} s", file=sys.stderr)
        if dist:
            dist.broadcast_object_list(names, 0)
        path = names[0]

    g = C.CDLL(lib_path("libggml_b200.so"))
    g.ggml_b200_get_stats.argtypes = [C.POINTER(_Stats)]
    g.ggml_b200_get_memory.argtypes = [C.POINTER(_Mem)]

    def stats():
        s = _Stats()
        g.ggml_b200_get_stats(C.byref(s))
        return s

    def sync():
        fl.check(fl.lib.fl_sync())
        if dist:
            dist.barrier()

    greedy = dict(temp=0.0, top_k=1, top_p=1.0, repeat_penalty=1.0)
    m = Model(path, num_threads=1, n_ctx=512, n_batch=128, logger=QuietLogger(), library_path=lib_path("pyfastllama.so"))
    assert m.ingest(_text(128 + 1 - 2))                      # shard uploads, plan builds and first launches, untimed
    m.generate(lambda s: None, num_tokens=4, **greedy)
    assert m.reset()
    sync()
    s0, t0 = stats(), time.perf_counter()
    assert m.ingest(_text(2 * 128 + 1 - 2, salt=3))          # two 128-token evals; the last token is left to the first generate call
    sync()
    s1, t1 = stats(), time.perf_counter()
    prompt_mode = int(g.ggml_b200_prompt_mode())
    m.generate(lambda s: None, num_tokens=1, **greedy)        # the prompt's last token
    sync()
    s2, t2 = stats(), time.perf_counter()
    m.generate(lambda s: None, num_tokens=args.tokens, **greedy)
    sync()
    s3, t3 = stats(), time.perf_counter()
    decode_mode = int(g.ggml_b200_decode_mode())
    mem = _Mem()
    g.ggml_b200_get_memory(C.byref(mem))
    free, total = torch.cuda.mem_get_info(local)
    m.close()

    n_embd, n_head, _ = LLAMA_SIZES[args.size]
    ff = n_ff(n_embd, 256)
    p_evals, d_evals = int(s1.n_evals - s0.n_evals), int(s3.n_evals - s2.n_evals)
    p_dev, d_dev = (s1.total_device_us - s0.total_device_us) * 1e-6, (s3.total_device_us - s2.total_device_us) * 1e-6
    res = {"rank": rank, "world": world,
           "partition": {"n_embd": tp_split(n_embd, n_embd // n_head, world, rank), "n_ff": tp_split(ff, 32, world, rank),
                         "n_vocab": tp_split(args.vocab, 2, world, rank)},
           "decode_mode": decode_mode, "prompt_mode": prompt_mode,
           "prompt_evals": p_evals, "prompt_tokens_per_s_device": p_evals * 128 / p_dev if p_dev else 0.0,
           "prompt_tokens_per_s_wall": p_evals * 128 / (t1 - t0),
           "decode_steps": d_evals, "decode_tokens_per_s_device": d_evals / d_dev if d_dev else 0.0, "decode_tokens_per_s_wall": d_evals / (t3 - t2),
           "weight_mirror_bytes": int(mem.weight_mirror_bytes), "shard_bytes": int(mem.shard_bytes), "mirror_bytes": int(mem.mirror_bytes),
           "kv_gathers": int(mem.kv_gathers), "device_used_bytes": int(total - free), **_card(local)}
    reports = [None] * world
    if dist:
        dist.all_gather_object(reports, res)
        dist.destroy_process_group()
    else:
        reports = [res]
    if rank == 0:
        print(json.dumps({"size": args.size, "n_vocab": args.vocab, "layers": args.layers, "world": world,
                          "decode_tokens_per_s": min(r["decode_tokens_per_s_device"] for r in reports),
                          "prompt_tokens_per_s": min(r["prompt_tokens_per_s_device"] for r in reports), "ranks": reports}), flush=True)
        if not args.model:
            import shutil

            shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
