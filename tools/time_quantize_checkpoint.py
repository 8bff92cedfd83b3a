"""Wall clock, input GB/s and peak host memory of quantising a LLaMA-7B-shaped f16 checkpoint to q4_0, in one pass
(fastllama_b200.quantize.quantize_model on the checkpoint) and in the reference's two steps (the f16 GGJT file its
converter writes, here written by tests/checkpoint_files.write_converted, its numpy restatement, then quantize_model
on that file), for the checkpoint as one Meta .pth (consolidated.00.pth) and as two Hugging Face safetensors files.

The checkpoints are generated into a temporary directory (or --dir): the safetensors files tensor by tensor, and the
.pth by torch.save over memory maps of them (the same data under the Meta names, q / k rows not permuted: a different
model, the same bytes to read).  Every configuration runs in its own process, from a warm page cache, and reports
its own peak resident set (VmHWM or ru_maxrss, which count the pages of memory-mapped inputs it touched) and the peak
of its anonymous memory (RssAnon, sampled every 10 ms; null where /proc does not report it).  The one-pass and
two-step outputs of each checkpoint are checked to be the same bytes.  Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/time_quantize_checkpoint.py [--layers 32] [--dir DIR]
"""
import argparse
import json
import os
import resource
import shutil
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402

from tests.checkpoint_files import (TOKENIZER, hf_names, make_tensor, meta_shapes, permute, write_converted,  # noqa: E402
                                    write_safetensors)
from time_quantize import card, same_bytes  # noqa: E402

SEVEN_B = dict(n_vocab=32000, n_embd=4096)


def generate(d, n_layer):
    shapes = dict(meta_shapes(n_layer=n_layer, **SEVEN_B))
    names = hf_names(shapes)                                # (hf name, meta name, permuted) over the shapes' keys
    os.makedirs(os.path.join(d, "hf"), exist_ok=True)
    half = -(-len(names) // 2)
    files = []
    for j in range(2):
        path = os.path.join(d, "hf", f"model-{j + 1:05}-of-00002.safetensors")
        write_safetensors(path, [(h, np.float16, shapes[m], (lambda m=m: make_tensor(m, shapes[m], np.float16, 1)))
                                 for h, m, _ in names[j * half:(j + 1) * half]])
        files.append(path)
    with open(TOKENIZER, "rb") as f, open(os.path.join(d, "tokenizer.model"), "wb") as g:
        g.write(f.read())
    with open(os.path.join(d, "added_tokens.json"), "w") as f:
        json.dump({f"<extra_{i}>": i for i in range(300, SEVEN_B["n_vocab"])}, f)

    import torch

    from fastllama_b200.quantize import read_checkpoint

    os.makedirs(os.path.join(d, "meta"), exist_ok=True)
    hf = {t.name: t for t in read_checkpoint(files[0], "f16", d).tensors}
    maps = [np.memmap(p, dtype=np.uint8, mode="c") for p in files]
    sd = {}
    for _, m, _ in names:
        sh = hf[m].shards[0]
        sd[m] = torch.from_numpy(maps[sh.part][sh.offset:sh.offset + sh.nbytes].view(np.float16).reshape(shapes[m]))
    torch.save(sd, os.path.join(d, "meta", "consolidated.00.pth"))
    return {"pth": os.path.join(d, "meta"), "safetensors": files[0]}


def meta_view(kind, path, n_layer):
    """The joined Meta-named model of a checkpoint, one callable per tensor, for the numpy restatement."""
    if kind == "pth":
        import torch

        sd = torch.load(os.path.join(path, "consolidated.00.pth"), mmap=True, weights_only=True)
        return {n: (lambda t=t: t.numpy()) for n, t in sd.items()}
    from safetensors import safe_open

    d = os.path.dirname(path)
    handles = [safe_open(os.path.join(d, f), "np") for f in sorted(os.listdir(d)) if f.endswith(".safetensors")]
    where = {k: h for h in handles for k in h.keys()}
    n_head = SEVEN_B["n_embd"] // 128
    shapes = dict(meta_shapes(n_layer=n_layer, **SEVEN_B))
    return {m: (lambda h=h, p=p: permute(where[h].get_tensor(h), n_head) if p else where[h].get_tensor(h))
            for h, m, p in hf_names(shapes)}


def run_one(kind, mode, path, d, n_layer):
    from fastllama_b200.cuda_abi import FlCuda
    from fastllama_b200.quantize import quantize_model

    peak_anon = [0]
    done = threading.Event()

    def sample():
        while not done.wait(0.01):
            peak_anon[0] = max(peak_anon[0], status("RssAnon"))

    fl = FlCuda()
    inputs = [os.path.join(path, "consolidated.00.pth")] if kind == "pth" else \
        [os.path.join(os.path.dirname(path), f) for f in sorted(os.listdir(os.path.dirname(path))) if f.endswith(".safetensors")]
    for p in inputs:                                        # warm page cache: every run reads cached input
        with open(p, "rb") as f:
            while f.read(256 << 20):
                pass
    out = os.path.join(d, f"{kind}-{mode}.q4_0.bin")
    res = {"input_bytes": sum(os.path.getsize(p) for p in inputs)}
    th = threading.Thread(target=sample, daemon=True)
    th.start()
    t0 = time.perf_counter()
    if mode == "one_pass":
        quantize_model(path, out, 2, fl=fl, verbose=False, vocab_dir=d)
    else:
        ggjt = os.path.join(d, f"{kind}-f16.ggjt.bin")
        write_converted(ggjt, meta_view(kind, path, n_layer), os.path.join(d, "tokenizer.model"), "f16")
        res["convert_s"] = round(time.perf_counter() - t0, 2)
        res["f16_file_bytes"] = os.path.getsize(ggjt)
        quantize_model(ggjt, out, 2, fl=fl, verbose=False)
        os.unlink(ggjt)
    dt = time.perf_counter() - t0
    done.set()
    th.join()
    res.update(seconds=round(dt, 2), input_GB_per_s=round(res["input_bytes"] / dt / 1e9, 2),
               peak_rss_MB=round(max(status("VmHWM"), resource.getrusage(resource.RUSAGE_SELF).ru_maxrss) / 1024),
               peak_anon_rss_MB=round(peak_anon[0] / 1024) if peak_anon[0] else None, output=out)
    print(json.dumps(res))


def status(key):
    with open("/proc/self/status") as f:
        for line in f:
            if line.startswith(key + ":"):
                return int(line.split()[1])                 # kB
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--dir", default=None)
    ap.add_argument("--run", nargs=3, metavar=("KIND", "MODE", "PATH"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.run:
        return run_one(*args.run, args.dir, args.layers)
    d = args.dir or tempfile.mkdtemp(prefix="time_quantize_checkpoint_")
    try:
        t0 = time.perf_counter()
        paths = generate(d, args.layers)
        res = {"layers": args.layers, "generate_s": round(time.perf_counter() - t0, 1), "runs": {}}
        for kind, path in paths.items():
            for mode in ("one_pass", "two_step"):
                p = subprocess.run([sys.executable, os.path.abspath(__file__), "--dir", d, "--layers", str(args.layers),
                                    "--run", kind, mode, path], capture_output=True, text=True)
                if p.returncode != 0:
                    raise RuntimeError(f"{kind} {mode} failed: {p.stderr[-3000:]}")
                res["runs"][f"{kind}_{mode}"] = json.loads(p.stdout.strip().splitlines()[-1])
            r = res["runs"]
            res[f"{kind}_outputs_identical"] = same_bytes(r[f"{kind}_one_pass"].pop("output"), r[f"{kind}_two_step"].pop("output"))
        res["gpu"], res["power_limit"] = card()
        res["cpu_threads"] = os.cpu_count()
        print(json.dumps(res))
    finally:
        if args.dir is None:
            shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
