"""Wall-clock time and input GB/s of quantising a LLaMA-7B-shaped f16 file to q4_0, three ways:

  * fastllama_b200.quantize.quantize_model (k_quantize_q4_file, streamed through pinned staging buffers)
  * the drop-in fastllama_b200/lib/quantize (the reference's threaded tool over libggml_b200)
  * oracle/_ref/quantize_ref (the reference's tool over its own lib/ggml.c, on the CPU)

The input is generated into a temporary directory (or --dir), read once so every tool starts from a warm page
cache, and the three outputs are checked to be the same bytes.  Prints one JSON line with the card's name and
power limit, read in the same run.

    python tools/time_quantize.py [--layers 32] [--dir DIR]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from fastllama_b200.build import lib_path  # noqa: E402
from fastllama_b200.cuda_abi import FlCuda  # noqa: E402
from fastllama_b200.ggjt import F16, Q4_0, write_synthetic_float  # noqa: E402
from fastllama_b200.quantize import quantize_model  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().splitlines() or ["?, ?"])[0].split(", ")
    return name, power


def same_bytes(a, b):
    with open(a, "rb") as fa, open(b, "rb") as fb:
        while True:
            x, y = fa.read(64 << 20), fb.read(64 << 20)
            if x != y:
                return False
            if not x:
                return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--dir", default=None)
    args = ap.parse_args()
    fl = FlCuda()
    d = args.dir or tempfile.mkdtemp(prefix="time_quantize_")
    try:
        src = os.path.join(d, "7b-f16.bin")
        t0 = time.perf_counter()
        write_synthetic_float(src, F16, n_vocab=32000, n_embd=4096, n_mult=256, n_head=32, n_layer=args.layers, seed=1, std=0.02)
        t_gen = time.perf_counter() - t0
        size = os.path.getsize(src)
        with open(src, "rb") as f:                         # warm the page cache: every tool reads the same cached file
            while f.read(256 << 20):
                pass
        res = {"input_bytes": size, "layers": args.layers, "generate_s": round(t_gen, 1)}
        outs = {}
        runs = [("quantize_model", None),
                ("dropin_quantize", [lib_path("quantize")]),
                ("quantize_ref_cpu", [os.path.join(ROOT, "oracle", "_ref", "quantize_ref")])]
        for name, exe in runs:
            out = os.path.join(d, f"{name}.bin")
            t0 = time.perf_counter()
            if exe is None:
                quantize_model(src, out, Q4_0, fl=fl, verbose=False)
            else:
                p = subprocess.run(exe + [src, out, str(Q4_0)], capture_output=True, text=True)
                if p.returncode != 0:
                    raise RuntimeError(f"{name} failed: {p.stderr[-2000:]}")
            dt = time.perf_counter() - t0
            res[name] = {"seconds": round(dt, 2), "input_GB_per_s": round(size / dt / 1e9, 2)}
            outs[name] = out
        res["outputs_identical"] = all(same_bytes(outs["quantize_ref_cpu"], o) for o in outs.values())
        name, power = card()
        res["gpu"] = name
        res["power_limit"] = power
        res["cpu_threads"] = os.cpu_count()
        print(json.dumps(res))
    finally:
        if args.dir is None:
            shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
