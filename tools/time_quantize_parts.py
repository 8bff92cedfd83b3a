"""Wall-clock time and input GB/s of quantising a LLaMA-13B-shaped f16 model to q4_0 with
fastllama_b200.quantize.quantize_model, the same model written two ways: as 2 parts (write_synthetic_parts, the layout
the reference's converter writes for 13B) and as one file (write_synthetic_joined).

Both inputs are generated into a temporary directory (or --dir) and read once before every run, so each run starts
from a warm page cache; the runs alternate (one file, parts, one file, parts, ...) --repeats times, and the two outputs
are checked to be the same bytes.  Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/time_quantize_parts.py [--layers 40] [--repeats 2] [--dir DIR]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from fastllama_b200.cuda_abi import FlCuda  # noqa: E402
from fastllama_b200.ggjt import F16, Q4_0, write_synthetic_joined, write_synthetic_parts  # noqa: E402
from fastllama_b200.quantize import quantize_model  # noqa: E402
from time_quantize import card, same_bytes  # noqa: E402

THIRTEEN_B = dict(n_vocab=32000, n_embd=5120, n_mult=256, n_head=40)


def warm(paths):
    for p in paths:
        with open(p, "rb") as f:
            while f.read(256 << 20):
                pass


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=40)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--dir", default=None)
    args = ap.parse_args()
    fl = FlCuda()
    d = args.dir or tempfile.mkdtemp(prefix="time_quantize_parts_")
    try:
        t0 = time.perf_counter()
        part0 = write_synthetic_parts(os.path.join(d, "13b-f16.bin"), ["ggjt", "ggjt"], F16, n_layer=args.layers, seed=1,
                                      **THIRTEEN_B)
        single = write_synthetic_joined(os.path.join(d, "13b-f16-single.bin"), 2, F16, n_layer=args.layers, seed=1,
                                        **THIRTEEN_B)
        t_gen = time.perf_counter() - t0
        inputs = {"single_file": [single], "two_parts": [part0, part0 + ".1"]}
        size = {k: sum(os.path.getsize(p) for p in v) for k, v in inputs.items()}
        res = {"layers": args.layers, "input_bytes": size, "generate_s": round(t_gen, 1), "runs": {k: [] for k in inputs}}
        outs = {}
        for _ in range(args.repeats):
            for name, paths in inputs.items():
                warm(paths)
                outs[name] = os.path.join(d, f"{name}.bin")
                t0 = time.perf_counter()
                quantize_model(paths[0], outs[name], Q4_0, fl=fl, verbose=False)
                dt = time.perf_counter() - t0
                res["runs"][name].append({"seconds": round(dt, 2), "input_GB_per_s": round(size[name] / dt / 1e9, 2)})
        res["outputs_identical"] = same_bytes(outs["single_file"], outs["two_parts"])
        res["gpu"], res["power_limit"] = card()
        res["cpu_threads"] = os.cpu_count()
        print(json.dumps(res))
    finally:
        if args.dir is None:
            shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
