"""tools/time_exact_ingest.py -- what the reference's bits cost in prompt ingest.

1. Per-matmul CUDA-event times (fl_dev_time_mul_mat_q, warmed up, the kernels alternating in one process) of
     impl 8  k_mul_mat_q_ref        (reference order, 8 rows per warp, operands through L1/L2)
     impl 9  k_mul_mat_q_ref_tiled  (reference order, shared-memory tiles)
     impl 4  k_mul_mat_q_umma       (wgmma GEMM: the default above 15 columns, block terms in another fp32 order)
   at the 7B q4_0 and 13B q4_1 matrix shapes, for N in --ns.  FL_REF_TILED_MIN_N (fl_quant_kernels.cu) comes from this table.
2. Whole-eval prompt tokens/s through Model.ingest on bench.py's 32-layer 7B q4_0 file, n_batch 16 and 128, with
   FASTLLAMA_B200_INGEST=exact and without, in the same process.
Prints the card's name and power limit first, then one JSON line per measurement.  Asserts nothing about speed.

    python tools/time_exact_ingest.py [--ns 4,8,...] [--iters 20] [--no-model]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {  # name: (type, [(matrix, M, K, count per layer or per model)])
    "7B q4_0": (2, [("wq|wk|wv|wo", 4096, 4096, 4), ("w1|w3", 11008, 4096, 2), ("w2", 4096, 11008, 1), ("output", 32000, 4096, 0)]),
    "13B q4_1": (3, [("wq|wk|wv|wo", 5120, 5120, 4), ("w1|w3", 13824, 5120, 2), ("w2", 5120, 13824, 1), ("output", 32000, 5120, 0)]),
}
IMPLS = {8: "ref", 9: "ref_tiled", 4: "wgmma"}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=60).stdout.strip()
    except Exception as e:  # noqa: BLE001
        out = f"nvidia-smi unavailable: {e}"
    return out


def time_matmuls(ns, iters):
    from fastllama_b200.cuda_abi import FlCuda

    fl = FlCuda()
    rng = np.random.default_rng(0)
    for model, (t, mats) in SHAPES.items():
        bb = 20 if t == 2 else 24
        for name, M, K, _ in mats:
            nb = K // 32
            qs = rng.integers(0, 256, size=(M, nb, 16), dtype=np.uint8)
            d = (rng.random((M, nb, 1), dtype=np.float32) * 0.02 + 1e-3).view(np.uint8).reshape(M, nb, 4)
            parts = [d] if t == 2 else [d, (rng.standard_normal((M, nb, 1), dtype=np.float32) * 0.05).view(np.uint8).reshape(M, nb, 4)]
            w = np.ascontiguousarray(np.concatenate(parts + [qs], axis=2).reshape(M, nb * bb))
            nmax = max(ns)
            dW = fl.to_device(w)
            dX = fl.to_device(rng.standard_normal((nmax, K)).astype(np.float32))
            dY, dD = fl.alloc(nmax * nb * 40), fl.alloc(nmax * M * 4)
            fl.check(fl.lib.fl_dev_quantize_q8_0(dX, K * 4, dY, K, nmax))
            for N in ns:
                ms = {}
                for impl in IMPLS:                                   # warm-up: module load, tensor maps, buffers
                    fl.check(fl.lib.fl_dev_mul_mat_q(t, dW, nb * bb, M, K, dY, N, dD, M, impl))
                for rep in range(2):                                 # alternate the kernels, keep each one's best batch
                    for impl in IMPLS:
                        v = C.c_float()
                        fl.check(fl.lib.fl_dev_time_mul_mat_q(t, dW, nb * bb, M, K, dY, N, dD, M, impl, iters, 0, C.byref(v)))
                        ms[impl] = min(ms.get(impl, 1e30), v.value)
                print(json.dumps({"model": model, "matrix": name, "M": M, "K": K, "N": N,
                                  **{f"us_{IMPLS[i]}": round(ms[i] * 1e3, 2) for i in IMPLS},
                                  "tiled_over_ref": round(ms[8] / ms[9], 3), "tiled_over_wgmma": round(ms[9] / ms[4], 3)}), flush=True)
            for dv in (dW, dX, dY, dD):
                fl.free(dv)


def time_model(batches):
    import bench

    be = bench.Backend(0)
    path = bench.ensure_model("7B", "q4_0")
    n_tok = batches * 128
    prompt = bench._long_prompt(n_tok + 1 - 2, salt=3)     # n_tok tokens in ingest(); the last one is left to the first generate()
    for n_batch in (16, 128):
        m = be.model(path, n_batch=n_batch)
        res = {}
        for rep in range(3):
            for mode in ("default", "exact"):
                if mode == "exact":
                    os.environ["FASTLLAMA_B200_INGEST"] = "exact"
                else:
                    os.environ.pop("FASTLLAMA_B200_INGEST", None)
                assert m.reset()
                be.fl.check(be.fl.lib.fl_sync())
                t0 = time.perf_counter()
                assert m.ingest(prompt)
                be.fl.check(be.fl.lib.fl_sync())
                dt = time.perf_counter() - t0
                if rep > 0:                                          # rep 0 warms up both modes
                    res[mode] = min(res.get(mode, 1e30), dt)
        os.environ.pop("FASTLLAMA_B200_INGEST", None)
        m.close()
        print(json.dumps({"model": "7B q4_0 (32 layers)", "n_batch": n_batch, "prompt_tokens": n_tok,
                          "default_tokens_per_s": round(n_tok / res["default"], 1), "exact_tokens_per_s": round(n_tok / res["exact"], 1),
                          "exact_over_default_time": round(res["exact"] / res["default"], 3)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ns", default="4,8,12,16,32,64,128,256,512")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--batches", type=int, default=3, help="128-token chunks of the timed prompt (n_ctx is 512)")
    ap.add_argument("--no-model", action="store_true", help="skip the whole-model part")
    args = ap.parse_args()
    print("card:", card(), flush=True)
    time_matmuls([int(x) for x in args.ns.split(",")], args.iters)
    if not args.no_model:
        time_model(args.batches)


if __name__ == "__main__":
    main()
