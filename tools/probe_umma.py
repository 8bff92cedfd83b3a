"""GPU probe: the wgmma prompt-ingest GEMM (fl_umma_kernel.cu; impl 5 / 6 / 7 = column tiles of 32 / 64 / 64) against the plain
kernel (impl 1) and the exact oracle, then timings at the LLaMA-7B shapes.

  python tools/probe_umma.py [check|time|all]
"""
import ctypes as C
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fastllama_b200.cuda_abi import FlCuda  # noqa: E402
from oracle.pyoracle import Oracle, np_quantize_q4_0, np_quantize_q4_1  # noqa: E402

mode = sys.argv[1] if len(sys.argv) > 1 else "all"
fl = FlCuda()
orc = Oracle()
BUDGET = 2e-6


def check(t, m, k, n, impl):
    rng = np.random.default_rng(m + 3 * k + 7 * n)
    w = (rng.standard_normal((m, k)) * 0.03).astype(np.float32)
    wq = (np_quantize_q4_0 if t == 2 else np_quantize_q4_1)(w)
    x = rng.standard_normal((n, k)).astype(np.float32)
    ex, mag = orc.mul_mat_q_exact(wq, x, t)
    q8 = orc.quantize_q8_0(x)
    dW, dY, dD = fl.to_device(wq), fl.to_device(q8), fl.alloc(m * n * 4)
    fl.check(fl.lib.fl_dev_memset(dD, 0xFF, m * n * 4))
    rc = fl.lib.fl_dev_mul_mat_q(t, dW, wq.shape[1], m, k, dY, n, dD, m, impl)
    if rc != 0:
        print(f"  type {t} {m}x{k}xN{n} impl {impl}: launch failed: {fl.lib.fl_last_error().decode()}")
        return False
    rc = fl.lib.fl_sync()
    if rc != 0:
        print(f"  type {t} {m}x{k}xN{n} impl {impl}: SYNC FAILED: {fl.lib.fl_last_error().decode()}")
        return False
    got = fl.to_host(dD, (n, m), np.float32)
    err = np.abs(got.astype(np.float64) - ex) / np.maximum(mag, 1e-30)
    bad = ~(err <= BUDGET)
    ok = not bad.any()
    print(f"  type {t} {m}x{k}xN{n} impl {impl}: max err {np.nanmax(err):.3e} of sum|dq|  {'OK' if ok else 'FAIL'}  nan {np.isnan(got).sum()}")
    if not ok:
        idx = np.argwhere(bad)
        print(f"    {bad.sum()} of {bad.size} wrong; first (col,row) {idx[:6].tolist()}; rows wrong {np.unique(idx[:, 1])[:16].tolist()} cols wrong {np.unique(idx[:, 0])[:16].tolist()}")
        c, r = idx[0]
        print(f"    got {got[c, r]:.6g} want {ex[c, r]:.6g}; ratio {got[c, r] / ex[c, r] if ex[c, r] else float('nan'):.4g}")
        # is the result a permutation / transposition of the right answer?
        if got.shape[0] == got.shape[1]:
            e2 = np.abs(got.T.astype(np.float64) - ex) / np.maximum(mag, 1e-30)
            print(f"    transposed match: {np.nanmax(e2):.3e}")
    for d in (dW, dY, dD):
        fl.free(d)
    return ok


if mode in ("check", "all"):
    allok = True
    for t in (2, 3):
        for (m, k, n) in [(128, 128, 32), (128, 128, 128), (256, 512, 64), (300, 256, 5), (1000, 11008, 37), (1024, 4096, 128), (514, 4096, 200)]:
            for impl in (5, 6, 7):
                if impl == 7 and t == 3:
                    continue
                allok &= check(t, m, k, n, impl)
    print("CHECK", "PASSED" if allok else "FAILED")
    if not allok and mode == "all":
        sys.exit(1)

if mode in ("time", "all"):
    N = 128
    rng = np.random.default_rng(0)
    SHAPES = [("wq/wk/wv/wo", 4096, 4096, 4 * 32), ("w1/w3", 11008, 4096, 2 * 32), ("w2", 4096, 11008, 32), ("output", 32000, 4096, 1)]
    total = {}
    for name, m, k, count in SHAPES:
        nb = k // 32
        w = rng.integers(0, 256, size=(m, nb, 20), dtype=np.uint8)
        w[:, :, 0:4] = np.frombuffer(np.float32(0.01).tobytes(), dtype=np.uint8)
        w = w.reshape(m, nb * 20)
        q8 = fl.quantize_q8_0(rng.standard_normal((N, k)).astype(np.float32))
        dW, dY, dD = fl.to_device(w), fl.to_device(q8), fl.alloc(m * N * 4)
        for impl in (5, 6, 7, 4, 3):
            ms = C.c_float()
            fl.check(fl.lib.fl_dev_time_mul_mat_q(2, dW, nb * 20, m, k, dY, N, dD, m, impl, 10, 0, C.byref(ms)))
            total[impl] = total.get(impl, 0.0) + ms.value * count
            print(f"{name:12s} {m:6d} x {k:6d} x N={N}: impl {impl}: {ms.value:8.3f} ms  {m * k * N / ms.value / 1e9:8.2f} TMAC/s  {2 * m * k * N / ms.value / 1e9:9.1f} TFLOP/s")
        for d in (dW, dY, dD):
            fl.free(d)
    for impl, v in total.items():
        print(f"impl {impl}: all quantised matmuls of a {N}-token 7B batch: {v:8.2f} ms -> {2 * 6607077376 * N / v / 1e9:8.1f} TFLOP/s")
