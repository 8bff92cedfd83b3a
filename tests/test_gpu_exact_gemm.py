"""GPU: the tiled reference-order GEMM (k_mul_mat_q_ref_tiled, fl_exact_kernels.cu; fl_dev_mul_mat_q impl 9) carries the same bits
as k_mul_mat_q_ref (impl 8) and the C oracle, at every LLaMA matrix shape, on ragged shapes and on row slices, and a whole model
ingested under FASTLLAMA_B200_INGEST=exact gives the reference's tokens and logits bit for bit.  Every comparison is on uint32 views:
no tolerance anywhere."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

IMPL_REF, IMPL_TILED = 8, 9
TYPES = [pytest.param(2, id="q4_0"), pytest.param(3, id="q4_1")]


@pytest.fixture(scope="module")
def fl():
    from fastllama_b200.cuda_abi import FlCuda

    return FlCuda()


@pytest.fixture
def exact_ingest():
    old = os.environ.get("FASTLLAMA_B200_INGEST")
    os.environ["FASTLLAMA_B200_INGEST"] = "exact"
    yield
    if old is None:
        del os.environ["FASTLLAMA_B200_INGEST"]
    else:
        os.environ["FASTLLAMA_B200_INGEST"] = old


def _random_q4(rng, t, M, K):
    """M rows of K/32 random q4 blocks: random nibble bytes, small positive fp32 scales (and signed mins for q4_1)"""
    nb = K // 32
    qs = rng.integers(0, 256, size=(M, nb, 16), dtype=np.uint8)
    d = (rng.random((M, nb, 1), dtype=np.float32) * 0.02 + 1e-3).view(np.uint8).reshape(M, nb, 4)
    parts = [d] if t == 2 else [d, (rng.standard_normal((M, nb, 1), dtype=np.float32) * 0.05).view(np.uint8).reshape(M, nb, 4)]
    return np.ascontiguousarray(np.concatenate(parts + [qs], axis=2).reshape(M, -1))


def _first_diff(got, want):
    g, w = got.view(np.uint32), want.view(np.uint32)
    bad = np.argwhere(g != w)
    if bad.size == 0:
        return None
    i = tuple(bad[0])
    return f"{bad.shape[0]} of {g.size} differ; first (column, row) {i}: {got[i]!r} (0x{int(g[i]):08x}) vs {want[i]!r} (0x{int(w[i]):08x})"


SHAPES = [  # (M, K): 7B, 13B, 65B attention / feed-forward / output matrices
    (4096, 4096), (11008, 4096), (4096, 11008), (32000, 4096),
    (5120, 5120), (13824, 5120), (5120, 13824), (32000, 5120),
    (8192, 8192), (22016, 8192), (8192, 22016),
]
NS = (1, 2, 15, 16, 17, 64, 127, 128, 129, 512)


@pytest.mark.parametrize("t", TYPES)
@pytest.mark.parametrize("M,K", SHAPES, ids=[f"{m}x{k}" for m, k in SHAPES])
def test_tiled_equals_reference_order_kernel_at_model_shapes(fl, t, M, K):
    rng = np.random.default_rng(M * 7 + K + t)
    w = _random_q4(rng, t, M, K)
    wrs = w.shape[1]
    ns = NS + ((2048,) if (M, K) == (4096, 4096) else ())
    nmax = max(ns)
    dW = fl.to_device(w)
    dX = fl.to_device((rng.standard_normal((nmax, K)) * 0.5).astype(np.float32))
    dY = fl.alloc(nmax * (K // 32) * 40)
    dA, dB = fl.alloc(nmax * M * 4), fl.alloc(nmax * M * 4)
    try:
        fl.check(fl.lib.fl_dev_quantize_q8_0(dX, K * 4, dY, K, nmax))
        for N in ns:
            fl.check(fl.lib.fl_dev_memset(dA, 0xFF, N * M * 4))
            fl.check(fl.lib.fl_dev_memset(dB, 0x7F, N * M * 4))
            fl.check(fl.lib.fl_dev_mul_mat_q(t, dW, wrs, M, K, dY, N, dA, M, IMPL_REF))
            fl.check(fl.lib.fl_dev_mul_mat_q(t, dW, wrs, M, K, dY, N, dB, M, IMPL_TILED))
            want = fl.to_host(dA, (N, M), np.float32)
            got = fl.to_host(dB, (N, M), np.float32)
            assert np.isfinite(want).all(), N
            msg = _first_diff(got, want)
            assert msg is None, f"N={N}: {msg}"
    finally:
        for d in (dW, dX, dY, dA, dB):
            fl.free(d)


# K: 32, 96, 4128 give rows that are not 16-byte aligned (q4_0 and q4_1) and go to k_mul_mat_q_ref; the others are aligned, and
# their block counts leave a short last chunk (KC = 12 blocks for q4_0, 10 for q4_1), fill less than one chunk, or fill whole chunks.
RAGGED_K = (32, 96, 4128, 256, 384, 640, 1152, 1408)
RAGGED_M = (1, 7, 31, 33, 63, 65, 130, 515)
RAGGED_N = (1, 7, 8, 9, 31, 32, 33, 64, 65)        # both sides of the 8-column warp and 32-column CTA edges


@pytest.mark.parametrize("t", TYPES)
@pytest.mark.parametrize("K", RAGGED_K)
def test_ragged_shapes_against_the_oracle(fl, oracle, exact_ingest, t, K):
    from fastllama_b200.cuda_abi import FlCudaError

    rng = np.random.default_rng(K + 31 * t)
    nmax = max(RAGGED_N)
    x = rng.standard_normal((nmax, K)).astype(np.float32)
    dY = fl.to_device(oracle.quantize_q8_0(x))
    for M in RAGGED_M:
        w = oracle.quantize_q4((rng.standard_normal((M, K)) * 0.05).astype(np.float32), t)
        wrs = w.shape[1]
        aligned = wrs % 16 == 0
        assert aligned == (K not in (32, 96, 4128))
        drs = M + 3
        dW, dD = fl.to_device(w), fl.alloc(nmax * drs * 4)
        try:
            for N in RAGGED_N:
                want = oracle.mul_mat_q(w, x[:N], t)
                for impl in (0, IMPL_TILED):
                    fl.check(fl.lib.fl_dev_memset(dD, 0xFF, N * drs * 4))
                    if impl == IMPL_TILED and not aligned:
                        with pytest.raises(FlCudaError):
                            fl.check(fl.lib.fl_dev_mul_mat_q(t, dW, wrs, M, K, dY, N, dD, drs, impl))
                        continue
                    fl.check(fl.lib.fl_dev_mul_mat_q(t, dW, wrs, M, K, dY, N, dD, drs, impl))
                    out = fl.to_host(dD, (N, drs), np.float32)
                    msg = _first_diff(np.ascontiguousarray(out[:, :M]), want)
                    assert msg is None, f"impl {impl} M={M} N={N}: {msg}"
                    assert (out[:, M:].view(np.uint32) == 0xFFFFFFFF).all(), f"impl {impl} M={M} N={N}: wrote past row M"
        finally:
            fl.free(dW)
            fl.free(dD)
    fl.free(dY)


@pytest.mark.parametrize("t", TYPES)
@pytest.mark.parametrize("M,K", [(4096, 4096), (11008, 4096), (4096, 11008)])
def test_row_slices_carry_the_full_product_bits(fl, exact_ingest, t, M, K):
    """Rows [r * M/p, (r + 1) * M/p) computed on their own (the weight pointer starts inside the matrix, as the tensor-parallel
    plan's row slices do) and written with the full row stride equal the full product, for impl 9 and impl 0 in exact mode."""
    rng = np.random.default_rng(M + K + t)
    w = _random_q4(rng, t, M, K)
    wrs = w.shape[1]
    nmax = 129
    dW = fl.to_device(w)
    dX = fl.to_device((rng.standard_normal((nmax, K)) * 0.5).astype(np.float32))
    dY = fl.alloc(nmax * (K // 32) * 40)
    dFull, dParts = fl.alloc(nmax * M * 4), fl.alloc(nmax * M * 4)
    try:
        fl.check(fl.lib.fl_dev_quantize_q8_0(dX, K * 4, dY, K, nmax))
        for N in (16, 48, 128, 129):
            fl.check(fl.lib.fl_dev_mul_mat_q(t, dW, wrs, M, K, dY, N, dFull, M, IMPL_REF))
            full = fl.to_host(dFull, (N, M), np.float32)
            for impl in (0, IMPL_TILED):
                for p in (2, 4, 8):
                    ms = M // p
                    fl.check(fl.lib.fl_dev_memset(dParts, 0xFF, N * M * 4))
                    for r in range(p):
                        fl.check(fl.lib.fl_dev_mul_mat_q(t, dW + r * ms * wrs, wrs, ms, K, dY, N, dParts + r * ms * 4, M, impl))
                    msg = _first_diff(fl.to_host(dParts, (N, M), np.float32), full)
                    assert msg is None, f"impl {impl} N={N} p={p}: {msg}"
    finally:
        for d in (dW, dX, dY, dFull, dParts):
            fl.free(d)


# ---- whole models through fastllama_b200.Model, exact mode, against the reference library ----------------------------------------
N_STEPS = 8
PROMPT_CHARS = {"p40": 38, "p200": 198}      # bench._long_prompt: one token per character with the synthetic vocabulary, plus 2


def _model_file(size, wtype):
    import bench
    from fastllama_b200.ggjt import write_synthetic_gpu

    path = os.path.join(bench.bench_dir(), f"fastllama_b200_synth_{size}_{'q4_0' if wtype == 2 else 'q4_1'}_4layers_seed0.bin")
    if not os.path.exists(path):
        write_synthetic_gpu(path + ".tmp", size=size, wtype=wtype, seed=0, std=0.02, n_layer=4)
        os.replace(path + ".tmp", path)
    return path


def _ours(path, prompt, n_batch, profile=False):
    import bench

    be = bench.Backend(0)
    m = be.model(path, n_batch=n_batch)
    kernels = None
    if profile:
        import torch
        from torch.profiler import ProfilerActivity, profile as tprofile

        torch.cuda.init()
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            assert m.ingest(prompt)
            torch.cuda.synchronize()
        kernels = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    else:
        assert m.ingest(prompt)
    toks, logits = [], []
    for _ in range(N_STEPS):
        got = []
        m.generate(lambda s: got.append(s), num_tokens=1, **bench.GREEDY)
        if not got:
            break
        toks.append("".join(got))
        logits.append(m.get_logits_array())
    m.close()
    return toks, np.stack(logits), kernels


@pytest.mark.parametrize("n_batch", [16, 128])
@pytest.mark.parametrize("prompt", sorted(PROMPT_CHARS))
@pytest.mark.parametrize("size,wtype", [("7B", 2), ("13B", 3)], ids=["7B_q4_0", "13B_q4_1"])
def test_exact_ingest_gives_the_reference_bits(tmp_path, exact_ingest, size, wtype, prompt, n_batch):
    import bench
    from oracle.pyoracle import REF_PYFASTLLAMA_SO

    if not os.path.exists(REF_PYFASTLLAMA_SO):
        pytest.skip("oracle/_ref not built")
    path = _model_file(size, wtype)
    text = bench._long_prompt(PROMPT_CHARS[prompt])
    lp = str(tmp_path / "ref_logits.npy")
    r = bench.run_ref_worker({"path": path, "threads": min(32, os.cpu_count() or 1), "prompt": text, "n_parity": N_STEPS,
                              "logits_out": lp, "n_batch": n_batch})
    ref_tokens, ref_logits = r["parity_tokens"], np.load(lp)
    profile = (size, prompt, n_batch) == ("7B", "p200", 128)
    our_tokens, our_logits, kernels = _ours(path, text, n_batch, profile=profile)
    if profile:
        assert any("k_mul_mat_q_ref_tiled" in k for k in kernels), sorted(kernels)
        assert not any("k_mul_mat_q_umma" in k for k in kernels), sorted(kernels)
    par = bench.compare_parity(ref_tokens, ref_logits, our_tokens, our_logits)
    print("parity:", par)
    assert par["tokens_compared"] >= N_STEPS // 2
    assert par["greedy_ids_equal"], par
    assert par["logits_bit_identical"] and par["logits_maxabs_over_range"] == 0.0, par
