"""GPU: the hot-path row functions through the C ABI (include/fl_cuda.h, host buffers) against
  * the committed golden vectors (outputs of the reference's own kernels, tests/golden/),
  * the C oracle (oracle/q4_oracle.c) on fresh seeded inputs up to the full 7B shapes,
  * the live reference library where oracle/_ref was built.
Bar: bit-exact for q8_0 / q4 quantisation, dequantisation and get_rows (byte/integer work and
single fp32 operations); for the dot products the per-block integers are exact and only the fp32
summation ORDER differs, so the result must sit within 2e-6 * sum_i |d_i q_i| of the order-free
(double) value -- the same budget tests/test_oracle.py shows the reference's own AVX2 order needs.
"""
import numpy as np
import pytest

from oracle.pyoracle import GGML_TYPE_Q4_0, GGML_TYPE_Q4_1

pytestmark = pytest.mark.gpu
TYPES = [("q4_0", GGML_TYPE_Q4_0), ("q4_1", GGML_TYPE_Q4_1)]
REORDER_BUDGET = 2e-6


@pytest.fixture(scope="module")
def fl():
    from fastllama_b200.cuda_abi import FlCuda

    return FlCuda()           # raises (no skip) when the library or the device is missing


def _dot_ok(got, exact, mag):
    return np.all(np.abs(got.astype(np.float64) - exact) <= REORDER_BUDGET * mag + 1e-30)


def test_device_is_h100(fl):
    p = fl.device_props()
    assert p["cc"] == (9, 0) and p["sm_count"] >= 100, p


def test_q8_0_golden_bit_exact(fl, golden_rowfns):
    k, g = golden_rowfns
    assert np.array_equal(fl.quantize_q8_0(g["x"]), g["q8"])


@pytest.mark.parametrize("k", [64, 4096, 11008])
def test_q8_0_oracle_bit_exact(fl, oracle, k):
    rng = np.random.default_rng(k)
    x = (rng.standard_normal((257, k)) * rng.uniform(1e-3, 50.0, (257, 1))).astype(np.float32)
    x[3] = 0
    x[5, :32] = np.arange(32) - 15.5       # exact ties at id = 1
    x[5, 0] = 127.0
    assert np.array_equal(fl.quantize_q8_0(x), oracle.quantize_q8_0(x))


@pytest.mark.parametrize("name,t", TYPES)
def test_q4_quantize_dequantize_golden(fl, golden_rowfns, name, t):
    k, g = golden_rowfns
    assert np.array_equal(fl.quantize_q4(g["w"], t), g[f"{name}_w"])
    got = fl.dequantize_q4(g[f"{name}_w"], t, k)
    assert np.array_equal(got.view(np.uint32), g[f"{name}_deq"].view(np.uint32))
    ids = np.array([2, 0, 2, g["w"].shape[0] - 1], dtype=np.int32)
    rows = fl.get_rows_q(g[f"{name}_w"], ids, t, k)
    assert np.array_equal(rows.view(np.uint32), g[f"{name}_deq"][ids].view(np.uint32))


@pytest.mark.parametrize("name,t", TYPES)
def test_mul_mat_golden(fl, oracle, golden_rowfns, name, t):
    k, g = golden_rowfns
    got = fl.mul_mat_q(g[f"{name}_w"], g["x"], t)
    ex, mag = oracle.mul_mat_q_exact(g[f"{name}_w"], g["x"], t)
    assert _dot_ok(got, ex, mag)
    # and against the reference's own numbers (N < 16: the reference-order kernel): the same bits
    assert np.array_equal(got.view(np.uint32), g[f"{name}_mul_mat"].astype(np.float32).view(np.uint32))


@pytest.mark.parametrize("name,t", TYPES)
def test_vec_dot_hook(fl, oracle, golden_rowfns, name, t):
    k, g = golden_rowfns
    ex, mag = oracle.mul_mat_q_exact(g[f"{name}_w"][:3], g["x"][:1], t)
    for m in range(3):
        s = fl.vec_dot(g[f"{name}_w"][m], g["q8"][0], t, k)
        assert abs(float(s) - ex[0, m]) <= REORDER_BUDGET * mag[0, m] + 1e-30
        assert np.float32(s).view(np.uint32) == np.float32(oracle.vec_dot(g[f"{name}_w"][m], g["q8"][0], t, k)).view(np.uint32)


# LLaMA-7B (q4_0) and 13B (q4_1) matvec shapes, M x K (SURVEY.md 8a row a7)
FULL_SHAPES = [(GGML_TYPE_Q4_0, 4096, 4096), (GGML_TYPE_Q4_0, 11008, 4096), (GGML_TYPE_Q4_0, 4096, 11008),
               (GGML_TYPE_Q4_0, 32000, 4096), (GGML_TYPE_Q4_1, 5120, 5120), (GGML_TYPE_Q4_1, 13824, 5120),
               (GGML_TYPE_Q4_1, 5120, 13824), (GGML_TYPE_Q4_0, 8192, 8192), (GGML_TYPE_Q4_0, 8192, 22016)]


@pytest.mark.parametrize("t,m,k", FULL_SHAPES)
def test_decode_matvec_full_shapes(fl, oracle, t, m, k):
    """N = 1 at the real shapes: the reference-order kernel (impl 8 and the default, impl 0) must give the oracle's (= the reference's)
    bits; the TMA ring kernel (impl 2) and the plain kernel (impl 1) of round 1 stay within the reordering budget of the order-free
    value, and the ring kernel must be run-to-run deterministic."""
    import ctypes as C

    rng = np.random.default_rng(m * 7 + k)
    from oracle.pyoracle import np_quantize_q4_0, np_quantize_q4_1

    w = (rng.standard_normal((m, k)) * 0.02).astype(np.float32)
    wq = (np_quantize_q4_0 if t == GGML_TYPE_Q4_0 else np_quantize_q4_1)(w)
    x = rng.standard_normal((1, k)).astype(np.float32)
    ex, mag = oracle.mul_mat_q_exact(wq, x, t)
    q8 = oracle.quantize_q8_0(x)
    dW, dY, dD = fl.to_device(wq), fl.to_device(q8), fl.alloc(m * 4)
    outs = {}
    want = oracle.mul_mat_q(wq, x, t)
    for impl in (1, 2, 2, 8, 0):
        fl.check(fl.lib.fl_dev_memset(dD, 0xFF, m * 4))
        fl.check(fl.lib.fl_dev_mul_mat_q(t, dW, wq.shape[1], m, k, dY, 1, dD, m, impl))
        got = fl.to_host(dD, (1, m), np.float32)
        assert _dot_ok(got, ex, mag), f"impl {impl}"
        if impl in (0, 8):
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"impl {impl}: {int((got != want).sum())} of {m} differ"
        outs.setdefault(impl, []).append(got)
    assert np.array_equal(outs[2][0].view(np.uint32), outs[2][1].view(np.uint32))
    for d in (dW, dY, dD):
        fl.free(d)


@pytest.mark.parametrize("name,t", TYPES)
@pytest.mark.parametrize("m,k,n", [(1, 64, 1), (7, 64, 3), (300, 256, 5), (1000, 4096, 2), (33, 11008, 1), (9, 96, 15), (130, 320, 37), (515, 4096, 128)])
def test_mul_mat_ragged_shapes(fl, oracle, name, t, m, k, n):
    """Any M, K, N through the reference-order kernel (impl 8): the oracle's bits.  The default dispatch (impl 0) is the same kernel
    below 16 columns and the wgmma GEMM (reordering budget) from 16 columns on."""
    rng = np.random.default_rng(m + k + n)
    w = oracle.quantize_q4((rng.standard_normal((m, k)) * 0.05).astype(np.float32), t)
    x = rng.standard_normal((n, k)).astype(np.float32)
    ex, mag = oracle.mul_mat_q_exact(w, x, t)
    want = oracle.mul_mat_q(w, x, t)
    got0 = fl.mul_mat_q(w, x, t)
    assert _dot_ok(got0, ex, mag)
    if n < 16:
        assert np.array_equal(got0.view(np.uint32), want.view(np.uint32))
    dW, dY, dD = fl.to_device(w), fl.to_device(oracle.quantize_q8_0(x)), fl.alloc(m * n * 4)
    fl.check(fl.lib.fl_dev_memset(dD, 0xFF, m * n * 4))
    fl.check(fl.lib.fl_dev_mul_mat_q(t, dW, w.shape[1], m, k, dY, n, dD, m, 8))
    got = fl.to_host(dD, (n, m), np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"{int((got != want).sum())} of {got.size} differ"
    for d in (dW, dY, dD):
        fl.free(d)


def test_empty_and_invalid_inputs(fl):
    from fastllama_b200.cuda_abi import FlCudaError

    w = np.zeros((0, 40), dtype=np.uint8)
    assert fl.mul_mat_q(w, np.zeros((2, 64), dtype=np.float32), GGML_TYPE_Q4_0).shape == (2, 0)
    assert fl.quantize_q8_0(np.zeros((0, 64), dtype=np.float32)).shape == (0, 80)
    with pytest.raises(FlCudaError):
        fl.quantize_q8_0(np.zeros((1, 48), dtype=np.float32))          # k not a multiple of 32
    with pytest.raises(FlCudaError):
        fl.mul_mat_q(np.zeros((2, 20), dtype=np.uint8), np.zeros((1, 32), dtype=np.float32), 6)   # q8_0 weights
    with pytest.raises(FlCudaError):
        fl.get_rows_q(np.zeros((2, 40), dtype=np.uint8), np.array([5], dtype=np.int32), GGML_TYPE_Q4_0, 64)


def test_live_reference_q8_and_dots(fl, ref, oracle):
    rng = np.random.default_rng(99)
    k = 4096
    x = rng.standard_normal((9, k)).astype(np.float32)
    assert np.array_equal(fl.quantize_q8_0(x), ref.quantize_q8_0(x))
    for name, t in TYPES:
        w = ref.quantize_q4_reference((rng.standard_normal((64, k)) * 0.02).astype(np.float32), t)
        r = ref.mul_mat_q(w, x, t)
        ex, mag = oracle.mul_mat_q_exact(w, x, t)
        got = fl.mul_mat_q(w, x, t)
        assert _dot_ok(got, ex, mag)
        assert np.all(np.abs(got.astype(np.float64) - r) <= 2 * REORDER_BUDGET * mag + 1e-30)


@pytest.mark.parametrize("t", [GGML_TYPE_Q4_0, GGML_TYPE_Q4_1])
@pytest.mark.parametrize("m,k,n", [(33, 64, 9), (300, 256, 5), (1000, 11008, 37), (1024, 4096, 128), (514, 4096, 200), (16, 32, 1)])
def test_prompt_ingest_tensor_core_kernel(fl, oracle, t, m, k, n):
    """N > 1 (impl 3): integer block sums on the tensor cores (mma.sync m16n8k32 u8 x s8), scales in fp32 -- same budget
    as every other dot product against the order-free oracle, ragged M / N tails included; and it must agree with the
    plain kernel (impl 1) to within twice the budget and be run-to-run deterministic."""
    rng = np.random.default_rng(m + 3 * k + 7 * n)
    from oracle.pyoracle import np_quantize_q4_0, np_quantize_q4_1

    w = (rng.standard_normal((m, k)) * 0.03).astype(np.float32)
    wq = (np_quantize_q4_0 if t == GGML_TYPE_Q4_0 else np_quantize_q4_1)(w)
    x = rng.standard_normal((n, k)).astype(np.float32)
    ex, mag = oracle.mul_mat_q_exact(wq, x, t)
    q8 = oracle.quantize_q8_0(x)
    dW, dY, dD = fl.to_device(wq), fl.to_device(q8), fl.alloc(m * n * 4)
    outs = {}
    for impl in (3, 3, 1):
        fl.check(fl.lib.fl_dev_memset(dD, 0xFF, m * n * 4))
        fl.check(fl.lib.fl_dev_mul_mat_q(t, dW, wq.shape[1], m, k, dY, n, dD, m, impl))
        got = fl.to_host(dD, (n, m), np.float32)
        assert _dot_ok(got, ex, mag), f"impl {impl}"
        outs.setdefault(impl, []).append(got)
    assert np.array_equal(outs[3][0].view(np.uint32), outs[3][1].view(np.uint32))
    assert np.all(np.abs(outs[3][0].astype(np.float64) - outs[1][0]) <= 2 * REORDER_BUDGET * mag + 1e-30)
    for d in (dW, dY, dD):
        fl.free(d)


@pytest.mark.parametrize("t", [GGML_TYPE_Q4_0, GGML_TYPE_Q4_1])
@pytest.mark.parametrize("m,k,n", [(128, 128, 32), (300, 256, 5), (1000, 11008, 37), (1024, 4096, 128), (514, 4096, 200), (4096, 4096, 128)])
def test_prompt_ingest_tcgen05_kernel(fl, oracle, t, m, k, n):
    """N > 1 on the Hopper tensor cores (impl 4 = tile width chosen; 5 / 6 / 7 = column tiles of 32 / 64 / 64): one wgmma with 8-bit operands
    per quant block into registers, exact fp32 block scaling -- the same budget against the order-free oracle as every other dot
    product, ragged M / N / K-block tails included (TMA zero fill), run-to-run deterministic, and every tile width gives the same bits
    (the per-output arithmetic does not depend on the tiling)."""
    rng = np.random.default_rng(m + 3 * k + 7 * n)
    from oracle.pyoracle import np_quantize_q4_0, np_quantize_q4_1

    w = (rng.standard_normal((m, k)) * 0.03).astype(np.float32)
    wq = (np_quantize_q4_0 if t == GGML_TYPE_Q4_0 else np_quantize_q4_1)(w)
    x = rng.standard_normal((n, k)).astype(np.float32)
    ex, mag = oracle.mul_mat_q_exact(wq, x, t)
    q8 = oracle.quantize_q8_0(x)
    dW, dY, dD = fl.to_device(wq), fl.to_device(q8), fl.alloc(m * n * 4)
    outs = []
    for impl in (4, 4, 5, 6, 7):
        if impl == 7 and t == GGML_TYPE_Q4_1:
            continue
        fl.check(fl.lib.fl_dev_memset(dD, 0xFF, m * n * 4))
        fl.check(fl.lib.fl_dev_mul_mat_q(t, dW, wq.shape[1], m, k, dY, n, dD, m, impl))
        got = fl.to_host(dD, (n, m), np.float32)
        assert _dot_ok(got, ex, mag), f"impl {impl}"
        outs.append(got)
    for o in outs[1:]:
        assert np.array_equal(outs[0].view(np.uint32), o.view(np.uint32))
    for d in (dW, dY, dD):
        fl.free(d)
