"""GPU: every position-dependent kernel out to a full 2048-token context, bit for bit against the CPU stand-in of the device layer
(tests/mock, libfl_cpumodel.so: plain C over the oracle's row functions, pinned to the reference library by
tests/test_long_context_mock.py and tests/test_nodes_mock.py).

Part A runs the f32 ops of a multi-token eval through fl_dev_* on the views Model::eval makes (tests/llama_graph.py), with identical
seeded inputs on both sides: rope while its cos/sin table grows past 512 positions, diag_mask_inf + soft_max on rows up to 2048 long,
K.Q and V.P at every n_pos % 32 leftover form, rms_norm at subnormal and overflowing magnitudes, the KV cache writes near the end of
the cache, silu over every fp16 input, add / mul / repeat.  Part B runs the persistent token kernel at n_ctx 2048 for the attention
shapes of LLaMA 7B..65B and the other head dimensions it accepts.  Comparisons are on the uint32 bits.

FASTLLAMA_TEST_FL_LIB=<path of libfl_cpumodel.so> runs the file with the stand-in in place of the H100 library: the comparisons are
then trivially equal, but the views, shapes, offsets and canaries are exercised without a GPU."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from fastllama_b200.cuda_abi import FlCuda
from oracle.pyoracle import GGML_TYPE_Q4_0, GGML_TYPE_Q4_1
from tests.long_context_cases import (N_CTX, attn_input, bits, diff_report, put, rope_input, run_kq, run_mask_soft_max, run_rope, run_vp,
                                      scores_input, view)
from tests.mockbuild import ensure_mock
from tests.test_gpu_fused import test_token_kernel_has_the_reference_bits as token_kernel_check

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fl():
    path = os.environ.get("FASTLLAMA_TEST_FL_LIB")
    return FlCuda(path=path) if path else FlCuda()


@pytest.fixture(scope="module")
def cpu_model():
    path = os.path.join(ensure_mock(), "libfl_cpumodel.so")
    assert os.path.exists(path), f"{path} is missing: the CPU stand-in (tests/mock) did not build"
    return FlCuda(path=path)


def check(fails):
    assert not fails, "\n".join(fails)


# ---- A.1 rope -------------------------------------------------------------------------------------------------------------------
ROPE_HEADS = [(128, 32), (64, 32), (128, 40)]           # (head dim, heads), interleaved so that the hd 64 and hd 128 tables coexist
ROPE_NS = (1, 7, 128)


def rope_calls():
    """(N, n_past) in the order that grows the table: positions < 512 (the first table), one call that needs 513 positions (rebuilt
    at 1024), n_past 1000 (N = 128 needs 1128: rebuilt at 2048), then up to position 2047."""
    low = [(n, p) for n in ROPE_NS for p in (0, 511 - n, 512 - n)]
    return low + [(1, 512)] + [(n, 1000) for n in ROPE_NS] + [(n, p) for n in ROPE_NS for p in (1920, 2048 - n)]


def test_rope_while_its_table_grows_to_2048_positions(fl, cpu_model):
    fails, first = [], {}
    for n, n_past in rope_calls():
        for hd, n_head in ROPE_HEADS:
            x = rope_input(hd, n_head, n, n_past)
            got = run_rope(fl, x, n_past)
            first.setdefault((hd, n_head), (n, n_past, got))
            msg = diff_report(got, run_rope(cpu_model, x, n_past), ("position", "head", "column"), (n_past, 0, 0))
            if msg:
                fails.append(f"rope hd {hd} x {n_head} heads, N {n}, n_past {n_past}: {msg}")
    hd, n_head, n, n_past = 128, 32, 128, 1920                      # a permuted, non-contiguous view
    x = rope_input(hd, n_head, n, n_past)
    msg = diff_report(run_rope(fl, x, n_past, permuted=True), run_rope(cpu_model, x, n_past), ("position", "head", "column"), (n_past, 0, 0))
    if msg:
        fails.append(f"rope on a permuted view, hd {hd} x {n_head} heads, N {n}, n_past {n_past}: {msg}")
    for (hd, n_head), (n, n_past, got0) in first.items():           # after the rebuilds: the first call's bits again
        msg = diff_report(run_rope(fl, rope_input(hd, n_head, n, n_past), n_past), got0, ("position", "head", "column"), (n_past, 0, 0))
        if msg:
            fails.append(f"rope hd {hd} x {n_head} heads, N {n}, n_past {n_past} repeated after the table grew: {msg}")
    check(fails)


# ---- A.2 diag_mask_inf + soft_max -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sigma", [1, 30])
@pytest.mark.parametrize("n", ROPE_NS)
def test_mask_and_soft_max_on_rows_up_to_2048(fl, cpu_model, n, sigma):
    fails = []
    for n_past in (0, 511 - n, 512 - n, 1000, 1920, 2048 - n):
        s = scores_input(n_past, n, 8, sigma)
        (gm, gs), (wm, ws) = run_mask_soft_max(fl, s, n_past), run_mask_soft_max(cpu_model, s, n_past)
        for what, g, w in (("diag_mask_inf", gm, wm), ("soft_max", gs, ws)):
            msg = diff_report(g, w, ("head", "position", "column"), (0, n_past, 0))
            if msg:
                fails.append(f"{what}, n_past {n_past}, N {n}, sigma {sigma}: {msg}")
        assert np.abs(ws.sum(-1) - 1.0).max() < 1e-3 and (ws[:, ::5, 1:] == 0).all()       # the inputs reach the edges they are for
    check(fails)


# ---- A.3 mul_mat f32: K.Q and V.P on the cache views --------------------------------------------------------------------------------
def kq_vp_fails(fl, cpu_model, hd, n_head, n, n_pos):
    kc, q, vt, p = attn_input(hd, n_head, n, n_pos)
    fails = []
    for what, f in (("K.Q", lambda be: run_kq(be, kc, q, n_pos)), ("V.P", lambda be: run_vp(be, vt, p, hd))):
        msg = diff_report(f(fl), f(cpu_model), ("head", "token", "column"))
        if msg:
            fails.append(f"{what}, {n_head} heads of {hd}, N {n}, n_pos {n_pos} (n_pos % 32 = {n_pos % 32}): {msg}")
    return fails


def test_mul_mat_f32_at_every_leftover_form(fl, cpu_model):
    """n_pos = 2016 + r for every r in 0..31: V.P's inner length takes every leftover form of ggml_vec_dot_f32 (groups of 8 and 4 as
    product + add, up to 3 fmas), N = 5 columns is not a multiple of the kernel's 8-column tile."""
    check([f for r in range(32) for f in kq_vp_fails(fl, cpu_model, 128, 2, 5, 2016 + r)])


@pytest.mark.parametrize("n_pos", [2048, 1937])
def test_mul_mat_f32_at_7b_geometry(fl, cpu_model, n_pos):
    check(kq_vp_fails(fl, cpu_model, 128, 32, 128, n_pos))


# ---- A.4 rms_norm ---------------------------------------------------------------------------------------------------------------
def near_float_midpoint(row, n):
    """True when the exactly rounded double sum of the row's fp32 squares puts the float mean within 2^-40 relative of a rounding
    midpoint of float32: only there may a sum in another order round the mean to the neighbouring float."""
    sq = (row * row).astype(np.float64)
    m = math.fsum(sq.tolist()) / n
    if not math.isfinite(m) or m == 0.0:
        return False
    f = np.float32(m)
    other = np.nextafter(f, np.float32(np.inf) if float(f) < m else np.float32(-np.inf))
    mid = (float(f) + float(other)) / 2
    return abs(m - mid) <= abs(m) * 2.0 ** -40


@pytest.mark.parametrize("n", [1, 128, 512])
@pytest.mark.parametrize("n_embd", [4096, 5120, 6656, 8192])
def test_rms_norm_at_extreme_magnitudes(fl, cpu_model, n_embd, n):
    """Rows of magnitude 1e-30 (squares are 0 in fp32: the build has no flush-to-zero, so 1e-30 * 1000 must come out), 1e-19 (squares
    subnormal), 1, 1e18 and 1e20 (squares overflow to inf), and rows mixing them.  The double sum is added in another order than the
    stand-in's scalar loop, so a row may differ by 1 ulp where the exact sum puts the float mean within 2^-40 of a rounding midpoint;
    the test prints how many rows used that allowance (expected: none)."""
    rng = np.random.default_rng([4, n_embd, n])
    mags = np.array([1e-30, 1e-19, 1.0, 1e18, 1e20], dtype=np.float64)
    x = rng.standard_normal((n, n_embd))
    kind = (np.arange(n) + n_embd // 1024) % 6                              # 0..4: one magnitude, 5: every element picks one
    scale = np.where(kind[:, None] < 5, mags[np.minimum(kind, 4)][:, None], mags[rng.integers(0, 5, (n, n_embd))])
    x = (x * scale).astype(np.float32)

    def run(be):
        d, o = put(be, x), be.alloc(x.nbytes)
        be.check(be.lib.fl_dev_rms_norm(*(C.byref(view(be, p, (n_embd, n))) for p in (d, o))))
        out = be.to_host(o, x.shape, np.float32)
        be.free(d)
        be.free(o)
        return out

    got, want = run(fl), run(cpu_model)
    gb, wb = bits(got).astype(np.int64), bits(want).astype(np.int64)
    rows = np.flatnonzero((gb != wb).any(axis=1))
    allowed = [r for r in rows if np.abs(gb[r] - wb[r]).max() <= 1 and near_float_midpoint(x[r], n_embd)]
    print(f"rms_norm [{n_embd}, {n}]: {len(allowed)} rows used the 1-ulp allowance")
    bad = [r for r in rows if r not in allowed]
    assert not bad, f"rms_norm [{n_embd}, {n}], row {bad[0]} (kind {kind[bad[0]]}): {len(bad)} rows differ; " + \
        diff_report(got[bad], want[bad], ("row of the differing", "column"))
    assert np.isfinite(want).all() and (want[kind == 0] != 0).all()  # 1e-30 rows: mean 0, scale 1/sqrt(1e-6), not flushed


# ---- A.5 cpy_f32 into the KV cache -----------------------------------------------------------------------------------------------
KV_EMBD, KV_HEAD = 4096, 32


@pytest.mark.parametrize("n,n_past", [(1, 0), (1, 511), (1, 2047), (7, 504), (7, 1000), (7, 2041), (128, 0), (128, 384), (128, 1920)])
def test_kv_cache_writes_touch_only_their_window(fl, cpu_model, n, n_past):
    """K: Kcur [hd, n_head, N] into view_1d(k, N * n_embd, n_past * n_embd * 4).  V: transpose(Vcur [n_embd, N]) into
    view_2d(v, N, n_embd, n_ctx * 4, n_past * 4).  The caches start as a canary; nothing outside the window may change."""
    rng = np.random.default_rng([5, n, n_past])
    hd = KV_EMBD // KV_HEAD
    kcur = rng.standard_normal((n, KV_HEAD, hd)).astype(np.float32)
    vcur = rng.standard_normal((n, KV_EMBD)).astype(np.float32)
    k_canary = rng.standard_normal((N_CTX, KV_EMBD)).astype(np.float32)
    v_canary = rng.standard_normal((KV_EMBD, N_CTX)).astype(np.float32)

    def run(be):
        dk, dv, dkc, dvc = put(be, kcur), put(be, vcur), put(be, k_canary), put(be, v_canary)
        src_k, dst_k = view(be, dk, (hd, KV_HEAD, n)), view(be, dkc + n_past * KV_EMBD * 4, (n * KV_EMBD,))
        src_v = view(be, dv, (n, KV_EMBD), (KV_EMBD * 4, 4))
        dst_v = view(be, dvc + n_past * 4, (n, KV_EMBD), (4, N_CTX * 4))
        be.check(be.lib.fl_dev_cpy_f32(C.byref(src_k), C.byref(dst_k)))
        be.check(be.lib.fl_dev_cpy_f32(C.byref(src_v), C.byref(dst_v)))
        out = be.to_host(dkc, k_canary.shape, np.float32), be.to_host(dvc, v_canary.shape, np.float32)
        for d in (dk, dv, dkc, dvc):
            be.free(d)
        return out

    (gk, gv), (wk, wv) = run(fl), run(cpu_model)
    ek, ev = k_canary.copy(), v_canary.copy()
    ek[n_past:n_past + n] = kcur.reshape(n, KV_EMBD)
    ev[:, n_past:n_past + n] = vcur.T
    fails = [f"{what} vs {other}: {m}" for what, g, w, other, axes in
             (("K cache", gk, wk, "the CPU model", ("position", "column")), ("K cache", gk, ek, "canary + window", ("position", "column")),
              ("V cache", gv, wv, "the CPU model", ("column", "position")), ("V cache", gv, ev, "canary + window", ("column", "position")))
             for m in [diff_report(g, w, axes)] if m]
    check(fails)


def test_kqv_merge_at_128_tokens(fl, cpu_model):
    """cpy(permute(KQV [hd, N, n_head], 0, 2, 1, 3), [n_embd, N]) at N = 128."""
    n, hd = 128, KV_EMBD // KV_HEAD
    kqv = np.random.default_rng(6).standard_normal((KV_HEAD, n, hd)).astype(np.float32)

    def run(be):
        d, o = put(be, kqv), be.alloc(kqv.nbytes)
        be.check(be.lib.fl_dev_cpy_f32(C.byref(view(be, d, (hd, KV_HEAD, n), (4, hd * n * 4, hd * 4))), C.byref(view(be, o, (KV_EMBD, n)))))
        out = be.to_host(o, (n, KV_EMBD), np.float32)
        be.free(d)
        be.free(o)
        return out

    got = run(fl)
    check([f"KQV merge vs {w}: {m}" for w, ref in (("the CPU model", run(cpu_model)), ("numpy", kqv.transpose(1, 0, 2).reshape(n, KV_EMBD)))
           for m in [diff_report(got, ref, ("token", "column"))] if m])


# ---- A.6 silu, add, mul, repeat --------------------------------------------------------------------------------------------------
def test_silu_over_every_fp16_input_and_midpoint(fl, cpu_model):
    """Every fp16 bit pattern widened to fp32, and every fp32 value halfway between two neighbouring fp16 values (round-half-even
    decides which table entry it reads; 65520 rounds to inf).  NaN outputs are only checked to be NaN: the NaN inputs, because the
    kernel's __float2half_rn and the stand-in's F16C conversion give them different payloads and so read different (all NaN) table
    entries, and silu(-inf) (also from -65520), the table's -inf / inf, whose NaN the GPU's fp16 -> fp32 conversion does not carry
    over bit for bit."""
    h = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16).view(np.float16)
    f = h.astype(np.float32)
    fin = np.sort(f[np.isfinite(f)].astype(np.float64))
    fin = np.unique(np.concatenate([fin, [65536.0, -65536.0]]))     # the midpoints above 65504 and below -65504 as well
    mids = ((fin[:-1] + fin[1:]) / 2).astype(np.float32)
    x = np.concatenate([f, mids]).astype(np.float32)

    def run(be):
        d, o = put(be, x), be.alloc(x.nbytes)
        be.check(be.lib.fl_dev_silu(C.byref(view(be, d, (x.size,))), C.byref(view(be, o, (x.size,)))))
        out = be.to_host(o, x.shape, np.float32)
        be.free(d)
        be.free(o)
        return out

    got, want = run(fl), run(cpu_model)
    nan = np.isnan(want)
    assert np.array_equal(nan, np.isnan(got)) and np.array_equal(np.flatnonzero(nan), np.flatnonzero(np.isnan(x) | (x <= -65520)))
    msg = diff_report(got[~nan], want[~nan], ("input",))
    assert msg is None, f"silu: {msg}"


def test_add_mul_repeat_at_ffn_width(fl, cpu_model):
    """[11008, 512]: the FFN activations of a 512-token chunk; repeat broadcasts an [11008] row over the 512 columns."""
    rng = np.random.default_rng(7)
    a, b = (rng.standard_normal((512, 11008)) * 3).astype(np.float32), rng.standard_normal((512, 11008)).astype(np.float32)
    row = rng.standard_normal(11008).astype(np.float32)
    ne = (11008, 512)

    def run(be):
        da, db, dr, do = put(be, a), put(be, b), put(be, row), be.alloc(a.nbytes)
        va, vb, vo = view(be, da, ne), view(be, db, ne), view(be, do, ne)
        out = {}
        for name, call in (("add", lambda: be.lib.fl_dev_add(C.byref(va), C.byref(vb), C.byref(vo))),
                           ("mul", lambda: be.lib.fl_dev_mul(C.byref(va), C.byref(vb), C.byref(vo))),
                           ("repeat", lambda: be.lib.fl_dev_repeat(C.byref(view(be, dr, (11008, 1))), C.byref(vo)))):
            be.check(call())
            out[name] = be.to_host(do, a.shape, np.float32)
        for d in (da, db, dr, do):
            be.free(d)
        return out

    got, want = run(fl), run(cpu_model)
    check([f"{k}: {m}" for k in got for m in [diff_report(got[k], want[k], ("column", "row"))] if m])
    assert np.array_equal(bits(want["repeat"]), bits(np.broadcast_to(row, a.shape)))


# ---- B. the token kernel at n_ctx 2048 --------------------------------------------------------------------------------------------
# (type, n_embd, n_head, n_ff, n_past): one layer, a 320-entry vocabulary, random K/V caches of 2048 positions, two launches
TOKEN_CASES = (
    [(GGML_TYPE_Q4_0, 4096, 32, 11008, p) for p in (511, 512, 1023, 2047, 2015, 2023, 2027, 2028, 2031, 2046)]   # 7B, head_split 4
    + [(GGML_TYPE_Q4_1, 5120, 40, 13824, p) for p in (2047, 1300)]                                               # 13B, split 2
    + [(GGML_TYPE_Q4_0, 6656, 52, 1024, 2047), (GGML_TYPE_Q4_0, 8192, 64, 1024, 2047)]                           # 30B / 65B heads
    + [(GGML_TYPE_Q4_0, 2048, 32, 1024, 2047), (GGML_TYPE_Q4_0, 4096, 16, 1024, 2047),                           # hd 64, hd 256
       (GGML_TYPE_Q4_0, 256, 8, 1024, 2047), (GGML_TYPE_Q4_0, 256, 8, 1024, 2028),                               # hd 32: split 1
       (GGML_TYPE_Q4_1, 6144, 96, 1024, 2047)])                                                                  # 96 x 64: split 1
N_VOCAB = 320


class Recorder:
    """A backend that keeps every array it copies back to the host, in order.  The CPU model's one run and each GPU launch of
    test_token_kernel_has_the_reference_bits copy back the same buffers in the same order, so a mismatch it reports can be located."""

    def __init__(self, be):
        self.be, self.out = be, []

    def __getattr__(self, name):
        return getattr(self.be, name)

    def to_host(self, d, shape, dtype):
        a = self.be.to_host(d, shape, dtype)
        self.out.append(a)
        return a


def located_diffs(want, got, n_embd, n_head):
    """diff_report of every buffer of every GPU launch against the CPU model's, with the caches and n_embd vectors split by head."""
    hd, fails = n_embd // n_head, []
    for j, g in enumerate(got):
        w = want[j % len(want)]
        shape, names = {(N_CTX, n_embd): ((N_CTX, n_head, hd), ("position", "head", "column")),
                         (n_embd, N_CTX): ((n_head, hd, N_CTX), ("head", "column", "position")),
                         (n_embd,): ((n_head, hd), ("head", "column"))}.get(w.shape, (w.shape, ("element",)))
        msg = diff_report(g.reshape(shape), w.reshape(shape), names)
        if msg:
            fails.append(f"launch {j // len(want)}, buffer {j % len(want)} of shape {w.shape}: {msg}")
    return fails


@pytest.mark.parametrize("t,n_embd,n_head,n_ff,n_past", TOKEN_CASES)
def test_token_kernel_at_2048_positions(fl, cpu_model, t, n_embd, n_head, n_ff, n_past):
    """tests/test_gpu_fused.py::test_token_kernel_has_the_reference_bits at n_ctx 2048: the scores buffer and the weight ring share
    shared memory, the attention loops run over up to 2048 cached positions with every n_pos % 32 leftover form of V.P, and the rope
    table covers 2048 positions.  Logits, q, attention output and both caches: the CPU model's bits, on both launches.  A failure
    also lists every differing buffer with its first differing position, head and column."""
    gpu, cpu = Recorder(fl), Recorder(cpu_model)
    try:
        token_kernel_check(gpu, cpu, t, n_embd, n_head, n_ff, N_VOCAB, N_CTX, n_past, 1)
    except AssertionError as e:
        raise AssertionError("\n".join([str(e)] + located_diffs(cpu.out, gpu.out, n_embd, n_head))) from None
