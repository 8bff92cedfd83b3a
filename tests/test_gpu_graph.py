"""GPU: boundary B1 end to end.  The same ggml-API script runs on the reference library (CPU,
oracle/_ref/libggml_ref.so) and on libggml_b200 (H100); results are compared op by op and for whole
LLaMA eval graphs (prompt + decode steps, KV cache carried across ggml_graph_compute calls).

Bar: the reference library's BITS, op by op and at the logits of whole eval graphs -- every fp32 operation follows the reference's
order (fl_exact.cuh).  The one op with a stated tolerance is rms_norm, whose double-precision sum of squares is added in another order
(one ulp of the float mean when the double sum sits on a rounding boundary; never observed in these graphs).
"""
import math
import os

import numpy as np
import pytest

os.environ.setdefault("FASTLLAMA_B200_SYNC_ALL", "1")     # copy every node back so all of them can be compared

from fastllama_b200.build import lib_path  # noqa: E402
from oracle.pyoracle import REF_GGML_SO, Oracle  # noqa: E402
from tests import ggml_api as G  # noqa: E402
from tests.llama_graph import HParams, MiniLlama, make_weights  # noqa: E402

pytestmark = pytest.mark.gpu
OURS = os.environ.get("FASTLLAMA_TEST_OURS", lib_path("libggml_b200.so"))


@pytest.fixture(scope="module")
def libs(ref):            # `ref` skips when oracle/_ref is absent
    return G.Ggml(REF_GGML_SO), G.Ggml(OURS)


def run(g, build, seed=0, mem=32 << 20):
    """build(g, arena, rng) -> list of output tensors; returns their host values after compute."""
    a = g.context(mem)
    outs = build(g, a, np.random.default_rng(seed))
    gf = G.new_graph()
    for o in outs:
        g.build_forward_expand(gf, o)
    g.graph_compute(a.ctx, gf)
    vals = [a.numpy(o).copy() for o in outs]
    a.free()
    return vals


def both(libs, build, seed=0):
    return run(libs[0], build, seed), run(libs[1], build, seed)


def f32(g, a, rng, *ne, scale=1.0):
    t = {1: g.new_tensor_1d, 2: g.new_tensor_2d, 3: g.new_tensor_3d}[len(ne)](a.ctx, G.F32, *ne)
    a.set(t, (rng.standard_normal(ne[::-1]) * scale).astype(np.float32))
    return t


def bits(x):
    return np.ascontiguousarray(x).view(np.uint32)


def test_elementwise_exact(libs):
    def build(g, a, rng):
        x, y, row = f32(g, a, rng, 96, 5), f32(g, a, rng, 96, 5), f32(g, a, rng, 96)
        return [g.add(a.ctx, x, y), g.mul(a.ctx, g.repeat(a.ctx, row, x), x), g.scale(a.ctx, g.add(a.ctx, y, y), g.new_f32(a.ctx, 0.125)),
                g.silu(a.ctx, g.mul(a.ctx, x, y))]
    r, o = both(libs, build)
    for i, (a_, b_) in enumerate(zip(r, o)):
        assert np.array_equal(bits(a_), bits(b_)), f"output {i}"


def test_silu_table_exact_over_range(libs):
    def build(g, a, rng):
        x = g.new_tensor_1d(a.ctx, G.F32, 8192)
        a.set(x, np.linspace(-20, 20, 8192).astype(np.float32))
        return [g.silu(a.ctx, x)]
    r, o = both(libs, build)
    assert np.array_equal(bits(r[0]), bits(o[0]))


def test_rms_norm(libs):
    def build(g, a, rng):
        return [g.rms_norm(a.ctx, f32(g, a, rng, 4096, 3, scale=2.0)), g.rms_norm(a.ctx, f32(g, a, rng, 160, 7, scale=1e-3))]
    r, o = both(libs, build)
    for a_, b_ in zip(r, o):          # double-precision sum in a different order: at most 1 ulp through the float mean
        assert np.allclose(a_, b_, rtol=2.5e-7, atol=0)


def test_rope_and_mask_and_softmax(libs):
    def build(g, a, rng):
        q = g.rope(a.ctx, f32(g, a, rng, 32, 4, 6), 9, 32, 0)                 # [head_dim, heads, tokens], n_past 9
        kq = f32(g, a, rng, 15, 6, 4, scale=3.0)                               # [n_past+N, N, heads]
        sm = g.soft_max(a.ctx, g.diag_mask_inf(a.ctx, kq, 9))
        return [q, sm]
    r, o = both(libs, build)
    assert np.array_equal(bits(r[0]), bits(o[0])), "rope"              # host-built cos/sin table (libm), the reference build's fma contraction
    assert np.array_equal(r[1] == 0, o[1] == 0), "mask pattern"
    assert np.array_equal(bits(r[1]), bits(o[1])), "soft_max"          # fp16 table values: the double sum is exact in any order
    assert np.allclose(o[1].sum(-1), 1.0, atol=1e-3)


def test_cpy_strided_and_mul_mat_f32(libs):
    def build(g, a, rng):
        x = f32(g, a, rng, 24, 5)                                             # [n_embd, N]
        dst = g.new_tensor_2d(a.ctx, G.F32, 5, 24)
        xt = g.cpy(a.ctx, g.transpose(a.ctx, x), dst)                          # transposed copy (the V-cache write)
        k = f32(g, a, rng, 16, 11, 3)
        q = f32(g, a, rng, 16, 4, 3)
        kq = g.mul_mat(a.ctx, k, q)                                           # [11, 4, 3]
        p3 = g.permute(a.ctx, f32(g, a, rng, 8, 3, 5), 0, 2, 1, 3)
        merged = g.cpy(a.ctx, p3, g.new_tensor_2d(a.ctx, G.F32, 24, 5))
        return [xt, kq, merged]
    r, o = both(libs, build)
    assert np.array_equal(bits(r[0]), bits(o[0]))
    assert np.array_equal(bits(r[1]), bits(o[1]))          # mul_mat f32: ggml_vec_dot_f32's order, inner length 16 = leftovers only
    assert np.array_equal(bits(r[2]), bits(o[2]))


def test_mul_mat_f32_attention_shapes_of_a_prompt_eval(libs):
    """K*Q and V*P of a multi-token eval with the strided operands Model::eval uses (K as a permuted view of the cache, V^T with n_ctx
    row stride); inner lengths 128 (no leftovers) and 205 (13 leftovers: 8 + 4 products-then-adds and one fma in the reference build):
    the same bits as the reference library."""
    def build(g, a, rng):
        hd, n_pos, n, heads, n_ctx = 128, 205, 96, 3, 256
        kc = f32(g, a, rng, hd * heads, n_pos)                                                    # cache rows [pos][n_embd]
        k = g.permute(a.ctx, g.reshape_3d(a.ctx, kc, hd, heads, n_pos), 0, 2, 1, 3)               # [hd, n_pos, heads]
        q = f32(g, a, rng, hd, n, heads)
        kq = g.mul_mat(a.ctx, k, q)                                                               # [n_pos, n, heads]
        vt = f32(g, a, rng, n_ctx, hd * heads)                                                    # V^T [n_embd][n_ctx]
        v = g.view_3d(a.ctx, vt, n_pos, hd, heads, n_ctx * 4, n_ctx * 4 * hd, 0)                  # [n_pos, hd, heads]
        p = f32(g, a, rng, n_pos, n, heads)
        kqv = g.mul_mat(a.ctx, v, p)                                                              # [hd, n, heads]
        return [kq, kqv]
    r, o = both(libs, build)
    assert np.array_equal(bits(r[0]), bits(o[0]))
    assert np.array_equal(bits(r[1]), bits(o[1]))


@pytest.mark.parametrize("t", [G.Q4_0, G.Q4_1])
def test_get_rows_and_quantised_mul_mat(libs, t):
    orc = Oracle()

    def build(g, a, rng):
        w = orc.quantize_q4((rng.standard_normal((48, 256)) * 0.05).astype(np.float32), t)
        wt = g.new_tensor_2d(a.ctx, t, 256, 48)
        a.set(wt, w)
        ids = g.new_tensor_1d(a.ctx, G.I32, 3)
        a.set(ids, np.array([47, 0, 13], dtype=np.int32))
        x = f32(g, a, rng, 256, 3)
        return [g.get_rows(a.ctx, wt, ids), g.mul_mat(a.ctx, wt, x)]
    r, o = both(libs, build)
    assert np.array_equal(bits(r[0]), bits(o[0]))
    assert np.array_equal(bits(r[1]), bits(o[1]))


@pytest.mark.parametrize("t", [G.Q4_0, G.Q4_1])
@pytest.mark.parametrize("dims", ["generic", "fused"])
def test_llama_eval_prompt_then_decode(libs, t, dims):
    """Model::eval semantics: a 5-token prompt (N = 5), then three decode steps (N = 1) that read the
    KV cache written by the earlier graphs.  "generic": n_ff = 352 rows are not 16-byte multiples, so the decode steps
    run node by node; "fused": shapes the decode plan accepts, so they run as the persistent token kernel."""
    orc = Oracle()
    hp = HParams(n_vocab=96, n_embd=128, n_head=4, n_layer=3, n_mult=32, n_ctx=32) if dims == "generic" else \
        HParams(n_vocab=96, n_embd=256, n_head=4, n_layer=3, n_mult=256, n_ctx=32)
    w = make_weights(hp, t, lambda x, tt: orc.quantize_q4(x, tt), seed=3)
    models = [MiniLlama(g, hp, w, compute_mb=32) for g in libs]
    steps = [([5, 17, 3, 80, 41], 0), ([7], 5), ([60], 6), ([2], 7)]
    for tokens, n_past in steps:
        outs = []
        for m in models:
            c, gf, named = m.eval(tokens, n_past)
            m.compute(c, gf)
            outs.append((c.numpy(named["logits"]).copy(), c.numpy(named["embeddings"]).copy()))
        (rl, re), (ol, oe) = outs
        assert np.isfinite(ol).all()
        nd = int((bits(rl) != bits(ol)).sum()), int((bits(re) != bits(oe)).sum())
        assert nd == (0, 0), (n_past, nd, rl.size, float(np.abs(rl - ol).max()), float(np.abs(rl).max()))      # the reference library's bits
    import ctypes as C
    assert C.CDLL(OURS).ggml_b200_decode_mode() == (2 if dims == "fused" else 0)


def test_unsupported_op_aborts_loudly():
    """No CPU fallback: an f16 KV cache copy (outside the supported set) must abort, not fall back."""
    import subprocess
    import sys

    code = (
        "import numpy as np\n"
        "from tests import ggml_api as G\n"
        f"g = G.Ggml({OURS!r})\n"
        "a = g.context(1 << 20)\n"
        "x = g.new_tensor_1d(a.ctx, G.F32, 64)\n"
        "h = g.new_tensor_1d(a.ctx, G.F16, 64)\n"
        "gf = G.new_graph(); g.build_forward_expand(gf, g.cpy(a.ctx, x, h)); g.graph_compute(a.ctx, gf)\n"
        "print('survived')\n"
    )
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert res.returncode != 0 and "survived" not in res.stdout
    assert "GGML_B200_ASSERT" in res.stderr
