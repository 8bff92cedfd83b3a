"""CPU: the stand-in of the device layer (tests/mock) against the reference library at a 2048-position context, bit for bit, on the
inputs of tests/test_gpu_long_context.py (tests/long_context_cases.py): rope at n_past 1920 for head dims 128 and 64, diag_mask_inf +
soft_max on [2048, 128, n_head], K.Q and V.P of a 7B layer with 128 tokens over all 2048 positions, and V.P at every n_pos % 32
leftover form.  The GPU tests compare the H100 with the stand-in; this file makes that a comparison with the reference."""
import os

import numpy as np
import pytest

from oracle.pyoracle import REF_GGML_SO
from tests import ggml_api as G
from tests.long_context_cases import N_CTX, attn_input, diff_report, rope_input, run_kq, run_mask_soft_max, run_rope, run_vp, scores_input
from tests.mockbuild import ensure_mock

pytestmark = pytest.mark.skipif(not os.path.exists(REF_GGML_SO), reason="oracle/_ref not built")


@pytest.fixture(scope="module")
def libs():
    from fastllama_b200.cuda_abi import FlCuda

    path = os.path.join(ensure_mock(), "libfl_cpumodel.so")
    if not os.path.exists(path):
        pytest.skip("tests/mock not built")
    return G.Ggml(REF_GGML_SO), FlCuda(path=path)


def ref_run(g, nbytes, build):
    """build(g, arena) -> output tensor of one graph on the reference library; its values after compute."""
    a = g.context(nbytes + (16 << 20))
    out = build(g, a)
    gf = G.new_graph()
    g.build_forward_expand(gf, out)
    g.graph_compute(a.ctx, gf)
    v = a.numpy(out).copy()
    a.free()
    return v


def tensor(g, a, x, ne):
    t = {1: g.new_tensor_1d, 2: g.new_tensor_2d, 3: g.new_tensor_3d}[len(ne)](a.ctx, G.F32, *ne)
    a.set(t, x)
    return t


def ref_rope(g, x, n_past):
    n, n_head, hd = x.shape
    return ref_run(g, 2 * x.nbytes, lambda g, a: g.rope(a.ctx, tensor(g, a, x, (hd, n_head, n)), n_past, hd, 0))


def ref_mask_soft_max(g, s, n_past):
    return ref_run(g, 2 * s.nbytes, lambda g, a: g.soft_max(a.ctx, g.diag_mask_inf(a.ctx, tensor(g, a, s, s.shape[::-1]), n_past)))


def ref_kq(g, kc, q, n_pos):
    n, n_head, hd = q.shape
    n_embd = hd * n_head

    def build(g, a):
        k = tensor(g, a, kc, (kc.size,))
        kv = g.permute(a.ctx, g.reshape_3d(a.ctx, g.view_1d(a.ctx, k, n_pos * n_embd, 0), hd, n_head, n_pos), 0, 2, 1, 3)
        return g.mul_mat(a.ctx, kv, g.permute(a.ctx, tensor(g, a, q, (hd, n_head, n)), 0, 2, 1, 3))
    return ref_run(g, kc.nbytes + 2 * q.nbytes + n_pos * n * n_head * 4, build)


def ref_vp(g, vt, p, hd):
    n_head, n, n_pos = p.shape

    def build(g, a):
        v = g.view_3d(a.ctx, tensor(g, a, vt, (N_CTX, vt.shape[0])), n_pos, hd, n_head, N_CTX * 4, N_CTX * 4 * hd, 0)
        return g.mul_mat(a.ctx, v, tensor(g, a, p, (n_pos, n, n_head)))
    return ref_run(g, vt.nbytes + 2 * p.nbytes, build)


@pytest.mark.parametrize("hd,n_head", [(128, 32), (64, 32)])
def test_rope_at_position_1920(libs, hd, n_head):
    ref, mock = libs
    x = rope_input(hd, n_head, 128, 1920)
    msg = diff_report(run_rope(mock, x, 1920), ref_rope(ref, x, 1920), ("position", "head", "column"), (1920, 0, 0))
    assert msg is None, msg


@pytest.mark.parametrize("sigma", [1, 30])
def test_mask_and_soft_max_at_2048_positions(libs, sigma):
    ref, mock = libs
    s = scores_input(1920, 128, 8, sigma)
    msg = diff_report(run_mask_soft_max(mock, s, 1920)[1], ref_mask_soft_max(ref, s, 1920), ("head", "position", "column"), (0, 1920, 0))
    assert msg is None, msg


@pytest.mark.parametrize("hd,n_head,n,n_pos", [(128, 32, 128, 2048)] + [(128, 2, 5, 2016 + r) for r in range(32)])
def test_attention_products(libs, hd, n_head, n, n_pos):
    ref, mock = libs
    kc, q, vt, p = attn_input(hd, n_head, n, n_pos)
    for what, got, want in (("K.Q", run_kq(mock, kc, q, n_pos), ref_kq(ref, kc, q, n_pos)), ("V.P", run_vp(mock, vt, p, hd), ref_vp(ref, vt, p, hd))):
        msg = diff_report(got, want, ("head", "token", "column"))
        assert msg is None, f"{what}: {msg}"
