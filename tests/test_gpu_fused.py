"""GPU: the fused decode kernels through the C ABI (fl_dev_mv_fused, fl_dev_attn_decode) against the
oracle: every prologue (plain / rms_norm*gamma / silu*mul) and epilogue (store / residual / rope+KV)
on small, ragged and full LLaMA shapes.  Prologue arithmetic is single fp32 operations + the bit-exact
q8_0 quantiser, so the q8 vector the kernel builds equals the oracle's and the dot products must sit in
the same 2e-6 * sum|d q| reordering budget as the plain matvec; rope/residual add a few ulp."""
import ctypes as C
import math

import numpy as np
import pytest

from oracle.pyoracle import GGML_TYPE_Q4_0, GGML_TYPE_Q4_1, np_quantize_q4_0, np_quantize_q4_1

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fl():
    from fastllama_b200.cuda_abi import FlCuda

    return FlCuda()


def silu_tab(x):
    h = x.astype(np.float16).astype(np.float32)
    return (h / (1.0 + np.exp(-h, dtype=np.float32))).astype(np.float16).astype(np.float32)


def quant(w, t):
    return (np_quantize_q4_0 if t == GGML_TYPE_Q4_0 else np_quantize_q4_1)(w)


def rope_ref(v, pos, hd):
    """mode-0 rope of a [n_embd] vector at absolute position pos (reference lib/ggml.c:8655-8682)."""
    out = v.copy()
    ts = np.float32(10000.0) ** np.float32(-2.0 / hd)
    for h0 in range(0, v.size, hd):
        theta = np.float32(pos)
        for i in range(0, hd, 2):
            c, s = np.cos(theta, dtype=np.float32), np.sin(theta, dtype=np.float32)
            x0, x1 = v[h0 + i], v[h0 + i + 1]
            out[h0 + i] = x0 * c - x1 * s
            out[h0 + i + 1] = x0 * s + x1 * c
            theta = np.float32(theta * ts)
    return out


@pytest.mark.parametrize("t", [GGML_TYPE_Q4_0, GGML_TYPE_Q4_1])
@pytest.mark.parametrize("k,rows", [(128, (2,)), (256, (6, 10)), (4096, (4096,)), (4096, (11008, 11008)), (11008, (4096,)), (5120, (5120, 5120, 5120))])
@pytest.mark.parametrize("pro", [0, 1, 2])
def test_mv_fused_prologues_and_segments(fl, oracle, t, k, rows, pro):
    from fastllama_b200.cuda_abi import EPI_RESADD, EPI_STORE, FlMvArgs

    rng = np.random.default_rng(k + sum(rows) + pro)
    ws = [quant((rng.standard_normal((m, k)) * 0.02).astype(np.float32), t) for m in rows]
    x = (rng.standard_normal(k) * 1.5).astype(np.float32)
    gamma = (1.0 + 0.1 * rng.standard_normal(k)).astype(np.float32)
    b = rng.standard_normal(k).astype(np.float32)
    res = rng.standard_normal(rows[0]).astype(np.float32)
    if pro == 0:
        v = x
    elif pro == 1:
        scale = np.float32(1.0) / np.sqrt(np.float32((x.astype(np.float64) ** 2).sum() / k) + np.float32(1e-6), dtype=np.float32)
        v = gamma * (x * scale)
    else:
        v = silu_tab(x) * b
    epi = EPI_RESADD if len(rows) == 1 else EPI_STORE
    a = FlMvArgs()
    a.type, a.K, a.nseg, a.pro, a.epi = t, k, len(rows), pro, epi
    dws, douts = [], []
    for i, (w, m) in enumerate(zip(ws, rows)):
        dws.append(fl.to_device(w))
        douts.append(fl.alloc(m * 4))
        a.seg_w[i], a.seg_rows[i], a.seg_dst[i] = dws[-1], m, douts[-1]
    dx, dg, db, dr, dn = fl.to_device(x), fl.to_device(gamma), fl.to_device(b), fl.to_device(res), fl.alloc(k * 4)
    a.x, a.gamma, a.b, a.res, a.normed_out = dx, dg, db, dr, dn
    fl.check(fl.lib.fl_dev_mv_fused(C.byref(a)))
    for i, (w, m) in enumerate(zip(ws, rows)):
        got = fl.to_host(douts[i], (m,), np.float32)
        ex, mag = oracle.mul_mat_q_exact(w, v[None, :], t)
        ex, mag = ex[0], mag[0]
        if epi == EPI_RESADD:
            ex = ex + res
        # 2e-6 reordering budget + 1 ulp of the residual add
        assert np.all(np.abs(got - ex) <= 2e-6 * mag + 2.4e-7 * (np.abs(ex) + np.abs(res if epi == EPI_RESADD else 0)) + 1e-30), (i, np.abs(got - ex).max())
    if pro == 1:
        assert np.allclose(fl.to_host(dn, (k,), np.float32), v, rtol=3e-7, atol=0)
    for d in dws + douts + [dx, dg, db, dr, dn]:
        fl.free(d)


@pytest.mark.parametrize("t", [GGML_TYPE_Q4_0, GGML_TYPE_Q4_1])
@pytest.mark.parametrize("n_embd,hd,n_ctx,n_past", [(256, 64, 32, 0), (256, 64, 32, 17), (4096, 128, 512, 300)])
def test_mv_fused_qkv_epilogue(fl, oracle, t, n_embd, hd, n_ctx, n_past):
    from fastllama_b200.cuda_abi import EPI_QKV, PRO_RMSNORM, FlMvArgs

    rng = np.random.default_rng(n_embd + n_past)
    ws = [quant((rng.standard_normal((n_embd, n_embd)) * 0.03).astype(np.float32), t) for _ in range(3)]
    x = rng.standard_normal(n_embd).astype(np.float32)
    gamma = (1.0 + 0.1 * rng.standard_normal(n_embd)).astype(np.float32)
    scale = np.float32(1.0) / np.sqrt(np.float32((x.astype(np.float64) ** 2).sum() / n_embd) + np.float32(1e-6), dtype=np.float32)
    v = gamma * (x * scale)
    kc = rng.standard_normal((n_ctx, n_embd)).astype(np.float32)
    vc = rng.standard_normal((n_embd, n_ctx)).astype(np.float32)
    a = FlMvArgs()
    a.type, a.K, a.nseg, a.pro, a.epi = t, n_embd, 3, PRO_RMSNORM, EPI_QKV
    dws = [fl.to_device(w) for w in ws]
    dq, dk, dv = fl.alloc(n_embd * 4), fl.to_device(kc), fl.to_device(vc)
    dnp = fl.to_device(np.array([n_past], dtype=np.int32))
    dx, dg = fl.to_device(x), fl.to_device(gamma)
    for i in range(3):
        a.seg_w[i], a.seg_rows[i] = dws[i], n_embd
    a.seg_dst[0] = dq
    a.x, a.gamma, a.n_past, a.n_ctx, a.n_embd, a.head_dim, a.kcache, a.vcache = dx, dg, dnp, n_ctx, n_embd, hd, dk, dv
    fl.check(fl.lib.fl_dev_rope_table(hd, n_ctx))
    fl.check(fl.lib.fl_dev_mv_fused(C.byref(a)))
    raw = [oracle.mul_mat_q_exact(w, v[None, :], t) for w in ws]
    q_ref, k_ref, v_ref = rope_ref(raw[0][0][0].astype(np.float32), n_past, hd), rope_ref(raw[1][0][0].astype(np.float32), n_past, hd), raw[2][0][0]
    tol = lambda mag: 4e-6 * mag.max() + 1e-6
    assert np.abs(fl.to_host(dq, (n_embd,), np.float32) - q_ref).max() <= tol(raw[0][1])
    kc2 = fl.to_host(dk, (n_ctx, n_embd), np.float32)
    vc2 = fl.to_host(dv, (n_embd, n_ctx), np.float32)
    assert np.abs(kc2[n_past] - k_ref).max() <= tol(raw[1][1])
    assert np.abs(vc2[:, n_past] - v_ref).max() <= tol(raw[2][1])
    mask = np.ones(n_ctx, bool)
    mask[n_past] = False
    assert np.array_equal(kc2[mask], kc[mask]) and np.array_equal(vc2[:, mask], vc[:, mask])      # nothing else touched
    for d in dws + [dq, dk, dv, dnp, dx, dg]:
        fl.free(d)


@pytest.mark.parametrize("n_embd,n_head,n_ctx,n_past", [(256, 4, 32, 0), (256, 4, 32, 31), (4096, 32, 512, 200)])
def test_attn_decode(fl, n_embd, n_head, n_ctx, n_past):
    rng = np.random.default_rng(n_past + n_embd)
    hd = n_embd // n_head
    q = rng.standard_normal(n_embd).astype(np.float32)
    kc = rng.standard_normal((n_ctx, n_embd)).astype(np.float32)
    vc = rng.standard_normal((n_embd, n_ctx)).astype(np.float32)
    scale = np.float32(1.0 / math.sqrt(hd))
    dq, dk, dv, do = fl.to_device(q), fl.to_device(kc), fl.to_device(vc), fl.alloc(n_embd * 4)
    dnp = fl.to_device(np.array([n_past], dtype=np.int32))
    fl.check(fl.lib.fl_dev_attn_decode(dq, dk, dv, do, dnp, n_embd, n_head, hd, n_ctx, scale))
    got = fl.to_host(do, (n_embd,), np.float32)
    want = np.zeros(n_embd, dtype=np.float32)
    n_pos = n_past + 1
    for h in range(n_head):
        s = (kc[:n_pos, h * hd:(h + 1) * hd].astype(np.float64) @ q[h * hd:(h + 1) * hd].astype(np.float64)).astype(np.float32) * scale
        e = np.exp((s - s.max()).astype(np.float16).astype(np.float32), dtype=np.float32).astype(np.float16).astype(np.float32)
        p = e * np.float32(1.0 / e.astype(np.float64).sum())
        want[h * hd:(h + 1) * hd] = (vc[h * hd:(h + 1) * hd, :n_pos].astype(np.float64) @ p.astype(np.float64)).astype(np.float32)
    # scores differ in the last ulps from the double-precision restatement; an fp16 table flip moves one
    # probability by <= 2^-11 relative, so 2e-3 of the output scale bounds it
    assert np.abs(got - want).max() <= 2e-3 * np.abs(want).max()
    for d in (dq, dk, dv, do, dnp):
        fl.free(d)


@pytest.fixture(scope="module")
def cpu_model():
    """The CPU stand-in of the device layer (tests/mock: the oracle's row functions behind the same C ABI), built under its own
    soname so that it can sit next to the real libfl_cuda.so in this process."""
    import os

    from fastllama_b200.cuda_abi import FlCuda
    from tests.mockbuild import ensure_mock

    path = os.path.join(ensure_mock(), "libfl_cpumodel.so")
    if not os.path.exists(path):
        pytest.skip("tests/mock not built")
    return FlCuda(path=path)


@pytest.mark.parametrize("t", [GGML_TYPE_Q4_0, GGML_TYPE_Q4_1])
@pytest.mark.parametrize("n_embd,n_head,n_ff,n_vocab,n_ctx,n_past,n_layer",
                         [(256, 4, 768, 512, 32, 5, 2), (512, 4, 1408, 300, 64, 40, 2), (4096, 32, 11008, 32000, 512, 37, 2), (4096, 32, 11008, 2000, 512, 300, 1),
                          (5120, 40, 13824, 32000, 512, 300, 1)])
def test_token_kernel_has_the_reference_bits(fl, cpu_model, t, n_embd, n_head, n_ff, n_vocab, n_ctx, n_past, n_layer):
    """The persistent token kernel (fl_token_plan_*) against the CPU model of the same steps, which is built from the oracle's
    row functions (the reference's AVX2 accumulation order, pinned to the reference library in tests/test_oracle.py): logits, q,
    attention output and the KV cache rows must be IDENTICAL, bit for bit."""
    from fastllama_b200.cuda_abi import EPI_QKV, EPI_RESADD, EPI_STORE, PRO_RMSNORM, PRO_SILUMUL, FlMvArgs, FlTokenStep

    rng = np.random.default_rng(n_embd + n_past)
    hd = n_embd // n_head
    scale = np.float32(1.0 / math.sqrt(hd))

    def wq(m, k, s=0.03):
        return quant((rng.standard_normal((m, k)) * s).astype(np.float32), t)

    def gam(n):
        return (1.0 + 0.1 * rng.standard_normal(n)).astype(np.float32)

    x0 = rng.standard_normal(n_embd).astype(np.float32)
    layers = []
    for _ in range(n_layer):
        layers.append(dict(wq=wq(n_embd, n_embd), wk=wq(n_embd, n_embd), wv=wq(n_embd, n_embd), wo=wq(n_embd, n_embd), w1=wq(n_ff, n_embd), w3=wq(n_ff, n_embd),
                           w2=wq(n_embd, n_ff), g1=gam(n_embd), g2=gam(n_embd), kc=rng.standard_normal((n_ctx, n_embd)).astype(np.float32),
                           vc=rng.standard_normal((n_embd, n_ctx)).astype(np.float32)))
    w_out, g_out = wq(n_vocab, n_embd), gam(n_embd)

    def run(be, relaunches):
        keep = []

        def dev(a):
            p = be.to_device(a)
            keep.append(p)
            return p

        def buf(n):
            p = be.alloc(n * 4)
            be.check(be.lib.fl_dev_memset(p, 0, n * 4))
            keep.append(p)
            return p

        be.check(be.lib.fl_dev_rope_table(hd, n_ctx))
        dnp = dev(np.array([n_past], dtype=np.int32))
        W = [{k: dev(v) for k, v in L.items() if k not in ("kc", "vc")} for L in layers]
        d_out, d_gout = dev(w_out), dev(g_out)
        results = []
        for _ in range(relaunches):
            xa, xb, q, att, m1, m3, emb, logits = buf(n_embd), buf(n_embd), buf(n_embd), buf(n_embd), buf(n_ff), buf(n_ff), buf(n_embd), buf(n_vocab)
            be.check(be.lib.fl_h2d(xa, x0.ctypes.data, n_embd * 4))
            steps, kvs = [], []
            for L, Lh in zip(W, layers):
                kc, vc = dev(Lh["kc"]), dev(Lh["vc"])
                kvs.append((kc, vc))
                a = FlMvArgs()
                a.type, a.K, a.nseg, a.pro, a.epi = t, n_embd, 3, PRO_RMSNORM, EPI_QKV
                for i, w in enumerate((L["wq"], L["wk"], L["wv"])):
                    a.seg_w[i], a.seg_rows[i] = w, n_embd
                a.seg_dst[0] = q
                a.x, a.gamma, a.n_past, a.n_ctx, a.n_embd, a.head_dim, a.kcache, a.vcache = xa, L["g1"], dnp, n_ctx, n_embd, hd, kc, vc
                steps.append(("mv", a))
                steps.append(("attn", (q, kc, vc, att)))
                a = FlMvArgs()
                a.type, a.K, a.nseg, a.pro, a.epi = t, n_embd, 1, 0, EPI_RESADD
                a.seg_w[0], a.seg_rows[0], a.seg_dst[0], a.x, a.res = L["wo"], n_embd, xb, att, xa
                steps.append(("mv", a))
                a = FlMvArgs()
                a.type, a.K, a.nseg, a.pro, a.epi = t, n_embd, 2, PRO_RMSNORM, EPI_STORE
                a.seg_w[0], a.seg_rows[0], a.seg_dst[0] = L["w1"], n_ff, m1
                a.seg_w[1], a.seg_rows[1], a.seg_dst[1] = L["w3"], n_ff, m3
                a.x, a.gamma = xb, L["g2"]
                steps.append(("mv", a))
                a = FlMvArgs()
                a.type, a.K, a.nseg, a.pro, a.epi = t, n_ff, 1, PRO_SILUMUL, EPI_RESADD
                a.seg_w[0], a.seg_rows[0], a.seg_dst[0], a.x, a.b, a.res = L["w2"], n_embd, xa, m1, m3, xb
                steps.append(("mv", a))
            a = FlMvArgs()
            a.type, a.K, a.nseg, a.pro, a.epi = t, n_embd, 1, PRO_RMSNORM, EPI_STORE
            a.seg_w[0], a.seg_rows[0], a.seg_dst[0], a.x, a.gamma, a.normed_out = d_out, n_vocab, logits, xa, d_gout, emb
            steps.append(("mv", a))
            arr = (FlTokenStep * len(steps))()
            for i, (kind, s) in enumerate(steps):
                if kind == "mv":
                    arr[i].kind, arr[i].mv = 0, s
                else:
                    arr[i].kind = 1
                    arr[i].q, arr[i].kcache, arr[i].vcache, arr[i].out, arr[i].n_past = s[0], s[1], s[2], s[3], dnp
                    arr[i].k_row_stride, arr[i].n_head, arr[i].head_dim, arr[i].n_ctx, arr[i].scale = n_embd, n_head, hd, n_ctx, scale
            plan = C.c_void_p()
            be.check(be.lib.fl_token_plan_create(arr, len(steps), C.byref(plan)))
            be.check(be.lib.fl_token_plan_launch(plan))
            be.check(be.lib.fl_sync())
            assert be.lib.fl_token_plan_error(plan) == 0
            r = {k: be.to_host(p, (n,), np.float32) for k, (p, n) in dict(xa=(xa, n_embd), q=(q, n_embd), att=(att, n_embd), emb=(emb, n_embd), logits=(logits, n_vocab)).items()}
            for i, (kc, vc) in enumerate(kvs):
                r[f"k{i}"] = be.to_host(kc, (n_ctx, n_embd), np.float32)
                r[f"v{i}"] = be.to_host(vc, (n_embd, n_ctx), np.float32)
            be.check(be.lib.fl_token_plan_destroy(plan))
            results.append(r)
        for d in keep:
            be.free(d)
        return results

    want = run(cpu_model, 1)[0]
    assert np.isfinite(want["logits"]).all() and np.abs(want["logits"]).max() > 0
    for got in run(fl, 2):                       # a second plan over fresh buffers must give the same bits again
        for k in want:
            nd = int((got[k] != want[k]).sum())
            assert nd == 0, (k, nd, got[k].size, np.abs(got[k] - want[k]).max())
