"""The LLaMA eval graph, built through the ggml C API exactly as the reference's Model::eval builds it
(reference lib/llama.cpp:297-474), so the same script can run on the reference library (CPU) and on
libggml_b200 (H100) and every node can be compared.  Three arenas like the reference: weights
(Model::ctx), KV cache (kv_self.ctx), compute (buf_compute, re-initialised per eval).
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

from tests import ggml_api as G


@dataclass
class HParams:
    n_vocab: int = 64
    n_embd: int = 128
    n_head: int = 4
    n_layer: int = 2
    n_mult: int = 32
    n_ctx: int = 32

    @property
    def n_ff(self) -> int:          # reference lib/llama.cpp:129
        return ((2 * (4 * self.n_embd) // 3 + self.n_mult - 1) // self.n_mult) * self.n_mult


def make_weights(hp: HParams, wtype: int, quantize, seed: int = 0) -> dict:
    """name -> (ggml_type, shape_ne, bytes).  2-D tensors ~ N(0, 0.02^2) quantised with `quantize`
    (the oracle's quantize_row_q4_*_reference restatement); norms f32 around 1."""
    rng = np.random.default_rng(seed)
    out = {}

    def mat(name, k, m, scale=0.02):
        w = (rng.standard_normal((m, k)) * scale).astype(np.float32)
        out[name] = (wtype, (k, m), quantize(w, wtype))

    def vec(name, n):
        out[name] = (G.F32, (n,), (1.0 + 0.1 * rng.standard_normal(n)).astype(np.float32))

    mat("tok_embeddings.weight", hp.n_embd, hp.n_vocab, 1.0)
    vec("norm.weight", hp.n_embd)
    mat("output.weight", hp.n_embd, hp.n_vocab, 0.1)
    for i in range(hp.n_layer):
        vec(f"layers.{i}.attention_norm.weight", hp.n_embd)
        for w in ("wq", "wk", "wv", "wo"):
            mat(f"layers.{i}.attention.{w}.weight", hp.n_embd, hp.n_embd, 0.04)
        vec(f"layers.{i}.ffn_norm.weight", hp.n_embd)
        mat(f"layers.{i}.feed_forward.w1.weight", hp.n_embd, hp.n_ff, 0.04)
        mat(f"layers.{i}.feed_forward.w2.weight", hp.n_ff, hp.n_embd, 0.04)
        mat(f"layers.{i}.feed_forward.w3.weight", hp.n_embd, hp.n_ff, 0.04)
    return out


class MiniLlama:
    def __init__(self, g: G.Ggml, hp: HParams, weights: dict, compute_mb: int = 64):
        self.g, self.hp = g, hp
        wbytes = sum(np.asarray(v[2]).nbytes + 256 for v in weights.values())
        self.wctx = g.context(wbytes + 4096)
        self.w = {}
        for name, (t, ne, data) in weights.items():
            tt = g.new_tensor_1d(self.wctx.ctx, t, ne[0]) if len(ne) == 1 else g.new_tensor_2d(self.wctx.ctx, t, ne[0], ne[1])
            self.wctx.set(tt, np.asarray(data))
            self.w[name] = tt
        n_el = hp.n_layer * hp.n_ctx * hp.n_embd
        self.kvctx = g.context(2 * n_el * 4 + (2 << 20))      # reference lib/llama.cpp:24-46
        self.k = g.new_tensor_1d(self.kvctx.ctx, G.F32, n_el)
        self.v = g.new_tensor_1d(self.kvctx.ctx, G.F32, n_el)
        self.compute_bytes = compute_mb << 20
        self.cbuf = None

    def eval(self, tokens, n_past: int):
        """One Model::eval.  Returns (compute arena, graph, named tensors of interest)."""
        g, hp = self.g, self.hp
        if self.cbuf is not None:
            self.cbuf.free()
        # same buffer every call, like buf_compute
        if not hasattr(self, "_cmem"):
            self._cmem = g.context(self.compute_bytes)
            self._cmem.free()
        c = self._cmem
        c.ctx = g.init(G.InitParams(self.compute_bytes, c.base, False))
        self.cbuf = c
        ctx = c.ctx
        N = len(tokens)
        n_embd, n_head, n_ctx = hp.n_embd, hp.n_head, hp.n_ctx
        hd = n_embd // n_head
        gf = G.new_graph()
        named = {}

        embd = g.new_tensor_1d(ctx, G.I32, N)
        c.set(embd, np.asarray(tokens, dtype=np.int32))
        inpL = g.get_rows(ctx, self.w["tok_embeddings.weight"], embd)
        for il in range(hp.n_layer):
            L = lambda s: self.w[f"layers.{il}.{s}.weight"]
            inpSA = inpL
            cur = g.rms_norm(ctx, inpL)
            cur = g.mul(ctx, g.repeat(ctx, L("attention_norm"), cur), cur)
            Qcur = g.rope(ctx, g.reshape_3d(ctx, g.mul_mat(ctx, L("attention.wq"), cur), hd, n_head, N), n_past, hd, 0)
            Kcur = g.rope(ctx, g.reshape_3d(ctx, g.mul_mat(ctx, L("attention.wk"), cur), hd, n_head, N), n_past, hd, 0)
            Vcur = g.transpose(ctx, g.reshape_2d(ctx, g.mul_mat(ctx, L("attention.wv"), cur), n_embd, N))
            k = g.view_1d(ctx, self.k, N * n_embd, 4 * n_embd * (il * n_ctx + n_past))
            v = g.view_2d(ctx, self.v, N, n_embd, n_ctx * 4, (il * n_ctx) * 4 * n_embd + n_past * 4)
            g.build_forward_expand(gf, g.cpy(ctx, Kcur, k))
            g.build_forward_expand(gf, g.cpy(ctx, Vcur, v))
            Q = g.permute(ctx, Qcur, 0, 2, 1, 3)
            K = g.permute(ctx, g.reshape_3d(ctx, g.view_1d(ctx, self.k, (n_past + N) * n_embd, il * n_ctx * 4 * n_embd), hd, n_head, n_past + N), 0, 2, 1, 3)
            KQ = g.mul_mat(ctx, K, Q)
            KQ_scaled = g.scale(ctx, KQ, g.new_f32(ctx, 1.0 / math.sqrt(float(n_embd) / n_head)))
            KQ_masked = g.diag_mask_inf(ctx, KQ_scaled, n_past)
            KQ_soft = g.soft_max(ctx, KQ_masked)
            V = g.view_3d(ctx, self.v, n_past + N, hd, n_head, n_ctx * 4, n_ctx * 4 * hd, il * n_ctx * 4 * n_embd)
            KQV = g.mul_mat(ctx, V, KQ_soft)
            KQV_merged = g.permute(ctx, KQV, 0, 2, 1, 3)
            cur = g.cpy(ctx, KQV_merged, g.new_tensor_2d(ctx, G.F32, n_embd, N))
            cur = g.mul_mat(ctx, L("attention.wo"), cur)
            inpFF = g.add(ctx, cur, inpSA)
            cur = g.rms_norm(ctx, inpFF)
            cur = g.mul(ctx, g.repeat(ctx, L("ffn_norm"), cur), cur)
            tmp = g.mul_mat(ctx, L("feed_forward.w3"), cur)
            cur = g.mul_mat(ctx, L("feed_forward.w1"), cur)
            cur = g.silu(ctx, cur)
            cur = g.mul(ctx, cur, tmp)
            cur = g.mul_mat(ctx, L("feed_forward.w2"), cur)
            cur = g.add(ctx, cur, inpFF)
            inpL = cur
        inpL = g.rms_norm(ctx, inpL)
        inpL = g.mul(ctx, g.repeat(ctx, self.w["norm.weight"], inpL), inpL)
        named["embeddings"] = inpL
        inpL = g.mul_mat(ctx, self.w["output.weight"], inpL)
        named["logits"] = inpL
        g.build_forward_expand(gf, inpL)
        return c, gf, named

    def compute(self, c, gf):
        self.g.graph_compute(c.ctx, gf)


def graph_signature(c: G.Arena, gf: G.CGraph, arenas=()):
    """Library-independent description of a built graph: per node (op, type, ne, nb, data location)."""
    bases = [("c", c.base, c.buf.nbytes)] + [(f"a{i}", a.base, a.buf.nbytes) for i, a in enumerate(arenas)]

    def loc(p):
        for tag, b, n in bases:
            if b <= p < b + n:
                return (tag, p - b)
        return ("?", 0)

    sig = []
    for i in range(gf.n_nodes):
        t = gf.nodes[i].contents
        sig.append((G.OP_NAMES[t.op], t.type, tuple(t.ne), tuple(t.nb), loc(t.data)))
    leafs = []
    for i in range(gf.n_leafs):
        t = gf.leafs[i].contents
        leafs.append((t.type, tuple(t.ne), loc(t.data)))
    return sig, leafs
