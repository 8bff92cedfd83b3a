"""Generate tests/golden/lora_f16_ops.npz from the REFERENCE itself (oracle/_ref/libggml_ref.so): the ops of attaching and detaching a
cached f16 LoRA adapter, as oracle/gen_golden.py does for the f32 forms (lora_ops.npz).

Run in the build container (where /root/reference exists):  python -m oracle.gen_golden_lora_f16
"""
import os

import numpy as np

from oracle.gen_golden import OUT, lora_inputs
from oracle.pyoracle import RefGgml, build_oracle

LORA_F16_SHAPES = ((64, 8), (256, 24), (4096, 6))          # (K, M) of the adapted weight
LORA_F16_SCALE = 0.3712                                    # a factor other than -1, to pin scale_f16's rounding


def lora_f16_delta(rng, m, k):
    """A cached f16 adapter matrix (BA * scale as convert-lora-to-ggml.py --dtype fp16 stores it): values large enough to move many
    nibbles of every block, f16 subnormals, signed zeros, and rows that push a block's range far out or cancel it."""
    x = (rng.standard_normal((m, k)) * 0.3).astype(np.float16)
    x[0, :64] = (rng.standard_normal(64) * 2e-5).astype(np.float16)                 # subnormal in f16 (|x| < 6.1e-5)
    x[0, 64:] = np.float16(0.0)
    x[0, 1::7] = np.float16(-0.0)
    x[1, :32] = np.float16(5.96e-8)                                                 # the smallest f16 subnormal
    x[2] *= np.float16(8.0)                                                         # big moves: most codes of the row change
    x[3, :32] = np.linspace(-40.0, 40.0, 32).astype(np.float16)
    return x


def lora_f16_ops():
    """Outputs of the reference LIBRARY for a cached f16 adapter (convert-lora-to-ggml.py --dtype fp16): attach is
    add_inplace(W_q4, X_f16) -> ggml_compute_forward_add_q_f16 (lib/ggml.c:12372-12483); detach is
    add_inplace(W_q4, scale(X_f16, -1)), where the scale runs ggml_compute_forward_scale_f16 (:12485-12524) in place on X.
    Also scale_f16 with a factor that rounds."""
    from oracle.pyoracle import REF_GGML_SO
    from tests import ggml_api as G

    ref = RefGgml()
    g = G.Ggml(REF_GGML_SO)
    rng = np.random.default_rng(1616)
    out = {}
    for k, m in LORA_F16_SHAPES:
        w = lora_inputs(rng, m, k)
        x = lora_f16_delta(rng, m, k)
        out[f"x_{k}x{m}"] = x
        for name, t in (("q4_0", G.Q4_0), ("q4_1", G.Q4_1)):
            base = ref.quantize_q4_reference(w, t)
            out[f"{name}_base_{k}x{m}"] = base
            ar = g.context(16 << 20)
            tw = g.new_tensor_2d(ar.ctx, t, k, m); ar.set(tw, base)
            tx = g.new_tensor_2d(ar.ctx, G.F16, k, m); ar.set(tx, x)
            res = g.add_inplace(ar.ctx, tw, tx)
            gf = G.new_graph()
            g.build_forward_expand(gf, res)
            g.graph_compute(ar.ctx, gf)
            out[f"{name}_merged_{k}x{m}"] = ar.numpy(tw).reshape(m, -1).copy()
            neg = g.scale(ar.ctx, tx, g.new_f32(ar.ctx, -1.0))
            res2 = g.add_inplace(ar.ctx, tw, neg)
            gf2 = G.new_graph()
            g.build_forward_expand(gf2, res2)
            g.graph_compute(ar.ctx, gf2)
            out[f"{name}_detached_{k}x{m}"] = ar.numpy(tw).reshape(m, -1).copy()
            ar.free()
        ar = g.context(16 << 20)
        tx = g.new_tensor_2d(ar.ctx, G.F16, k, m); ar.set(tx, x)
        sc = g.scale(ar.ctx, tx, g.new_f32(ar.ctx, LORA_F16_SCALE))
        gf = G.new_graph()
        g.build_forward_expand(gf, sc)
        g.graph_compute(ar.ctx, gf)
        out[f"x_scaled_{k}x{m}"] = ar.numpy(tx).view(np.float16).reshape(m, k).copy()
        ar.free()
    path = os.path.join(OUT, "lora_f16_ops.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    build_oracle()
    lora_f16_ops()
