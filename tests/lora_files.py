"""LoRA adapter files for tests, in the on-disk format the reference's loader reads (include/file_loader.hpp) and its converter
scripts/convert-lora-to-ggml.py writes:

    u32 magic 'ggla', u32 version 1, u8 cache flag, u32 r, u32 alpha
    per tensor: i32 n_dims, i32 name length, i32 ftype (0 = f32, 1 = f16), the dims reversed (ne0 first), the name,
                zero padding to a multiple of 32 bytes, the data

Tensor names are `<base>.lora` (cached: the whole delta BA * scale, ne = [K, M] like the base weight) or `<base>.loraA`
(ne = [r, K], already scaled) and `<base>.loraB` (ne = [r, M]) when uncached; the loader merges mul_mat(loraA, loraB)."""
import struct

import numpy as np

GGLA_MAGIC = 0x67676C61
FTYPE = {np.dtype(np.float32): 0, np.dtype(np.float16): 1}
FORMS = ("cached_f32", "uncached_f32", "cached_f16")
TARGETS = ("attention.wq", "attention.wk", "attention.wv", "attention.wo", "feed_forward.w1", "feed_forward.w2", "feed_forward.w3")


def write_lora(path, tensors, r, alpha, cached):
    """tensors: (name, 2-D numpy array of float32 or float16) in file order; an array of shape (rows, cols) is a tensor with
    ne = [cols, rows]."""
    with open(path, "wb") as f:
        f.write(struct.pack("<IIBII", GGLA_MAGIC, 1, 1 if cached else 0, r, alpha))
        for name, a in tensors:
            a = np.ascontiguousarray(a)
            nm = name.encode()
            f.write(struct.pack("<iii", a.ndim, len(nm), FTYPE[a.dtype]))
            f.write(struct.pack(f"<{a.ndim}i", *a.shape[::-1]))
            f.write(nm)
            f.write(b"\0" * (-f.tell() & 31))
            f.write(a.tobytes())


def weight_shape(target, n_embd, n_ff):
    """(K, M) = (ne0, ne1) of a layer's weight."""
    return {"feed_forward.w1": (n_embd, n_ff), "feed_forward.w3": (n_embd, n_ff), "feed_forward.w2": (n_ff, n_embd)}.get(target, (n_embd, n_embd))


def write_adapter(path, form, n_embd, n_ff, layers, seed, r=8, alpha=16, std=0.02, targets=TARGETS):
    """An adapter on `targets` of each layer in `layers`, in one of FORMS, or "uncached_f16" (which the reference refuses) or
    "mismatch" (a cached delta whose shape fits no weight: [M, K] instead of [K, M] for w1)."""
    rng = np.random.default_rng(seed)
    scale = alpha / r
    tensors = []
    for il in layers:
        for tg in targets:
            k, m = weight_shape(tg, n_embd, n_ff)
            base = f"layers.{il}.{tg}.weight"
            a = (rng.standard_normal((k, r)) * std).astype(np.float32) * np.float32(scale)     # loraA * scale, ne = [r, K]
            b = (rng.standard_normal((m, r)) * std * 4).astype(np.float32)                      # loraB, ne = [r, M]
            if form == "mismatch":
                if tg == "feed_forward.w1":
                    tensors.append((base + ".lora", np.zeros((k, m), dtype=np.float32)))
                continue
            if form.startswith("uncached"):
                dt = np.float16 if form.endswith("f16") else np.float32
                tensors += [(base + ".loraA", a.astype(dt)), (base + ".loraB", b.astype(dt))]
            else:
                ba = b @ a.T                                                                    # [M, K]
                tensors.append((base + ".lora", ba.astype(np.float16 if form.endswith("f16") else np.float32)))
    write_lora(path, tensors, r, alpha, cached=not form.startswith("uncached"))
