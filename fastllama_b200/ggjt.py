"""Synthetic GGJT-v1 model files (bench / test tooling; no real weights are available offline).

File layout (reference include/file_loader.hpp:94-250 reader, scripts/convert.py:903-928 writer):
  u32 magic 'ggjt', u32 version 1, 7 x i32 {n_vocab, n_embd, n_mult, n_head, n_layer, n_rot, ftype},
  n_vocab x {i32 len, bytes, f32 score}, then per tensor
  {i32 n_dims, i32 name_len, i32 type, i32 ne[n_dims] (ne0 = K first), name, pad to 32 B, data}.
Tensor names / shapes: reference lib/llama.cpp:223-245.  2-D tensors ~ N(0, std^2) quantised row by row with
quantize_row_q4_{0,1}_reference semantics; norms = 1.0 (f32).
"""
from __future__ import annotations

import struct
from typing import Callable, Iterator, Tuple

import numpy as np

GGJT_MAGIC = 0x67676A74
F32, Q4_0, Q4_1 = 0, 2, 3
FTYPE = {Q4_0: 2, Q4_1: 3}
BLOCK_BYTES = {Q4_0: 20, Q4_1: 24}

LLAMA_SIZES = {     # n_embd, n_head, n_layer (n_mult 256, n_vocab 32000); reference lib/llama.cpp:129-139
    "toy": (256, 4, 2), "7B": (4096, 32, 32), "13B": (5120, 40, 40), "30B": (6656, 52, 60), "65B": (8192, 64, 80),
}


def n_ff(n_embd: int, n_mult: int) -> int:
    return ((2 * (4 * n_embd) // 3 + n_mult - 1) // n_mult) * n_mult


def vocab_entries(n_vocab: int):
    """ids 0-2 specials, 3-258 the byte-fallback tokens (the tokenizer maps byte b to id b+3,
    reference include/tokenizer.hpp:130-133), the rest unique ASCII dummies with decreasing scores.
    Every string is ASCII so the Python stream callback can always decode it."""
    for i in range(n_vocab):
        if i == 0:
            tok = b"<unk>"
        elif i == 1:
            tok = b"<s>"
        elif i == 2:
            tok = b"</s>"
        elif i < 259:
            tok = b"<0x%02X>" % (i - 3)
        else:
            tok = b"~t%05d" % i
        yield tok, -float(i)


def tensor_plan(n_vocab, n_embd, n_mult, n_head, n_layer) -> Iterator[Tuple[str, Tuple[int, ...]]]:
    """(name, ne) with ne0 = K (input features) first."""
    ff = n_ff(n_embd, n_mult)
    yield "tok_embeddings.weight", (n_embd, n_vocab)
    yield "norm.weight", (n_embd,)
    yield "output.weight", (n_embd, n_vocab)
    for i in range(n_layer):
        yield f"layers.{i}.attention.wq.weight", (n_embd, n_embd)
        yield f"layers.{i}.attention.wk.weight", (n_embd, n_embd)
        yield f"layers.{i}.attention.wv.weight", (n_embd, n_embd)
        yield f"layers.{i}.attention.wo.weight", (n_embd, n_embd)
        yield f"layers.{i}.attention_norm.weight", (n_embd,)
        yield f"layers.{i}.feed_forward.w1.weight", (n_embd, ff)
        yield f"layers.{i}.feed_forward.w2.weight", (ff, n_embd)
        yield f"layers.{i}.feed_forward.w3.weight", (n_embd, ff)
        yield f"layers.{i}.ffn_norm.weight", (n_embd,)


def write_ggjt(path: str, wtype: int, n_vocab: int, n_embd: int, n_mult: int, n_head: int, n_layer: int,
               matrix_bytes: Callable[[str, int, int, int], bytes]) -> int:
    """matrix_bytes(name, K, M, wtype) -> the M*K/32*block_bytes quantised bytes of that tensor."""
    with open(path, "wb") as f:
        f.write(struct.pack("<II", GGJT_MAGIC, 1))
        f.write(struct.pack("<7i", n_vocab, n_embd, n_mult, n_head, n_layer, n_embd // n_head, FTYPE[wtype]))
        for tok, score in vocab_entries(n_vocab):
            f.write(struct.pack("<i", len(tok)) + tok + struct.pack("<f", score))
        for name, ne in tensor_plan(n_vocab, n_embd, n_mult, n_head, n_layer):
            nm = name.encode()
            t = F32 if len(ne) == 1 else wtype
            f.write(struct.pack("<iii", len(ne), len(nm), t))
            f.write(struct.pack(f"<{len(ne)}i", *ne))
            f.write(nm)
            f.write(b"\0" * (-f.tell() & 31))
            if len(ne) == 1:
                f.write(np.ones(ne[0], dtype=np.float32).tobytes())
            else:
                data = matrix_bytes(name, ne[0], ne[1], wtype)
                assert len(data) == ne[1] * (ne[0] // 32) * BLOCK_BYTES[wtype], name
                f.write(data)
        return f.tell()


GGML_MAGIC, GGMF_MAGIC = 0x67676D6C, 0x67676D66
F16 = 1
FLOAT_DTYPE = {F32: np.float32, F16: np.float16}


def write_model_file(path: str, fmt: str, hparams, vocab, tensors) -> int:
    """Any single-file model the reference's reader accepts (include/file_loader.hpp:94-250).  fmt: "ggjt"
    (version 1, tensor data 32-byte aligned), "ggmf" (version 1, no padding) or "ggml" (no version, vocab
    without scores).  hparams: the 7 header integers; vocab: (bytes, score) pairs; tensors: (name, ne, type,
    data bytes) with ne0 first."""
    with open(path, "wb") as f:
        if fmt == "ggml":
            f.write(struct.pack("<I", GGML_MAGIC))
        else:
            f.write(struct.pack("<II", {"ggjt": GGJT_MAGIC, "ggmf": GGMF_MAGIC}[fmt], 1))
        f.write(struct.pack("<7i", *hparams))
        for tok, score in vocab:
            f.write(struct.pack("<i", len(tok)) + tok + (b"" if fmt == "ggml" else struct.pack("<f", score)))
        for name, ne, t, data in tensors:
            nm = name.encode()
            f.write(struct.pack("<iii", len(ne), len(nm), t))
            f.write(struct.pack(f"<{len(ne)}i", *ne))
            f.write(nm)
            if fmt == "ggjt":
                f.write(b"\0" * (-f.tell() & 31))
            f.write(data)
        return f.tell()


def write_synthetic_float(path, ftype=F16, n_vocab=512, n_embd=256, n_mult=64, n_head=4, n_layer=2, seed=0, std=0.02,
                          fmt="ggjt") -> int:
    """An unquantised model as the reference's scripts/convert.py writes it: every 2-D tensor f16 (ftype 1) or
    f32 (ftype 0), ~ N(0, std^2) (token embeddings N(0, 1)); 1-D norms f32 ones.  The input of the quantiser
    (fastllama_b200/quantize.py).  Tensors are generated one at a time, so the host holds one at most."""
    rng = np.random.default_rng(seed)
    dt = FLOAT_DTYPE[ftype]

    def tensors():
        for name, ne in tensor_plan(n_vocab, n_embd, n_mult, n_head, n_layer):
            if len(ne) == 1:
                yield name, ne, F32, np.ones(ne[0], dtype=np.float32).tobytes()
                continue
            scale = 1.0 if name.startswith("tok_embeddings") else std
            w = rng.standard_normal((ne[1], ne[0]), dtype=np.float32)
            w *= np.float32(scale)
            yield name, ne, ftype, w.astype(dt, copy=False).tobytes()

    return write_model_file(path, fmt, (n_vocab, n_embd, n_mult, n_head, n_layer, n_embd // n_head, ftype),
                            vocab_entries(n_vocab), tensors())


def splits_by_columns(name: str) -> bool:
    """The tensors the reference's reader joins from column ranges when a model comes in parts (the token embeddings,
    wo and w2: include/tensor/utils.hpp:101-106); every other matrix is joined from row ranges."""
    return name.startswith("tok_embeddings.") or name.endswith((".attention.wo.weight", ".feed_forward.w2.weight"))


def _shard(name, idx, ne, ftype, n_parts, j, seed, std):
    """Part j's shard of tensor idx (tensor_plan order) of a split synthetic model: (shard ne, type, bytes).  Each
    shard is its own Gaussian stream; vectors are ones, whole in every part."""
    if len(ne) == 1:
        return ne, F32, np.ones(ne[0], dtype=np.float32).tobytes()
    k, m = ne
    shape = (m, k // n_parts) if splits_by_columns(name) else (m // n_parts, k)
    w = np.random.default_rng([seed, idx, j]).standard_normal(shape, dtype=np.float32)
    w *= np.float32(1.0 if name.startswith("tok_embeddings") else std)
    return (shape[1], shape[0]), ftype, w.astype(FLOAT_DTYPE[ftype], copy=False).tobytes()


def write_synthetic_parts(base, fmts, ftype=F16, n_vocab=512, n_embd=256, n_mult=64, n_head=4, n_layer=2, seed=0, std=0.02,
                          edit=None) -> str:
    """An unquantised model split into len(fmts) parts the way the reference's converter writes one per checkpoint
    shard: part j, in format fmts[j], goes to base (j = 0) or base.j, every part with the full model's header and
    vocab.  edit(j, hparams, tensors) -> (hparams, tensors) changes a part before it is written (tests).  Shards are
    generated one at a time unless edit needs a part's list."""
    hp = (n_vocab, n_embd, n_mult, n_head, n_layer, n_embd // n_head, ftype)
    plan = list(tensor_plan(n_vocab, n_embd, n_mult, n_head, n_layer))
    for j, fmt in enumerate(fmts):
        tensors = ((name, *_shard(name, i, ne, ftype, len(fmts), j, seed, std)) for i, (name, ne) in enumerate(plan))
        hp_j = hp
        if edit is not None:
            hp_j, tensors = edit(j, hp, list(tensors))
        write_model_file(base if j == 0 else f"{base}.{j}", fmt, hp_j, vocab_entries(n_vocab), tensors)
    return base


def write_synthetic_joined(path, n_parts, ftype=F16, n_vocab=512, n_embd=256, n_mult=64, n_head=4, n_layer=2, seed=0,
                           std=0.02, fmt="ggjt") -> str:
    """The model write_synthetic_parts splits into n_parts parts, as one file: every matrix its shards joined by
    columns or by rows (splits_by_columns), every vector part 0's."""
    def tensors():
        for i, (name, ne) in enumerate(tensor_plan(n_vocab, n_embd, n_mult, n_head, n_layer)):
            shards = [_shard(name, i, ne, ftype, n_parts, j, seed, std) for j in range(n_parts)]
            if len(ne) == 1:
                yield name, ne, F32, shards[0][2]
                continue
            arrs = [np.frombuffer(b, dtype=FLOAT_DTYPE[ftype]).reshape(sne[1], sne[0]) for sne, _, b in shards]
            yield name, ne, ftype, np.concatenate(arrs, axis=1 if splits_by_columns(name) else 0).tobytes()

    write_model_file(path, fmt, (n_vocab, n_embd, n_mult, n_head, n_layer, n_embd // n_head, ftype), vocab_entries(n_vocab),
                     tensors())
    return path


def write_synthetic_numpy(path, wtype=Q4_0, n_vocab=512, n_embd=256, n_mult=64, n_head=4, n_layer=2, seed=0, std=0.02,
                          quantize=None) -> int:
    """CPU generator for toy models (tests).  `quantize(w_f32[M,K], wtype) -> uint8` must follow the
    reference's quantize_row_q4_*_reference; the tests pass the oracle's."""
    rng = np.random.default_rng(seed)

    def gen(name, k, m, t):
        scale = 1.0 if name.startswith("tok_embeddings") else std * (4.0 if n_embd < 1024 else 1.0)
        w = (rng.standard_normal((m, k)) * scale).astype(np.float32)
        return np.ascontiguousarray(quantize(w, t)).tobytes()

    return write_ggjt(path, wtype, n_vocab, n_embd, n_mult, n_head, n_layer, gen)


def write_synthetic_gpu(path, size="7B", wtype=Q4_0, seed=0, std=0.02, n_vocab=32000, n_mult=256, fl=None, n_layer=None) -> int:
    """GPU generator for full-size models: a counter-based Gaussian filled on the device and quantised
    by the library's bit-exact quantize_row_q4_*_reference kernel, streamed to the file per tensor."""
    import ctypes as C

    from .cuda_abi import FlCuda

    fl = fl or FlCuda()
    n_embd, n_head, layers = LLAMA_SIZES[size]
    n_layer = n_layer or layers
    ff = n_ff(n_embd, n_mult)
    max_el = max(n_vocab, ff) * max(n_embd, ff) if False else max(n_vocab * n_embd, ff * n_embd)
    d_f32 = fl.alloc(max_el * 4)
    d_q = fl.alloc(max_el // 32 * BLOCK_BYTES[wtype])
    counter = [0]

    def gen(name, k, m, t):
        n = k * m
        fl.check(fl.lib.fl_dev_fill_normal(d_f32, n, C.c_uint64(seed * 1000003 + counter[0]), C.c_float(std)))
        counter[0] += 1
        fl.check(fl.lib.fl_dev_quantize_q4(t, d_f32, d_q, k, m))
        return fl.to_host(d_q, (n // 32 * BLOCK_BYTES[t],), np.uint8).tobytes()

    try:
        return write_ggjt(path, wtype, n_vocab, n_embd, n_mult, n_head, n_layer, gen)
    finally:
        fl.free(d_f32)
        fl.free(d_q)
