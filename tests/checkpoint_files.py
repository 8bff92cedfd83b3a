"""Synthetic LLaMA checkpoints in the layouts the reference's converter (scripts/convert.py) reads, and a numpy
restatement of the f16 / f32 GGJT file it writes from them (tests and tools/time_quantize_checkpoint.py).

Layouts:
  * Meta: consolidated.00.pth, .01.pth, ... (torch.save zips), every tensor in every file; vectors whole, the token
    embeddings, wo and w2 cut into column ranges, every other matrix into row ranges.
  * Hugging Face: pytorch_model-0000j-of-0000N.bin (torch.save) or model-0000j-of-0000N.safetensors, each tensor whole
    in one file, under the Hugging Face names, with wq / wk rows in the Hugging Face order (the converter's permute
    undone), so they convert to the same file as the Meta layout of the same weights.

Shapes follow torch: (rows, columns).  The converter guesses n_head = n_embd // 128, so toy models need head_dim 128.
"""
from __future__ import annotations

import json
import os
import struct

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOKENIZER = os.path.join(ROOT, "tests", "golden", "tokenizer_toy.model")      # sentencepiece BPE, byte fallback, 300 pieces
GGJT_MAGIC = 0x67676A74


def n_ff(n_embd: int) -> int:
    return ((2 * (4 * n_embd) // 3 + 255) // 256) * 256                      # n_mult 256, as the converter writes


def layer_shapes(n_embd: int):
    ff = n_ff(n_embd)
    return [("attention.wq", (n_embd, n_embd)), ("attention.wk", (n_embd, n_embd)), ("attention.wv", (n_embd, n_embd)),
            ("attention.wo", (n_embd, n_embd)), ("attention_norm", (n_embd,)), ("feed_forward.w1", (ff, n_embd)),
            ("feed_forward.w2", (n_embd, ff)), ("feed_forward.w3", (ff, n_embd)), ("ffn_norm", (n_embd,))]


def meta_shapes(n_vocab: int, n_embd: int, n_layer: int):
    """(name, torch shape) of a LLaMA checkpoint in the converter's order."""
    out = [("tok_embeddings.weight", (n_vocab, n_embd)), ("norm.weight", (n_embd,)), ("output.weight", (n_vocab, n_embd))]
    for i in range(n_layer):
        out += [(f"layers.{i}.{t}.weight", s) for t, s in layer_shapes(n_embd)]
    return out


def make_tensor(name, shape, dtype, seed, std=0.02):
    """A tensor of the synthetic model: vectors 1 + N(0, 0.1^2), matrices N(0, std^2), the token embeddings N(0, 1);
    its own seeded stream, so any tensor can be made on its own."""
    rng = np.random.default_rng([seed, hash_name(name)])
    if len(shape) == 1:
        w = 1.0 + 0.1 * rng.standard_normal(shape, dtype=np.float32)
    else:
        w = rng.standard_normal(shape, dtype=np.float32) * np.float32(1.0 if name.startswith("tok_") else std)
    return w.astype(dtype)


def hash_name(name: str) -> int:
    h = 0
    for c in name.encode():
        h = (h * 131 + c) % (1 << 31)
    return h


def meta_model(n_vocab=300, n_embd=256, n_layer=2, dtype=np.float16, seed=0, std=0.02) -> dict:
    return {name: make_tensor(name, shape, dtype, seed, std) for name, shape in meta_shapes(n_vocab, n_embd, n_layer)}


def splits_by_columns(name: str) -> bool:
    return name.startswith("tok_embeddings.") or name.endswith((".attention.wo.weight", ".feed_forward.w2.weight"))


def permute(w, n_head):
    """The converter's q / k row order from the Hugging Face one: within a head, row 2i + p <- row p * hd/2 + i."""
    return w.reshape(n_head, 2, w.shape[0] // n_head // 2, *w.shape[1:]).swapaxes(1, 2).reshape(w.shape)


def unpermute(w, n_head):
    return w.reshape(n_head, w.shape[0] // n_head // 2, 2, *w.shape[1:]).swapaxes(1, 2).reshape(w.shape)


def _torch_save(path, tensors):
    import torch

    torch.save({n: torch.from_numpy(np.ascontiguousarray(a)) for n, a in tensors.items()}, path)


def write_meta(d, model: dict, n_shards=1, extra=True) -> str:
    """consolidated.0j.pth for j < n_shards; extra adds rope.freqs, which the converter drops.  The tensors are saved
    in an order other than the converter's (norm last), so the output order is the converter's, not the file's."""
    os.makedirs(d, exist_ok=True)
    names = [n for n in model if n != "norm.weight"] + ["norm.weight"]
    for j in range(n_shards):
        shard = {}
        if extra:
            shard["rope.freqs"] = np.linspace(0, 1, 64, dtype=np.float32)
        for n in names:
            a = model[n]
            if a.ndim == 1 or n_shards == 1:
                shard[n] = a
            elif splits_by_columns(n):
                shard[n] = np.split(a, n_shards, axis=1)[j]
            else:
                shard[n] = np.split(a, n_shards, axis=0)[j]
        _torch_save(os.path.join(d, f"consolidated.{j:02}.pth"), shard)
    return d


_HF = {"attention.wq": "self_attn.q_proj", "attention.wk": "self_attn.k_proj", "attention.wv": "self_attn.v_proj",
       "attention.wo": "self_attn.o_proj", "feed_forward.w1": "mlp.gate_proj", "feed_forward.w2": "mlp.down_proj",
       "feed_forward.w3": "mlp.up_proj", "attention_norm": "input_layernorm", "ffn_norm": "post_attention_layernorm"}


def hf_names(model: dict):
    """(Hugging Face name, Meta name, needs unpermute) in the Hugging Face files' order."""
    out = [("model.embed_tokens.weight", "tok_embeddings.weight", False)]
    i = 0
    while f"layers.{i}.attention.wq.weight" in model:
        for t, h in _HF.items():
            out.append((f"model.layers.{i}.{h}.weight", f"layers.{i}.{t}.weight", t in ("attention.wq", "attention.wk")))
        i += 1
    return out + [("model.norm.weight", "norm.weight", False), ("lm_head.weight", "output.weight", False)]


def hf_model(model: dict, n_head: int) -> dict:
    return {h: (unpermute(model[m], n_head) if p else model[m]) for h, m, p in hf_names(model)}


def write_hf(d, hf: dict, n_files=2, form="bin", extra=True, dtype_names=None) -> str:
    """The Hugging Face tensors in n_files files, consecutive runs of names; returns the first file.  dtype_names:
    see write_safetensors."""
    os.makedirs(d, exist_ok=True)
    names = list(hf)
    per = -(-len(names) // n_files)
    first = None
    for j in range(n_files):
        part = {n: hf[n] for n in names[j * per:(j + 1) * per]}
        if extra and j == 0:
            part["model.layers.0.self_attn.rotary_emb.inv_freq"] = np.linspace(0, 1, 64, dtype=np.float32)
        stem = "pytorch_model" if form == "bin" else "model"
        path = os.path.join(d, f"{stem}-{j + 1:05}-of-{n_files:05}.{'bin' if form == 'bin' else 'safetensors'}")
        if form == "bin":
            _torch_save(path, part)
        else:
            write_safetensors(path, [(n, a.dtype, a.shape, (lambda a=a: a)) for n, a in part.items()], dtype_names)
        first = first or path
    return first


ST_DTYPES = {np.dtype(np.float16): "F16", np.dtype(np.float32): "F32", np.dtype(np.int32): "I32"}


def write_safetensors(path, entries, dtype_names=None) -> None:
    """entries: (name, numpy dtype, shape, make() -> array), written one tensor at a time.  dtype_names overrides the
    header's dtype of a name (tests: "BF16" over 2-byte data)."""
    header, off = {}, 0
    for name, dt, shape, _ in entries:
        n = int(np.prod(shape)) * np.dtype(dt).itemsize
        header[name] = {"dtype": (dtype_names or {}).get(name, ST_DTYPES[np.dtype(dt)]), "shape": list(shape),
                        "data_offsets": [off, off + n]}
        off += n
    h = json.dumps(header, separators=(",", ":")).encode()
    h += b" " * (-len(h) % 8)
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(h)) + h)
        for name, dt, shape, make in entries:
            a = np.ascontiguousarray(make(), dtype=dt)
            assert a.shape == tuple(shape), name
            a.tofile(f)


def converter_vocab(tokenizer_path, n_vocab):
    """(bytes, score) as the converter writes them: tokenizer.model's pieces, then added_tokens.json's tokens beside
    it with score -1000 unless the model has the base size."""
    import sentencepiece

    sp = sentencepiece.SentencePieceProcessor(model_file=str(tokenizer_path))
    out = []
    for i in range(sp.vocab_size()):
        if sp.is_unknown(i):
            out.append((" ⁇ ".encode(), sp.get_score(i)))
        elif sp.is_control(i):
            out.append((b"", sp.get_score(i)))
        elif sp.is_byte(i):
            out.append((bytes([int(sp.id_to_piece(i)[3:5], 16)]), sp.get_score(i)))
        else:
            out.append((sp.id_to_piece(i).replace("▁", " ").encode(), sp.get_score(i)))
    added = os.path.join(os.path.dirname(str(tokenizer_path)), "added_tokens.json")
    if n_vocab != len(out) and os.path.exists(added):
        with open(added) as f:
            out += [(t.encode(), -1000.0) for t, _ in sorted(json.load(f).items(), key=lambda kv: kv[1])]
    assert len(out) == n_vocab, (len(out), n_vocab)
    return out


def write_converted(path, model: dict, tokenizer_path, outtype="f16") -> str:
    """The GGJT file the converter writes for the Meta-named, joined model (name -> array, or a callable returning
    it, so that a large model is read one tensor at a time): header {1, n_vocab, n_embd, 256, n_embd // 128, n_layer,
    rot, ftype}, the vocab, then the tensors in the converter's order, vectors f32, matrices f16 or f32."""
    get = {n: (v if callable(v) else (lambda v=v: v)) for n, v in model.items()}
    n_vocab, n_embd = (model["tok_embeddings.weight"].shape if not callable(model["tok_embeddings.weight"])
                       else get["tok_embeddings.weight"]().shape)
    n_layer = 0
    while f"layers.{n_layer}.attention.wq.weight" in model:
        n_layer += 1
    n_head = n_embd // 128
    ftype = {"f32": 0, "f16": 1}[outtype]
    with open(path, "wb") as f:
        f.write(struct.pack("<I7i", GGJT_MAGIC, 1, n_vocab, n_embd, 256, n_head, n_layer, n_embd // n_head) +
                struct.pack("<i", ftype))
        for text, score in converter_vocab(tokenizer_path, n_vocab):
            f.write(struct.pack("<i", len(text)) + text + struct.pack("<f", score))
        for name, _ in meta_shapes(n_vocab, n_embd, n_layer):
            a = np.asarray(get[name]())
            dt = np.float32 if a.ndim == 1 or outtype == "f32" else np.float16
            nm = name.encode()
            f.write(struct.pack(f"<iii{a.ndim}i", a.ndim, len(nm), 0 if dt == np.float32 else 1, *a.shape[::-1]) + nm)
            f.write(b"\0" * (-f.tell() & 31))
            a.astype(dt).tofile(f)
    return path
