"""Quantise an f32 / f16 model file to q4_0 or q4_1 on the GPU: the middle step of the reference's pipeline
(scripts/convert.py -> quantize -> model), writing byte for byte the file the reference's quantize tool writes.

    python -m fastllama_b200.quantize IN OUT TYPE        TYPE: 2 = q4_0, 3 = q4_1 (the reference CLI's arguments)

Input: one single-file model the reference's reader accepts (include/file_loader.hpp:94-250): GGML (no version,
vocab without scores: the score becomes 0.0), GGMF v1 or GGJT v1 (tensor data 32-byte aligned), with 1-D or 2-D
f32 / f16 tensors.  Output: what the reference's FileSaver writes (include/file_loader.hpp:254-375): GGJT v1, the
input's hyperparameters, the vocab as {u32 len, bytes, f32 score}, then the tensors in input order, each padded
with zeros to 32 bytes before its data.  Every 2-D tensor is quantised (lib/llama.cpp:558-572 never excludes one)
by k_quantize_q4_file (fl_dev_quantize_q4_file), 1-D tensors are copied unchanged.

Streaming: the input is memory-mapped and read one tensor at a time through two pinned staging chunks, so a read
from the file overlaps the previous chunk's host-to-device copy, and a tensor's file reads overlap the previous
tensor's kernel and device-to-host copy; the previous tensor is written to the output while this one's copies run.
Host memory stays bounded (two 64 MiB input chunks plus one pinned buffer of the largest quantised tensor); the
device holds the largest input tensor and its quantised form.
"""
from __future__ import annotations

import ctypes as C
import os
import struct
import sys
from typing import NamedTuple

import numpy as np

from .cuda_abi import FlCuda

GGML_MAGIC, GGMF_MAGIC, GGJT_MAGIC, GGLA_MAGIC = 0x67676D6C, 0x67676D66, 0x67676A74, 0x67676C61
F32, F16, Q4_0, Q4_1 = 0, 1, 2, 3
TYPE_NAMES = ["f32", "f16", "q4_0", "q4_1", "q4_2", "q4_3"]         # the types the reader accepts (0..5)
ELEM_BYTES = {F32: 4, F16: 2}
BLOCK_BYTES = {Q4_0: 20, Q4_1: 24}
QK = 32
CHUNK_BYTES = 64 << 20                                                # one pinned staging chunk of input


class QuantizeError(ValueError):
    pass


class Tensor(NamedTuple):
    name: str
    ne: tuple          # ne0 (row length) first
    type: int
    offset: int        # of the data in the input file
    nbytes: int


class ModelFile(NamedTuple):
    version: str       # "ggml", "ggmf" or "ggjt"
    hparams: bytes     # the 7 header integers, raw: n_vocab, n_embd, n_mult, n_head, n_layer, n_rot, ftype
    vocab: list        # (token bytes, raw f32 score bytes)
    tensors: list


def _read(f, n: int) -> bytes:
    b = f.read(n)
    if len(b) != n:
        raise QuantizeError(f"{f.name}: unexpected end of file")
    return b


def read_model(path: str) -> ModelFile:
    """Parse the header, vocab and tensor table and reject every input the tool would otherwise have to guess about."""
    size = os.path.getsize(path)
    with open(path, "rb") as f:
        (magic,) = struct.unpack("<I", _read(f, 4))
        if magic == GGLA_MAGIC:
            raise QuantizeError(f"{path} is a LoRA adapter (ggla magic); only model files can be quantised")
        if magic == GGML_MAGIC:
            version = "ggml"
        elif magic in (GGMF_MAGIC, GGJT_MAGIC):
            (ver,) = struct.unpack("<I", _read(f, 4))
            if ver != 1:
                raise QuantizeError(f"{path}: unsupported file version {ver} for magic {magic:08x} (expected 1)")
            version = "ggmf" if magic == GGMF_MAGIC else "ggjt"
        else:
            raise QuantizeError(f"{path}: bad magic {magic:08x} (not a ggml / ggmf / ggjt model file)")
        hparams = _read(f, 28)
        n_vocab, n_embd = struct.unpack("<7i", hparams)[:2]
        vocab = []
        for _ in range(n_vocab):
            (n,) = struct.unpack("<I", _read(f, 4))
            tok = _read(f, n)
            vocab.append((tok, b"\0\0\0\0" if version == "ggml" else _read(f, 4)))      # GGML has no scores: 0.0
        tensors, names = [], set()
        while f.tell() < size:
            n_dims, name_len, t = struct.unpack("<III", _read(f, 12))
            if n_dims < 1 or n_dims > 2:
                raise QuantizeError(f"{path}: a tensor has {n_dims} dimensions (1 or 2 expected)")
            ne = struct.unpack(f"<{n_dims}I", _read(f, 4 * n_dims))
            name = _read(f, name_len).decode("utf-8", errors="replace")
            if t >= len(TYPE_NAMES):
                raise QuantizeError(f"{path}: tensor '{name}' has unrecognised type {t}")
            if t not in (F32, F16):
                raise QuantizeError(f"{path}: tensor '{name}' is already quantised ({TYPE_NAMES[t]}); only f32 and f16 "
                                    "tensors can be quantised (the reference: unsupported for integer quantization)")
            if name in names:
                raise QuantizeError(f"{path}: tensor '{name}' appears twice")
            names.add(name)
            if n_dims == 2 and ne[0] % QK:
                raise QuantizeError(f"{path}: tensor '{name}' has rows of {ne[0]} elements, not a multiple of {QK}")
            if version == "ggjt":
                f.seek(-f.tell() & 31, os.SEEK_CUR)
            nbytes = int(np.prod(ne, dtype=np.int64)) * ELEM_BYTES[t]
            off = f.tell()
            if off + nbytes > size:
                raise QuantizeError(f"{path}: tensor '{name}' extends past the end of the file")
            tensors.append(Tensor(name, tuple(ne), t, off, nbytes))
            f.seek(nbytes, os.SEEK_CUR)
    # the reader takes n_embd / tok_embeddings.ne[0] as the number of parts of a split model
    # (include/file_loader.hpp:443-453); only single-file models are accepted
    tok = next((t for t in tensors if t.name == "tok_embeddings.weight"), None)
    if tok is None:
        raise QuantizeError(f"{path}: tok_embeddings.weight not found")
    n_parts = n_embd // tok.ne[0]
    if n_parts != 1:
        raise QuantizeError(f"{path}: multi-part model ({n_parts} parts by n_embd / tok_embeddings.ne[0] = {n_embd} / "
                            f"{tok.ne[0]}); only single-file models can be quantised")
    return ModelFile(version, hparams, vocab, tensors)


def _tensor_header(t: Tensor, new_type: int) -> bytes:
    nm = t.name.encode()
    return struct.pack(f"<III{len(t.ne)}I", len(t.ne), len(nm), new_type, *t.ne) + nm


def _pinned(fl: FlCuda, nbytes: int):
    p = fl.lib.fl_host_alloc_pinned(nbytes)
    if not p:
        raise MemoryError(fl.lib.fl_last_error().decode())
    return p, np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(p))


def quantize_model(in_path: str, out_path: str, wtype: int, fl: FlCuda | None = None, verbose: bool = True) -> dict:
    """Quantise in_path (f32 / f16) to out_path (q4_0 for wtype 2, q4_1 for 3).  Returns per-tensor and total sizes
    and the 16-bin histograms of the stored nibbles (counts), as the reference's tool reports them."""
    if wtype not in (Q4_0, Q4_1):
        hint = " (q4_2 / q4_3 / mostly-q4_1-some-f16 are not supported)" if wtype in (4, 5, 6) else ""
        raise QuantizeError(f"invalid quantization type {wtype}{hint}: use 2 (q4_0) or 3 (q4_1)")
    model = read_model(in_path)
    fl = fl or FlCuda()
    quantize_file = fl.fn("fl_dev_quantize_q4_file")
    bb = BLOCK_BYTES[wtype]
    mats = [t for t in model.tensors if len(t.ne) == 2]
    max_in = max((t.nbytes for t in mats), default=0)
    max_out = max((t.ne[0] // QK * t.ne[1] * bb for t in mats), default=0)

    src = np.memmap(in_path, dtype=np.uint8, mode="r")
    dev_in = fl.alloc(max(max_in, 16))
    dev_out = fl.alloc(max(max_out, 16))
    dev_hist = fl.alloc(16 * 8)
    chunk = min(CHUNK_BYTES, max(max_in, 16))
    stage = [_pinned(fl, chunk) for _ in range(2)]
    outbuf = _pinned(fl, max(max_out, 16))
    hist_host = _pinned(fl, 16 * 8)
    ev_stage = [fl.lib.fl_event_create() for _ in range(2)]
    ev_out = fl.lib.fl_event_create()
    stage_busy = [False, False]
    n_chunks = 0

    report = {"tensors": [], "total_size_org": 0, "total_size_new": 0, "hist": [0] * 16}

    def record(i, t, new_type, size_new, hist):
        report["tensors"].append({"name": t.name, "ne": t.ne, "type": TYPE_NAMES[t.type], "new_type": TYPE_NAMES[new_type],
                                  "size_org": t.nbytes, "size_new": size_new, "hist": hist})
        report["total_size_org"] += t.nbytes
        report["total_size_new"] += size_new
        if verbose:
            line = (f"[{i:4d}/{len(model.tensors):4d}] {t.name:>36s} - {'x '.join(f'{e:5d}' for e in t.ne):>16s}, "
                    f"type = {TYPE_NAMES[t.type]:>6s}, ")
            if hist is None:
                print(line + f"size = {t.nbytes / 1024 / 1024:8.3f} MB", flush=True)
            else:
                n_el = t.ne[0] * t.ne[1]
                print(line + f"size = {t.nbytes / 1024 / 1024:8.2f} MB -> {size_new / 1024 / 1024:8.2f} MB | hist: "
                      + " ".join(f"{h / n_el:5.3f}" for h in hist), flush=True)

    try:
        with open(out_path, "wb") as out:
            out.write(struct.pack("<II", GGJT_MAGIC, 1))
            # the input's hyperparameters, ftype included: the reference's FileSaver::write_hyperparams writes the
            # loader's ftype, not the new one (include/file_loader.hpp:328-341), and its files are what we reproduce
            out.write(model.hparams)
            for tok, score in model.vocab:
                out.write(struct.pack("<I", len(tok)) + tok + score)

            def write_tensor(t: Tensor, new_type: int, data) -> None:
                out.write(_tensor_header(t, new_type))
                out.write(b"\0" * (-out.tell() & 31))
                out.write(data)

            pending = None          # (index, tensor, bytes): quantised, its kernel and copies back possibly still running

            def flush_pending():
                nonlocal pending
                if pending is None:
                    return
                i, t, nbytes = pending
                fl.check(fl.lib.fl_event_sync(ev_out))
                write_tensor(t, wtype, outbuf[1][:nbytes])
                hist = [int(v) for v in hist_host[1].view(np.uint64)]
                for j in range(16):
                    report["hist"][j] += hist[j]
                record(i, t, wtype, nbytes, hist)
                pending = None

            for i, t in enumerate(model.tensors):
                if len(t.ne) == 1:
                    flush_pending()
                    write_tensor(t, t.type, src[t.offset:t.offset + t.nbytes])
                    record(i, t, t.type, t.nbytes, None)
                    continue
                # stage the rows into the device input buffer, one pinned chunk at a time; these copies queue behind
                # the previous tensor's kernel and copies on the library stream, so reusing dev_in / dev_out is safe
                for off in range(0, t.nbytes, chunk):
                    n = min(chunk, t.nbytes - off)
                    s = n_chunks % 2
                    if stage_busy[s]:
                        fl.check(fl.lib.fl_event_sync(ev_stage[s]))      # the chunk staged there before is on the device
                    stage[s][1][:n] = src[t.offset + off:t.offset + off + n]
                    fl.check(fl.lib.fl_h2d(dev_in + off, stage[s][0], n))
                    fl.check(fl.lib.fl_event_record(ev_stage[s]))
                    stage_busy[s] = True
                    n_chunks += 1
                # the previous quantised tensor goes to the file while this one's copies run
                flush_pending()
                k, nrows = t.ne
                nbytes = k // QK * nrows * bb
                fl.check(fl.lib.fl_dev_memset(dev_hist, 0, 16 * 8))
                fl.check(quantize_file(wtype, t.type, dev_in, dev_out, k, nrows, dev_hist))
                fl.check(fl.lib.fl_d2h(outbuf[0], dev_out, nbytes))
                fl.check(fl.lib.fl_d2h(hist_host[0], dev_hist, 16 * 8))
                fl.check(fl.lib.fl_event_record(ev_out))
                pending = (i, t, nbytes)
            flush_pending()
    finally:
        fl.check(fl.lib.fl_sync())
        for e in ev_stage + [ev_out]:
            fl.lib.fl_event_destroy(e)
        for p, _ in stage + [outbuf, hist_host]:
            fl.lib.fl_host_free_pinned(p)
        for d in (dev_in, dev_out, dev_hist):
            fl.free(d)
        del src
    if verbose:
        tot = sum(report["hist"]) or 1
        print(f"model size  = {report['total_size_org'] / 1024 / 1024:8.2f} MB")
        print(f"quant size  = {report['total_size_new'] / 1024 / 1024:8.2f} MB")
        print("hist: " + " ".join(f"{h / tot:5.3f}" for h in report["hist"]), flush=True)
    return report


def main(argv=None) -> int:
    argv = sys.argv[1:] if argv is None else argv
    if len(argv) != 3:
        print("usage: python -m fastllama_b200.quantize model-f32.bin model-quant.bin type\n  type = 2 - q4_0\n  type = 3 - q4_1",
              file=sys.stderr)
        return 1
    try:
        quantize_model(argv[0], argv[1], int(argv[2]))
    except QuantizeError as e:
        print(f"quantize: {e}", file=sys.stderr)
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
