"""Quantise an f32 / f16 model file to q4_0 or q4_1 on the GPU: the middle step of the reference's pipeline
(scripts/convert.py -> quantize -> model), writing byte for byte the file the reference's quantize tool writes.

    python -m fastllama_b200.quantize IN OUT TYPE        TYPE: 2 = q4_0, 3 = q4_1 (the reference CLI's arguments)

Input: a model the reference's reader accepts (include/file_loader.hpp:94-250, 387-453), as one file or as the
parts IN, IN.1, IN.2, ... that the reference's converter writes per checkpoint shard (LLaMA-13B, 30B and 65B:
2, 4 and 8 parts).  IN is part 0; the number of parts is n_embd / tok_embeddings.ne[0] of part 0.  Every part is
GGML (no version, vocab without scores: the score becomes 0.0), GGMF v1 or GGJT v1 (tensor data 32-byte aligned)
on its own, with 1-D or 2-D f32 / f16 tensors and the same hyperparameters as part 0.  Every part holds every
tensor; a tensor's shards (its entries in the parts) must agree in type and extents and are joined as the
reference's reader joins them (include/tensor/utils.hpp:93-150, file_loader.hpp:597-637): a vector is part 0's;
the token embeddings, wo and w2 are split by columns (row r is every shard's row r, in part order); every other
matrix is split by rows (the shards back to back).

Output: what the reference's FileSaver writes (include/file_loader.hpp:254-375): GGJT v1, part 0's
hyperparameters, its vocab as {u32 len, bytes, f32 score}, then the joined tensors in part 0's order, each
padded with zeros to 32 bytes before its data.  Every 2-D tensor is quantised (lib/llama.cpp:558-572 never
excludes one) by k_quantize_q4_file (fl_dev_quantize_q4_file), 1-D tensors are copied unchanged.  For a part set
that is the reference tool's output for the joined model written as one file.  The reference's tool itself
aborts on every part set: its File move constructor (include/detail/file.hpp:55-58) copies the FILE pointer
without clearing it, so when ModelLoader's vector of loaders grows to take part 1, the moved-from loader closes
part 0's file and the first read from part 0 fails.

Streaming: each part is memory-mapped once and read one shard at a time through two pinned staging chunks, so a
read from a file overlaps the previous chunk's host-to-device copy, and a tensor's file reads overlap the previous
tensor's kernel and device-to-host copy; the previous tensor is written to the output while this one's copies run.
Row-split shards are copied to their place in the device input buffer; a column-split shard is copied to a device
scratch buffer and from there, with one pitched device copy, into its column range.  Host memory stays bounded
(two 64 MiB input chunks plus one pinned buffer of the largest quantised tensor); the device holds the largest
joined input tensor, its quantised form and, for split models, one column-split shard.
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
SPLIT_NONE, SPLIT_ROWS, SPLIT_COLUMNS = 0, 1, 2                       # how a tensor's shards are joined


class QuantizeError(ValueError):
    pass


class Shard(NamedTuple):
    part: int          # index of the part file that holds it
    offset: int        # of the data in that file
    nbytes: int


class Tensor(NamedTuple):
    name: str
    ne: tuple          # joined extents, ne0 (row length) first
    type: int
    split: int         # SPLIT_NONE, SPLIT_ROWS or SPLIT_COLUMNS
    shards: tuple      # one Shard per part, in part order; SPLIT_NONE reads shards[0] only
    nbytes: int        # of the joined tensor


class ModelFile(NamedTuple):
    paths: list        # the part files, part 0 (the path the user names) first
    hparams: bytes     # part 0's 7 header integers, raw: n_vocab, n_embd, n_mult, n_head, n_layer, n_rot, ftype
    vocab: list        # part 0's (token bytes, raw f32 score bytes)
    tensors: list      # in part 0's order


class _Part(NamedTuple):
    hparams: bytes
    vocab: list
    entries: list      # (name, ne, type, offset, nbytes) in file order


def _read(f, n: int) -> bytes:
    b = f.read(n)
    if len(b) != n:
        raise QuantizeError(f"{f.name}: unexpected end of file")
    return b


def _read_part(path: str) -> _Part:
    """Parse one file's header, vocab and tensor table, rejecting every entry the tool would otherwise have to guess
    about."""
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
        (n_vocab,) = struct.unpack_from("<i", hparams)
        vocab = []
        for _ in range(n_vocab):
            (n,) = struct.unpack("<I", _read(f, 4))
            tok = _read(f, n)
            vocab.append((tok, b"\0\0\0\0" if version == "ggml" else _read(f, 4)))      # GGML has no scores: 0.0
        entries, names = [], set()
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
            if version == "ggjt":
                f.seek(-f.tell() & 31, os.SEEK_CUR)
            nbytes = int(np.prod(ne, dtype=np.int64)) * ELEM_BYTES[t]
            off = f.tell()
            if off + nbytes > size:
                raise QuantizeError(f"{path}: tensor '{name}' extends past the end of the file")
            entries.append((name, tuple(ne), t, off, nbytes))
            f.seek(nbytes, os.SEEK_CUR)
    return _Part(hparams, vocab, entries)


def split_type(name: str, n_dims: int, n_parts: int) -> int:
    """How the reference joins a tensor's shards (include/tensor/utils.hpp:93-114): the token embeddings and the
    matrices whose input is split across parts (wo, w2) are cut into column ranges, every other matrix into row
    ranges; a vector, or any tensor of a single-file model, is taken whole from part 0."""
    if n_dims == 1 or n_parts == 1:
        return SPLIT_NONE
    if name.startswith("tok_embeddings.") or ".attention.wo.weight" in name or ".feed_forward.w2.weight" in name:
        return SPLIT_COLUMNS
    return SPLIT_ROWS


def read_model(path: str) -> ModelFile:
    """Parse a model stored as one file or as parts path, path.1, path.2, ... (as the reference's converter writes a
    model per checkpoint shard), join every tensor's shards by the reference's rules and reject every input the tool
    would otherwise have to guess about, naming the file and the tensor."""
    part0 = _read_part(path)
    n_embd = struct.unpack_from("<7i", part0.hparams)[1]
    # the reader takes n_embd / tok_embeddings.ne[0] of part 0 as the number of parts (include/file_loader.hpp:387-453)
    tok = next((e for e in part0.entries if e[0] == "tok_embeddings.weight"), None)
    if tok is None:
        raise QuantizeError(f"{path}: tok_embeddings.weight not found")
    if not 0 < tok[1][0] <= n_embd:
        raise QuantizeError(f"{path}: tok_embeddings.weight has rows of {tok[1][0]} elements, not a part of n_embd {n_embd}")
    n_parts = n_embd // tok[1][0]
    paths, parts = [path], [part0]
    for i in range(1, n_parts):
        p = f"{path}.{i}"
        if not os.path.exists(p):
            raise QuantizeError(f"{path}: multi-part model ({n_parts} parts by n_embd / tok_embeddings.ne[0] = {n_embd} / "
                                f"{tok[1][0]}), but part {i}, {p}, does not exist")
        part = _read_part(p)
        if part.hparams != part0.hparams:
            raise QuantizeError(f"{p}: hyperparameters {struct.unpack('<7i', part.hparams)} differ from those of {path} "
                                f"{struct.unpack('<7i', part0.hparams)}")
        paths.append(p)
        parts.append(part)

    # Every part must hold every tensor.  The reference's reader would join whatever shards a tensor has, so a tensor
    # missing from a part would come out as a part-sized matrix whose extents contradict the hyperparameters.
    shards = {name: [] for name, *_ in part0.entries}      # name -> [(ne, type, Shard)] in part order
    for i, part in enumerate(parts):
        for name, ne, t, off, nbytes in part.entries:
            if name not in shards:
                raise QuantizeError(f"{paths[i]}: tensor '{name}' is not in part 0, {path}")
            shards[name].append((ne, t, Shard(i, off, nbytes)))
    tensors = []
    for name, sh in shards.items():
        if len(sh) < n_parts:
            i = min(set(range(n_parts)) - {s.part for *_, s in sh})
            raise QuantizeError(f"{paths[i]}: tensor '{name}' of part 0 is missing")
        ne, t, _ = sh[0]
        for ne_i, t_i, s in sh[1:]:
            if t_i != t:
                raise QuantizeError(f"{paths[s.part]}: tensor '{name}' is {TYPE_NAMES[t_i]} there but {TYPE_NAMES[t]} in "
                                    f"{path} (inconsistent tensor shard type)")
            if ne_i != ne:
                raise QuantizeError(f"{paths[s.part]}: tensor '{name}' has extents {ne_i} there but {ne} in {path} "
                                    "(inconsistent tensor shard extents)")
        split = split_type(name, len(ne), n_parts)
        if split == SPLIT_COLUMNS:
            ne = (ne[0] * n_parts, ne[1])
        elif split == SPLIT_ROWS:
            ne = (ne[0], ne[1] * n_parts)
        if max(ne) >= 1 << 32:
            raise QuantizeError(f"{path}: the joined extents {ne} of tensor '{name}' overflow 32 bits")
        if len(ne) == 2 and ne[0] % QK:
            raise QuantizeError(f"{path}: tensor '{name}' has rows of {ne[0]} elements, not a multiple of {QK}")
        tensors.append(Tensor(name, ne, t, split, tuple(s for *_, s in sh), int(np.prod(ne, dtype=np.int64)) * ELEM_BYTES[t]))
    return ModelFile(paths, part0.hparams, part0.vocab, tensors)


def _tensor_header(t: Tensor, new_type: int) -> bytes:
    nm = t.name.encode()
    return struct.pack(f"<III{len(t.ne)}I", len(t.ne), len(nm), new_type, *t.ne) + nm


def _pinned(fl: FlCuda, nbytes: int):
    p = fl.lib.fl_host_alloc_pinned(nbytes)
    if not p:
        raise MemoryError(fl.lib.fl_last_error().decode())
    return p, np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(p))


def quantize_model(in_path: str, out_path: str, wtype: int, fl: FlCuda | None = None, verbose: bool = True) -> dict:
    """Quantise in_path (f32 / f16; for a model in parts, part 0's path) to out_path (q4_0 for wtype 2, q4_1 for 3).
    Returns the number of parts read, per-tensor and total sizes and the 16-bin histograms of the stored nibbles
    (counts), as the reference's tool reports them."""
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

    # a column-split shard lands in dev_cols first, then a pitched device copy puts it into its column range of dev_in
    max_cols = max((t.shards[0].nbytes for t in mats if t.split == SPLIT_COLUMNS), default=0)

    srcs = [np.memmap(p, dtype=np.uint8, mode="r") for p in model.paths]
    dev_in = fl.alloc(max(max_in, 16))
    dev_cols = fl.alloc(max_cols) if max_cols else None
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

    report = {"n_parts": len(model.paths), "tensors": [], "total_size_org": 0, "total_size_new": 0, "hist": [0] * 16}

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
                    sh = t.shards[0]
                    write_tensor(t, t.type, srcs[sh.part][sh.offset:sh.offset + sh.nbytes])
                    record(i, t, t.type, t.nbytes, None)
                    continue
                # stage the shards into the device input buffer, one pinned chunk at a time, so that it holds the joined
                # tensor: row-split shards back to back, each column-split shard in its column range of every row.
                # These copies queue behind the previous tensor's kernel and copies on the library stream, so reusing
                # dev_in / dev_cols / dev_out is safe
                shards = t.shards[:1] if t.split == SPLIT_NONE else t.shards
                for j, sh in enumerate(shards):
                    dst = dev_cols if t.split == SPLIT_COLUMNS else dev_in + j * sh.nbytes
                    src = srcs[sh.part]
                    for off in range(0, sh.nbytes, chunk):
                        n = min(chunk, sh.nbytes - off)
                        s = n_chunks % 2
                        if stage_busy[s]:
                            fl.check(fl.lib.fl_event_sync(ev_stage[s]))      # the chunk staged there before is on the device
                        stage[s][1][:n] = src[sh.offset + off:sh.offset + off + n]
                        fl.check(fl.lib.fl_h2d(dst + off, stage[s][0], n))
                        fl.check(fl.lib.fl_event_record(ev_stage[s]))
                        stage_busy[s] = True
                        n_chunks += 1
                    if t.split == SPLIT_COLUMNS:
                        w = sh.nbytes // t.ne[1]
                        fl.check(fl.lib.fl_d2d_2d(dev_in + j * w, w * len(shards), dev_cols, w, w, t.ne[1]))
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
        for d in (dev_in, dev_cols, dev_out, dev_hist):
            if d is not None:
                fl.free(d)
        del srcs
    if verbose:
        tot = sum(report["hist"]) or 1
        print(f"model size  = {report['total_size_org'] / 1024 / 1024:8.2f} MB")
        print(f"quant size  = {report['total_size_new'] / 1024 / 1024:8.2f} MB")
        print("hist: " + " ".join(f"{h / tot:5.3f}" for h in report["hist"]), flush=True)
    return report


def main(argv=None) -> int:
    argv = sys.argv[1:] if argv is None else argv
    if len(argv) != 3:
        print("usage: python -m fastllama_b200.quantize model-f32.bin model-quant.bin type\n  type = 2 - q4_0\n  type = 3 - q4_1\n"
              "  a model in parts: give part 0; the others are read from model-f32.bin.1, model-f32.bin.2, ...", file=sys.stderr)
        return 1
    try:
        quantize_model(argv[0], argv[1], int(argv[2]))
    except QuantizeError as e:
        print(f"quantize: {e}", file=sys.stderr)
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
