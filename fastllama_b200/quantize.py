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

Input may also be a PyTorch (torch.save zip) or safetensors checkpoint, Meta or Hugging Face layout, given as a
directory or its first file: it is quantised as the f16 (outtype "f16", the default) or f32 file the reference's
scripts/convert.py writes from it (read_checkpoint), in one pass and without writing that file.

Streaming: each part is memory-mapped once and read one shard at a time through two pinned staging chunks, so a
read from a file overlaps the previous chunk's host-to-device copy, and a tensor's file reads overlap the previous
tensor's kernel and device-to-host copy; the previous tensor is written to the output while this one's copies run.
Row-split shards are copied to their place in the device input buffer; a column-split shard is copied to a device
scratch buffer and from there, with one pitched device copy, into its column range.  Host memory stays bounded
(two 64 MiB input chunks plus one pinned buffer of the largest quantised tensor); the device holds the largest
joined input tensor, its quantised form and, for split models, one column-split shard.
"""
from __future__ import annotations

import collections
import ctypes as C
import io
import json
import os
import pathlib
import pickle
import re
import struct
import sys
import zipfile
import zlib
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
    src_type: int = -1     # checkpoints: the type the shards store (F32 / F16) when it is not `type`
    permute_heads: int = 0  # checkpoints: n_head of the Hugging Face q / k row order to undo while staging


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


# ------------------------------------------------------------------------------------------------------- checkpoints
# PyTorch (torch.save zip) and safetensors checkpoints, read as the reference's converter reads them
# (scripts/convert.py: load_some_model, find_multifile_paths, lazy_load_file, merge_sharded,
# convert_transformers_to_orig, filter_and_sort_tensors, Params.guessed, SentencePieceVocab) and described as the
# f16 / f32 GGJT file it writes, so that quantising them gives that file's q4 file.  Nothing is loaded: every tensor
# is a Shard of a memory-mapped checkpoint file, staged like the tensors of a model file.
OUTTYPES = {"f32": F32, "f16": F16}
CKPT_ITEMSIZE = {"F16": 2, "F32": 4}
CKPT_TYPE = {"F16": F16, "F32": F32}
MAX_LAYERS = 80            # the converter's tensor list stops there


class _Stored(NamedTuple):
    """One tensor of a checkpoint file: its dtype name, shape (torch order, rows first) and data, or why its data
    cannot be read (`bad`, reported only if the tensor is kept)."""
    dtype: str
    shape: tuple
    shard: Shard
    bad: str = ""


class _StorageKind(NamedTuple):
    name: str                                   # torch.HalfStorage -> "HalfStorage"


class _Storage(NamedTuple):
    kind: _StorageKind
    entry: str
    offset: int                                 # of the entry's data in the file
    nbytes: int
    bad: str                                    # why the entry cannot be read in place ("" if it can)


class _TorchTensor(NamedTuple):
    storage: _Storage
    offset: int                                 # storage_offset, elements
    size: tuple
    stride: tuple


_TORCH_DTYPES = {"HalfStorage": "F16", "FloatStorage": "F32", "BFloat16Storage": "BF16", "IntStorage": "I32"}


def _rebuild_tensor_v2(storage, storage_offset, size, stride, requires_grad=False, backward_hooks=None, metadata=None):
    return _TorchTensor(storage, storage_offset, tuple(size), tuple(stride))


class _CheckpointUnpickler(pickle.Unpickler):
    """data.pkl of a torch.save zip without running it: the only globals it may name are the tensor rebuilder, the
    torch storage classes and OrderedDict, each replaced by a description; every tensor's storage is resolved to its
    entry of the zip, which is read in place later.  A checkpoint is untrusted input: anything else is refused."""

    def __init__(self, f, path, entries):
        super().__init__(f)
        self.path, self.entries = path, entries

    def find_class(self, module, name):
        if (module, name) == ("torch._utils", "_rebuild_tensor_v2"):
            return _rebuild_tensor_v2
        if (module, name) == ("collections", "OrderedDict"):
            return collections.OrderedDict
        if module == "torch" and name.endswith("Storage") and name.isidentifier():
            return _StorageKind(name)
        raise QuantizeError(f"{self.path}: data.pkl names the global {module}.{name}; a checkpoint's pickle may name "
                            "only torch._utils._rebuild_tensor_v2, torch storage classes and collections.OrderedDict")

    def persistent_load(self, pid):
        if not (isinstance(pid, tuple) and len(pid) >= 3 and pid[0] == "storage" and isinstance(pid[1], _StorageKind)):
            raise QuantizeError(f"{self.path}: data.pkl has an unrecognised persistent id {pid!r:.80}")
        key = str(pid[2])
        if key not in self.entries:
            raise QuantizeError(f"{self.path}: data.pkl refers to storage '{key}', which the archive does not hold")
        return _Storage(pid[1], *self.entries[key])


def _read_torch_zip(path: str, part: int) -> dict:
    """name -> _Stored of a torch.save zip.  The zip's central directory gives each entry; its data is found from the
    entry's local header and read in place, never through ZipFile.open (some Python versions report false overlap and
    CRC errors there for entries read at an offset)."""
    size = os.path.getsize(path)
    with open(path, "rb") as f:
        try:
            infos = zipfile.ZipFile(f).infolist()
        except zipfile.BadZipFile as e:
            raise QuantizeError(f"{path}: not a readable zip archive ({e})") from None
        pkls = [i for i in infos if i.filename.endswith(".pkl")]
        if len(pkls) != 1:
            raise QuantizeError(f"{path}: {len(pkls)} pickles in the archive, expected one data.pkl")
        data_dir = pkls[0].filename[:-4] + "/"          # <archive>/data.pkl -> its storages <archive>/data/<key>

        def locate(info):
            f.seek(info.header_offset)
            hdr = f.read(30)
            if len(hdr) != 30 or hdr[:4] != b"PK\x03\x04":
                raise QuantizeError(f"{path}: entry '{info.filename}' has no local header at {info.header_offset}")
            n, m = struct.unpack_from("<HH", hdr, 26)
            off = info.header_offset + 30 + n + m
            bad = ""
            if info.compress_type != zipfile.ZIP_STORED:
                bad = f"is compressed (method {info.compress_type}); only stored entries can be read in place"
            elif off + info.file_size > size:
                bad = "extends past the end of the file"
            return off, info.file_size, bad

        entries = {}
        for info in infos:
            if info.filename.startswith(data_dir):
                entries[info.filename[len(data_dir):]] = (info.filename, *locate(info))
            elif info.filename.endswith("/byteorder"):
                off, n, bad = locate(info)
                f.seek(off)
                if bad or f.read(n) != b"little":
                    raise QuantizeError(f"{path}: the archive's byteorder is not little-endian")
        off, n, bad = locate(pkls[0])
        if bad:
            raise QuantizeError(f"{path}: entry '{pkls[0].filename}' {bad}")
        f.seek(off)
        raw = f.read(n)
    if zlib.crc32(raw) != pkls[0].CRC:
        raise QuantizeError(f"{path}: CRC-32 of '{pkls[0].filename}' does not match the archive's directory")
    try:
        obj = _CheckpointUnpickler(io.BytesIO(raw), path, entries).load()
    except QuantizeError:
        raise
    except Exception as e:
        raise QuantizeError(f"{path}: data.pkl cannot be read as a state dict ({type(e).__name__}: {e})") from None
    if not isinstance(obj, dict):
        raise QuantizeError(f"{path}: data.pkl holds a {type(obj).__name__}, not a state dict")
    out = {}
    for name, t in obj.items():
        if not isinstance(t, _TorchTensor):
            continue
        st = t.storage
        dtype = _TORCH_DTYPES.get(st.kind.name, st.kind.name)
        item = CKPT_ITEMSIZE.get(dtype, 1)
        numel = int(np.prod(t.size, dtype=np.int64))
        want = [int(np.prod(t.size[d + 1:], dtype=np.int64)) for d in range(len(t.size))]
        bad = f"entry '{st.entry}' {st.bad}" if st.bad else ""
        if not bad and any(s != w and n != 1 for s, w, n in zip(t.stride, want, t.size)):
            bad = f"has strides {t.stride} for shape {t.size}, not row-major contiguous"
        elif not bad and (t.offset < 0 or (t.offset + numel) * item > st.nbytes):
            bad = (f"needs elements [{t.offset}, {t.offset + numel}) of storage '{st.entry}', which holds "
                   f"{st.nbytes // item}")
        out[str(name)] = _Stored(dtype, t.size, Shard(part, st.offset + t.offset * item, numel * item), bad)
    return out


def _read_safetensors(path: str, part: int) -> dict:
    size = os.path.getsize(path)
    with open(path, "rb") as f:
        (n,) = struct.unpack("<Q", _read(f, 8))
        try:
            header = json.loads(_read(f, n))
        except ValueError as e:
            raise QuantizeError(f"{path}: the safetensors header is not JSON ({e})") from None
    base = 8 + n
    out = {}
    for name, info in header.items():
        if name == "__metadata__":
            continue
        try:
            dtype, shape, (begin, end) = info["dtype"], tuple(int(d) for d in info["shape"]), info["data_offsets"]
        except (KeyError, TypeError, ValueError):
            raise QuantizeError(f"{path}: tensor '{name}' has a malformed header entry") from None
        if not 0 <= begin <= end <= size - base:
            raise QuantizeError(f"{path}: tensor '{name}' has data offsets [{begin}, {end}) outside the file's "
                                f"{size - base} data bytes")
        bad = ""
        if dtype in CKPT_ITEMSIZE and end - begin != int(np.prod(shape, dtype=np.int64)) * CKPT_ITEMSIZE[dtype]:
            bad = f"has {end - begin} data bytes, not the {int(np.prod(shape, dtype=np.int64)) * CKPT_ITEMSIZE[dtype]} of shape {shape}"
        out[name] = _Stored(dtype, shape, Shard(part, base + begin, end - begin), bad)
    return out


def checkpoint_kind(path: str):
    """'torch', 'safetensors' or None (a model file, or nothing the converter recognises): the converter's tests on a
    file's first bytes."""
    with open(path, "rb") as f:
        first8 = f.read(8)
    if len(first8) >= 4 and struct.unpack_from("<I", first8)[0] in (GGML_MAGIC, GGMF_MAGIC, GGJT_MAGIC, GGLA_MAGIC):
        return None
    if first8[:2] == b"PK":
        return "torch"
    if len(first8) == 8 and struct.unpack("<Q", first8)[0] < 16 << 20:
        return "safetensors"
    return None


def checkpoint_files(path: str) -> list:
    """The files of the checkpoint at path: a directory's consolidated.00.pth, pytorch_model-00001-of-*.bin or *.pt
    (exactly one), and from that first file its siblings x.01.pth, x.02.pth, ... or x-00002-of-N, ... (or x.1, x.2)."""
    p = pathlib.Path(path)
    if p.is_dir():
        found = [f for g in ("consolidated.00.pth", "pytorch_model-00001-of-*.bin", "*.pt") for f in sorted(p.glob(g))]
        if not found:
            raise QuantizeError(f"{path}: no consolidated.00.pth, pytorch_model-00001-of-*.bin or *.pt in the directory")
        if len(found) > 1:
            raise QuantizeError(f"{path}: several checkpoints in the directory, not sure which to pick: "
                                f"{', '.join(f.name for f in found)}")
        p = found[0]

    def nth(n):
        for pattern, repl in ((r"\.[0-9]{2}\.pth$", f".{n:02}.pth"), (r"-[0-9]{5}-of-(.*)$", rf"-{n:05}-of-\1"),
                              (r"(\.[0-9]+)?$", r"\1" if n == 0 else rf"\1.{n}")):
            if re.search(pattern, p.name):
                q = p.with_name(re.sub(pattern, repl, p.name))
                if q.exists():
                    return q
        return None

    # n counts up until no n-th file exists.  For x-00001-of-N the converter's rules also give x-00001-of-N for n = 0
    # (the x.bin, x.bin.1 rule), so the first file comes twice; it is read once here
    files, n = [], 0
    while (q := nth(n)) is not None:
        if q not in files:
            files.append(q)
        n += 1
    return [str(q) for q in files] or [str(p)]


def _read_vocab(vocab_path: pathlib.Path, n_vocab: int) -> list:
    """(token bytes, f32 score bytes) as the converter writes them from tokenizer.model and added_tokens.json."""
    import sentencepiece

    if vocab_path.is_dir():
        for cand in (vocab_path / "tokenizer.model", vocab_path.parent / "tokenizer.model"):
            if cand.exists():
                vocab_path = cand
                break
        else:
            raise QuantizeError(f"no tokenizer.model in {vocab_path} or its parent; name the directory that holds it "
                                "with --vocab-dir")
    sp = sentencepiece.SentencePieceProcessor()
    if not sp.Load(str(vocab_path)):
        raise QuantizeError(f"{vocab_path}: not a sentencepiece model")
    vocab = []
    for i in range(sp.GetPieceSize()):
        piece = sp.IdToPiece(i)
        if sp.IsUnknown(i):
            text = " ⁇ ".encode()
        elif sp.IsControl(i):
            text = b""
        elif sp.IsByte(i):
            if len(piece) != 6:
                raise QuantizeError(f"{vocab_path}: byte token {i} is '{piece}', not <0xXX>")
            text = bytes([int(piece[3:-1], 16)])
        else:
            text = piece.replace("▁", " ").encode()
        vocab.append((text, struct.pack("<f", sp.GetScore(i))))
    base = len(vocab)
    added_path = vocab_path.parent / "added_tokens.json"
    added = {}
    if added_path.exists():
        with open(added_path) as f:
            added = json.load(f)
        if sorted(added.values()) != list(range(base, base + len(added))):
            raise QuantizeError(f"{added_path}: added token ids {sorted(added.values())} do not follow the "
                                f"{base} of {vocab_path} in sequence")
    if n_vocab == base:
        return vocab                     # the model has the base size: added_tokens.json does not apply
    if n_vocab != base + len(added):
        more = f" combined with {added_path}" if added else ""
        raise QuantizeError(f"vocab size mismatch: the model has {n_vocab} tokens, but {vocab_path}{more} has "
                            f"{base + len(added)}")
    return vocab + [(text.encode(), struct.pack("<f", -1000.0)) for text, _ in sorted(added.items(), key=lambda kv: kv[1])]


_HF_LAYER = {"self_attn.q_proj": "attention.wq", "self_attn.k_proj": "attention.wk", "self_attn.v_proj": "attention.wv",
             "self_attn.o_proj": "attention.wo", "mlp.gate_proj": "feed_forward.w1", "mlp.down_proj": "feed_forward.w2",
             "mlp.up_proj": "feed_forward.w3", "input_layernorm": "attention_norm",
             "post_attention_layernorm": "ffn_norm"}
_LAYER_TENSORS = ["attention.wq", "attention.wk", "attention.wv", "attention.wo", "attention_norm", "feed_forward.w1",
                  "feed_forward.w2", "feed_forward.w3", "ffn_norm"]


def read_checkpoint(path: str, outtype: str = "f16", vocab_dir: str | None = None) -> ModelFile:
    """Describe the f16 (outtype "f16") or f32 GGJT file the reference's converter writes from the checkpoint at path
    (a directory or its first file), without writing it: the hyperparameters and vocab as bytes, and every kept
    tensor, in the converter's order, as shards of the checkpoint's files.  Refuses, naming the file and the tensor,
    every checkpoint the converter would reject or turn into a file the LLaMA loader cannot load."""
    if outtype not in OUTTYPES:
        raise QuantizeError(f"outtype {outtype!r}: use f16 or f32")
    paths = checkpoint_files(path)
    files = []
    for part, p in enumerate(paths):
        kind = checkpoint_kind(p)
        if kind is None:
            raise QuantizeError(f"{p}: not a torch zip or safetensors checkpoint")
        files.append(_read_torch_zip(p, part) if kind == "torch" else _read_safetensors(p, part))
        gptq = next((n for n in files[-1] if n.endswith(".qweight")), None)
        if gptq:
            raise QuantizeError(f"{p}: tensor '{gptq}' is GPTQ-quantised; only f16 / f32 checkpoints can be quantised")

    # name -> [(file index, _Stored)]: a Hugging Face checkpoint keeps each tensor whole in one file and is renamed to
    # the original names; the original checkpoints hold a shard of every tensor in every file
    hf = any("model.embed_tokens.weight" in f for f in files)
    if hf:
        merged = {}
        for i, f in enumerate(files):
            merged.update({n: [(i, s)] for n, s in f.items()})
        if "lm_head.weight" in merged:
            by_hf = merged
            merged = {"tok_embeddings.weight": by_hf["model.embed_tokens.weight"],
                      "norm.weight": by_hf.get("model.norm.weight"), "output.weight": by_hf["lm_head.weight"]}
            i = 0
            while f"model.layers.{i}.self_attn.q_proj.weight" in by_hf:
                for src, dst in _HF_LAYER.items():
                    merged[f"layers.{i}.{dst}.weight"] = by_hf.get(f"model.layers.{i}.{src}.weight")
                i += 1
            merged = {n: s for n, s in merged.items() if s is not None}
    else:
        merged = {}
        for f in files:
            for n in f:
                merged.setdefault(n, None)
        merged = {n: [(i, f[n]) for i, f in enumerate(files) if n in f] for n in merged}

    def missing(name, i=0):
        return QuantizeError(f"{paths[i]}: tensor '{name}' not found; the LLaMA loader needs it")

    if "tok_embeddings.weight" not in merged:
        raise missing("tok_embeddings.weight")
    n_layer = 0
    while f"layers.{n_layer}.attention.wq.weight" in merged:
        n_layer += 1
    if n_layer > MAX_LAYERS:
        raise QuantizeError(f"{paths[0]}: {n_layer} layers; the converter writes at most {MAX_LAYERS}")
    names = ["tok_embeddings.weight", "norm.weight", "output.weight"] + [
        f"layers.{i}.{t}.weight" for i in range(n_layer) for t in _LAYER_TENSORS]

    tok = merged["tok_embeddings.weight"]
    tok_shape = list(tok[0][1].shape)
    if len(tok_shape) != 2:
        raise QuantizeError(f"{paths[tok[0][0]]}: tensor 'tok_embeddings.weight' has shape {tuple(tok_shape)}, not 2-D")
    if len(tok) > 1:
        tok_shape[1] *= len(tok)                        # joined by columns
    n_vocab, n_embd = tok_shape
    n_head = n_embd // 128
    if n_head < 1:
        raise QuantizeError(f"{paths[0]}: n_embd {n_embd}; the converter's n_head = n_embd // 128 needs at least 128")
    ftype = OUTTYPES[outtype]

    tensors = []
    for name in names:
        if name not in merged:
            raise missing(name)
        shards = merged[name]
        if not hf and len(shards) < len(files):
            raise missing(name, min(set(range(len(files))) - {i for i, _ in shards}))
        (i0, s0), n = shards[0], len(shards)
        for i, s in shards:
            where = f"{paths[i]}: tensor '{name}'"
            if s.dtype not in CKPT_TYPE:
                raise QuantizeError(f"{where} is {s.dtype}; only F16 and F32 checkpoints can be quantised")
            if s.bad:
                raise QuantizeError(f"{where} {s.bad}")
            if (s.dtype, s.shape) != (s0.dtype, s0.shape):
                raise QuantizeError(f"{where} is {s.dtype} {s.shape} there but {s0.dtype} {s0.shape} in {paths[i0]}")
        if len(s0.shape) not in (1, 2):
            raise QuantizeError(f"{paths[i0]}: tensor '{name}' has {len(s0.shape)} dimensions (1 or 2 expected)")
        split = split_type(name, len(s0.shape), n)
        ne = tuple(reversed(s0.shape))
        if split == SPLIT_COLUMNS:
            ne = (ne[0] * n, ne[1])
        elif split == SPLIT_ROWS:
            ne = (ne[0], ne[1] * n)
        if max(ne) >= 1 << 32:
            raise QuantizeError(f"{paths[i0]}: the extents {ne} of tensor '{name}' overflow 32 bits")
        if len(ne) == 2 and ne[0] % QK:
            raise QuantizeError(f"{paths[i0]}: tensor '{name}' has rows of {ne[0]} elements, not a multiple of {QK}")
        t = F32 if len(ne) == 1 else ftype             # the converter writes vectors as f32
        src = CKPT_TYPE[s0.dtype]
        heads = 0
        if hf and name.endswith((".attention.wq.weight", ".attention.wk.weight")):
            heads = merged["layers.0.attention.wq.weight"][0][1].shape[1] // 128
            if heads < 1 or ne[1] % (2 * heads):
                raise QuantizeError(f"{paths[i0]}: tensor '{name}' has {ne[1]} rows, which cannot be permuted for "
                                    f"{heads} heads")
        tensors.append(Tensor(name, ne, t, split, tuple(s.shard for _, s in shards),
                              int(np.prod(ne, dtype=np.int64)) * ELEM_BYTES[t], src, heads))
    hparams = struct.pack("<7i", n_vocab, n_embd, 256, n_head, n_layer, n_embd // n_head, ftype)
    vocab = _read_vocab(pathlib.Path(vocab_dir) if vocab_dir else pathlib.Path(paths[0]).parent, n_vocab)
    return ModelFile(paths, hparams, vocab, tensors)


def _tensor_header(t: Tensor, new_type: int) -> bytes:
    nm = t.name.encode()
    return struct.pack(f"<III{len(t.ne)}I", len(t.ne), len(nm), new_type, *t.ne) + nm


def _pinned(fl: FlCuda, nbytes: int):
    p = fl.lib.fl_host_alloc_pinned(nbytes)
    if not p:
        raise MemoryError(fl.lib.fl_last_error().decode())
    return p, np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(p))


def _src_type(t: Tensor) -> int:
    """The type of t's data as staged: its shards' type."""
    return t.type if t.src_type < 0 else t.src_type


def quantize_model(in_path: str, out_path: str, wtype: int, fl: FlCuda | None = None, verbose: bool = True, *,
                   outtype: str | None = None, vocab_dir: str | None = None) -> dict:
    """Quantise in_path to out_path (q4_0 for wtype 2, q4_1 for 3).  in_path is an f32 / f16 model file (for a model
    in parts, part 0's path) or a PyTorch / safetensors checkpoint (a directory or its first file, see
    read_checkpoint).  A checkpoint is quantised as the f16 (outtype None or "f16") or f32 ("f32") file the reference's
    converter writes from it; vocab_dir is where its tokenizer.model is, if not beside the checkpoint or in its parent.
    outtype and vocab_dir are refused for model files, which carry their types and vocab.  Returns the number of parts
    read, per-tensor and total sizes and the 16-bin histograms of the stored nibbles (counts), as the reference's tool
    reports them (sizes and types of a checkpoint's tensors are those of the converter's file)."""
    if wtype not in (Q4_0, Q4_1):
        hint = " (q4_2 / q4_3 / mostly-q4_1-some-f16 are not supported)" if wtype in (4, 5, 6) else ""
        raise QuantizeError(f"invalid quantization type {wtype}{hint}: use 2 (q4_0) or 3 (q4_1)")
    if os.path.isdir(in_path) or checkpoint_kind(in_path):
        model = read_checkpoint(in_path, outtype or "f16", vocab_dir)
    else:
        if outtype is not None or vocab_dir is not None:
            raise QuantizeError(f"{in_path} is a model file: --outtype and --vocab-dir apply only to checkpoints")
        model = read_model(in_path)
    fl = fl or FlCuda()
    quantize_file = fl.fn("fl_dev_quantize_q4_file")
    bb = BLOCK_BYTES[wtype]
    mats = [t for t in model.tensors if len(t.ne) == 2]
    staged = {t.name: int(np.prod(t.ne, dtype=np.int64)) * ELEM_BYTES[_src_type(t)] for t in mats}
    max_in = max(staged.values(), default=0)
    max_out = max((t.ne[0] // QK * t.ne[1] * bb for t in mats), default=0)

    # a column-split shard, or a Hugging Face q / k matrix, lands in dev_cols first; then pitched device copies put it
    # into its column range of dev_in, or its rows into the converter's order
    max_cols = max((t.shards[0].nbytes for t in mats if t.split == SPLIT_COLUMNS or t.permute_heads), default=0)

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
                    data = srcs[sh.part][sh.offset:sh.offset + sh.nbytes]
                    if _src_type(t) != t.type:          # an f16 checkpoint's vector, which the converter widens
                        data = data.view(np.float16).astype(np.float32).view(np.uint8)
                    write_tensor(t, t.type, data)
                    record(i, t, t.type, t.nbytes, None)
                    continue
                # stage the shards into the device input buffer, one pinned chunk at a time, so that it holds the joined
                # tensor: row-split shards back to back, each column-split shard in its column range of every row.
                # These copies queue behind the previous tensor's kernel and copies on the library stream, so reusing
                # dev_in / dev_cols / dev_out is safe
                shards = t.shards[:1] if t.split == SPLIT_NONE else t.shards
                for j, sh in enumerate(shards):
                    dst = dev_cols if t.split == SPLIT_COLUMNS or t.permute_heads else dev_in + j * sh.nbytes
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
                if t.permute_heads:
                    # the converter's permute: within head h, output row 2i + p is input row p * hd/2 + i, so each
                    # (head, p) is hd/2 consecutive rows put every other row
                    rb, hd = sh.nbytes // t.ne[1], t.ne[1] // t.permute_heads
                    for h in range(t.permute_heads):
                        for p in range(2):
                            fl.check(fl.lib.fl_d2d_2d(dev_in + (h * hd + p) * rb, 2 * rb, dev_cols + (h * hd + p * hd // 2) * rb,
                                                      rb, rb, hd // 2))
                # the previous quantised tensor goes to the file while this one's copies run
                flush_pending()
                k, nrows = t.ne
                nbytes = k // QK * nrows * bb
                # src 2: an f32 checkpoint's values as the converter's f16 file holds them
                src = 2 if (_src_type(t), t.type) == (F32, F16) else _src_type(t)
                fl.check(fl.lib.fl_dev_memset(dev_hist, 0, 16 * 8))
                fl.check(quantize_file(wtype, src, dev_in, dev_out, k, nrows, dev_hist))
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


USAGE = """usage: python -m fastllama_b200.quantize IN OUT TYPE [--outtype f16|f32] [--vocab-dir DIR]
  TYPE = 2 - q4_0, 3 - q4_1
  IN: an f16 / f32 model file (a model in parts: part 0; the others are read from IN.1, IN.2, ...), or a
      PyTorch / safetensors checkpoint (a directory, or its first file), quantised as the f16 (--outtype f16, the
      default) or f32 file the reference's scripts/convert.py writes from it; tokenizer.model is read from
      --vocab-dir, else from beside the checkpoint, else from its parent directory"""


def main(argv=None) -> int:
    argv = list(sys.argv[1:] if argv is None else argv)
    opts, args = {}, []
    while argv:
        a = argv.pop(0)
        key, eq, val = a.partition("=")
        if key in ("--outtype", "--vocab-dir"):
            if not eq:
                if not argv:
                    print(USAGE, file=sys.stderr)
                    return 1
                val = argv.pop(0)
            opts[key[2:].replace("-", "_")] = val
        else:
            args.append(a)
    if len(args) != 3 or opts.get("outtype", "f16") not in OUTTYPES:
        print(USAGE, file=sys.stderr)
        return 1
    try:
        quantize_model(args[0], args[1], int(args[2]), **opts)
    except QuantizeError as e:
        print(f"quantize: {e}", file=sys.stderr)
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
