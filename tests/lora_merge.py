"""The file quantize_model(..., lora=ADAPTER) must write, built from the reference alone: the reference's attach_lora
graphs (lib/llama.cpp:867-873: BA = mul_mat(loraA, loraB) for an uncached adapter, then ggml_add_inplace(W, BA or the
cached delta)) run on the reference's ggml library (oracle/_ref/libggml_ref.so) for every tensor the adapter names,
written back into a copy of the f16 / f32 model file, which the reference's quantize tool (oracle/_ref/quantize_ref)
then quantises.  tests/test_quantize_lora.py pins these graphs against the reference's real attach on the same f16
model; tools/time_quantize_lora.py uses them too.
"""
import ctypes as C
import shutil
import struct

import numpy as np

from fastllama_b200.quantize import read_model
from oracle.pyoracle import REF_GGML_SO
from tests import ggml_api as G
from tests.test_quantize_model import QUANTIZE_REF, run_tool

DTYPE = {G.F32: np.float32, G.F16: np.float16}


def read_ggla(path):
    """(cached, r, alpha, [(name, ne, type, array of shape (ne1, ne0))]) of an adapter file, in file order."""
    raw = np.memmap(path, dtype=np.uint8, mode="r")
    magic, version, cached, r, alpha = struct.unpack_from("<IIBII", raw, 0)
    assert (magic, version) == (0x67676C61, 1)
    off, out = 17, []
    while off < raw.size:
        n_dims, name_len, t = struct.unpack_from("<iii", raw, off)
        ne = struct.unpack_from(f"<{n_dims}i", raw, off + 12)
        off += 12 + 4 * n_dims
        name = bytes(raw[off:off + name_len]).decode()
        off += name_len
        off += -off & 31
        n = int(np.prod(ne))
        out.append((name, ne, t, np.frombuffer(raw, dtype=DTYPE[t], count=n, offset=off).reshape(ne[1], ne[0])))
        off += n * np.dtype(DTYPE[t]).itemsize
    return bool(cached), r, alpha, out


def merge_reference(model_path, adapter_path, out_path, lib=REF_GGML_SO):
    """Copy the single-file f16 / f32 model at model_path to out_path with the adapter merged into it by the
    reference's attach graphs on the ggml library at lib.  Returns the names of the merged tensors."""
    shutil.copyfile(model_path, out_path)
    tensors = {t.name: t for t in read_model(model_path).tensors}
    cached, _, _, entries = read_ggla(adapter_path)
    groups = {}
    for name, ne, t, a in entries:
        base, key = (name[:-5], "lora") if cached else (name[:-6], name[-1])
        groups.setdefault(base, {})[key] = (ne, t, a)
    g = G.Ggml(lib)
    src = np.memmap(model_path, dtype=np.uint8, mode="r")
    with open(out_path, "r+b") as f:
        for base, parts in groups.items():
            w = tensors[base]
            k, m = w.ne
            off = w.shards[0].offset
            ar = g.context(w.nbytes + sum(a.nbytes for *_, a in parts.values()) + k * m * 4 + (1 << 20))
            tw = g.new_tensor_2d(ar.ctx, w.type, k, m)
            ar.set(tw, src[off:off + w.nbytes])
            if cached:
                ne, t, a = parts["lora"]
                delta = g.new_tensor_2d(ar.ctx, t, ne[0], ne[1])
                ar.set(delta, a)
            else:
                ops = []
                for key in "AB":
                    ne, t, a = parts[key]
                    ops.append(g.new_tensor_2d(ar.ctx, t, ne[0], ne[1]))
                    ar.set(ops[-1], a)
                delta = g.mul_mat(ar.ctx, ops[0], ops[1])
            res = g.add_inplace(ar.ctx, tw, delta)
            gf = G.new_graph()
            g.build_forward_expand(gf, res)
            g.graph_compute(ar.ctx, gf)
            f.seek(off)
            f.write(C.string_at(tw.contents.data, w.nbytes))
            ar.free()
    return sorted(groups)


def expected_q4(model_path, adapter_path, wtype, tmp_dir, tag="ref"):
    """quantize_ref's output for the model at model_path after the reference's attach of the adapter."""
    merged = str(tmp_dir / f"{tag}-merged.bin")
    merge_reference(model_path, adapter_path, merged)
    return run_tool(QUANTIZE_REF, merged, str(tmp_dir / f"{tag}-q{wtype}.bin"), wtype)
