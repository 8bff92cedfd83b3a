"""Model-file quantisation (fastllama_b200/quantize.py, k_quantize_q4_file) against the reference's own quantize tool
(oracle/_ref/quantize_ref: src/quantize.cpp over the reference's lib/ggml.c, CPU): the output files must be equal
byte for byte.

CPU tests run the tool over the stand-in device layer (tests/mock, the oracle's quantisers).  GPU tests run it on
the H100 at toy size and at LLaMA-7B matrix shapes, run the reference's threaded tool over libggml_b200 (the
drop-in fastllama_b200/lib/quantize) once, and decode greedily from a quantised file with the drop-in library and
with the reference library.
"""
import os
import struct
import subprocess

import numpy as np
import pytest

from fastllama_b200.build import lib_path
from fastllama_b200.ggjt import F16, F32, GGJT_MAGIC, Q4_0, Q4_1, vocab_entries, write_model_file, write_synthetic_float
from fastllama_b200.quantize import QuantizeError, main, quantize_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
QUANTIZE_REF = os.path.join(ROOT, "oracle", "_ref", "quantize_ref")
DROPIN_QUANTIZE = lib_path("quantize")
TOY = dict(n_vocab=300, n_embd=256, n_mult=64, n_head=4, n_layer=2)
need_ref = pytest.mark.skipif(not os.path.exists(QUANTIZE_REF), reason="oracle/_ref/quantize_ref not built (no reference sources at build time)")


def run_tool(exe, src, dst, wtype):
    p = subprocess.run([exe, src, dst, str(wtype)], capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, (exe, p.returncode, p.stdout[-2000:], p.stderr[-2000:])
    return dst


def file_hist(path):
    """16-bin histogram of every stored nibble of the q4 tensors of a GGJT file, counted with numpy."""
    raw = np.memmap(path, dtype=np.uint8, mode="r")
    magic, version = struct.unpack_from("<II", raw, 0)
    assert (magic, version) == (GGJT_MAGIC, 1)
    n_vocab = struct.unpack_from("<i", raw, 8)[0]
    off = 36
    for _ in range(n_vocab):
        off += 4 + struct.unpack_from("<I", raw, off)[0] + 4
    hist = np.zeros(16, dtype=np.int64)
    while off < raw.size:
        n_dims, name_len, t = struct.unpack_from("<III", raw, off)
        ne = struct.unpack_from(f"<{n_dims}I", raw, off + 12)
        off += 12 + 4 * n_dims + name_len
        off += -off & 31
        n = int(np.prod(ne))
        if t in (Q4_0, Q4_1):
            bb, qoff = (20, 4) if t == Q4_0 else (24, 8)
            qs = raw[off:off + n // 32 * bb].reshape(-1, bb)[:, qoff:qoff + 16]
            hist += np.bincount((qs & 0xF).ravel(), minlength=16) + np.bincount((qs >> 4).ravel(), minlength=16)
            off += n // 32 * bb
        else:
            off += n * (4 if t == F32 else 2)
    return hist


@pytest.fixture(scope="module")
def mock_fl(tmp_path_factory):
    """The CPU stand-in of the device layer (tests/mock/mock_fl_cuda.c) plus its fl_dev_quantize_q4_file
    (tests/mock/mock_quantize_file.c), built as one library in a temporary directory with the stand-in's flags."""
    from fastllama_b200.cuda_abi import FlCuda

    mock = os.path.join(ROOT, "tests", "mock")
    path = str(tmp_path_factory.mktemp("mockq") / "libfl_cuda.so")
    subprocess.run(["/usr/bin/gcc", "-O2", "-mavx2", "-mfma", "-mf16c", "-ffp-contract=off", "-fPIC", "-shared", "-w",
                    "-I" + os.path.join(ROOT, "include"), "-o", path, os.path.join(mock, "mock_fl_cuda.c"),
                    os.path.join(mock, "mock_quantize_file.c"), os.path.join(ROOT, "oracle", "q4_oracle.c"), "-lm", "-lrt"],
                   check=True, capture_output=True, timeout=300)
    return FlCuda(path)


def check_against_reference(fl, tmp_path, fmt, ftype, wtype, **shape):
    src = str(tmp_path / f"in-{fmt}-{ftype}.bin")
    write_synthetic_float(src, ftype, seed=3, std=0.02, fmt=fmt, **shape)
    ours = str(tmp_path / "ours.bin")
    rep = quantize_model(src, ours, wtype, fl=fl, verbose=False)
    want = run_tool(QUANTIZE_REF, src, str(tmp_path / "ref.bin"), wtype)
    a, b = np.memmap(ours, dtype=np.uint8, mode="r"), np.memmap(want, dtype=np.uint8, mode="r")
    assert a.size == b.size, (a.size, b.size)
    nd = int(np.count_nonzero(a != b))
    assert nd == 0, f"{nd} bytes differ from the reference's quantize output (first at {int(np.argmax(a != b))})"
    return rep, ours


# ---------------------------------------------------------------------------------------------------------------- CPU
@need_ref
@pytest.mark.parametrize("wtype", [Q4_0, Q4_1])
@pytest.mark.parametrize("fmt,ftype", [("ggjt", F32), ("ggjt", F16), ("ggmf", F16), ("ggml", F32)])
def test_mock_output_is_the_reference_file(mock_fl, tmp_path, fmt, ftype, wtype):
    rep, ours = check_against_reference(mock_fl, tmp_path, fmt, ftype, wtype, **TOY)
    hist = file_hist(ours)
    assert rep["hist"] == hist.tolist()
    assert sum(h for t in rep["tensors"] if t["hist"] for h in t["hist"]) == int(hist.sum())
    n_q = sum(int(np.prod(t["ne"])) for t in rep["tensors"] if len(t["ne"]) == 2)
    assert int(hist.sum()) == n_q
    assert rep["total_size_new"] < rep["total_size_org"]


def _write(path, tok_ne0=64, tok_type=F32, extra=()):
    """A minimal model (n_embd 64): a token embedding, a norm and `extra` tensors."""
    n_embd, n_vocab = 64, 8
    tok_bytes = {F32: 4 * tok_ne0, F16: 2 * tok_ne0, Q4_0: tok_ne0 // 32 * 20}[tok_type] * n_vocab
    tensors = [("tok_embeddings.weight", (tok_ne0, n_vocab), tok_type, bytes(tok_bytes)),
               ("norm.weight", (n_embd,), F32, np.ones(n_embd, np.float32).tobytes()), *extra]
    write_model_file(path, "ggjt", (n_vocab, n_embd, 64, 2, 1, 32, 0), vocab_entries(n_vocab), tensors)
    return path


@pytest.mark.parametrize("wtype", [4, 5, 6, 0, 1, 7])
def test_rejects_target_types(tmp_path, wtype):
    path = _write(str(tmp_path / "in.bin"))
    with pytest.raises(QuantizeError, match="invalid quantization type"):
        quantize_model(path, str(tmp_path / "out.bin"), wtype)
    assert not os.path.exists(tmp_path / "out.bin")


def test_rejects_multi_part(tmp_path):
    path = _write(str(tmp_path / "in.bin"), tok_ne0=32)              # n_embd 64 / 32: the reader would look for in.bin.1
    with pytest.raises(QuantizeError, match="multi-part model"):
        quantize_model(path, str(tmp_path / "out.bin"), Q4_0)


def test_rejects_lora_adapter(tmp_path):
    path = str(tmp_path / "adapter.bin")
    with open(path, "wb") as f:
        f.write(struct.pack("<IIIi", 0x67676C61, 1, 8, 16))           # 'ggla', version 1, r, alpha
    with pytest.raises(QuantizeError, match="LoRA adapter"):
        quantize_model(path, str(tmp_path / "out.bin"), Q4_0)


def test_rejects_quantised_input(tmp_path):
    path = _write(str(tmp_path / "in.bin"), tok_type=Q4_0)
    with pytest.raises(QuantizeError, match="already quantised"):
        quantize_model(path, str(tmp_path / "out.bin"), Q4_1)


def test_rejects_rows_not_a_multiple_of_32(tmp_path):
    odd = ("layers.0.attention.wq.weight", (48, 4), F32, bytes(48 * 4 * 4))
    path = _write(str(tmp_path / "in.bin"), extra=[odd])
    with pytest.raises(QuantizeError, match="not a multiple of 32"):
        quantize_model(path, str(tmp_path / "out.bin"), Q4_0)


def test_cli_usage():
    assert main(["only-one-argument"]) == 1


# ---------------------------------------------------------------------------------------------------------------- GPU
SEVEN_B_2L = dict(n_vocab=32000, n_embd=4096, n_mult=256, n_head=32, n_layer=2)


@pytest.fixture(scope="module")
def fl_gpu():
    from fastllama_b200.cuda_abi import FlCuda

    return FlCuda()


@pytest.mark.gpu
@need_ref
@pytest.mark.parametrize("wtype", [Q4_0, Q4_1])
@pytest.mark.parametrize("fmt,ftype", [("ggjt", F32), ("ggjt", F16), ("ggmf", F16)])
def test_gpu_toy_output_is_the_reference_file(fl_gpu, tmp_path, fmt, ftype, wtype):
    rep, ours = check_against_reference(fl_gpu, tmp_path, fmt, ftype, wtype, **TOY)
    assert rep["hist"] == file_hist(ours).tolist()


@pytest.fixture(scope="module")
def seven_b_inputs(tmp_path_factory):
    """2-layer files with LLaMA-7B shapes: the full 32000 x 4096 embedding and output matrices (each far above one
    staging chunk and one ggml_quantize_chunk), f16 and f32."""
    d = tmp_path_factory.mktemp("q7b")
    paths = {}
    for ftype in (F16, F32):
        paths[ftype] = str(d / f"7b-2l-{ftype}.bin")
        write_synthetic_float(paths[ftype], ftype, seed=7, std=0.02, **SEVEN_B_2L)
    yield paths
    for p in paths.values():
        os.unlink(p)


@pytest.mark.gpu
@need_ref
@pytest.mark.parametrize("wtype", [Q4_0, Q4_1])
@pytest.mark.parametrize("ftype", [F16, F32])
def test_gpu_7b_shapes_output_is_the_reference_file(fl_gpu, seven_b_inputs, tmp_path, ftype, wtype):
    src = seven_b_inputs[ftype]
    ours = str(tmp_path / "ours.bin")
    rep = quantize_model(src, ours, wtype, fl=fl_gpu, verbose=False)
    want = run_tool(QUANTIZE_REF, src, str(tmp_path / "ref.bin"), wtype)
    a, b = np.memmap(ours, dtype=np.uint8, mode="r"), np.memmap(want, dtype=np.uint8, mode="r")
    assert a.size == b.size
    nd = int(np.count_nonzero(a != b))
    assert nd == 0, f"{nd} bytes differ from the reference's quantize output"
    assert rep["hist"] == file_hist(ours).tolist()
    if ftype == F16 and wtype == Q4_0:
        # the reference's own threaded tool over libggml_b200: eight threads call ggml_quantize_chunk at once, each
        # staging through the library's shared buffers.  One run; its output must be the reference's file too.
        assert os.path.exists(DROPIN_QUANTIZE), "drop-in quantize not built"
        got = run_tool(DROPIN_QUANTIZE, src, str(tmp_path / "dropin.bin"), wtype)
        c = np.memmap(got, dtype=np.uint8, mode="r")
        assert c.size == b.size
        nd = int(np.count_nonzero(c != b))
        assert nd == 0, f"the drop-in quantize wrote {nd} bytes unlike the reference's"


@pytest.mark.gpu
@need_ref
@pytest.mark.parametrize("wtype", [Q4_0, Q4_1])
def test_gpu_quantised_file_decodes_like_the_reference(fl_gpu, tmp_path, wtype):
    from oracle.pyoracle import REF_PYFASTLLAMA_SO
    from tests.test_gpu_e2e import DROPIN, _run

    assert os.path.exists(REF_PYFASTLLAMA_SO) and os.path.exists(DROPIN)
    src = str(tmp_path / "f16.bin")
    write_synthetic_float(src, F16, n_vocab=512, n_embd=256, n_mult=64, n_head=4, n_layer=3, seed=11, std=0.01)
    path = str(tmp_path / "q.bin")
    quantize_model(src, path, wtype, fl=fl_gpu, verbose=False)
    ref_toks, ref_logits = _run(REF_PYFASTLLAMA_SO, path, 8)
    our_toks, our_logits = _run(DROPIN, path, 8)
    assert len(ref_toks) > 4
    assert our_toks == ref_toks, (our_toks, ref_toks)
    nd = int((our_logits.view(np.uint32) != ref_logits.view(np.uint32)).sum())
    assert nd == 0, (nd, our_logits.size, float(np.abs(our_logits - ref_logits).max()))
