"""Quantising PyTorch and Hugging Face checkpoints in one pass (fastllama_b200/quantize.py, read_checkpoint): the output
must be byte for byte what the reference's two steps write, its converter (scripts/convert.py --outtype f16 / f32) and
then its quantize tool (oracle/_ref/quantize_ref).

CPU tests run the converter itself, in a subprocess.  On some Python versions (3.12.3 among them) its reads of
torch.save zips fail: zipfile reports overlapping entries, and with that check cleared, CRC errors.  Those come from
the converter reading every tensor from eight threads through one ZipFile: the threads' seeks inside stored entries
race on the shared file position, so with the CRC check cleared as well, the output changes from run to run.  The
oracle run clears both checks and gives the converter's thread pool one worker (PATCHED_CONVERT), which makes its
output repeatable; test_reference_converter_fails_unpatched records the failure.  GPU tests, where the reference's
scripts are not available, quantise with the tool from the file tests/checkpoint_files.write_converted writes, a numpy
restatement of the converter's output that test_restatement_is_the_converter pins byte for byte.  CPU tests run
quantize_model over the stand-in device layer (tests/mock, with mock_quantize_file_f16round.c for source type 2); GPU
tests on the H100.
"""
import json
import os
import pickle
import struct
import subprocess
import sys
import zipfile

import numpy as np
import pytest

from fastllama_b200.quantize import QuantizeError, main, quantize_model
from tests.checkpoint_files import (TOKENIZER, hf_model, meta_model, permute, write_converted, write_hf, write_meta,
                                    write_safetensors)
from tests.test_quantize_model import QUANTIZE_REF, file_hist, need_ref, run_tool
from tests.test_quantize_parts import same_file

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REFERENCE_SCRIPTS = os.path.join(os.environ.get("REF", "/root/reference"), "scripts")
need_convert = pytest.mark.skipif(not os.path.exists(os.path.join(REFERENCE_SCRIPTS, "convert.py")),
                                  reason="the reference's scripts/convert.py is not available")
TOY = dict(n_vocab=300, n_embd=256, n_layer=2)              # head_dim 128: the converter's n_head = n_embd // 128
PATCHED_CONVERT = r"""
import concurrent.futures, runpy, sys, zipfile
_pool = concurrent.futures.ThreadPoolExecutor.__init__
concurrent.futures.ThreadPoolExecutor.__init__ = lambda self, *a, **k: _pool(self, max_workers=1)
_contents = zipfile.ZipFile._RealGetContents
def _no_end_offsets(self):
    _contents(self)
    for info in self.filelist:
        info._end_offset = None
zipfile.ZipFile._RealGetContents = _no_end_offsets
zipfile.ZipExtFile._update_crc = lambda self, newdata: None
sys.argv = ["convert.py"] + sys.argv[1:]
runpy.run_path("convert.py", run_name="__main__")
"""


def run_convert(model_path, out, outtype, vocab_dir=None, patched=True):
    args = ["--outtype", outtype, "--outfile", str(out)] + (["--vocab-dir", str(vocab_dir)] if vocab_dir else [])
    cmd = [sys.executable, "-c", PATCHED_CONVERT] if patched else [sys.executable, "convert.py"]
    return subprocess.run(cmd + args + [str(model_path)], cwd=REFERENCE_SCRIPTS, capture_output=True, text=True,
                          timeout=900)


def converted(model_path, out, outtype, vocab_dir=None):
    p = run_convert(model_path, out, outtype, vocab_dir)
    assert p.returncode == 0, (p.stdout[-2000:], p.stderr[-3000:])
    return str(out)


@pytest.fixture(scope="module")
def mock_fl(tmp_path_factory):
    """The CPU stand-in of the device layer (tests/mock/mock_fl_cuda.c) plus its fl_dev_quantize_q4_file with every
    source type (tests/mock/mock_quantize_file_f16round.c)."""
    from fastllama_b200.cuda_abi import FlCuda

    mock = os.path.join(ROOT, "tests", "mock")
    path = str(tmp_path_factory.mktemp("mockckpt") / "libfl_cuda.so")
    subprocess.run(["/usr/bin/gcc", "-O2", "-mavx2", "-mfma", "-mf16c", "-ffp-contract=off", "-fPIC", "-shared", "-w",
                    "-I" + os.path.join(ROOT, "include"), "-o", path, os.path.join(mock, "mock_fl_cuda.c"),
                    os.path.join(mock, "mock_quantize_file_f16round.c"), os.path.join(ROOT, "oracle", "q4_oracle.c"), "-lm",
                    "-lrt"],
                   check=True, capture_output=True, timeout=300)
    return FlCuda(path)


def write_layout(root, layout, model, vocab="parent", added=None, dtype_names=None):
    """A checkpoint of `model` (Meta names, joined) in layout pth1 / pth2 / pth4 / hf-bin / hf-safetensors under root,
    tokenizer.model beside it ("beside"), in its parent ("parent") or in root/vocab ("dir", for --vocab-dir).  Returns
    (the path to quantise, the --vocab-dir or None)."""
    d = root / "model"
    vocab_dir = {"beside": d, "parent": root, "dir": root / "vocab"}[vocab]
    os.makedirs(vocab_dir, exist_ok=True)
    with open(TOKENIZER, "rb") as f, open(vocab_dir / "tokenizer.model", "wb") as g:
        g.write(f.read())
    if added is not None:
        with open(vocab_dir / "added_tokens.json", "w") as f:
            json.dump(added, f)
    if layout.startswith("pth"):
        path = write_meta(str(d), model, int(layout[3:]))
    else:
        n_head = model["tok_embeddings.weight"].shape[1] // 128
        first = write_hf(str(d), hf_model(model, n_head), 2, layout[3:], dtype_names=dtype_names)
        path = str(d) if layout == "hf-bin" else first
    return path, (str(vocab_dir) if vocab == "dir" else None)


def quantise_both(fl, path, out_dir, outtype, wtypes=(2, 3), vocab_dir=None):
    outs = {}
    for w in wtypes:
        outs[w] = str(out_dir / f"ours-{outtype}-{w}.bin")
        rep = quantize_model(path, outs[w], w, fl=fl, verbose=False, outtype=outtype, vocab_dir=vocab_dir)
        assert rep["hist"] == file_hist(outs[w]).tolist()
    return outs


def check_two_steps(fl, tmp_path, path, outtype, ggjt, vocab_dir=None, wtypes=(2, 3)):
    """quantize_model on the checkpoint against quantize_ref on the converter's (or the restatement's) file ggjt."""
    ours = quantise_both(fl, path, tmp_path, outtype, wtypes, vocab_dir)
    for w in wtypes:
        same_file(ours[w], run_tool(QUANTIZE_REF, ggjt, str(tmp_path / f"ref-{outtype}-{w}.bin"), w))
    return ours


LAYOUTS = ["pth1", "pth2", "pth4", "hf-bin", "hf-safetensors"]
VOCAB_AT = {"pth1": "parent", "pth2": "beside", "pth4": "dir", "hf-bin": "beside", "hf-safetensors": "dir"}


# ---------------------------------------------------------------------------------------------------------------- CPU
@need_ref
@need_convert
@pytest.mark.parametrize("outtype", ["f16", "f32"])
@pytest.mark.parametrize("dtype", ["f16", "f32"])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_mock_checkpoint_output_is_the_two_step_file(mock_fl, tmp_path, layout, dtype, outtype):
    model = meta_model(**TOY, dtype=np.float16 if dtype == "f16" else np.float32, seed=5)
    path, vd = write_layout(tmp_path, layout, model, VOCAB_AT[layout])
    ggjt = converted(path, tmp_path / "conv.bin", outtype, vd)
    check_two_steps(mock_fl, tmp_path, path, outtype, ggjt, vd)


@need_ref
@need_convert
@pytest.mark.parametrize("case", ["one-added-token", "added-tokens-ignored"])
def test_mock_added_tokens(mock_fl, tmp_path, case):
    """added_tokens.json adds its tokens (score -1000) after tokenizer.model's when the model has room for them, and is
    ignored when the model has tokenizer.model's size."""
    n_vocab = 301 if case == "one-added-token" else 300
    model = meta_model(n_vocab=n_vocab, n_embd=256, n_layer=2, seed=6)
    path, vd = write_layout(tmp_path, "pth1", model, "parent", added={"<pad>": 300})
    ggjt = converted(path, tmp_path / "conv.bin", "f16", vd)
    check_two_steps(mock_fl, tmp_path, path, "f16", ggjt, vd)
    with open(ggjt, "rb") as f:
        assert struct.unpack_from("<i", f.read(12), 8)[0] == n_vocab


@need_convert
@pytest.mark.parametrize("layout,dtype,outtype", [("pth2", np.float16, "f16"), ("pth1", np.float32, "f16"),
                                                  ("hf-safetensors", np.float16, "f32"), ("pth4", np.float32, "f32")])
def test_restatement_is_the_converter(tmp_path, layout, dtype, outtype):
    """tests/checkpoint_files.write_converted, which the GPU tests use in place of the converter, writes its bytes."""
    model = meta_model(**TOY, dtype=dtype, seed=7)
    path, vd = write_layout(tmp_path, layout, model, VOCAB_AT[layout])
    ours = write_converted(str(tmp_path / "restated.bin"), model, TOKENIZER, outtype)
    same_file(ours, converted(path, tmp_path / "conv.bin", outtype, vd))


@need_convert
def test_reference_converter_fails_unpatched(tmp_path, mock_fl):
    """On this Python the reference's converter cannot read a torch.save checkpoint without the two zipfile checks
    cleared.  Should it succeed on another Python, its file must quantise to quantize_model's."""
    model = meta_model(**TOY, seed=8)
    path, _ = write_layout(tmp_path, "pth1", model, "parent")
    p = run_convert(path, tmp_path / "conv.bin", "f16", patched=False)
    if p.returncode == 0:
        ours = quantize_model(path, str(tmp_path / "ours.bin"), 2, fl=mock_fl, verbose=False)
        assert ours and os.path.exists(QUANTIZE_REF)
        same_file(tmp_path / "ours.bin", run_tool(QUANTIZE_REF, str(tmp_path / "conv.bin"), str(tmp_path / "ref.bin"), 2))
    else:
        assert "BadZipFile" in p.stderr and ("Overlapped entries" in p.stderr or "Bad CRC-32" in p.stderr), p.stderr[-2000:]


def test_mock_layouts_give_one_file(mock_fl, tmp_path):
    """The same weights as 1, 2 and 4 Meta shards and as Hugging Face .bin and safetensors files quantise to the same
    bytes: the joins and the q / k row permutation on the way to the device are the converter's."""
    model = meta_model(**TOY, seed=9)
    outs = []
    for layout in LAYOUTS:
        path, vd = write_layout(tmp_path / layout, layout, model, VOCAB_AT[layout])
        outs.append(quantise_both(mock_fl, path, tmp_path / layout, "f16", (3,), vd)[3])
    for o in outs[1:]:
        same_file(outs[0], o)
    assert np.array_equal(permute(hf_model(model, 2)["model.layers.1.self_attn.k_proj.weight"], 2),
                          model["layers.1.attention.wk.weight"])


def special_block_model(n_embd=256, n_vocab=300, seed=10):
    """An f32 model whose matrix blocks carry their minimum (q4_1 stores it in m as the f16 step leaves it) at values
    that test the f16 rounding: halfway between two f16 values (ties to even, both parities), the f16 subnormal range
    and its halfway points, and just under +-65504; the rest of each block lies above the minimum."""
    rng = np.random.default_rng(seed)
    model = meta_model(n_vocab=n_vocab, n_embd=n_embd, n_layer=2, dtype=np.float32, seed=seed)
    for name, a in model.items():
        if a.ndim != 2:
            continue
        blocks = a.reshape(-1, 32)
        nb = blocks.shape[0]
        kind = rng.integers(0, 4, nb)
        h = rng.uniform(-4, 4, nb).astype(np.float16)
        ulp = np.spacing(np.abs(h).astype(np.float16)).astype(np.float32)
        tie = h.astype(np.float32) + ulp / 2                                    # halfway between two f16 values
        sub = (rng.integers(-1024, 1024, nb) * 2.0 ** -24 + 2.0 ** -25).astype(np.float32)   # subnormal halfway points
        small = rng.uniform(-2.0 ** -14, 2.0 ** -14, nb).astype(np.float32)
        big = (rng.choice([-1, 1], nb) * (65504 - rng.uniform(0, 16, nb))).astype(np.float32)
        mn = np.select([kind == 0, kind == 1, kind == 2], [tie, sub, small], big)
        span = np.select([kind == 0, kind == 1, kind == 2], [np.abs(tie) * 0.5, np.full(nb, 2.0 ** -16), np.full(nb, 2.0 ** -14)],
                         np.full(nb, 8.0)).astype(np.float32)
        rest = mn[:, None] + rng.uniform(0, 1, (nb, 32)).astype(np.float32) * span[:, None]
        rest = np.minimum(rest, np.float32(65504))
        rest[:, 0] = mn
        rng.permuted(rest, axis=1, out=rest)
        blocks[:] = rest
    return model


@need_ref
@need_convert
@pytest.mark.parametrize("layout", ["pth2", "hf-safetensors"])
def test_mock_f32_checkpoint_f16_rounding(mock_fl, tmp_path, layout):
    model = special_block_model()
    path, vd = write_layout(tmp_path, layout, model, VOCAB_AT[layout])
    ggjt = converted(path, tmp_path / "conv.bin", "f16", vd)
    check_two_steps(mock_fl, tmp_path, path, "f16", ggjt, vd)


# ------------------------------------------------------------------------------------------------------- rejections
def _zip_entries(path):
    """name -> bytes of a torch.save zip, read from each entry's local header (zipfile's reader fails on them here)."""
    raw = open(path, "rb").read()
    out = {}
    for info in zipfile.ZipFile(path).infolist():
        n, m = struct.unpack_from("<HH", raw, info.header_offset + 26)
        off = info.header_offset + 30 + n + m
        out[info.filename] = raw[off:off + info.file_size]
    return out


def _rezip(path, entries, deflate=()):
    with zipfile.ZipFile(path, "w") as z:
        for name, data in entries.items():
            z.writestr(name, data, zipfile.ZIP_DEFLATED if name in deflate else zipfile.ZIP_STORED)


class _System:
    def __init__(self, cmd):
        self.cmd = cmd

    def __reduce__(self):
        return (os.system, (self.cmd,))


def _reject_case(tmp_path, case):
    """(path to quantise, vocab_dir, pattern the QuantizeError must match)."""
    model = meta_model(**TOY, seed=12)
    if case == "bf16":
        path, vd = write_layout(tmp_path, "hf-safetensors", model, "beside",
                                dtype_names={"model.layers.0.self_attn.v_proj.weight": "BF16"})
        return path, vd, r"model-00001-of-00002\.safetensors: tensor 'layers\.0\.attention\.wv\.weight' is BF16"
    if case == "gptq":
        path, vd = write_layout(tmp_path, "hf-safetensors", model, "beside")
        q = tmp_path / "model" / "model-00002-of-00002.safetensors"
        write_safetensors(str(q), [("model.layers.1.mlp.up_proj.qweight", np.int32, (32, 768), lambda: np.zeros((32, 768), np.int32))])
        return path, vd, r"model-00002-of-00002\.safetensors: tensor 'model\.layers\.1\.mlp\.up_proj\.qweight' is GPTQ"
    if case in ("compressed", "pickle-global"):
        path, vd = write_layout(tmp_path, "pth1", model, "parent")
        pth = os.path.join(path, "consolidated.00.pth")
        entries = _zip_entries(pth)
        pkl = next(n for n in entries if n.endswith("data.pkl"))
        if case == "compressed":
            _rezip(pth, entries, deflate={n for n in entries if "/data/" in n})
            return path, vd, r"consolidated\.00\.pth: tensor 'tok_embeddings\.weight' entry '.*/data/\d+' is compressed"
        marker = tmp_path / "marker"
        entries[pkl] = pickle.dumps({"tok_embeddings.weight": _System(f"touch {marker}")}, protocol=2)
        _rezip(pth, entries)
        return path, vd, r"consolidated\.00\.pth: data\.pkl names the global (posix|os)\.system"
    if case == "strides":
        import torch

        path, vd = write_layout(tmp_path, "pth1", model, "parent")
        sd = {n: torch.from_numpy(a) for n, a in model.items()}
        sd["layers.1.attention.wo.weight"] = torch.from_numpy(np.ascontiguousarray(model["layers.1.attention.wo.weight"].T)).t()
        torch.save(sd, os.path.join(path, "consolidated.00.pth"))
        return path, vd, r"consolidated\.00\.pth: tensor 'layers\.1\.attention\.wo\.weight' has strides \(1, 256\)"
    if case == "no-output":
        del model["output.weight"]
        path, vd = write_layout(tmp_path, "pth2", model, "parent")
        return path, vd, r"consolidated\.00\.pth: tensor 'output\.weight' not found"
    if case == "vocab-size":
        model = meta_model(n_vocab=305, n_embd=256, n_layer=1, seed=12)
        path, vd = write_layout(tmp_path, "pth1", model, "parent", added={"<pad>": 300})
        return path, vd, r"vocab size mismatch: the model has 305 tokens, but .*tokenizer\.model combined with .*added_tokens\.json has 301"
    if case == "no-tokenizer":
        path, vd = write_layout(tmp_path, "pth1", model, "dir")
        return path, None, r"no tokenizer\.model in .*model or its parent"
    raise AssertionError(case)


REJECT_CASES = ["bf16", "gptq", "compressed", "pickle-global", "strides", "no-output", "vocab-size", "no-tokenizer"]


@pytest.mark.parametrize("case", REJECT_CASES)
def test_rejects_checkpoint(tmp_path, case):
    path, vd, match = _reject_case(tmp_path, case)
    out = tmp_path / "out.bin"
    with pytest.raises(QuantizeError, match=match):
        quantize_model(path, str(out), 2, vocab_dir=vd)
    assert not out.exists()
    assert not (tmp_path / "marker").exists()


def test_rejects_checkpoint_options_for_model_files(tmp_path):
    from fastllama_b200.ggjt import F16, write_synthetic_float

    src = str(tmp_path / "in.bin")
    write_synthetic_float(src, F16, n_vocab=64, n_embd=64, n_mult=32, n_head=2, n_layer=1)
    with pytest.raises(QuantizeError, match=r"in\.bin is a model file: --outtype and --vocab-dir apply only to checkpoints"):
        quantize_model(src, str(tmp_path / "out.bin"), 2, outtype="f16")
    assert main([src, str(tmp_path / "out.bin"), "2", "--outtype", "f16"]) == 1
    assert main([src, str(tmp_path / "out.bin"), "2", "--vocab-dir", str(tmp_path)]) == 1
    assert main([src, str(tmp_path / "out.bin"), "2", "--outtype", "bf16"]) == 1
    assert not (tmp_path / "out.bin").exists()


def test_directory_with_two_checkpoints_is_refused(tmp_path):
    model = meta_model(**TOY, seed=13)
    path, _ = write_layout(tmp_path, "pth1", model, "parent")
    os.link(os.path.join(path, "consolidated.00.pth"), os.path.join(path, "extra.pt"))
    with pytest.raises(QuantizeError, match="several checkpoints"):
        quantize_model(path, str(tmp_path / "out.bin"), 2)


def test_safetensors_writer_is_read_by_the_library(tmp_path):
    """The tests' safetensors writer against the safetensors package's reader."""
    from safetensors.numpy import load_file

    a, b = np.arange(12, dtype=np.float16).reshape(3, 4), np.ones(5, np.float32)
    write_safetensors(str(tmp_path / "x.safetensors"), [("a", a.dtype, a.shape, lambda: a), ("b", b.dtype, b.shape, lambda: b)])
    got = load_file(str(tmp_path / "x.safetensors"))
    assert np.array_equal(got["a"], a) and np.array_equal(got["b"], b)


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def fl_gpu():
    from fastllama_b200.cuda_abi import FlCuda

    return FlCuda()


@pytest.mark.gpu
@need_ref
@pytest.mark.parametrize("outtype", ["f16", "f32"])
@pytest.mark.parametrize("dtype", ["f16", "f32"])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_gpu_checkpoint_output_is_the_two_step_file(fl_gpu, tmp_path, layout, dtype, outtype):
    model = meta_model(**TOY, dtype=np.float16 if dtype == "f16" else np.float32, seed=5)
    path, vd = write_layout(tmp_path, layout, model, VOCAB_AT[layout])
    ggjt = write_converted(str(tmp_path / "conv.bin"), model, TOKENIZER, outtype)
    check_two_steps(fl_gpu, tmp_path, path, outtype, ggjt, vd)


@pytest.mark.gpu
@need_ref
def test_gpu_added_token(fl_gpu, tmp_path):
    model = meta_model(n_vocab=301, n_embd=256, n_layer=2, seed=6)
    path, vd = write_layout(tmp_path, "hf-bin", model, "beside", added={"<pad>": 300})
    ggjt = write_converted(str(tmp_path / "conv.bin"), model, os.path.join(path, "tokenizer.model"), "f16")
    check_two_steps(fl_gpu, tmp_path, path, "f16", ggjt, vd)


@pytest.fixture(scope="module")
def seven_b_model():
    """LLaMA-7B matrix shapes over 2 layers with a 32000-token vocabulary (31700 added tokens after the toy
    tokenizer's 300), f16."""
    return meta_model(n_vocab=32000, n_embd=4096, n_layer=2, seed=14)


@pytest.mark.gpu
@need_ref
@pytest.mark.parametrize("layout", ["pth2", "hf-safetensors"])
def test_gpu_7b_shapes_checkpoint(fl_gpu, seven_b_model, tmp_path, layout):
    added = {f"<extra_{i}>": i for i in range(300, 32000)}
    path, vd = write_layout(tmp_path, layout, seven_b_model, "parent" if layout == "pth2" else "dir", added=added)
    tok = os.path.join(vd or str(tmp_path), "tokenizer.model")
    ggjt = write_converted(str(tmp_path / "conv.bin"), seven_b_model, tok, "f16")
    check_two_steps(fl_gpu, tmp_path, path, "f16", ggjt, vd)


@pytest.mark.gpu
@need_ref
@pytest.mark.parametrize("layout", ["pth2", "hf-safetensors"])
def test_gpu_f32_checkpoint_f16_rounding(fl_gpu, mock_fl, tmp_path, layout):
    """src_type 2 on the device against the stand-in's (_Float16) rounding and the reference's tool on the f16 file."""
    model = special_block_model()
    path, vd = write_layout(tmp_path, layout, model, VOCAB_AT[layout])
    ggjt = write_converted(str(tmp_path / "conv.bin"), model, TOKENIZER, "f16")
    ours = check_two_steps(fl_gpu, tmp_path, path, "f16", ggjt, vd)
    (tmp_path / "mock").mkdir()
    stand_in = quantise_both(mock_fl, path, tmp_path / "mock", "f16", vocab_dir=vd)
    for w in ours:
        same_file(ours[w], stand_in[w])


def signed_zero_model(seed=16):
    """An f16 model whose matrix blocks are non-negative with a zero minimum held as +0 and as -0, in either order:
    the reference's q4_1 m is the first of them."""
    rng = np.random.default_rng(seed)
    model = meta_model(**TOY, seed=seed)
    for a in model.values():
        if a.ndim == 2:
            blocks = a.reshape(-1, 32)
            blocks[:] = np.abs(blocks)
            for b in range(blocks.shape[0]):
                i, j = rng.choice(32, 2, replace=False)
                blocks[b, i], blocks[b, j] = np.float16(0.0), np.float16(-0.0)
    return model


@pytest.mark.gpu
@need_ref
@pytest.mark.parametrize("layout", ["pth1", "hf-bin"])
def test_gpu_signed_zero_minimum(fl_gpu, tmp_path, layout):
    """k_quantize_q4_file keeps the sign of a q4_1 block's first zero minimum, for checkpoints and model files."""
    model = signed_zero_model()
    path, vd = write_layout(tmp_path, layout, model, VOCAB_AT[layout])
    ggjt = write_converted(str(tmp_path / "conv.bin"), model, TOKENIZER, "f16")
    check_two_steps(fl_gpu, tmp_path, path, "f16", ggjt, vd)
    ours = quantize_model(ggjt, str(tmp_path / "file.bin"), 3, fl=fl_gpu, verbose=False)
    assert ours["hist"] == file_hist(str(tmp_path / "file.bin")).tolist()
    same_file(tmp_path / "file.bin", tmp_path / "ref-f16-3.bin")


@pytest.mark.gpu
@need_ref
@pytest.mark.parametrize("wtype", [2, 3])
def test_gpu_quantised_checkpoint_decodes_like_the_reference(fl_gpu, tmp_path, wtype):
    from oracle.pyoracle import REF_PYFASTLLAMA_SO
    from tests.test_gpu_e2e import DROPIN, _run

    assert os.path.exists(REF_PYFASTLLAMA_SO) and os.path.exists(DROPIN)
    model = meta_model(**TOY, seed=15, std=0.01)
    path, _ = write_layout(tmp_path, "pth2", model, "parent")
    out = str(tmp_path / "q.bin")
    quantize_model(path, out, wtype, fl=fl_gpu, verbose=False)
    ref_toks, ref_logits = _run(REF_PYFASTLLAMA_SO, out, 8, n_gen=16)
    our_toks, our_logits = _run(DROPIN, out, 8, n_gen=16)
    assert len(ref_toks) > 4
    assert our_toks == ref_toks, (our_toks, ref_toks)
    nd = int((our_logits.view(np.uint32) != ref_logits.view(np.uint32)).sum())
    assert nd == 0, (nd, our_logits.size, float(np.abs(our_logits - ref_logits).max()))
