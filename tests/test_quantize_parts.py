"""Quantising models stored as several part files (fastllama_b200/quantize.py, part 0's path and the parts PATH.1,
PATH.2, ... beside it) against the reference's own quantize tool (oracle/_ref/quantize_ref): the output must be byte for
byte the tool's output for the same model joined into one file.

The part sets are written here by splitting a synthetic float model the way the reference's reader joins one: vectors
whole in every part, the token embeddings, wo and w2 cut into column ranges, every other matrix into row ranges, each
shard its own Gaussian stream; write_joined writes the model they join to.  The reference's tool cannot read the part
sets themselves (test_reference_tool_aborts_on_part_sets records that), so it quantises the joined file.  CPU tests run
the tool over the stand-in device layer (tests/mock); GPU tests run it on the H100 at toy size and at LLaMA-13B matrix
shapes, and decode greedily from a quantised 2-part model with the drop-in library and with the reference library.
"""
import os
import struct
import subprocess

import numpy as np
import pytest

from fastllama_b200.ggjt import (F16, F32, Q4_0, Q4_1, splits_by_columns, tensor_plan, write_synthetic_joined,
                                 write_synthetic_parts)
from fastllama_b200.quantize import QuantizeError, quantize_model
from tests.test_quantize_model import QUANTIZE_REF, file_hist, need_ref, run_tool

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# n_embd 96 and n_ff 288: over 2 parts the token-embedding and wo shards are 48 wide and the w2 shards 144, over 4
# parts 24 and 72 -- column shards whose width is not a multiple of 32, joined into rows that are
TOY = dict(n_vocab=300, n_embd=96, n_mult=96, n_head=3, n_layer=2)


def same_file(a, b):
    x, y = np.memmap(a, dtype=np.uint8, mode="r"), np.memmap(b, dtype=np.uint8, mode="r")
    assert x.size == y.size, (x.size, y.size)
    nd = int(np.count_nonzero(x != y))
    assert nd == 0, f"{nd} bytes differ (first at {int(np.argmax(x != y))})"


def check_against_reference(fl, out_dir, fmts, ftype, wtype, **kw):
    """Quantise a part set written by write_synthetic_parts(fmts, ftype, **kw) and compare with the reference tool's
    output for the joined model, written as one file in part 0's format."""
    part0 = write_synthetic_parts(str(out_dir / "in.bin"), fmts, ftype, **kw)
    ours = str(out_dir / "ours.bin")
    rep = quantize_model(part0, ours, wtype, fl=fl, verbose=False)
    joined = write_synthetic_joined(str(out_dir / "joined.bin"), len(fmts), ftype, fmt=fmts[0], **kw)
    ref = run_tool(QUANTIZE_REF, joined, str(out_dir / "ref.bin"), wtype)
    for p in [joined, part0] + [f"{part0}.{j}" for j in range(1, len(fmts))]:
        os.unlink(p)
    same_file(ours, ref)
    assert rep["hist"] == file_hist(ours).tolist()
    assert rep["n_parts"] == len(fmts)
    return rep, ours, ref


@pytest.fixture(scope="module")
def mock_fl(tmp_path_factory):
    """The CPU stand-in of the device layer (tests/mock/mock_fl_cuda.c) plus its fl_dev_quantize_q4_file
    (tests/mock/mock_quantize_file.c), built as one library in a temporary directory with the stand-in's flags."""
    from fastllama_b200.cuda_abi import FlCuda

    mock = os.path.join(ROOT, "tests", "mock")
    path = str(tmp_path_factory.mktemp("mockparts") / "libfl_cuda.so")
    subprocess.run(["/usr/bin/gcc", "-O2", "-mavx2", "-mfma", "-mf16c", "-ffp-contract=off", "-fPIC", "-shared", "-w",
                    "-I" + os.path.join(ROOT, "include"), "-o", path, os.path.join(mock, "mock_fl_cuda.c"),
                    os.path.join(mock, "mock_quantize_file.c"), os.path.join(ROOT, "oracle", "q4_oracle.c"), "-lm", "-lrt"],
                   check=True, capture_output=True, timeout=300)
    return FlCuda(path)


# part sets: the format of each part, the float type
SETS = [
    (["ggjt", "ggjt"], F16),
    (["ggjt", "ggjt"], F32),
    (["ggmf", "ggmf", "ggmf"], F16),
    (["ggml", "ggml", "ggml"], F32),
    (["ggjt"] * 4, F16),
    (["ggmf"] * 4, F32),
    (["ggml", "ggjt", "ggmf"], F16),
    (["ggjt", "ggml", "ggmf", "ggjt"], F32),
]
SET_IDS = [f"{len(f)}parts-{'-'.join(f)}-{'f16' if t == F16 else 'f32'}" for f, t in SETS]


# ---------------------------------------------------------------------------------------------------------------- CPU
@need_ref
@pytest.mark.parametrize("wtype", [Q4_0, Q4_1])
@pytest.mark.parametrize("fmts,ftype", SETS, ids=SET_IDS)
def test_mock_parts_output_is_the_reference_file(mock_fl, tmp_path, fmts, ftype, wtype):
    rep, ours, _ = check_against_reference(mock_fl, tmp_path, fmts, ftype, wtype, **TOY)
    hist = file_hist(ours)
    assert sum(h for t in rep["tensors"] if t["hist"] for h in t["hist"]) == int(hist.sum())
    assert int(hist.sum()) == sum(int(np.prod(t["ne"])) for t in rep["tensors"] if len(t["ne"]) == 2)
    want = dict(tensor_plan(**TOY))
    assert [(t["name"], tuple(t["ne"])) for t in rep["tensors"]] == list(want.items())      # joined extents, part 0's order


@pytest.mark.parametrize("wtype", [Q4_0, Q4_1])
@pytest.mark.parametrize("n_parts", [2, 3, 4])
def test_mock_parts_equal_the_joined_single_file(mock_fl, tmp_path, n_parts, wtype):
    part0 = write_synthetic_parts(str(tmp_path / "in.bin"), ["ggjt"] * n_parts, F16, **TOY)
    single = write_synthetic_joined(str(tmp_path / "single.bin"), n_parts, F16, **TOY)
    a = quantize_model(part0, str(tmp_path / "a.bin"), wtype, fl=mock_fl, verbose=False)
    b = quantize_model(single, str(tmp_path / "b.bin"), wtype, fl=mock_fl, verbose=False)
    same_file(tmp_path / "a.bin", tmp_path / "b.bin")
    assert (a["n_parts"], b["n_parts"]) == (n_parts, 1)
    assert a["hist"] == b["hist"] and a["tensors"] == b["tensors"]


@need_ref
def test_mock_shards_span_staging_chunks(mock_fl, tmp_path, monkeypatch):
    """Chunks of 1000 bytes: every shard spans several, and chunks alternate between the two pinned buffers across
    shard and tensor boundaries."""
    import fastllama_b200.quantize as q

    monkeypatch.setattr(q, "CHUNK_BYTES", 1000)
    check_against_reference(mock_fl, tmp_path, ["ggjt", "ggmf", "ggml"], F16, Q4_1, **TOY)


@need_ref
def test_reference_tool_aborts_on_part_sets(mock_fl, tmp_path):
    """The reference's tool fails on every part set: its File move constructor (include/detail/file.hpp) copies the
    FILE pointer without clearing it, so when ModelLoader's vector of file loaders grows to take part 1, the moved-from
    loader closes part 0's file and the first read from part 0 fails.  Should a fixed reference read part sets, its
    output must be this tool's."""
    part0 = write_synthetic_parts(str(tmp_path / "in.bin"), ["ggjt", "ggjt"], F16, **TOY)
    p = subprocess.run([QUANTIZE_REF, part0, str(tmp_path / "ref.bin"), "2"], capture_output=True, text=True, timeout=300)
    if p.returncode == 0:
        quantize_model(part0, str(tmp_path / "ours.bin"), Q4_0, fl=mock_fl, verbose=False)
        same_file(tmp_path / "ours.bin", tmp_path / "ref.bin")
    else:
        assert "failed to read data" in p.stderr, p.stderr[-2000:]


def test_mock_memory_bounds(mock_fl, tmp_path, monkeypatch):
    """Device: the largest joined input, its quantised form, one column-split shard and the histogram.  Host (pinned):
    two staging chunks, the largest quantised tensor and the histogram."""
    part0 = write_synthetic_parts(str(tmp_path / "in.bin"), ["ggjt"] * 2, F32, **TOY)
    dev, host = [], []
    alloc, pinned = mock_fl.alloc, mock_fl.lib.fl_host_alloc_pinned
    monkeypatch.setattr(mock_fl, "alloc", lambda n: dev.append(n) or alloc(n))
    monkeypatch.setattr(mock_fl.lib, "fl_host_alloc_pinned", lambda n: host.append(n) or pinned(n))
    quantize_model(part0, str(tmp_path / "out.bin"), Q4_0, fl=mock_fl, verbose=False)
    mats = [(name, ne[0] * ne[1]) for name, ne in tensor_plan(**TOY) if len(ne) == 2]
    largest = max(n for _, n in mats) * 4               # joined, f32
    q_largest = max(n for _, n in mats) // 32 * 20
    col_shard = max(n for name, n in mats if splits_by_columns(name)) // 2 * 4
    assert sorted(dev) == sorted([largest, q_largest, col_shard, 128])
    assert sorted(host) == sorted([largest, largest, q_largest, 128])       # toy tensors fit a chunk: chunk = largest


def _swap(tensors, name, ne, t, data):
    return [(name, ne, t, data) if x[0] == name else x for x in tensors]


WQ = "layers.0.attention.wq.weight"
REJECTIONS = {
    # case: (edit of the part set, message)
    "hyperparameters": (lambda j, hp, ts: ((hp[:2] + (32,) + hp[3:]) if j == 1 else hp, ts), r"in\.bin\.1: hyperparameters"),
    "shard-extents": (lambda j, hp, ts: (hp, _swap(ts, WQ, (96, 32), F16, bytes(96 * 32 * 2)) if j == 1 else ts),
                      r"in\.bin\.1: tensor 'layers\.0\.attention\.wq\.weight' has extents .*inconsistent tensor shard extents"),
    "shard-type": (lambda j, hp, ts: (hp, _swap(ts, WQ, (96, 48), F32, bytes(96 * 48 * 4)) if j == 1 else ts),
                   r"in\.bin\.1: tensor 'layers\.0\.attention\.wq\.weight' is f32 there .*inconsistent tensor shard type"),
    # wo shards 40 wide: the joined rows are 80 elements, not whole q4 blocks (the check is on the joined row)
    "joined-row": (lambda j, hp, ts: (hp, _swap(ts, "layers.0.attention.wo.weight", (40, 96), F16, bytes(40 * 96 * 2))),
                   r"in\.bin: tensor 'layers\.0\.attention\.wo\.weight' has rows of 80 elements, not a multiple of 32"),
    "quantised-shard": (lambda j, hp, ts: (hp, _swap(ts, WQ, (96, 48), Q4_0, bytes(3 * 48 * 20)) if j == 1 else ts),
                        r"in\.bin\.1: tensor 'layers\.0\.attention\.wq\.weight' is already quantised"),
    "duplicate": (lambda j, hp, ts: (hp, ts + [ts[-1]] if j == 1 else ts),
                  r"in\.bin\.1: tensor 'layers\.1\.ffn_norm\.weight' appears twice"),
    # the reference's reader would join the shards a tensor has: part 0's alone here, a matrix half the size the
    # hyperparameters give, which no loader accepts
    "missing-tensor": (lambda j, hp, ts: (hp, [t for t in ts if t[0] != WQ] if j == 1 else ts),
                       r"in\.bin\.1: tensor 'layers\.0\.attention\.wq\.weight' of part 0 is missing"),
    "extra-tensor": (lambda j, hp, ts: (hp, ts + [("extra.weight", (64, 2), F16, bytes(256))] if j == 1 else ts),
                     r"in\.bin\.1: tensor 'extra\.weight' is not in part 0"),
}


@pytest.mark.parametrize("case", list(REJECTIONS))
def test_rejects_inconsistent_parts(tmp_path, case):
    edit, match = REJECTIONS[case]
    part0 = write_synthetic_parts(str(tmp_path / "in.bin"), ["ggjt"] * 2, F16, edit=edit, **TOY)
    with pytest.raises(QuantizeError, match=match):
        quantize_model(part0, str(tmp_path / "out.bin"), Q4_0)
    assert not os.path.exists(tmp_path / "out.bin")


@pytest.mark.parametrize("case", ["missing", "truncated", "lora"])
def test_rejects_unreadable_later_part(tmp_path, case):
    part0 = write_synthetic_parts(str(tmp_path / "in.bin"), ["ggjt"] * 3, F16, **TOY)
    later = part0 + ".2"
    if case == "missing":
        os.unlink(later)
        match = r"multi-part model \(3 parts .*part 2, .*in\.bin\.2, does not exist"
    elif case == "truncated":
        os.truncate(later, os.path.getsize(later) - 100)
        match = r"in\.bin\.2: tensor 'layers\.1\.ffn_norm\.weight' extends past the end of the file"
    else:
        with open(later, "wb") as f:
            f.write(struct.pack("<IIIi", 0x67676C61, 1, 8, 16))
        match = r"in\.bin\.2 is a LoRA adapter"
    with pytest.raises(QuantizeError, match=match):
        quantize_model(part0, str(tmp_path / "out.bin"), Q4_0)
    assert not os.path.exists(tmp_path / "out.bin")


# ---------------------------------------------------------------------------------------------------------------- GPU
THIRTEEN_B_2L = dict(n_vocab=8000, n_embd=5120, n_mult=256, n_head=40, n_layer=2)


@pytest.fixture(scope="module")
def fl_gpu():
    from fastllama_b200.cuda_abi import FlCuda

    return FlCuda()


@pytest.mark.gpu
@need_ref
@pytest.mark.parametrize("wtype", [Q4_0, Q4_1])
@pytest.mark.parametrize("fmts,ftype", [SETS[0], SETS[3], SETS[4], SETS[7]], ids=[SET_IDS[i] for i in (0, 3, 4, 7)])
def test_gpu_toy_parts_output_is_the_reference_file(fl_gpu, tmp_path, fmts, ftype, wtype):
    check_against_reference(fl_gpu, tmp_path, fmts, ftype, wtype, **TOY)


@pytest.mark.gpu
@need_ref
@pytest.mark.parametrize("wtype", [Q4_0, Q4_1])
def test_gpu_13b_shapes_two_parts_output_is_the_reference_file(fl_gpu, tmp_path, wtype):
    """A 2-part f16 model with LLaMA-13B matrix shapes (n_embd 5120, n_ff 13824) over two layers and an 8000-token
    vocabulary: the w1 / w3 shards and the column-split w2 shards (6912 x 5120) are each larger than one staging chunk."""
    rep, _, _ = check_against_reference(fl_gpu, tmp_path, ["ggjt", "ggjt"], F16, wtype, seed=13, **THIRTEEN_B_2L)
    assert {t["name"]: tuple(t["ne"]) for t in rep["tensors"]}["layers.0.feed_forward.w2.weight"] == (13824, 5120)


@pytest.mark.gpu
@need_ref
@pytest.mark.parametrize("wtype", [Q4_0, Q4_1])
def test_gpu_quantised_parts_decode_like_the_reference(fl_gpu, tmp_path, wtype):
    from oracle.pyoracle import REF_PYFASTLLAMA_SO
    from tests.test_gpu_e2e import DROPIN, _run

    assert os.path.exists(REF_PYFASTLLAMA_SO) and os.path.exists(DROPIN)
    _, ours, ref = check_against_reference(fl_gpu, tmp_path, ["ggjt", "ggmf"], F16, wtype, seed=11, std=0.01,
                                           n_vocab=512, n_embd=256, n_mult=64, n_head=4, n_layer=3)
    ref_toks, ref_logits = _run(REF_PYFASTLLAMA_SO, ref, 8)
    our_toks, our_logits = _run(DROPIN, ours, 8)
    assert len(ref_toks) > 4
    assert our_toks == ref_toks, (our_toks, ref_toks)
    nd = int((our_logits.view(np.uint32) != ref_logits.view(np.uint32)).sum())
    assert nd == 0, (nd, our_logits.size, float(np.abs(our_logits - ref_logits).max()))
