"""Quantising with a LoRA adapter merged in (quantize_model(..., lora=), --lora; fl_dev_quantize_q4_file_lora): the
output must be byte for byte the reference quantize tool's file for the f16 / f32 model after the reference's
attach_lora, built by tests/lora_merge.py from the reference alone (its attach graphs on oracle/_ref/libggml_ref.so,
then oracle/_ref/quantize_ref).

test_merge_graphs_are_the_reference_attach pins those graphs: on the reference product library, the f16 model with the
adapter attached and the merged f16 file with none decode to the same logit bits.  CPU tests run quantize_model over the
stand-in device layer (tests/mock, with mock_quantize_file_lora.c); GPU tests on the H100, at toy sizes and at LLaMA-7B
matrix shapes, and a merged q4 file decodes with the reference library's bits.
"""
import os
import subprocess

import numpy as np
import pytest

from fastllama_b200.ggjt import F16, F32, n_ff, write_synthetic_float, write_synthetic_joined, write_synthetic_parts
from fastllama_b200.quantize import QuantizeError, main, quantize_model
from tests.checkpoint_files import TOKENIZER, meta_model, write_converted
from tests.lora_files import FORMS, TARGETS, write_adapter, write_lora
from tests.lora_merge import expected_q4, merge_reference
from tests.test_quantize_checkpoint import VOCAB_AT, write_layout
from tests.test_quantize_model import file_hist, need_ref
from tests.test_quantize_parts import same_file

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOY = dict(n_vocab=300, n_embd=256, n_layer=2)                      # meta_model / write_converted: n_ff 768
SUBSET = ("attention.wq", "attention.wv")
TARGET_SETS = {"wq-wv": SUBSET, "all7": TARGETS}


@pytest.fixture(scope="module")
def mock_fl(tmp_path_factory):
    """The CPU stand-in of the device layer with fl_dev_quantize_q4_file for every source type and
    fl_dev_quantize_q4_file_lora.  -Bsymbolic: the stand-in's calls between its own entry points (the merge calls
    fl_dev_quantize_q4_file) must reach its own definitions, not those of a libfl_cuda.so another test of the same
    process loaded with RTLD_GLOBAL."""
    from fastllama_b200.cuda_abi import FlCuda

    mock = os.path.join(ROOT, "tests", "mock")
    path = str(tmp_path_factory.mktemp("mocklora") / "libfl_cuda.so")
    subprocess.run(["/usr/bin/gcc", "-O2", "-mavx2", "-mfma", "-mf16c", "-ffp-contract=off", "-fPIC", "-shared", "-w",
                    "-Wl,-Bsymbolic", "-I" + os.path.join(ROOT, "include"), "-o", path, os.path.join(mock, "mock_fl_cuda.c"),
                    os.path.join(mock, "mock_quantize_file_f16round.c"), os.path.join(mock, "mock_quantize_file_lora.c"),
                    os.path.join(ROOT, "oracle", "q4_oracle.c"), "-lm", "-lrt"],
                   check=True, capture_output=True, timeout=300)
    return FlCuda(path)


@pytest.fixture(scope="module")
def fl_gpu():
    from fastllama_b200.cuda_abi import FlCuda

    return FlCuda()


def toy_adapter(path, form, n_embd=256, ff=768, layers=(0, 1), targets=TARGETS, seed=31, r=8):
    write_adapter(str(path), form, n_embd, ff, layers, seed=seed, r=r, targets=targets)
    return str(path)


def check_merged(fl, tmp_path, in_path, adapter, wtype, merged_from, tag="ours", **kw):
    """quantize_model(in_path, lora=adapter) against quantize_ref on the reference-merged model merged_from (the f16 /
    f32 file in_path is, or stands for); returns the report."""
    ours = str(tmp_path / f"{tag}-{wtype}.bin")
    rep = quantize_model(in_path, ours, wtype, fl=fl, verbose=False, lora=adapter, **kw)
    same_file(ours, expected_q4(merged_from, adapter, wtype, tmp_path, tag=f"ref-{tag}"))
    assert rep["hist"] == file_hist(ours).tolist()
    return rep


def model_file(tmp_path, ftype, model=None, seed=30):
    """An f16 / f32 model file: the converter's file of a toy Meta model."""
    model = model if model is not None else meta_model(**TOY, seed=seed)
    outtype = "f16" if ftype == F16 else "f32"
    return write_converted(str(tmp_path / f"model-{outtype}.bin"), model, TOKENIZER, outtype)


def ftype_forms():
    """(ftype, form) pairs the reference merges: an f16 delta only into an f16 model."""
    return [(ft, form) for ft in (F16, F32) for form in FORMS if not (ft == F32 and form == "cached_f16")]


# ---------------------------------------------------------------------------------------------------------------- CPU
@need_ref
@pytest.mark.parametrize("wtype", [2, 3])
@pytest.mark.parametrize("targets", sorted(TARGET_SETS))
@pytest.mark.parametrize("ftype,form", ftype_forms())
def test_mock_file_with_adapter_is_the_reference_file(mock_fl, tmp_path, ftype, form, targets, wtype):
    src = model_file(tmp_path, ftype)
    adapter = toy_adapter(tmp_path / "lora.bin", form, targets=TARGET_SETS[targets])
    rep = check_merged(mock_fl, tmp_path, src, adapter, wtype, src)
    merged = {t["name"] for t in rep["tensors"] if t["lora"]}
    assert merged == {f"layers.{i}.{tg}.weight" for i in (0, 1) for tg in TARGET_SETS[targets]}
    # the adapter changes the file: without it the output is the reference tool's file of the plain model
    plain = str(tmp_path / "plain.bin")
    quantize_model(src, plain, wtype, fl=mock_fl, verbose=False)
    assert open(plain, "rb").read() != open(tmp_path / f"ours-{wtype}.bin", "rb").read()


@need_ref
@pytest.mark.parametrize("wtype", [2, 3])
@pytest.mark.parametrize("form", FORMS)
def test_mock_part_set_with_adapter(mock_fl, tmp_path, form, wtype):
    shape = dict(n_vocab=300, n_embd=256, n_mult=64, n_head=4, n_layer=2)
    base = write_synthetic_parts(str(tmp_path / "model-f16.bin"), ["ggjt", "ggmf"], F16, seed=32, **shape)
    joined = write_synthetic_joined(str(tmp_path / "joined.bin"), 2, F16, seed=32, **shape)
    adapter = toy_adapter(tmp_path / "lora.bin", form, ff=n_ff(256, 64))
    rep = check_merged(mock_fl, tmp_path, base, adapter, wtype, joined)
    assert rep["n_parts"] == 2 and sum(t["lora"] for t in rep["tensors"]) == 14


CKPT_CASES = [("pth2", np.float16, "f16", "cached_f16"), ("pth2", np.float32, "f16", "uncached_f32"),
              ("pth2", np.float16, "f32", "uncached_f32"), ("pth2", np.float32, "f32", "cached_f32"),
              ("hf-safetensors", np.float16, "f16", "uncached_f32"), ("hf-safetensors", np.float32, "f16", "cached_f16"),
              ("hf-safetensors", np.float16, "f32", "cached_f32"), ("hf-bin", np.float32, "f32", "uncached_f32")]


def check_checkpoint(fl, tmp_path, layout, dtype, outtype, form, wtype, model=None, adapter=None):
    model = model if model is not None else meta_model(**TOY, dtype=dtype, seed=33)
    path, vd = write_layout(tmp_path, layout, model, VOCAB_AT[layout])
    conv = write_converted(str(tmp_path / "conv.bin"), model, TOKENIZER, outtype)
    adapter = adapter or toy_adapter(tmp_path / "lora.bin", form)
    return check_merged(fl, tmp_path, path, adapter, wtype, conv, outtype=outtype, vocab_dir=vd)


@need_ref
@pytest.mark.parametrize("wtype", [2, 3])
@pytest.mark.parametrize("layout,dtype,outtype,form", CKPT_CASES, ids=[f"{c[0]}-{np.dtype(c[1]).name}-{c[2]}-{c[3]}" for c in CKPT_CASES])
def test_mock_checkpoint_with_adapter(mock_fl, tmp_path, layout, dtype, outtype, form, wtype):
    """Meta and Hugging Face checkpoints under outtype f16 and f32: the adapter is merged into the converter's file, q / k
    rows in the converter's order; an f16 checkpoint under outtype f32 merges in f32 (source type 3)."""
    check_checkpoint(mock_fl, tmp_path, layout, dtype, outtype, form, wtype)


def special_case(dtype, seed=34):
    """A model and a cached f32 adapter on all seven targets of both layers whose sums w + d land on f16 rounding ties
    (halfway to the next f16 value away from and towards zero) and, in blocks of f16 subnormal weights, in the f16
    subnormal range and across its edge; the other blocks get ordinary deltas."""
    rng = np.random.default_rng(seed)
    model = meta_model(**TOY, dtype=dtype, seed=seed)
    deltas = []
    for il in (0, 1):
        for tg in TARGETS:
            name = f"layers.{il}.{tg}.weight"
            w = model[name]
            w16 = w.astype(np.float16)
            blocks = w16.reshape(-1, 32)
            kind = rng.integers(0, 4, blocks.shape[0])
            sub = (rng.integers(-1023, 1024, blocks.shape) * 2.0 ** -24).astype(np.float16)        # subnormal f16 values
            blocks[kind == 2] = sub[kind == 2]
            if dtype == np.float16:
                model[name] = w16
            else:                                                                              # f32 values that round to w16
                model[name] = np.where((kind == 2)[:, None], blocks.astype(np.float32), w.reshape(-1, 32)).reshape(w.shape)
            wv = model[name].astype(np.float16).astype(np.float32).reshape(-1, 32)
            half_ulp = np.abs(np.spacing(wv.astype(np.float16)).astype(np.float32)) / 2
            sign = rng.choice([-1, 1], wv.shape).astype(np.float32) * np.sign(wv + (wv == 0))
            d = np.select([kind[:, None] == 0, kind[:, None] == 1, kind[:, None] == 2],
                          [sign * half_ulp, sign * half_ulp * 3,
                           (rng.integers(-2048, 2048, wv.shape) * 2.0 ** -26).astype(np.float32)],
                          (rng.standard_normal(wv.shape) * 0.002).astype(np.float32))
            deltas.append((name + ".lora", d.reshape(w.shape).astype(np.float32)))
    return model, deltas


@need_ref
@pytest.mark.parametrize("wtype", [2, 3])
@pytest.mark.parametrize("case", ["f16-file", "f32-checkpoint-f16"])
def test_mock_f16_rounding_ties_and_subnormal_sums(mock_fl, tmp_path, case, wtype):
    model, deltas = special_case(np.float16 if case == "f16-file" else np.float32)
    adapter = str(tmp_path / "lora.bin")
    write_lora(adapter, deltas, r=8, alpha=16, cached=True)
    if case == "f16-file":
        src = model_file(tmp_path, F16, model)
        check_merged(mock_fl, tmp_path, src, adapter, wtype, src)
    else:
        check_checkpoint(mock_fl, tmp_path, "pth1", None, "f16", None, wtype, model=model, adapter=adapter)


@need_ref
def test_merge_graphs_are_the_reference_attach(tmp_path):
    """The graphs tests/lora_merge.py restates are the reference's attach on an unquantised model: on the reference
    library, the f16 model with each adapter form attached and the reference-merged f16 file with no adapter decode
    greedily to the same tokens and logit bits."""
    from fastllama_b200.model import Model, QuietLogger
    from oracle.pyoracle import REF_PYFASTLLAMA_SO

    src = model_file(tmp_path, F16, meta_model(**TOY, seed=35, std=0.05))
    greedy = dict(temp=0.0, top_k=1, top_p=1.0, repeat_penalty=1.0)

    def decode(path, adapter=None):
        m = Model(path, num_threads=4, n_ctx=64, n_batch=4, logger=QuietLogger(), library_path=REF_PYFASTLLAMA_SO)
        if adapter:
            assert m.attach_lora(adapter)
        assert m.ingest("An adapter changes the weights.")
        toks = []
        assert m.generate(lambda s: toks.append(s), num_tokens=6, **greedy)
        out = (toks, m.get_logits_array().copy())
        m.close()
        return out

    plain_toks, plain_logits = decode(src)
    for form in FORMS:
        adapter = toy_adapter(tmp_path / f"lora-{form}.bin", form, seed=36, targets=TARGETS)
        merged = str(tmp_path / f"merged-{form}.bin")
        merge_reference(src, adapter, merged)
        att_toks, att_logits = decode(src, adapter)
        mer_toks, mer_logits = decode(merged)
        assert att_toks == mer_toks, form
        assert np.array_equal(att_logits.view(np.uint32), mer_logits.view(np.uint32)), form
        assert not np.array_equal(att_logits.view(np.uint32), plain_logits.view(np.uint32)), f"{form}: the adapter must matter"


# ------------------------------------------------------------------------------------------------------- rejections
def _reject_case(tmp_path, case):
    """(model path, adapter path, pattern the QuantizeError must match)."""
    src = model_file(tmp_path, F32 if case == "f16-delta-on-f32" else F16)
    adapter = str(tmp_path / "lora.bin")
    a = np.zeros((256, 8), np.float32)
    b = np.zeros((256, 8), np.float32)
    if case == "unknown-base":
        write_lora(adapter, [("layers.7.attention.wq.weight.lora", np.zeros((256, 256), np.float32))], 8, 16, True)
        return src, adapter, r"lora\.bin: tensor 'layers\.7\.attention\.wq\.weight\.lora': its base 'layers\.7\.attention\.wq\.weight' is not a tensor"
    if case == "1-d-base":
        write_lora(adapter, [("layers.0.ffn_norm.weight.lora", np.zeros((1, 256), np.float32))], 8, 16, True)
        return src, adapter, r"tensor 'layers\.0\.ffn_norm\.weight\.lora': its base 'layers\.0\.ffn_norm\.weight' is 1-D"
    if case == "cached-shape":
        write_adapter(adapter, "mismatch", 256, 768, (0,), seed=1)
        return src, adapter, r"tensor 'layers\.0\.feed_forward\.w1\.weight\.lora' has extents \(768, 256\), but .* \(incompatible tensor dimensions\)"
    if case == "uncached-shape":
        write_lora(adapter, [("layers.0.feed_forward.w2.weight.loraA", a), ("layers.0.feed_forward.w2.weight.loraB", b)], 8, 16, False)
        return src, adapter, r"tensors 'layers\.0\.feed_forward\.w2\.weight\.loraA' \(8, 256\) and .*\(incompatible tensor dimensions\)"
    if case == "rank":
        write_lora(adapter, [("layers.0.attention.wq.weight.loraA", a), ("layers.0.attention.wq.weight.loraB", b[:, :4])], 8, 16, False)
        return src, adapter, r"'layers\.0\.attention\.wq\.weight\.loraA' and '.*loraB' have ranks 8 and 4"
    if case == "unpaired":
        write_lora(adapter, [("layers.0.attention.wq.weight.loraA", a), ("layers.0.attention.wk.weight.loraB", b)], 8, 16, False)
        return src, adapter, r"tensor 'layers\.0\.attention\.wq\.weight\.loraA' has no 'layers\.0\.attention\.wq\.weight\.loraB'"
    if case == "uncached-f16":
        write_adapter(adapter, "uncached_f16", 256, 768, (0,), seed=1)
        return src, adapter, r"tensor 'layers\.0\.attention\.wq\.weight\.loraA' is f16 in an uncached adapter"
    if case == "f16-delta-on-f32":
        write_adapter(adapter, "cached_f16", 256, 768, (1,), seed=1)
        return src, adapter, r"tensor 'layers\.1\.attention\.wq\.weight\.lora' is f16 and 'layers\.1\.attention\.wq\.weight' is f32"
    if case == "not-lora-name":
        write_lora(adapter, [("layers.0.attention.wq.weight", np.zeros((256, 256), np.float32))], 8, 16, True)
        return src, adapter, r"tensor 'layers\.0\.attention\.wq\.weight' is not a LoRA tensor"
    if case == "not-an-adapter":
        return src, src, r"model-f16\.bin: bad magic 67676a74 \(not a ggla LoRA adapter\)"
    raise AssertionError(case)


REJECT_CASES = ["unknown-base", "1-d-base", "cached-shape", "uncached-shape", "rank", "unpaired", "uncached-f16", "f16-delta-on-f32",
                "not-lora-name", "not-an-adapter"]


@pytest.mark.parametrize("case", REJECT_CASES)
def test_rejects_adapter(tmp_path, case):
    src, adapter, match = _reject_case(tmp_path, case)
    out = tmp_path / "out.bin"
    with pytest.raises(QuantizeError, match=match):
        quantize_model(src, str(out), 2, lora=adapter)
    assert not out.exists()
    assert main([src, str(out), "2", "--lora", adapter]) == 1
    assert not out.exists()


@need_ref
def test_cli_lora(mock_fl, tmp_path, monkeypatch):
    import fastllama_b200.quantize as q

    src = model_file(tmp_path, F16)
    adapter = toy_adapter(tmp_path / "lora.bin", "uncached_f32", targets=SUBSET)
    monkeypatch.setattr(q, "FlCuda", lambda: mock_fl)
    out = str(tmp_path / "cli.bin")
    assert main([src, out, "3", f"--lora={adapter}"]) == 0
    same_file(out, expected_q4(src, adapter, 3, tmp_path))
    assert main([src, out, "3", "--lora"]) == 1                          # --lora without its argument: usage


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@need_ref
@pytest.mark.parametrize("wtype", [2, 3])
@pytest.mark.parametrize("ftype,form", ftype_forms())
def test_gpu_file_with_adapter_is_the_reference_file(fl_gpu, tmp_path, ftype, form, wtype):
    src = model_file(tmp_path, ftype)
    check_merged(fl_gpu, tmp_path, src, toy_adapter(tmp_path / "lora.bin", form), wtype, src)


@pytest.mark.gpu
@need_ref
@pytest.mark.parametrize("wtype", [2, 3])
def test_gpu_part_set_and_checkpoints_with_adapter(fl_gpu, tmp_path, wtype):
    shape = dict(n_vocab=300, n_embd=256, n_mult=64, n_head=4, n_layer=2)
    (tmp_path / "parts").mkdir()
    base = write_synthetic_parts(str(tmp_path / "parts" / "model-f16.bin"), ["ggjt", "ggjt"], F16, seed=32, **shape)
    joined = write_synthetic_joined(str(tmp_path / "parts" / "joined.bin"), 2, F16, seed=32, **shape)
    check_merged(fl_gpu, tmp_path / "parts", base, toy_adapter(tmp_path / "parts" / "lora.bin", "cached_f16", ff=n_ff(256, 64)),
                 wtype, joined)
    for i, (layout, dtype, outtype, form) in enumerate(CKPT_CASES):
        d = tmp_path / f"ckpt{i}"
        d.mkdir()
        check_checkpoint(fl_gpu, d, layout, dtype, outtype, form, wtype)


@pytest.mark.gpu
@need_ref
@pytest.mark.parametrize("wtype", [2, 3])
@pytest.mark.parametrize("case", ["f16-file", "f32-checkpoint-f16"])
def test_gpu_f16_rounding_ties_and_subnormal_sums(fl_gpu, mock_fl, tmp_path, case, wtype):
    """The device's fp16 merge (__float2half_rn) against the reference and the stand-in's F16C rounding."""
    model, deltas = special_case(np.float16 if case == "f16-file" else np.float32)
    adapter = str(tmp_path / "lora.bin")
    write_lora(adapter, deltas, r=8, alpha=16, cached=True)
    if case == "f16-file":
        src = model_file(tmp_path, F16, model)
        check_merged(fl_gpu, tmp_path, src, adapter, wtype, src)
        quantize_model(src, str(tmp_path / "mock.bin"), wtype, fl=mock_fl, verbose=False, lora=adapter)
    else:
        check_checkpoint(fl_gpu, tmp_path, "pth1", None, "f16", None, wtype, model=model, adapter=adapter)
        quantize_model(str(tmp_path / "model"), str(tmp_path / "mock.bin"), wtype, fl=mock_fl, verbose=False, lora=adapter)
    same_file(tmp_path / "mock.bin", tmp_path / f"ours-{wtype}.bin")


SEVEN_B_2L = dict(n_vocab=32000, n_embd=4096, n_mult=256, n_head=32, n_layer=2)


@pytest.fixture(scope="module")
def seven_b_f16(tmp_path_factory):
    d = tmp_path_factory.mktemp("q7blora")
    path = str(d / "7b-2l-f16.bin")
    write_synthetic_float(path, F16, seed=37, std=0.02, **SEVEN_B_2L)
    yield path
    os.unlink(path)


@pytest.mark.gpu
@need_ref
@pytest.mark.parametrize("wtype", [2, 3])
@pytest.mark.parametrize("form", ["uncached_f32_r16_wq_wv", "cached_f32_all7_layer1"])
def test_gpu_7b_shapes_with_adapter(fl_gpu, seven_b_f16, tmp_path, form, wtype):
    ff = n_ff(4096, 256)
    adapter = str(tmp_path / "lora.bin")
    if form.startswith("uncached"):
        write_adapter(adapter, "uncached_f32", 4096, ff, (0, 1), seed=38, r=16, alpha=32, targets=SUBSET)
    else:
        write_adapter(adapter, "cached_f32", 4096, ff, (1,), seed=39, r=16, alpha=32)
    rep = check_merged(fl_gpu, tmp_path, seven_b_f16, adapter, wtype, seven_b_f16)
    assert sum(t["lora"] for t in rep["tensors"]) == (4 if form.startswith("uncached") else 7)


def decode_steps(lib, path, n_gen=12):
    """Greedy tokens (each the argmax of the logits before it) and the logits after the prompt and after each step, from
    the library at lib.  Tokens are taken from the logits: the toy vocabulary's byte tokens are not all UTF-8 text."""
    from fastllama_b200.model import Model, QuietLogger
    from tests.test_gpu_e2e import PROMPT

    m = Model(path, num_threads=8, n_ctx=128, n_batch=8, logger=QuietLogger(), library_path=lib)
    assert m.ingest(PROMPT)
    logits = [m.get_logits_array().copy()]
    for _ in range(n_gen):
        assert m.generate(lambda s: None, num_tokens=1, temp=0.0, top_k=1, top_p=1.0, repeat_penalty=1.0)
        logits.append(m.get_logits_array().copy())
    m.close()
    return [int(np.argmax(x)) for x in logits[:-1]], np.stack(logits)


@pytest.mark.gpu
@need_ref
@pytest.mark.parametrize("wtype", [2, 3])
@pytest.mark.parametrize("form", FORMS)
def test_gpu_merged_file_decodes_like_the_reference(fl_gpu, tmp_path, form, wtype):
    """A q4 file quantised with the adapter merged in: the drop-in library on the H100 decodes it with the reference
    library's tokens and logit bits after the prompt and after each of 12 greedy steps."""
    from oracle.pyoracle import REF_PYFASTLLAMA_SO
    from tests.test_gpu_e2e import DROPIN

    assert os.path.exists(REF_PYFASTLLAMA_SO) and os.path.exists(DROPIN)
    src = model_file(tmp_path, F16, meta_model(**TOY, seed=40, std=0.01))
    adapter = toy_adapter(tmp_path / "lora.bin", form, seed=41)
    out = str(tmp_path / "q.bin")
    quantize_model(src, out, wtype, fl=fl_gpu, verbose=False, lora=adapter)
    ref_toks, ref_logits = decode_steps(REF_PYFASTLLAMA_SO, out)
    our_toks, our_logits = decode_steps(DROPIN, out)
    assert our_toks == ref_toks, (our_toks, ref_toks)
    nd = int((our_logits.view(np.uint32) != ref_logits.view(np.uint32)).sum())
    assert nd == 0, (nd, our_logits.size, float(np.abs(our_logits - ref_logits).max()))
