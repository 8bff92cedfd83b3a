"""Quantising with a LoRA adapter merged in (quantize_model(..., lora=)): wall clock at LLaMA-7B matrix shapes, and a
CPU-only quality report.

  python tools/time_quantize_lora.py --layers 2 [--repeats 3] [--out results.json]      (H100)
  python tools/time_quantize_lora.py --quality-only [--out results.json]                (CPU)

Timing: an f16 model file with 7B shapes over --layers layers, quantised to q4_0 in three cases: no adapter, an
uncached r = 16 adapter on wq / wv of every layer, and a cached f32 adapter on all seven targets of every layer.
Each case runs once to warm up and --repeats times timed (median reported); every output is compared byte for byte
with the reference's file (tests/lora_merge.py: the reference's attach graphs, then its quantize tool).  The card's
name and power limit are read in the same run.

Quality (reference library only, on the CPU: the merged q4 file written by quantize_model equals the reference's
file, so the reference library can stand in for it): on a small f16 model, the logits of the f16 model with the
adapter attached are the ground truth; against them the report gives, after a prompt and over greedy steps, the RMS
and max logit differences and the greedy agreement of (a) the q4 file with the adapter merged before quantisation and
(b) the plain q4 file with the adapter attached at load (the attach-on-q4 path).  Nothing is asserted.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from fastllama_b200.ggjt import F16, n_ff, write_synthetic_float  # noqa: E402
from tests.lora_files import TARGETS, write_adapter  # noqa: E402
from tests.lora_merge import expected_q4  # noqa: E402
from tests.test_quantize_model import QUANTIZE_REF, run_tool  # noqa: E402

SEVEN_B = dict(n_vocab=32000, n_embd=4096, n_mult=256, n_head=32)


def card():
    p = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return p.stdout.strip().splitlines()[0] if p.returncode == 0 and p.stdout.strip() else "unknown"


def timing(layers, repeats, tmp):
    import pathlib

    from fastllama_b200.cuda_abi import FlCuda
    from fastllama_b200.quantize import quantize_model

    tmp = pathlib.Path(tmp)
    fl = FlCuda()
    src = str(tmp / "7b-f16.bin")
    write_synthetic_float(src, F16, seed=50, std=0.02, n_layer=layers, **SEVEN_B)
    ff = n_ff(4096, 256)
    adapters = {"none": None, "uncached_r16_wq_wv": str(tmp / "uncached.bin"), "cached_f32_all": str(tmp / "cached.bin")}
    write_adapter(adapters["uncached_r16_wq_wv"], "uncached_f32", 4096, ff, range(layers), seed=51, r=16, alpha=32,
                  targets=("attention.wq", "attention.wv"))
    write_adapter(adapters["cached_f32_all"], "cached_f32", 4096, ff, range(layers), seed=52, r=16, alpha=32, targets=TARGETS)
    out, res = str(tmp / "out.bin"), {}
    for case, adapter in adapters.items():
        want = expected_q4(src, adapter, 2, tmp, tag=case) if adapter else run_tool(QUANTIZE_REF, src, str(tmp / "plain.bin"), 2)
        times = []
        for i in range(repeats + 1):
            t0 = time.perf_counter()
            quantize_model(src, out, 2, fl=fl, verbose=False, lora=adapter)
            dt = time.perf_counter() - t0
            if i:
                times.append(dt)
        same = open(out, "rb").read() == open(want, "rb").read()
        res[case] = {"median_s": float(np.median(times)), "runs_s": times, "identical_to_reference": same}
        print(f"{case:>20s}: median {np.median(times):.3f} s over {repeats} runs, identical to the reference's file: {same}", flush=True)
        os.unlink(want)
    return {"model_bytes": os.path.getsize(src), "layers": layers, "cases": res}


def quality(tmp):
    """Reference library only, on the CPU."""
    import pathlib

    from fastllama_b200.model import Model, QuietLogger
    from oracle.pyoracle import REF_PYFASTLLAMA_SO
    from tests.checkpoint_files import TOKENIZER, meta_model, write_converted

    tmp = pathlib.Path(tmp)
    n_embd, n_layer = 512, 4
    src = write_converted(str(tmp / "small-f16.bin"), meta_model(n_vocab=300, n_embd=n_embd, n_layer=n_layer, seed=60, std=0.05),
                          TOKENIZER, "f16")
    ff = ((2 * (4 * n_embd) // 3 + 255) // 256) * 256
    greedy = dict(temp=0.0, top_k=1, top_p=1.0, repeat_penalty=1.0)
    prompt = "An adapter changes the weights of every layer it names."
    n_gen = 16

    def run(path, adapter=None):
        m = Model(path, num_threads=8, n_ctx=128, n_batch=8, logger=QuietLogger(), library_path=REF_PYFASTLLAMA_SO)
        if adapter:
            assert m.attach_lora(adapter)
        assert m.ingest(prompt)
        logits = [m.get_logits_array().copy()]
        toks = []
        for _ in range(n_gen):
            assert m.generate(lambda s: None, num_tokens=1, **greedy)
            logits.append(m.get_logits_array().copy())
            toks.append(int(np.argmax(logits[-2])))
        m.close()
        return toks, np.stack(logits)

    def compare(truth, other):
        d = (other[1] - truth[1]).astype(np.float64)
        agree = next((i for i, (a, b) in enumerate(zip(truth[0], other[0])) if a != b), len(truth[0]))
        return {"rms_prompt": float(np.sqrt((d[0] ** 2).mean())), "max_prompt": float(np.abs(d[0]).max()),
                "rms_all_steps": float(np.sqrt((d ** 2).mean())), "max_all_steps": float(np.abs(d).max()),
                "greedy_tokens_equal": int(sum(a == b for a, b in zip(truth[0], other[0]))), "greedy_prefix_agreement": agree,
                "greedy_steps": len(truth[0])}

    out = {"model": f"f16, n_embd {n_embd}, n_layer {n_layer}, n_vocab 300", "prompt": prompt}
    for form in ("cached_f32", "uncached_f32"):
        adapter = str(tmp / f"{form}.bin")
        write_adapter(adapter, form, n_embd, ff, range(n_layer), seed=61, r=16, alpha=32, std=0.05)
        truth = run(src, adapter)
        res = {}
        for wtype, name in ((2, "q4_0"), (3, "q4_1")):
            merged = expected_q4(src, adapter, wtype, tmp, tag=f"{form}-{name}")          # = quantize_model(src, lora=adapter)
            plain = run_tool(QUANTIZE_REF, src, str(tmp / f"plain-{name}.bin"), wtype)
            res[name] = {"merged_before_q4": compare(truth, run(merged)), "attached_to_q4": compare(truth, run(plain, adapter)),
                         "no_adapter_q4": compare(truth, run(plain))}
        out[form] = res
        print(json.dumps({form: res}, indent=1), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--quality-only", action="store_true")
    ap.add_argument("--no-quality", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    res = {}
    with tempfile.TemporaryDirectory() as tmp:
        if not a.quality_only:
            res["card"] = card()
            print(f"card (name, power limit): {res['card']}", flush=True)
            res["timing"] = timing(a.layers, a.repeats, tmp)
        if not a.no_quality:
            res["quality"] = quality(tmp)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
