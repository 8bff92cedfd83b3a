"""CPU: the piece of bench.py that decides what the JSON line claims about parity, and the --dump-outputs writer, on synthetic
inputs (no GPU, no reference run)."""
import numpy as np

import bench


def _logits(n, seed):
    return np.random.default_rng(seed).standard_normal((n, 64)).astype(np.float32)


def test_parity_identical_runs_report_bit_identity():
    ref = _logits(5, 0)
    toks = ["a", "b", "c", "d", "e"]
    par = bench.compare_parity(toks, ref, list(toks), ref.copy())
    assert par["greedy_ids_equal"] and par["first_divergence"] is None and par["tokens_compared"] == 5
    assert par["logits_bit_identical"] and par["logits_maxabs_over_range"] == 0.0 and par["logits_steps_compared"] == 5
    assert "reference's bits" in par["note"]


def test_parity_one_ulp_is_not_bit_identity():
    ref = _logits(4, 1)
    ours = ref.copy()
    ours[2, 7] = np.nextafter(ours[2, 7], np.float32(np.inf))
    par = bench.compare_parity(list("abcd"), ref, list("abcd"), ours)
    assert par["greedy_ids_equal"] and not par["logits_bit_identical"] and 0.0 < par["logits_maxabs_over_range"] < 1e-6


def test_parity_divergence_is_reported_with_the_reference_gap():
    ref = _logits(6, 2)
    ours = ref + np.float32(1e-3)
    par = bench.compare_parity(list("abcdef"), ref, list("abXdef"), ours)
    assert not par["greedy_ids_equal"] and par["first_divergence"] == 2
    assert par["logits_steps_compared"] == 3                     # steps 0 .. 2: the last one both arms evaluated on the same tokens
    assert "reference_top1_top2_gap_at_divergence" in par and not par["logits_bit_identical"]


def test_dump_outputs_writes_float_arrays(tmp_path):
    logits = _logits(1, 3)[0]
    bench.dump_outputs(str(tmp_path / "out"), {"logits": logits})
    got = np.load(tmp_path / "out" / "logits.npy")
    assert got.dtype == np.float32 and np.array_equal(got, logits)
