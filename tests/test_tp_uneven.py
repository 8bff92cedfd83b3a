"""CPU: tensor parallelism at world sizes that do not divide the model's shapes.

The partition rule (ggml_b200.cpp tp_split / tp_partition) restated in Python and checked on the LLaMA shapes and toy shapes at worlds 1
to 8.  Then, over gloo on the CPU stand-in of the device layer (tests/mock/mock_fl_cuda.c with fl_dev_tp_unshard from
tests/mock/mock_tp_unshard.c and fl_dev_tp_unshard_v from tests/mock/mock_tp_unshard_v.c), a toy model with 5 heads, n_ff 1792 (56
groups of 32 rows) and a 515-token vocabulary at worlds 2, 3 and 4: decode steps, multi-token evals at n_batch 4, 8 and 32, a state file, all-logits, embeddings and
perplexity must give the single-rank tokens and logit bits, through the sharded plans (decode mode 2, prompt mode 1) and with no device
copy of the model.  An odd vocabulary on one rank keeps the token kernel (its last LM-head row runs as a row pair of its own) and the
reference library's bits."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "fastllama_b200", "lib")
HAVE_MOCK = all(os.path.exists(os.path.join(LIB, n)) for n in ("libggml_b200.so", "pyfastllama.so"))
needs_mock = pytest.mark.skipif(not HAVE_MOCK, reason="needs the built host libraries and the drop-in pyfastllama.so")


# ---- the partition rule ----------------------------------------------------------------------------------------------------------------
def tp_split(total, unit, world, rank):
    """(first, rows) of rank `rank`: `total` rows in whole units of `unit`, dealt out in order as evenly as possible, the first
    (units % world) ranks taking one more; the rows after the last whole unit go with the last rank"""
    base, extra = divmod(total // unit, world)
    u0, nu = rank * base + min(rank, extra), base + (1 if rank < extra else 0)
    first, end = u0 * unit, total if rank == world - 1 else (u0 + nu) * unit
    return first, end - first


def tp_partition(n_embd, hd, n_ff, n_vocab, world):
    """every rank's (first, rows) of n_embd (whole heads), n_ff (32-row groups) and n_vocab (row pairs); None when a rank owns nothing"""
    p = {k: [tp_split(t, u, world, r) for r in range(world)] for k, t, u in (("e", n_embd, hd), ("f", n_ff, 32), ("v", n_vocab, 2))}
    return p if all(rows > 0 for s in p.values() for _, rows in s) else None


# name: (n_embd, n_head, n_ff, n_vocab)
SHAPES = {"7B": (4096, 32, 11008, 32000), "13B": (5120, 40, 13824, 32000), "30B": (6656, 52, 17920, 32000), "65B": (8192, 64, 22016, 32000),
          "7B-32001": (4096, 32, 11008, 32001), "toy": (256, 4, 768, 512), "toy-uneven": (640, 5, 1792, 515), "toy-2head": (128, 2, 384, 33)}


@pytest.mark.parametrize("name", sorted(SHAPES))
@pytest.mark.parametrize("world", range(1, 9))
def test_partition_covers_every_row_once(name, world):
    n_embd, n_head, n_ff, n_vocab = SHAPES[name]
    hd = n_embd // n_head
    p = tp_partition(n_embd, hd, n_ff, n_vocab, world)
    if p is None:
        assert world > n_head or world > n_ff // 32 or world > n_vocab // 2 + n_vocab % 2
        return
    for k, total, unit in (("e", n_embd, hd), ("f", n_ff, 32), ("v", n_vocab, 2)):
        rows = [i for first, n in p[k] for i in range(first, first + n)]
        assert rows == list(range(total)), k                                    # in order, each once
        sizes = [n for _, n in p[k]]
        whole = [n - (total % unit if r == world - 1 else 0) for r, n in enumerate(sizes)]
        assert max(whole) - min(whole) <= unit                                  # whole units: as even as they allow ...
        assert whole == sorted(whole, reverse=True)                             # ... the larger shares first
        for r, (first, n) in enumerate(p[k]):
            assert first % unit == 0 and whole[r] % unit == 0                   # a slice is whole units, and the last rank's
            assert n - whole[r] < unit                                          # also the rows after the last whole unit
    assert all(n % hd == 0 for _, n in p["e"])                                  # heads are never split


def _old_split_applied(name, world):
    _, n_head, n_ff, n_vocab = SHAPES[name]
    return n_head % world == 0 and n_ff % (32 * world) == 0 and n_vocab % (2 * world) == 0


@pytest.mark.parametrize("name,world", [(n, w) for n in sorted(SHAPES) for w in range(1, 9) if _old_split_applied(n, w)])
def test_partition_is_the_even_split_wherever_that_applied(name, world):
    """Where the decode plan's old conditions hold (n_head, n_ff / 32 and n_vocab / 2 divisible by world), the rule is n / world per rank,
    so shard keys, shard sizes and every existing test stay as they were."""
    n_embd, n_head, n_ff, n_vocab = SHAPES[name]
    p = tp_partition(n_embd, n_embd // n_head, n_ff, n_vocab, world)
    for k, total in (("e", n_embd), ("f", n_ff), ("v", n_vocab)):
        assert p[k] == [(r * (total // world), total // world) for r in range(world)]


def test_partition_declines_when_a_rank_would_own_nothing():
    assert tp_partition(256, 64, 768, 512, 5) is None                           # 4 heads on 5 ranks
    assert tp_partition(128, 64, 384, 33, 3) is None                            # 2 heads on 3 ranks
    assert tp_partition(256, 64, 64, 512, 3) is None                            # 2 n_ff groups on 3 ranks
    assert tp_partition(6656, 128, 17920, 32000, 8) is not None                 # 30B on 8: 7, 7, 7, 7, 6, 6, 6, 6 heads
    assert [n // 128 for _, n in tp_partition(6656, 128, 17920, 32000, 8)["e"]] == [7, 7, 7, 7, 6, 6, 6, 6]
    assert tp_partition(4096, 128, 11008, 32001, 1)["v"] == [(0, 32001)]
    assert tp_partition(4096, 128, 11008, 32001, 8)["v"][-1] == (28000, 4001)    # 2000 pairs each, and the single last row
    assert tp_partition(4096, 128, 11008, 32001, 3)["v"] == [(0, 10668), (10668, 10666), (21334, 10667)]


# ---- the library over gloo -------------------------------------------------------------------------------------------------------------
WORKER = r'''
import ctypes as C, os, sys, numpy as np
sys.path.insert(0, sys.argv[1])
from fastllama_b200.model import Model, QuietLogger
so, path, out, n_batch, scenario = sys.argv[2], sys.argv[3], sys.argv[4], int(sys.argv[5]), sys.argv[6]
rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
mock = os.path.exists(os.path.join(os.path.dirname(so), "libfl_cuda.so"))
if mock:
    import torch, torch.distributed as dist
    if world > 1:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    lib = C.CDLL(os.path.join(os.path.dirname(so), "libfl_cuda.so"), mode=C.RTLD_GLOBAL)
    CB = C.CFUNCTYPE(None, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t)
    def coll(kind, send, recv, n):
        if kind == 0:
            t = torch.from_numpy(np.ctypeslib.as_array((C.c_float * n).from_address(send))); dist.all_reduce(t)
        else:
            s = torch.from_numpy(np.ctypeslib.as_array((C.c_float * n).from_address(send)).copy())
            r = np.ctypeslib.as_array((C.c_float * (n * world)).from_address(recv))
            parts = [torch.empty(n) for _ in range(world)]
            dist.all_gather(parts, s)
            r[:] = torch.cat(parts).numpy()
    cb = CB(coll)
    lib.fl_mock_set_collective(cb, rank, world)
    g = C.CDLL(os.path.join(os.path.dirname(so), "libggml_b200.so"))
class Mem(C.Structure):
    _fields_ = [("weight_mirror_bytes", C.c_uint64), ("shard_bytes", C.c_uint64), ("mirror_bytes", C.c_uint64), ("kv_gathers", C.c_uint64)]
def mem():
    m = Mem(); g.ggml_b200_get_memory(C.byref(m)); return np.array([m.weight_mirror_bytes, m.shard_bytes, m.mirror_bytes, m.kv_gathers], dtype=np.uint64)
greedy = dict(temp=0.0, top_k=1, top_p=1.0, repeat_penalty=1.0)
toks, logits, pmodes, dmodes, mems = [], [], [], [], []
def step(kind, keep=True):
    # the modes of the step's last eval: a decode step (decode mode 2: the token program) or a multi-token eval (decode mode 0; prompt
    # mode 1: the tensor-parallel prompt plan).  The first generate() after an ingest or load_state evaluates several tokens.
    if keep:
        logits.append(m.get_logits_array())
    if mock:
        pmodes.append(g.ggml_b200_prompt_mode()); dmodes.append(g.ggml_b200_decode_mode())
        mems.append(mem())
def gen(n):
    for _ in range(n):
        assert m.generate(lambda s: toks.append(s), num_tokens=1, **greedy); step("d")
res = {}
if scenario == "greedy16":
    # one rank: an ingest, then 16 greedy steps, the logits after every one
    m = Model(path, num_threads=2, n_ctx=64, n_batch=n_batch, logger=QuietLogger(), library_path=so)
    assert m.ingest("An odd vocabulary."); step("p")
    gen(16)
    m.close()
else:
    P1 = "Tensor parallel prompt ingest at an uneven world size."
    P2 = " A second prompt attends to all of it."
    m = Model(path, num_threads=2, n_ctx=128, n_batch=n_batch, logger=QuietLogger(), library_path=so)
    assert m.ingest(P1); step("p")
    gen(4)
    assert m.ingest(P2); step("p")
    gen(4)
    assert m.save_state(out + f".rank{rank}.state")
    gen(3)
    first = list(toks[-3:])
    assert m.load_state(out + f".rank{rank}.state")
    gen(3)
    assert list(toks[-3:]) == first, (toks[-3:], first)
    m.close()
    if scenario == "full":
        m = Model(path, num_threads=2, n_ctx=128, n_batch=n_batch, should_get_all_logits=True, embedding_eval_enabled=True, logger=QuietLogger(),
                  library_path=so)
        assert m.ingest(P1); step("p", keep=False)
        res["all_logits"], res["emb"] = m.get_logits_array(), np.array(m.get_embeddings(), dtype=np.float32)
        res["ppl"] = np.float64(m.perplexity("The quick brown fox jumps over the lazy dog. " * 6)); step("p", keep=False)
        m.close()
np.savez(out + f".rank{rank}.npz", toks=np.array(toks), logits=np.stack(logits), pmodes=np.array(pmodes), dmodes=np.array(dmodes),
         mems=np.array(mems, dtype=np.uint64).reshape(-1, 4), **res)
'''

# 5 heads of 128; n_mult 256 gives n_ff 1792 (56 groups of 32 rows: uneven on 3 ranks); 515 tokens (a single last row)
UNEVEN = dict(n_vocab=515, n_embd=640, n_mult=256, n_head=5, n_layer=2)
# the same with an even vocabulary: equal logit slices on 2 ranks, so the decode steps run from captured graphs on the stand-in too
UNEVEN_HEADS = dict(UNEVEN, n_vocab=512)
# 4 heads: more ranks than heads
FOUR_HEADS = dict(n_vocab=512, n_embd=256, n_mult=256, n_head=4, n_layer=2)


@pytest.fixture(scope="module")
def mock():
    """The CPU stand-in of the device layer with both unshard entry points, built as one libfl_cuda.so in a temporary directory with the
    stand-in's flags, next to copies of the host libraries (their $ORIGIN runpath resolves libfl_cuda.so there)."""
    import shutil
    import tempfile

    d = tempfile.mkdtemp(prefix="fl_mock_tpu_")
    src = os.path.join(ROOT, "tests", "mock")
    subprocess.run(["/usr/bin/gcc", "-O2", "-mavx2", "-mfma", "-mf16c", "-ffp-contract=off", "-fPIC", "-shared", "-w",
                    "-I" + os.path.join(ROOT, "include"), "-o", os.path.join(d, "libfl_cuda.so"), os.path.join(src, "mock_fl_cuda.c"),
                    os.path.join(src, "mock_tp_unshard.c"), os.path.join(src, "mock_tp_unshard_v.c"),
                    os.path.join(ROOT, "oracle", "q4_oracle.c"), "-lm", "-lrt"],
                   check=True, capture_output=True, timeout=300)
    for n in ("libggml_b200.so", "pyfastllama.so"):
        shutil.copy(os.path.join(LIB, n), d)
    yield d
    shutil.rmtree(d, ignore_errors=True)


@pytest.fixture(scope="module")
def models(tmp_path_factory, mock):
    from fastllama_b200.ggjt import Q4_0, write_synthetic_numpy
    from oracle.pyoracle import Oracle

    orc = Oracle()
    d = tmp_path_factory.mktemp("tp_uneven")
    paths = {}
    for name, dims in (("uneven", UNEVEN), ("heads", UNEVEN_HEADS), ("four", FOUR_HEADS)):
        paths[name] = str(d / f"{name}.bin")
        write_synthetic_numpy(paths[name], Q4_0, seed=7, std=0.01, quantize=lambda w, t: orc.quantize_q4(w, t), **dims)
    script = d / "worker.py"
    script.write_text(WORKER)
    return d, paths, script, {}, mock


def launch(models, model, world, n_batch, scenario="full", graphs=False, so=None):
    """world rank processes over gloo; the results of each rank.  Unless `graphs`, multi-rank runs execute every decode step eagerly
    (FASTLLAMA_B200_NO_GRAPH): the stand-in's graph capture records only the operations of mock_fl_cuda.c, so the logits compaction of
    uneven vocabulary slices (fl_dev_tp_unshard_v, mock_tp_unshard_v.c) would not replay there.  On the GPU it is captured like any kernel."""
    d, paths, script, cache, mock = models
    key = (model, world, n_batch, scenario, graphs, so)
    if key in cache:
        return cache[key]
    tag = f"{model}_w{world}_b{n_batch}_{scenario}{'_g' if graphs else ''}{'_ref' if so else ''}"
    out = str(d / tag)
    procs = []
    for r in range(world):
        e = dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT="29671", OMP_NUM_THREADS="2",
                 FL_MOCK_SESSION=f"{os.getpid()}_{tag}")
        if world > 1 and not graphs:
            e["FASTLLAMA_B200_NO_GRAPH"] = "1"
        procs.append(subprocess.Popen([sys.executable, str(script), ROOT, so or os.path.join(mock, "pyfastllama.so"), paths[model], out, str(n_batch),
                                       scenario], env=e, stdout=subprocess.DEVNULL, stderr=subprocess.PIPE))
    errs = [p.communicate(timeout=600)[1] for p in procs]
    for p, err in zip(procs, errs):
        assert p.returncode == 0, err.decode()[-3000:]
    cache[key] = [np.load(out + f".rank{r}.npz") for r in range(world)]
    return cache[key]


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def shard_bytes(dims, world, rank):
    """(bytes, tail): what a rank uploads -- its rows of every matrix (tp_partition), the embedding table, the norms and, once it has
    decoded, `tail`: the last row of an odd LM-head slice twice more"""
    E, H, V, L = dims["n_embd"], dims["n_head"], dims["n_vocab"], dims["n_layer"]
    F = ((2 * (4 * E) // 3 + dims["n_mult"] - 1) // dims["n_mult"]) * dims["n_mult"]
    q4 = lambda k: k // 32 * 20                                                  # bytes of one q4_0 row of k elements
    p = tp_partition(E, E // H, F, V, world)
    nl, fl, vl = p["e"][rank][1], p["f"][rank][1], p["v"][rank][1]
    tail = 2 * q4(E) if vl % 2 else 0
    return L * (4 * nl * q4(E) + 2 * fl * q4(E) + nl * q4(F)) + vl * q4(E) + tail + V * q4(E) + (2 * L + 1) * E * 4, tail


def check_like_single(runs, single, dims, world, full=True):
    for r, res in enumerate(runs):
        assert list(res["toks"]) == list(single["toks"])
        assert len(res["logits"]) == len(single["logits"])
        for i, (a, b) in enumerate(zip(res["logits"], single["logits"])):
            assert same_bits(a, b), (r, i)
        assert len(res["dmodes"]) == len(single["dmodes"])
        for i, d in enumerate(single["dmodes"]):
            if d == 2:
                assert res["dmodes"][i] == 2, (r, i, res["dmodes"])             # every decode step: the token program
            else:
                assert res["dmodes"][i] == 0 and res["pmodes"][i] == 1, (r, i, res["pmodes"])   # every multi-token eval: the prompt plan
        want, tail = shard_bytes(dims, world, r)
        for m in res["mems"]:
            assert int(m[0]) == 0                                               # no device copy of any weight
            assert int(m[1]) in (want, want - tail)                             # exactly this rank's rows, the table and the norms
        assert int(res["mems"][int(np.nonzero(single["dmodes"] == 2)[0][-1])][1]) == want       # after the last decode step
        if full:
            assert same_bits(res["all_logits"], single["all_logits"]) and res["all_logits"].size % dims["n_vocab"] == 0
            assert res["all_logits"].size > dims["n_vocab"]
            assert same_bits(res["emb"], single["emb"]) and res["emb"].size == dims["n_embd"]
            assert float(res["ppl"]) == float(single["ppl"]) and float(res["ppl"]) > 1.0


@needs_mock
@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("n_batch", [4, 8, 32])
def test_uneven_world_matches_single_rank(models, n_batch, world):
    """Ingest, decode, ingest, decode, save_state, decode, load_state, decode; then every column's logits, the embeddings and the
    perplexity: the single-rank tokens and logit bits at every step, through the sharded plans, with no weight mirrored on any rank."""
    single = launch(models, "uneven", 1, n_batch)[0]
    assert (single["dmodes"] == 2).sum() >= 12                                  # one rank with 515 rows: still the token program
    check_like_single(launch(models, "uneven", world, n_batch), single, UNEVEN, world)


@needs_mock
def test_uneven_heads_with_captured_graphs(models):
    """5 heads on 2 ranks (3 and 2) with equal vocabulary slices: the decode steps replay captured graphs on the stand-in as well."""
    single = launch(models, "heads", 1, 8, scenario="state")[0]
    check_like_single(launch(models, "heads", 2, 8, scenario="state", graphs=True), single, UNEVEN_HEADS, 2, full=False)


@needs_mock
@pytest.mark.parametrize("world", [5, 6])
def test_more_ranks_than_heads_stays_replicated(models, world):
    """4 heads on 5 or 6 ranks: a rank would own no head, so both plans decline; every rank runs the replicated executor and still
    computes the single-rank bits."""
    single = launch(models, "four", 1, 8, scenario="state")[0]
    for res in launch(models, "four", world, 8, scenario="state"):
        assert list(res["toks"]) == list(single["toks"])
        for a, b in zip(res["logits"], single["logits"]):
            assert same_bits(a, b)
        assert set(res["pmodes"].tolist()) == {0} and set(res["dmodes"].tolist()) == {0}


@needs_mock
def test_odd_vocabulary_on_one_rank_has_the_reference_bits(models):
    """515 LM-head rows on one rank: the token program (decode mode 2), and over 16 greedy steps the reference library's tokens and
    logit bits."""
    from oracle.pyoracle import REF_PYFASTLLAMA_SO

    if not os.path.exists(REF_PYFASTLLAMA_SO):
        pytest.skip("oracle/_ref not built")
    ours = launch(models, "uneven", 1, 8, scenario="greedy16")[0]
    ref = launch(models, "uneven", 1, 8, scenario="greedy16", so=REF_PYFASTLLAMA_SO)[0]
    assert list(ours["dmodes"][2:]) == [2] * 15                                  # after the ingest and generate()'s first eval
    assert len(ours["toks"]) == 16 and list(ours["toks"]) == list(ref["toks"])
    assert len(ours["logits"]) == len(ref["logits"]) == 17
    for a, b in zip(ours["logits"], ref["logits"]):
        assert same_bits(a, b) and a.size == UNEVEN["n_vocab"]


@needs_mock
def test_unshard_v_stand_in_against_numpy(mock):
    lib = C.CDLL(os.path.join(mock, "libfl_cuda.so"))
    fn = lib.fl_dev_tp_unshard_v
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_void_p, C.c_void_p]
    rng = np.random.default_rng(11)
    for counts, N in [([3, 2], 5), ([7, 7, 6], 3), ([258, 257], 1), ([4, 4, 4, 4, 4, 3, 3, 3], 2), ([1], 4)]:
        world, stride, n = len(counts), max(counts), sum(counts)
        first = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int32)
        g = rng.standard_normal((world, N * stride)).astype(np.float32)
        want = np.concatenate([g[r, :N * c].reshape(N, c) for r, c in enumerate(counts)], axis=1)
        res = rng.standard_normal((N, n)).astype(np.float32)
        for residual in (None, res):
            dst = np.full((N, n), np.nan, dtype=np.float32)
            f, c = (C.c_int * world)(*first.tolist()), (C.c_int * world)(*counts)
            assert fn(g.ctypes.data, world, N, stride, f, c, None if residual is None else residual.ctypes.data, dst.ctypes.data) == 0
            ref = want if residual is None else (want + residual).astype(np.float32)
            assert np.array_equal(dst.view(np.uint32), ref.view(np.uint32))
