"""CPU: what the compiled sm_90a code actually contains (cuobjdump of the in-tree objects).  The decode kernels must move
weights with the bulk-copy engine (UBLKCP) and do the block dots with IDP.4A; the prompt-ingest kernel must use the integer
tensor-core MMA; the persistent token kernel must stay (almost) spill-free, because local memory behind a grid barrier is an
L2 round trip (L1 is invalidated by every gpu-scope acquire)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "fastllama_b200", "lib")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


def sass(obj):
    path = os.path.join(LIB, obj)
    if not os.path.exists(path) or not os.path.exists(CUOBJDUMP):
        pytest.skip(f"{obj} or cuobjdump missing")
    out = subprocess.run([CUOBJDUMP, "-sass", path], capture_output=True, text=True, timeout=300).stdout
    funcs, cur = {}, None
    for ln in out.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur:
            funcs[cur].append(ln)
    assert "sm_90a" in out
    return {k: "\n".join(v) for k, v in funcs.items()}


def count(text, mnemonic):
    return len(re.findall(r"\b" + re.escape(mnemonic), text))


def test_token_kernel_uses_bulk_copies_and_dp4a_and_barely_spills():
    f = sass("fl_token_kernel.o")
    k = next(v for n, v in f.items() if "k_decode_token" in n)
    assert count(k, "UBLKCP") >= 1                   # weights: global -> shared through the TMA unit (one row piece per producer lane)
    assert count(k, "IDP.4A") >= 16                  # the four-product sums of the reference's eight accumulators (q4_0 and q4_1 loops, unrolled)
    assert count(k, "PRMT") >= 16                    # nibbles -> elements 4l .. 4l+3
    assert count(k, "SYNCS") >= 4                    # mbarrier ring
    assert count(k, "USETMAXREG") == 2, "producer / consumer register re-allocation (setmaxnreg) is missing"
    # the 64-register producer warps (setmaxnreg) may spill a word or two per tile; the consumer code must not
    assert count(k, "LDL") + count(k, "STL") <= 8, "the token kernel spills"


def test_fused_and_ring_matvecs_use_bulk_copies():
    f = sass("fl_decode_kernels.o")
    assert any("k_mv_fused" in n and count(v, "UBLKCP") >= 1 and count(v, "IDP.4A") >= 8 for n, v in f.items())
    g = sass("fl_quant_kernels.o")
    assert any("k_matvec_q4_ring" in n and count(v, "UBLKCP") >= 1 for n, v in g.items())


def test_prompt_ingest_kernel_uses_integer_tensor_core_mma():
    f = sass("fl_mma_kernel.o")
    assert all(count(v, "IMMA") >= 8 for n, v in f.items() if "k_mul_mat_q_mma" in n)
    assert sum(1 for n in f if "k_mul_mat_q_mma" in n) == 2      # q4_0 and q4_1


def test_prompt_ingest_gemm_is_a_wgmma_kernel():
    """The n_batch > 1 GEMM (fl_umma_kernel.cu): wgmma.mma_async with 8-bit integer operands (SASS IGMMA) into register
    accumulators, weights by a tensor-map TMA copy (UTMALDG), activations by bulk copies (UBLKCP), no local-memory spills."""
    f = sass("fl_umma_kernel.o")
    ks = {n: v for n, v in f.items() if "k_mul_mat_q_umma" in n}
    assert len(ks) == 4                                   # {q4_0, q4_1} x {32, 64} column tiles
    for n, v in ks.items():
        assert count(v, "IGMMA") >= 2, n
        assert count(v, "WARPGROUP.DEPBAR") >= 1, n
        assert count(v, "UTMALDG") >= 1, n
        assert count(v, "UBLKCP") >= 2, n
        assert count(v, "LDL") + count(v, "STL") == 0, n
        assert count(v, "HMMA") == 0 and count(v, "IMMA.") == 0, n      # no legacy mma.sync in this kernel
