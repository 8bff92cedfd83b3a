"""CPU: the tiled reference-order GEMM (k_mul_mat_q_ref_tiled, fastllama_b200/csrc/fl_exact_kernels.cu) restated in Python, and what
its compiled sm_90a code contains.

The tile constants are read from the kernel source, so a change there is checked here:
  * every (row, column) of any M x N output is owned by exactly one (CTA, warp, lane group, k, c), and the lanes that store are
    exactly the owners inside the operands;
  * each CTA's chunks cover blocks 0 .. nb-1 in order, each block once, the last chunk possibly short;
  * the shared-memory loads of one warp instruction (weight words, weight scales, activation entries and their (d, s) pairs) are
    free of bank conflicts, with the byte offsets the kernel computes."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "fastllama_b200", "csrc", "fl_exact_kernels.cu")
LIB = os.path.join(ROOT, "fastllama_b200", "lib")
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"

YX_BYTES = 80            # sizeof(fl_yx): q[4][4] words, d, s, 2 pad words
Q4_0, Q4_1 = 2, 3


def _consts():
    text = open(SRC).read()
    c = {}
    for name in ("QT_WR", "QT_WC", "QT_R", "QT_C", "QT_STAGES"):
        c[name] = int(re.search(rf"#define {name} (\d+)", text).group(1))
    m = re.search(r"KC = \(TYPE == FL_TYPE_Q4_0\) \? (\d+) : (\d+);", text)
    c["KC"] = {Q4_0: int(m.group(1)), Q4_1: int(m.group(2))}
    c["BM"] = c["QT_WR"] * 8 * c["QT_R"]
    c["BN"] = c["QT_WC"] * c["QT_C"]
    return c


C = _consts()
BB = {Q4_0: 20, Q4_1: 24}


def _owners(M, N):
    """(row, col) -> list of owners, over the kernel's grid and thread mapping; and the set of (row, col) that get stored"""
    BM, BN, R, Cc, WR = C["BM"], C["BN"], C["QT_R"], C["QT_C"], C["QT_WR"]
    ntn, ntm = -(-N // BN), -(-M // BM)
    own, stored = {}, set()
    for bid in range(ntm * ntn):
        tn, tm = bid % ntn, bid // ntn
        m0, n0 = tm * BM, tn * BN
        for warp in range(C["QT_WR"] * C["QT_WC"]):
            wr, wc = warp % WR, warp // WR
            active = m0 + wr * 8 * R < M and n0 + wc * Cc < N
            for lane in range(32):
                g, jj = lane >> 2, lane & 3
                rt, ct = wr * 8 * R + g, wc * Cc
                for k in range(R):
                    for c in range(Cc):
                        row, col = m0 + rt + 8 * k, n0 + ct + c
                        if jj == 0:
                            own.setdefault((row, col), []).append((bid, warp, lane, k, c))
                        if active and jj == 0 and row < M and col < N:
                            assert (row, col) not in stored
                            stored.add((row, col))
    return own, stored


@pytest.mark.parametrize("M,N", [(1, 1), (7, 9), (63, 31), (64, 32), (65, 33), (130, 65), (515, 8), (100, 129)])
def test_every_output_is_owned_and_stored_once(M, N):
    own, stored = _owners(M, N)
    for r in range(M):
        for n in range(N):
            assert len(own[(r, n)]) == 1, (r, n, own[(r, n)])
    assert stored == {(r, n) for r in range(M) for n in range(N)}


@pytest.mark.parametrize("t", [Q4_0, Q4_1])
@pytest.mark.parametrize("nb", [1, 2, 8, 10, 12, 13, 20, 36, 44, 128, 129, 344, 432])
def test_chunks_visit_every_block_once_in_order(t, nb):
    KC, S = C["KC"][t], C["QT_STAGES"]
    nchunks = -(-nb // KC)
    order, slots = [], []
    for ch in range(nchunks):
        s, parity = ch % S, (ch // S) & 1
        slots.append((s, parity))
        kn = min(KC, nb - ch * KC)
        assert 1 <= kn <= KC
        order += [ch * KC + i for i in range(kn)]          # tile word offset ch * RW + i * WPB is block ch * KC + i of the row
    assert order == list(range(nb))
    # producer and consumers agree on (slot, parity); a slot's phases alternate
    for ch, (s, p) in enumerate(slots):
        if ch >= S:
            assert slots[ch - S] == (s, p ^ 1)


def _banks_conflict_free(addrs, width):
    """addrs: byte address per lane of one warp load of `width` bytes.  Distinct addresses must map to distinct banks
    (a repeated address is a broadcast); for 16-byte loads the distinct addresses are 16-byte units over 4 banks each."""
    uniq = sorted(set(addrs))
    banks = []
    for a in uniq:
        assert a % width == 0
        banks += [((a // 4) + i) % 32 for i in range(width // 4)]
    return len(banks) == len(set(banks)) and len(banks) <= 32


@pytest.mark.parametrize("t", [Q4_0, Q4_1])
def test_shared_memory_loads_are_conflict_free(t):
    KC, R, Cc, WR = C["KC"][t], C["QT_R"], C["QT_C"], C["QT_WR"]
    WPB = BB[t] // 4
    RW = KC * WPB
    QW = WPB - 4
    A_BYTES = C["BM"] * RW * 4
    assert (KC * BB[t]) % 16 == 0 and RW <= 256 and KC * YX_BYTES // 4 <= 256      # TMA box
    assert RW % 8 == 4
    for warp in range(WR * C["QT_WC"]):
        wr, wc = warp % WR, warp // WR
        for i in range(KC):
            for k in range(R):
                word, scale, mins = [], [], []
                for lane in range(32):
                    g, jj = lane >> 2, lane & 3
                    row = wr * 8 * R + g + 8 * k
                    blk = (row * RW + i * WPB) * 4
                    word.append(blk + (QW + jj) * 4)
                    scale.append(blk)
                    mins.append(blk + 4)
                assert _banks_conflict_free(word, 4), (t, warp, i, k)
                assert len(set(word)) == 32
                assert _banks_conflict_free(scale, 4), (t, warp, i, k)
                if t == Q4_1:
                    assert _banks_conflict_free(mins, 4), (t, warp, i, k)
            for c in range(Cc):
                ent, ds = [], []
                for lane in range(32):
                    jj = lane & 3
                    yb = A_BYTES + ((wc * Cc + c) * KC + i) * YX_BYTES
                    ent.append(yb + 16 * jj)
                    ds.append(yb + 64)
                assert _banks_conflict_free(ent, 16), (t, warp, i, c)
                assert _banks_conflict_free(ds, 8), (t, warp, i, c)


def _sass(obj):
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


def _count(text, mnemonic):
    return len(re.findall(r"\b" + re.escape(mnemonic), text))


def test_tiled_kernel_sass():
    f = _sass("fl_exact_kernels.o")
    ks = {n: v for n, v in f.items() if "k_mul_mat_q_ref_tiled" in n}
    assert len(ks) == 2, sorted(f)                                          # q4_0 and q4_1
    R, Cc = C["QT_R"], C["QT_C"]
    for n, v in ks.items():
        assert _count(v, "IDP.4A") >= 2 * R * Cc, n                         # two four-product sums per (row, column) and block
        assert _count(v, "PRMT") >= 2 * R, n                                # nibbles -> elements, once per row and block
        assert _count(v, "PRMT") < 2 * R * Cc, n                            # ... not once per column
        assert _count(v, "UTMALDG") >= 2, n                                 # weights and activations by tensor-map copies
        assert _count(v, "SYNCS") >= 2, n                                   # mbarrier ring
        assert _count(v, "LDL") + _count(v, "STL") == 0, n                  # no spills
        assert _count(v, "IMMA") + _count(v, "IGMMA") + _count(v, "HMMA") == 0, n
