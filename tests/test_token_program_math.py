"""CPU: the closed-form bookkeeping of the persistent token kernel (fastllama_b200/csrc/fl_token_kernel.cu), restated in Python and
checked exhaustively for the shapes the kernel meets -- 7B / 13B / 30B / 65B matrices, whole and as the row shards of 2 / 4 / 8
tensor-parallel ranks:
  * tk_make_slice_u + tk_tile_of: every unit (row pair) of every segment belongs to exactly one task of exactly one CTA, tasks never
    straddle segments, and the 32-bit magic-number divisions are exact;
  * tk_stream_of + the producer / consumer enumerations: the producer of a tile group issues positions 0, 1, 2, ... of the group's
    stream, the four consumer warps of the group partition them, each in increasing order; slot reuse cannot deadlock for any ring
    depth the host may choose (a slot is refilled only after its tile was consumed).
The GPU tests prove the same for the shapes they run (bit-identical logits need every row exactly once); this covers the shapes they
do not (65B, 8-rank shards) without a GPU."""
import random

import pytest

GRID = 132                  # one CTA per SM of an H100 SXM


def magic(d):
    k = 0
    while (2 << k) <= d:
        k += 1
    return (0 if d & (d - 1) == 0 else ((1 << (32 + k)) + d - 1) // d), k


def div(n, m, sh):
    assert 0 <= n < 2 ** 32
    return ((n * m) >> 32 if m else n) >> sh


def seg_span(u0, u1, base, m):
    lo, hi = max(u0, base), min(u1, base + m)
    return lo - base, max(0, hi - lo)


def make_slice(m, cta, lgG=2):
    gm, gs = magic(GRID)
    U = sum(m)
    u0, u1 = div(U * cta, gm, gs), div(U * (cta + 1), gm, gs)
    assert u0 == U * cta // GRID and u1 == U * (cta + 1) // GRID          # the magic division is exact
    f, n = zip(*(seg_span(u0, u1, sum(m[:i]), m[i]) for i in range(3)))
    rnd = (1 << lgG) - 1
    t0 = (n[0] + rnd) >> lgG
    t1 = t0 + ((n[1] + rnd) >> lgG)
    return f, n, t0, t1, t1 + ((n[2] + rnd) >> lgG)


def tile_of(sl, t, G=4):
    f, n, t0, t1, _ = sl
    seg = 0 if t < t0 else 1 if t < t1 else 2
    j = t - (0, t0, t1)[seg]
    return seg, f[seg] + j * G, min(G, n[seg] - j * G)


def model_phases(n_embd, n_ff, n_vocab, world):
    nl, fl, vl = n_embd // world, n_ff // world, n_vocab // world
    return [(nl // 2,) * 3, (nl // 2, 0, 0), (fl, 0, 0), (nl // 2, 0, 0), (vl // 2, 0, 0)]      # qkv pairs, wo, w1|w3 (swiglu units), w2, head


@pytest.mark.parametrize("dims", [(4096, 11008, 32000), (5120, 13824, 32000), (6656, 17920, 32000), (8192, 22016, 32000), (256, 768, 512)])
@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_every_unit_belongs_to_exactly_one_task(dims, world):
    n_embd, n_ff, n_vocab = dims
    if n_ff % (32 * world) or (n_embd // world) % 32 or n_vocab % (2 * world):
        pytest.skip("not a shardable shape")
    for m in model_phases(n_embd, n_ff, n_vocab, world):
        seen = [[0] * m[s] for s in range(3)]
        for cta in range(GRID):
            sl = make_slice(m, cta)
            for t in range(sl[4]):
                seg, u0, nu = tile_of(sl, t)
                assert 1 <= nu <= 4 and 0 <= u0 and u0 + nu <= m[seg]
                for u in range(u0, u0 + nu):
                    seen[seg][u] += 1
        assert all(c == 1 for s in seen for c in s), m


def stream_of(g, T0, ntasks):
    first = ((g - (T0 & 3)) + 4) & 3
    return first, ((ntasks - first + 3) >> 2 if first < ntasks else 0)


def test_streams_of_a_group_are_consistent_and_never_deadlock():
    rnd = random.Random(7)
    for _ in range(200):
        phases = [(rnd.choice([0, 1, 2, 3, 4, 5, 7, 11, 19, 27, 40]), rnd.choice([1, 2, 3, 6, 11])) for _ in range(rnd.randint(1, 12))]
        for g in range(4):
            prod, cons, T0, cg = [], [[] for _ in range(4)], 0, 0
            for ntasks, C in phases:
                first, n_g = stream_of(g, T0, ntasks)
                for k0 in range(0, n_g, 4):
                    n_r = min(4, n_g - k0)
                    prod += [cg + k0 * C + c * n_r + wl for c in range(C) for wl in range(n_r)]
                for wl in range(4):
                    for k in range(wl, n_g, 4):
                        k0 = k - wl
                        cons[wl] += [cg + k0 * C + c * min(4, n_g - k0) + wl for c in range(C)]
                cg += n_g * C
                T0 += ntasks
            assert prod == list(range(len(prod)))
            assert sorted(sum(cons, [])) == prod and all(c == sorted(c) for c in cons)
            for Sg in (2, 3, 4):                      # ring slots of the group: tile idx may be issued once tile idx - Sg was consumed
                issued, freed, pos, done = 0, set(), [0] * 4, 0
                while done < len(prod):
                    moved = False
                    if issued < len(prod) and (issued < Sg or issued - Sg in freed):
                        issued += 1
                        moved = True
                    for wl in rnd.sample(range(4), 4):
                        if pos[wl] < len(cons[wl]) and cons[wl][pos[wl]] < issued and rnd.random() < 0.7:
                            freed.add(cons[wl][pos[wl]])
                            pos[wl] += 1
                            done += 1
                            moved = True
                    stuck = not moved and not any(pos[w] < len(cons[w]) and cons[w][pos[w]] < issued for w in range(4)) and \
                        not (issued < len(prod) and (issued < Sg or issued - Sg in freed))
                    assert not stuck, (phases, g, Sg)
