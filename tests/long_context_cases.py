"""Inputs and fl_dev_* runners of the long-context op tests (tests/test_gpu_long_context.py on the H100 against the CPU stand-in,
tests/test_long_context_mock.py on the stand-in against the reference library).  Every tensor is laid out and viewed the way
Model::eval does it (tests/llama_graph.py) in a 2048-position context, so one input generator serves all three implementations.

numpy shapes are ggml's ne reversed: rope input [hd, n_head, N] is (N, n_head, hd), scores [n_pos, N, n_head] are (n_head, N, n_pos)."""
import ctypes as C

import numpy as np

N_CTX = 2048


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def diff_report(got, want, axes, origin=None):
    """None when got and want carry the same bits; else the count of differing elements, the first one's index (named by axes,
    numpy order, plus origin: e.g. n_past on the token axis gives the absolute position) and bits, and the max |diff| over them."""
    gb, wb = bits(got), bits(want)
    bad = gb != wb
    nd = int(bad.sum())
    if nd == 0:
        return None
    i = int(np.flatnonzero(bad)[0])
    first = np.unravel_index(i, got.shape)
    origin = origin or (0,) * len(axes)
    where = ", ".join(f"{a} {int(j) + o}" for a, j, o in zip(axes, first, origin))
    with np.errstate(invalid="ignore", over="ignore"):
        md = float(np.max(np.abs(got[bad].astype(np.float64) - want[bad].astype(np.float64))))
    return f"{nd} of {got.size} elements differ, first at ({where}): {gb.flat[i]:#010x} vs {wb.flat[i]:#010x}, max |diff| {md:.6g}"


def put(be, a):
    return be.to_device(np.ascontiguousarray(a))


def view(be, d, ne, nb=None):
    """fl_view over device pointer d; ne fastest first, nb byte strides (default: contiguous f32)."""
    return be.view(d, ne, nb=None if nb is None else list(nb) + [0] * (4 - len(nb)))


# ---- rope, mode 0, in place on Qcur / Kcur [hd, n_head, N] ------------------------------------------------------------------------
def rope_input(hd, n_head, n, n_past):
    rng = np.random.default_rng([1, hd, n_head, n, n_past])
    return rng.standard_normal((n, n_head, hd)).astype(np.float32)


def run_rope(be, x, n_past, permuted=False):
    """permuted: the tensor sits in memory as [hd, N, n_head] and rope works on the permuted view [hd, n_head, N] of it."""
    n, n_head, hd = x.shape
    mem = np.ascontiguousarray(x.transpose(1, 0, 2)) if permuted else x
    d = put(be, mem)
    v = view(be, d, (hd, n_head, n), (4, n * hd * 4, hd * 4)) if permuted else view(be, d, (hd, n_head, n))
    be.check(be.lib.fl_dev_rope(C.byref(v), n_past, hd, 0))
    out = be.to_host(d, mem.shape, np.float32)
    be.free(d)
    return out.transpose(1, 0, 2) if permuted else out


# ---- diag_mask_inf + soft_max on KQ_scaled [n_past + N, N, n_head] ----------------------------------------------------------------
def scores_input(n_past, n, n_head, sigma):
    """Scores of σ 1 or 30.  In rows 0, 5, 10, .. column 0 (never masked) is 8e4, so x - max of every other entry is below -65520 and
    rounds to fp16 -inf (table value 0); in rows 3, 10, 17, .. it is 65510, so x - max straddles -65504 / -65520, fp16's largest
    finite value and its rounding midpoint to -inf.  With n_past 0, row 0 keeps one entry after the mask."""
    rng = np.random.default_rng([2, n_past, n, n_head, sigma])
    s = (rng.standard_normal((n_head, n, n_past + n)) * sigma).astype(np.float32)
    s[:, ::5, 0] = 8e4
    s[:, 3::7, 0] = 65510.0
    return s


def run_mask_soft_max(be, s, n_past):
    d = put(be, s)
    v = view(be, d, s.shape[::-1])
    be.check(be.lib.fl_dev_diag_mask_inf(C.byref(v), n_past))
    masked = be.to_host(d, s.shape, np.float32)
    be.check(be.lib.fl_dev_soft_max(C.byref(v)))
    out = be.to_host(d, s.shape, np.float32)
    be.free(d)
    return masked, out


# ---- K.Q and V.P of a multi-token eval on the caches of one layer ----------------------------------------------------------------
def attn_input(hd, n_head, n, n_pos):
    """K cache rows [pos][n_embd], Qcur (N, n_head, hd), V^T cache [n_embd][n_ctx], probabilities (n_head, N, n_pos)."""
    rng = np.random.default_rng([3, hd, n_head, n, n_pos])
    n_embd = hd * n_head
    kc = rng.standard_normal((N_CTX, n_embd)).astype(np.float32)
    q = rng.standard_normal((n, n_head, hd)).astype(np.float32)
    vt = rng.standard_normal((n_embd, N_CTX)).astype(np.float32)
    p = rng.random((n_head, n, n_pos)).astype(np.float32)
    return kc, q, vt, p


def run_kq(be, kc, q, n_pos):
    """K = permute(reshape_3d(view_1d(k, n_pos * n_embd), hd, n_head, n_pos), 0, 2, 1, 3), Q = permute(Qcur, 0, 2, 1, 3):
    KQ [n_pos, N, n_head], returned as (n_head, N, n_pos)."""
    n, n_head, hd = q.shape
    n_embd = hd * n_head
    dk, dq, do = put(be, kc), put(be, q), be.alloc(n_pos * n * n_head * 4)
    k = view(be, dk, (hd, n_pos, n_head), (4, n_embd * 4, hd * 4))
    qv = view(be, dq, (hd, n, n_head), (4, n_embd * 4, hd * 4))
    o = view(be, do, (n_pos, n, n_head))
    be.check(be.lib.fl_dev_mul_mat_f32(C.byref(k), C.byref(qv), C.byref(o)))
    out = be.to_host(do, (n_head, n, n_pos), np.float32)
    for d in (dk, dq, do):
        be.free(d)
    return out


def run_vp(be, vt, p, hd):
    """V = view_3d(v, n_pos, hd, n_head, n_ctx * 4, n_ctx * 4 * hd, 0) (row stride n_ctx: the inner length is n_pos with its
    n_pos % 32 leftovers), P = KQ_soft [n_pos, N, n_head]: KQV [hd, N, n_head], returned as (n_head, N, hd)."""
    n_head, n, n_pos = p.shape
    dv, dp, do = put(be, vt), put(be, p), be.alloc(hd * n * n_head * 4)
    v = view(be, dv, (n_pos, hd, n_head), (4, N_CTX * 4, N_CTX * 4 * hd))
    pv = view(be, dp, (n_pos, n, n_head))
    o = view(be, do, (hd, n, n_head))
    be.check(be.lib.fl_dev_mul_mat_f32(C.byref(v), C.byref(pv), C.byref(o)))
    out = be.to_host(do, (n_head, n, hd), np.float32)
    for d in (dv, dp, do):
        be.free(d)
    return out
