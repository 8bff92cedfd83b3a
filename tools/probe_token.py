"""Where does the persistent token kernel spend its time?  Builds an n-layer LLaMA-7B-shaped token plan with
random q4_0 blocks (values do not matter for timing), launches it with FASTLLAMA_B200_TOKEN_PROF=1 and prints,
per step kind, the time CTAs spend in the grid barrier, the activation prologue and the tile loop.

    python tools/probe_token.py [n_layer] [n_past]
"""
import ctypes as C
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault("FASTLLAMA_B200_TOKEN_PROF", "1")

from fastllama_b200.cuda_abi import EPI_QKV, EPI_RESADD, EPI_STORE, PRO_RMSNORM, PRO_SILUMUL, FlCuda, FlMvArgs, FlTokenStep  # noqa: E402

n_layer = int(sys.argv[1]) if len(sys.argv) > 1 else 8
n_past = int(sys.argv[2]) if len(sys.argv) > 2 else 64
# FASTLLAMA_B200_PROBE_SHAPE=13B / 30B / 65B: those models' dimensions; FASTLLAMA_B200_PROBE_TYPE=3: q4_1 blocks
SHAPES = {"7B": (4096, 32, 11008, 32000, 512), "13B": (5120, 40, 13824, 32000, 512), "30B": (6656, 52, 17920, 32000, 512), "65B": (8192, 64, 22016, 32000, 512)}
n_embd, n_head, n_ff, n_vocab, n_ctx = SHAPES[os.environ.get("FASTLLAMA_B200_PROBE_SHAPE", "7B")]
WT = int(os.environ.get("FASTLLAMA_B200_PROBE_TYPE", "2"))
BB = 20 if WT == 2 else 24
hd = n_embd // n_head
fl = FlCuda()
rng = np.random.default_rng(0)


def wq(m, k):
    nb = k // 32
    w = np.empty((m, nb, BB), dtype=np.uint8)
    w[..., :4] = (0.002 * rng.random((m, nb, 1), dtype=np.float32) + 0.0005).view(np.uint8).reshape(m, nb, 4)
    if WT == 3:
        w[..., 4:8] = (0.01 * rng.random((m, nb, 1), dtype=np.float32) - 0.005).view(np.uint8).reshape(m, nb, 4)
    w[..., BB - 16:] = rng.integers(0, 256, size=(m, nb, 16), dtype=np.uint8)
    return fl.to_device(w.reshape(-1))


def buf(n, init=None):
    p = fl.alloc(n * 4)
    if init is None:
        fl.check(fl.lib.fl_dev_memset(p, 0, n * 4))
    else:
        fl.check(fl.lib.fl_h2d(p, init.ctypes.data, n * 4))
    return p


gam = np.ones(n_embd, dtype=np.float32)
x0 = rng.standard_normal(n_embd).astype(np.float32)
xa, xb, q, att, m1, m3, emb, logits = buf(n_embd, x0), buf(n_embd), buf(n_embd), buf(n_embd), buf(n_ff), buf(n_ff), buf(n_embd), buf(n_vocab)
dg = fl.to_device(gam)
dnp = fl.to_device(np.array([n_past], dtype=np.int32))
fl.check(fl.lib.fl_dev_rope_table(hd, n_ctx))
steps, names = [], []
for il in range(n_layer):
    kc = fl.to_device((rng.standard_normal((n_ctx, n_embd)) * 0.1).astype(np.float32))
    vc = fl.to_device((rng.standard_normal((n_embd, n_ctx)) * 0.1).astype(np.float32))
    a = FlMvArgs()
    a.type, a.K, a.nseg, a.pro, a.epi = WT, n_embd, 3, PRO_RMSNORM, EPI_QKV
    for i in range(3):
        a.seg_w[i], a.seg_rows[i] = wq(n_embd, n_embd), n_embd
    a.seg_dst[0] = q
    a.x, a.gamma, a.n_past, a.n_ctx, a.n_embd, a.head_dim, a.kcache, a.vcache = xa, dg, dnp, n_ctx, n_embd, hd, kc, vc
    steps.append(("mv", a)); names.append("qkv")
    steps.append(("attn", (q, kc, vc, att))); names.append("attn")
    a = FlMvArgs()
    a.type, a.K, a.nseg, a.pro, a.epi = WT, n_embd, 1, 0, EPI_RESADD
    a.seg_w[0], a.seg_rows[0], a.seg_dst[0], a.x, a.res = wq(n_embd, n_embd), n_embd, xb, att, xa
    steps.append(("mv", a)); names.append("wo")
    a = FlMvArgs()
    a.type, a.K, a.nseg, a.pro, a.epi = WT, n_embd, 2, PRO_RMSNORM, EPI_STORE
    a.seg_w[0], a.seg_rows[0], a.seg_dst[0] = wq(n_ff, n_embd), n_ff, m1
    a.seg_w[1], a.seg_rows[1], a.seg_dst[1] = wq(n_ff, n_embd), n_ff, m3
    a.x, a.gamma = xb, dg
    steps.append(("mv", a)); names.append("w13")
    a = FlMvArgs()
    a.type, a.K, a.nseg, a.pro, a.epi = WT, n_ff, 1, PRO_SILUMUL, EPI_RESADD
    a.seg_w[0], a.seg_rows[0], a.seg_dst[0], a.x, a.b, a.res = wq(n_embd, n_ff), n_embd, xa, m1, m3, xb
    steps.append(("mv", a)); names.append("w2")
a = FlMvArgs()
a.type, a.K, a.nseg, a.pro, a.epi = WT, n_embd, 1, PRO_RMSNORM, EPI_STORE
a.seg_w[0], a.seg_rows[0], a.seg_dst[0], a.x, a.gamma, a.normed_out = wq(n_vocab, n_embd), n_vocab, logits, xa, dg, emb
steps.append(("mv", a)); names.append("head")

arr = (FlTokenStep * len(steps))()
scale = np.float32(1.0 / math.sqrt(hd))
for i, (kind, s) in enumerate(steps):
    if kind == "mv":
        arr[i].kind, arr[i].mv = 0, s
    else:
        arr[i].kind = 1
        arr[i].q, arr[i].kcache, arr[i].vcache, arr[i].out, arr[i].n_past = s[0], s[1], s[2], s[3], dnp
        arr[i].k_row_stride, arr[i].n_head, arr[i].head_dim, arr[i].n_ctx, arr[i].scale = n_embd, n_head, hd, n_ctx, scale
plan = C.c_void_p()
fl.check(fl.lib.fl_token_plan_create(arr, len(steps), C.byref(plan)))
ev0, ev1 = fl.lib.fl_event_create(), fl.lib.fl_event_create()
for _ in range(3):
    fl.check(fl.lib.fl_h2d(xa, x0.ctypes.data, n_embd * 4))
    fl.check(fl.lib.fl_token_plan_launch(plan))
fl.check(fl.lib.fl_sync())
if fl.lib.fl_token_plan_error(plan):
    print("TOKEN KERNEL ERROR:", fl.lib.fl_last_error().decode())
    sys.exit(3)
iters = 10
fl.check(fl.lib.fl_event_record(ev0))
for _ in range(iters):
    fl.check(fl.lib.fl_token_plan_launch(plan))
fl.check(fl.lib.fl_event_record(ev1))
fl.check(fl.lib.fl_event_sync(ev1))
ms = C.c_float()
fl.check(fl.lib.fl_event_elapsed_ms(ev0, ev1, C.byref(ms)))
wbytes = n_layer * (4 * n_embd * n_embd + 3 * n_ff * n_embd) // 32 * BB + n_vocab * n_embd // 32 * BB
print(f"{n_layer} layers + head: {ms.value / iters * 1e3:.1f} us per launch, {wbytes / (ms.value / iters * 1e-3) / 1e9:.0f} GB/s of weights")

n_cta = C.c_int()
n_sm = fl.device_props()["sm_count"]            # one CTA per SM
prof = np.zeros((len(steps), n_sm, 4), dtype=np.uint64)
fl.check(fl.lib.fl_token_plan_profile(plan, prof.ctypes.data, prof.size, C.byref(n_cta)))
t = prof.astype(np.int64)
t0 = t[0, :, 0].min()
t = (t - t0) / 1e3   # us
print(f"kernel span (first stamp to last): {t[-1, :, 3].max():.1f} us")
print(f"{'step':>5} {'name':>5} {'start':>8} | barrier: {'mean':>6} {'max':>6} | prologue {'mean':>6} {'max':>6} | tiles {'mean':>6} {'max':>6} | span")
agg = {}
for i, nm in enumerate(names):
    bar = t[i, :, 1] - t[i, :, 0]
    pro = t[i, :, 2] - t[i, :, 1]
    til = t[i, :, 3] - t[i, :, 2]
    start = t[i, :, 0].min()
    end = t[i + 1, :, 0].min() if i + 1 < len(names) else t[i, :, 3].max()
    agg.setdefault(nm, []).append((bar.mean(), bar.max(), pro.mean(), pro.max(), til.mean(), til.max(), end - start))
    if i < 12 or i == len(names) - 1:
        print(f"{i:5d} {nm:>5} {start:8.1f} | {bar.mean():15.2f} {bar.max():6.2f} | {pro.mean():15.2f} {pro.max():6.2f} | {til.mean():12.2f} {til.max():6.2f} | {end - start:6.2f}")
print("\nmean over layers (us):")
for nm, rows in agg.items():
    r = np.array(rows).mean(axis=0)
    print(f"{nm:>5}: barrier {r[0]:5.2f} (max {r[1]:5.2f})  prologue {r[2]:5.2f} (max {r[3]:5.2f})  tiles {r[4]:5.2f} (max {r[5]:5.2f})  span {r[6]:6.2f}")
# per-warp cycle breakdown of the tile loops (PROF kernel)
p2 = np.zeros((len(steps), n_sm, 16, 8), dtype=np.uint32)
fl.check(fl.lib.fl_token_plan_profile2(plan, p2.ctypes.data, p2.size))
print("\nper consumer warp, mean over CTAs and warps (SM cycles): activation fetch | waiting for tiles | dots | reduce+epilogue+loop | rounds | total | tiles per CTA")
agg2 = {}
for i, nm in enumerate(names):
    if nm == "attn":
        continue
    agg2.setdefault(nm, []).append(p2[i].reshape(-1, 8).astype(np.float64).mean(axis=0))
for nm, rows in agg2.items():
    r = np.array(rows).mean(axis=0)
    per = (r[2] / r[4], r[3] / r[4]) if r[4] else (0, 0)
    print(f"{nm:>5}: yfetch {r[0]:7.0f}  wait {r[1]:7.0f}  dots {r[2]:7.0f}  tail {r[3]:7.0f}  rounds {r[4]:5.2f}  total {r[5]:7.0f}  tiles/warp {r[6]:5.1f}  wait of round 1 {r[7]:6.0f}   per round: dots {per[0]:6.0f} tail {per[1]:6.0f}")
fl.check(fl.lib.fl_token_plan_destroy(plan))
