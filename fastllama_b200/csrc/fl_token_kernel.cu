// fl_token_kernel.cu -- the whole decode step of a LLaMA token as ONE persistent kernel.
//
// Why: with one kernel per matrix group the decode step is 160 launches of 3-18 us whose fixed costs
// (launch, barrier init, prologue, first-tile latency, drain) leave HBM idle ~70 % of the time
// (DESIGN.md section 4).  Here one CTA per SM (co-resident by cooperative launch) walk a
// "program" of phases -- per layer: wq|wk|wv, attention, wo, w1|w3, w2; then the LM head -- separated
// by grid-wide barriers, and each CTA's producer lane streams the weight tiles of ALL phases through one
// mbarrier ring, running ahead of the consumers across phase boundaries: while the grid synchronises
// and the next activation vector is quantised, the next matrices are already landing in shared memory.
//
// Work unit = a PAIR of rows (both rows against the same prepared activations):
//   * default: rows (2u, 2u+1) of a matrix;
//   * wq|wk|wv: the pair is a rope pair, so rope + KV-cache store need no cross-warp staging;
//   * w1|w3 ("SwiGLU" phases, detected at plan creation): the pair is (w1 row u, w3 row u) and the
//     epilogue writes silu(w1.x) * (w3.x) directly, so w2's prologue is a plain quantisation.
// ARITHMETIC: every fp32 operation happens in the reference's own order (fl_exact.cuh): a warp owns a TASK of four units (eight
// rows), four lanes per row, lane jj carrying the reference's accumulators 2jj and 2jj+1 through ALL blocks of the row in order;
// attention scores and the value mix follow ggml_vec_dot_f32's 32-lane order.  The logits of a token are therefore the bits the
// reference's x86 build produces (the one known exception: rms_norm's double sum, see fl_ops_kernels.cu).
// A task's rows are streamed in K-chunks of TK_CHB blocks: tile = (task, chunk) = 8 row pieces of <= 640 (q4_0) / 768 (q4_1)
// bytes, each copied by its own bulk copy to a row pitch of chunk + 16 bytes, which makes the 32 lanes' weight words fall into
// 32 different banks.  The four consumer warps of a tile group take the tiles of their group's stream in turn.
// Activations move between phases through L2: they are read with ld.global.cg (L1 is not coherent
// across SMs inside a kernel) and published by a gpu-scope release before the barrier arrive.
#include <cuda_fp16.h>
#include <stdlib.h>

#include <algorithm>
#include <vector>

#include "fl_common.cuh"
#include "fl_decode.h"
#include "fl_decode_dev.cuh"
#include "fl_exact.cuh"
#include "fl_kernels.h"

#define TK_CW 16                 // consumer warps
#define TK_NT (TK_CW * 32)
#define TK_TG 4                  // tile groups; ring slot s always belongs to group s % 4 (S is a multiple of 4)
#define TK_WPG 4                 // consumer warps per tile group
#define TK_GMAX 4                // units (row pairs) per task
#define TK_CHB 32                // blocks per K-chunk of a task (one tile = 8 row pieces of one chunk; see DESIGN.md section 3 for 32 vs 64)
#define TK_PW 4                  // producer warps: warp TK_CW + g streams the tiles of tile group g (its own slots, its own pace)
#define TK_THREADS (TK_NT + 32 * TK_PW)
#define TK_REGS_CONSUMER 104      // setmaxnreg: the producer warpgroup hands registers to the four consumer warpgroups.  The pool is the CTA's
                                  // LAUNCH allocation (96 x 640 = 61440 registers): 104 x 512 + 64 x 128 = 61440 is exactly the pool; a request beyond the pool
                                  // waits forever (checked on the host at plan creation)
#define TK_REGS_PRODUCER 64

enum { TK_PH_MATVEC = 0, TK_PH_ATTN = 1 };

struct tk_phase {
    int kind;
    int nb, nchunks;             // blocks per row, K-chunks per task
    uint32_t srow;               // pitch of a row piece in a ring slot: chunk bytes + 16
    int swiglu;                  // pair = (seg 0 row u, seg 1 row u); epilogue writes silu(a) * b to seg_dst[0][u]
    int units[3];                // pairs per segment (swiglu: one segment of seg_rows[0] pairs)
    uint32_t row_bytes;
    fl_mv_args a;
    // attention
    const float *q, *kcache, *vcache;
    float *out;
    int k_row_stride, n_head, head_dim, n_ctx;
    int head_split;              // CTAs per head (each owns head_dim / head_split output dimensions)
    int out_ll, out_seq, n_out_peer;
    float *out_peer[7];
    float scale;
};

struct tk_params {
    const tk_phase *phases;
    int n_phases;
    unsigned *grid_bar;              // [0] arrival counter (zeroed per launch)
    unsigned *err;                   // error block in pinned, device-mapped HOST memory: [0] flag, [1..4] details (the host reads it without a copy)
    int rank, world;
    unsigned *ll_count;              // running number of LL exchanges of all earlier launches (a device word that lives with the LL vectors)
    int n_ll;                        // LL exchanges per launch
    const uint16_t *exp_tab;
    unsigned long long *prof;      // optional: [n_phases][gridDim.x][4] globaltimer stamps of thread 0
    unsigned *prof2;               // optional (PROF kernel only): [n_phases][gridDim.x][TK_CW][8] cycle counts of every consumer warp's tile loop
    int S, Sg;                       // ring slots in total and per tile group (S = 4 * Sg)
    uint32_t grid_magic, grid_shift, s_magic, s_shift;  // n / d == umulhi(n, magic) >> shift (magic 0: d is a power of two, n >> shift); exact for n < 2^31; s_*: d = Sg
    uint32_t slot_bytes;
    int diag;                        // FASTLLAMA_B200_TK_DIAG (timing experiments only; results are garbage): 1 = no weight copies, 2 = no dot products, 4 = no grid barriers, 8 = no prologue
    uint32_t off_y, off_red, off_rowbuf, off_cnt, off_sc, off_stage0;
};

__device__ __forceinline__ unsigned long long tk_now() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void tk_bar_consumers(int id) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(TK_NT) : "memory"); }

// Every spin in this kernel is bounded: after 2 s (a peer GPU that never launched, a bug) the waiter raises the error flag
// and everybody falls through; the host reports it (fl_token_plan_error) instead of the GPU hanging.
__device__ __forceinline__ void tk_wait_ge(const unsigned *p, unsigned target, bool sys, unsigned *err, unsigned who) {
    unsigned long long t0 = 0;
    for (unsigned n = 1;; n++) {
        unsigned v;
        if (sys) asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");     // caller fences after the wait
        else asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
        if ((int)(v - target) >= 0) return;
        if ((n & 1023u) == 0) {
            if (*(volatile unsigned *)err) return;
            const unsigned long long t = tk_now();
            if (t0 == 0) t0 = t;
            else if (t - t0 > 2000000000ull) {
                if (atomicExch(err, 1u) == 0u) { err[1] = who; err[2] = target; err[3] = v; err[4] = blockIdx.x; }   // first failure, for the host's message
                return;
            }
        }
    }
}
// mbarrier wait of the weight ring, bounded like every other spin of this kernel: a protocol bug reports (who, slot, parity) instead of hanging the GPU
__device__ __forceinline__ void tk_mbar_wait(uint32_t bar, uint32_t parity, unsigned *err, unsigned who, unsigned slot) {
    unsigned long long t0 = 0;
    for (unsigned n = 1; !fl_mbar_try_wait(bar, parity); n++) {
        if ((n & 4095u) == 0) {
            if (*(volatile unsigned *)err) return;
            const unsigned long long t = tk_now();
            if (t0 == 0) t0 = t;
            else if (t - t0 > 2000000000ull) {
                if (atomicExch(err, 1u) == 0u) { err[1] = who; err[2] = slot; err[3] = parity; err[4] = blockIdx.x; }
                return;
            }
        }
    }
}
__device__ __forceinline__ void tk_tag_wait(volatile uint32_t *tag, uint32_t want, unsigned *err, unsigned who, unsigned slot) {
    unsigned long long t0 = 0;
    for (unsigned n = 1; *tag != want; n++) {
        if ((n & 4095u) == 0) {
            if (*(volatile unsigned *)err) return;
            const unsigned long long t = tk_now();
            if (t0 == 0) t0 = t;
            else if (t - t0 > 2000000000ull) {
                if (atomicExch(err, 1u) == 0u) { err[1] = who; err[2] = slot; err[3] = want; err[4] = blockIdx.x; }
                return;
            }
        }
    }
}
// Grid barrier: CTA barrier, then one thread publishes the CTA's writes with a gpu-scope release increment and spins on
// an acquire load; the second CTA barrier hands the acquired view to the other threads, which read shared activations
// with ld.global.cg only.  Only the step in front of the attention needs it (q and the KV rows of all CTAs); every other
// hand-over is a dataflow (LL) vector.
__device__ __forceinline__ void tk_grid_sync(const tk_params &prm, unsigned target, unsigned) {
    // One arrival per CTA.  (Per-warp arrivals -- 16 atomics per CTA on one address -- make every barrier slower.)
    tk_bar_consumers(13);
    if (threadIdx.x == 0) {
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(prm.grid_bar) : "memory");
        tk_wait_ge(prm.grid_bar, target, false, prm.err, 0x100u);
    }
    tk_bar_consumers(13);
}

// ---- the CTA's slice of a phase, in units (row pairs), cut into tiles of at most G units ------------
struct tk_slice {
    int f0, f1, f2, n0, n1, n2, t0, t1, ntiles;
};
__device__ __forceinline__ uint32_t tk_div(uint32_t n, uint32_t magic, uint32_t shift) { return (magic ? __umulhi(n, magic) : n) >> shift; }
// lgG = log2 of the units per tile (1, 2 or 4 units)
__device__ __forceinline__ tk_slice tk_make_slice_u(int m0, int m1, int m2, int lgG, uint32_t grid_magic, uint32_t grid_shift) {
    tk_slice sl;
    const unsigned U = (unsigned)(m0 + m1 + m2);            // U * gridDim.x < 2^32 (checked at plan creation)
    const int u0 = (int)tk_div(U * blockIdx.x, grid_magic, grid_shift);
    const int u1 = (int)tk_div(U * (blockIdx.x + 1), grid_magic, grid_shift);
    const int rnd = (1 << lgG) - 1;
    fd_seg_span(u0, u1, 0, m0, sl.f0, sl.n0);
    fd_seg_span(u0, u1, m0, m1, sl.f1, sl.n1);
    fd_seg_span(u0, u1, m0 + m1, m2, sl.f2, sl.n2);
    sl.t0 = (sl.n0 + rnd) >> lgG;
    sl.t1 = sl.t0 + ((sl.n1 + rnd) >> lgG);
    sl.ntiles = sl.t1 + ((sl.n2 + rnd) >> lgG);
    return sl;
}
__device__ __forceinline__ void tk_tile_of(const tk_slice &sl, int G, int t, int &seg, int &unit0, int &nunits) {
    seg = (t < sl.t0) ? 0 : (t < sl.t1) ? 1 : 2;
    const int j = t - (seg == 0 ? 0 : seg == 1 ? sl.t0 : sl.t1);
    const int first = seg == 0 ? sl.f0 : seg == 1 ? sl.f1 : sl.f2;
    const int n = seg == 0 ? sl.n0 : seg == 1 ? sl.n1 : sl.n2;
    unit0 = first + j * G;
    nunits = min(G, n - j * G);
}

// ---- prologue: the phase's activations, q8_0-quantised and prepared for the block dot, into shared memory ----
// Same arithmetic as quantize_row_q8_0 (bit-exact, tests/test_gpu_rowfns.py), different work split: one
// thread quantises one HALF block (16 consecutive values, two lanes per block), which needs one shuffle per
// reduction and two divisions per block pair instead of per float4 group -- 2.5x fewer issue slots than the
// float4-group scheme, and this code runs redundantly in every CTA behind every grid barrier.
// A prepared block is an fl_yx (fl_exact.cuh, 80 bytes): per lane-of-four jj the two 4-value words and their biases (one LDS.128),
// then the block's d and s (one LDS.64).
typedef fl_yx tk_yblock;

// A thread quantises E consecutive values (E = 8: four lanes per block, E = 16: two lanes per block, E = 32: a whole block).
template <int E>
__device__ __forceinline__ void tk_load_vals(const float4 *p4, int u, float v[E], bool cg) {
#pragma unroll
    for (int k = 0; k < E / 4; k++) {
        const float4 t = cg ? __ldcg(p4 + (E / 4) * u + k) : __ldg(p4 + (E / 4) * u + k);
        v[4 * k + 0] = t.x; v[4 * k + 1] = t.y; v[4 * k + 2] = t.z; v[4 * k + 3] = t.w;
    }
}
template <int E>
__device__ __forceinline__ void tk_zero_vals(float v[E]) {
#pragma unroll
    for (int k = 0; k < E; k++) v[k] = 0.f;
}
// E values of unit u from an LL slot ({value, epoch} words): all loads are issued, then re-issued until every word carries epoch e
template <int E>
__device__ __forceinline__ void tk_load_ll(const float *base, int u, float v[E], unsigned e, unsigned *err) {
    const uint4 *p = (const uint4 *)base + (size_t)(E / 2) * u;
    unsigned long long t0 = 0;
    for (unsigned n = 1;; n++) {
        uint4 t[E / 2];
#pragma unroll
        for (int k = 0; k < E / 2; k++)
            asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(t[k].x), "=r"(t[k].y), "=r"(t[k].z), "=r"(t[k].w) : "l"(p + k) : "memory");
        bool ok = true;
#pragma unroll
        for (int k = 0; k < E / 2; k++) {
            ok = ok && t[k].y == e && t[k].w == e;
            v[2 * k] = __uint_as_float(t[k].x);
            v[2 * k + 1] = __uint_as_float(t[k].z);
        }
        if (ok) return;
        // a failed round backs off: every CTA's 512 threads spinning on the same words would otherwise keep the L2 busy with the polls
        // themselves -- and with it the stores they are waiting for and the weight stream
        __nanosleep(n < 4 ? 40u : 200u);
        if ((n & 255u) == 0) {                       // bounded like every other spin of this kernel
            if (*(volatile unsigned *)err) return;
            const unsigned long long now = tk_now();
            if (t0 == 0) t0 = now;
            else if (now - t0 > 2000000000ull) {
                if (atomicExch(err, 1u) == 0u) { err[1] = 0x300u; err[2] = e; err[3] = t[0].y; err[4] = blockIdx.x; }
                return;
            }
        }
    }
}
// x (LL vector: polled until every word carries the epoch) (+ xadd) of unit u
template <int E>
__device__ __forceinline__ void tk_load_x(const fl_mv_args &A, int u, float v[E], unsigned ll_epoch, unsigned *err) {
    if (A.x_ll) tk_load_ll<E>(A.x, u, v, ll_epoch, err);
    else tk_load_vals<E>((const float4 *)A.x, u, v, true);
    if (A.xadd) {
        float w[E];
        tk_load_vals<E>((const float4 *)A.xadd, u, w, true);
#pragma unroll
        for (int k = 0; k < E; k++) v[k] = __fadd_rn(v[k], w[k]);
    }
}
template <int E>
__device__ __forceinline__ void tk_store_vals(float *dst, int u, const float v[E]) {
#pragma unroll
    for (int k = 0; k < E / 4; k++) ((float4 *)dst)[(E / 4) * u + k] = make_float4(v[4 * k], v[4 * k + 1], v[4 * k + 2], v[4 * k + 3]);
}
// v: the E final values of unit u (all lanes of the warp call this; `valid` lanes store); off = 8 for q4_0 weights, 0 for q4_1
template <int E>
__device__ __forceinline__ void tk_quant(const float v[E], int u, bool valid, tk_yblock *ysm, int off) {
    float m0 = 0.f, m1 = 0.f;                        // two chains: max is order-independent
#pragma unroll
    for (int k = 0; k < E; k += 2) { m0 = fmaxf(m0, fabsf(v[k])); m1 = fmaxf(m1, fabsf(v[k + 1])); }
    float amax = fmaxf(m0, m1);
    if (E <= 16) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
    if (E == 8) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
    const float d = __fdiv_rn(amax, 127.f);
    const float id = (amax != 0.0f) ? __fdiv_rn(127.f, amax) : 0.0f;
    int q[E], s0 = 0, s1 = 0;
#pragma unroll
    for (int k = 0; k < E; k += 2) {
        q[k] = max(-128, min(127, __float2int_rn(__fmul_rn(v[k], id))));
        q[k + 1] = max(-128, min(127, __float2int_rn(__fmul_rn(v[k + 1], id))));
        s0 += q[k]; s1 += q[k + 1];
    }
    int sum = s0 + s1;
    if (E <= 16) sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    if (E == 8) sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    if (valid) {
        constexpr int NW = E / 8;                    // 8-element groups of the block this thread owns
        constexpr int UPB = 32 / E;                  // units per block
        tk_yblock *yb = ysm + u / UPB;
        const int part = u % UPB;
#pragma unroll
        for (int j = 0; j < NW; j++) {
            const uint32_t ya = (uint32_t)(q[8 * j + 0] & 0xFF) | ((uint32_t)(q[8 * j + 1] & 0xFF) << 8) | ((uint32_t)(q[8 * j + 2] & 0xFF) << 16) | ((uint32_t)(q[8 * j + 3] & 0xFF) << 24);
            const uint32_t yb4 = (uint32_t)(q[8 * j + 4] & 0xFF) | ((uint32_t)(q[8 * j + 5] & 0xFF) << 8) | ((uint32_t)(q[8 * j + 6] & 0xFF) << 16) | ((uint32_t)(q[8 * j + 7] & 0xFF) << 24);
            const int sa = q[8 * j + 0] + q[8 * j + 1] + q[8 * j + 2] + q[8 * j + 3], sb = q[8 * j + 4] + q[8 * j + 5] + q[8 * j + 6] + q[8 * j + 7];
            *(uint4 *)yb->q[NW * part + j] = make_uint4(ya, yb4, (uint32_t)(FX_MAGIC_I - off * sa), (uint32_t)(FX_MAGIC_I - off * sb));
        }
        if (part == 0) *(float2 *)&yb->d = make_float2(d, __fmul_rn(d, (float)sum));
    }
}
// plain / silu*mul prologue body for one unit size
template <int E>
__device__ __forceinline__ void tk_prologue_nonorm(const fl_mv_args &A, int K, tk_yblock *ysm, int warp, int tid, unsigned lle, unsigned *err) {
    const int qoff = (A.type == FL_TYPE_Q4_0) ? 8 : 0;
    const int nu = K / E;
    if (E == 16 && A.pro != FL_PRO_SILUMUL && nu > TK_NT && nu <= 2 * TK_NT) {
        // two units per thread (K = 11008: 688 half blocks on 512 threads), BOTH loads in flight before either is quantised: one L2
        // round trip instead of two on the critical path behind the grid barrier
        const int ua = tid, ub = tid + TK_NT;
        const bool vb = ub < nu, wb = TK_NT + warp * 32 < nu;          // wb: warp-uniform
        float va[E], vv[E];
        tk_load_x<E>(A, ua, va, lle, err);
        if (vb) tk_load_x<E>(A, ub, vv, lle, err); else tk_zero_vals<E>(vv);
        if (A.sum_out && blockIdx.x == 0) { tk_store_vals<E>(A.sum_out, ua, va); if (vb) tk_store_vals<E>(A.sum_out, ub, vv); }
        tk_quant<E>(va, ua, true, ysm, qoff);
        if (wb) tk_quant<E>(vv, ub, vb, ysm, qoff);
        return;
    }
    for (int u0 = 0; u0 < nu; u0 += TK_NT) {
        if (u0 + warp * 32 >= nu) break;                 // warp-uniform
        const int u = u0 + tid;
        const bool valid = u < nu;
        float v[E];
        if (valid) tk_load_x<E>(A, u, v, lle, err); else tk_zero_vals<E>(v);
        if (A.sum_out && blockIdx.x == 0 && valid) tk_store_vals<E>(A.sum_out, u, v);
        if (A.pro == FL_PRO_SILUMUL) {
            float bm[E];
            if (valid) tk_load_vals<E>((const float4 *)A.b, u, bm, true); else tk_zero_vals<E>(bm);
#pragma unroll
            for (int k = 0; k < E; k++) {
                const uint16_t hh = __half_as_ushort(__float2half_rn(v[k]));
                v[k] = __fmul_rn(__half2float(__ushort_as_half(__ldg(A.silu_tab + hh))), bm[k]);
            }
        }
        tk_quant<E>(v, u, valid, ysm, qoff);
    }
}

// rms_norm * gamma prologue.  RES > 0: the thread's RES 8-element units stay in registers between the sum of squares
// and the quantisation (K <= 8 * RES * TK_NT); RES == 0: two passes over L2.
// Sum of squares: thread t adds the values of units t, t + NT, ... in order (k_mv_fused uses the same order).
template <int RES>
__device__ __forceinline__ void tk_prologue_norm(const fl_mv_args &A, int K, tk_yblock *ysm, double *red, int warp, int lane, int tid, unsigned lle, unsigned *err) {
    const int qoff = (A.type == FL_TYPE_Q4_0) ? 8 : 0;
    constexpr int E = 8, NR = RES > 0 ? RES : 1;
    const int nu = K >> 3;
    float v[NR][E], gm[NR][E];
    double acc = 0.0;
    if (RES > 0) {
#pragma unroll
        for (int r = 0; r < NR; r++) {
            const int u = tid + r * TK_NT;
            if (u < nu) { tk_load_x<E>(A, u, v[r], lle, err); tk_load_vals<E>((const float4 *)A.gamma, u, gm[r], false); }
            else { tk_zero_vals<E>(v[r]); tk_zero_vals<E>(gm[r]); }
        }
#pragma unroll
        for (int r = 0; r < NR; r++)
#pragma unroll
            for (int k = 0; k < E; k++) acc += (double)__fmul_rn(v[r][k], v[r][k]);
    } else {
        for (int u = tid; u < nu; u += TK_NT) {
            tk_load_x<E>(A, u, v[0], lle, err);
#pragma unroll
            for (int k = 0; k < E; k++) acc += (double)__fmul_rn(v[0][k], v[0][k]);
        }
    }
    acc = fl_warp_sum_d(acc);
    if (lane == 0) red[warp] = acc;
    tk_bar_consumers(15);
    if (warp == 0) {                                         // the double division is ~100 instructions: one warp, not sixteen
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < TK_CW; w++) t += red[w];
        const float mean = (float)(t / (double)K);
        if (lane == 0) ((float *)(red + 16))[0] = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(mean, 1e-6f)));
    }
    tk_bar_consumers(15);
    const float scale = ((float *)(red + 16))[0];
    if (RES > 0) {
#pragma unroll
        for (int r = 0; r < NR; r++) {
            if (r * TK_NT + warp * 32 < nu) {                // warp-uniform
                const int u = tid + r * TK_NT;
                const bool valid = u < nu;
                if (A.sum_out && blockIdx.x == 0 && valid) tk_store_vals<E>(A.sum_out, u, v[r]);
#pragma unroll
                for (int k = 0; k < E; k++) v[r][k] = __fmul_rn(gm[r][k], __fmul_rn(v[r][k], scale));
                if (A.normed_out && blockIdx.x == 0 && valid) tk_store_vals<E>(A.normed_out, u, v[r]);
                tk_quant<E>(v[r], u, valid, ysm, qoff);
            }
        }
    } else {
        for (int u0 = 0; u0 < nu; u0 += TK_NT) {
            if (u0 + warp * 32 >= nu) break;
            const int u = u0 + tid;
            const bool valid = u < nu;
            if (valid) { tk_load_x<E>(A, u, v[0], lle, err); tk_load_vals<E>((const float4 *)A.gamma, u, gm[0], false); }
            else { tk_zero_vals<E>(v[0]); tk_zero_vals<E>(gm[0]); }
            if (A.sum_out && blockIdx.x == 0 && valid) tk_store_vals<E>(A.sum_out, u, v[0]);
#pragma unroll
            for (int k = 0; k < E; k++) v[0][k] = __fmul_rn(gm[0][k], __fmul_rn(v[0][k], scale));
            if (A.normed_out && blockIdx.x == 0 && valid) tk_store_vals<E>(A.normed_out, u, v[0]);
            tk_quant<E>(v[0], u, valid, ysm, qoff);
        }
    }
}

__device__ __forceinline__ void tk_prologue(const fl_mv_args &A, int K, tk_yblock *ysm, double *red, int warp, int lane, int tid, unsigned lle, unsigned *err) {
    const int nu8 = K >> 3;
    if (A.pro == FL_PRO_RMSNORM) {
        if (nu8 <= TK_NT) tk_prologue_norm<1>(A, K, ysm, red, warp, lane, tid, lle, err);
        else if (nu8 <= 2 * TK_NT) tk_prologue_norm<2>(A, K, ysm, red, warp, lane, tid, lle, err);
        else tk_prologue_norm<0>(A, K, ysm, red, warp, lane, tid, lle, err);
    } else if (nu8 <= TK_NT) {
        tk_prologue_nonorm<8>(A, K, ysm, warp, tid, lle, err);          // short vectors: latency matters, spread over all threads
    } else {
        tk_prologue_nonorm<16>(A, K, ysm, warp, tid, lle, err);         // long vectors: issue slots matter (a whole block per thread was measured: slower)
    }
}

// ---- epilogue of one unit (lane 0 of the warp that holds the complete sums a, b) --------------------
// `pre` is what the epilogue needs from memory -- the residual pair (RESADD) or the rope (cos, sin) pair (QKV, q and k rows) --
// loaded by tk_epilogue_preload BEFORE the warp's dot products, so its L2 round trip hides behind them.
__device__ __forceinline__ void tk_store_ll(float *slot, int row, float v, unsigned e, float *const *peers, int n_peers) {
    const unsigned uv = __float_as_uint(v);
    asm volatile("st.relaxed.sys.global.v2.u32 [%0], {%1, %2};" ::"l"(slot + 2 * row), "r"(uv), "r"(e) : "memory");
    for (int r = 0; r < n_peers; r++)                                                                     // posted stores over NVLink
        asm volatile("st.relaxed.sys.global.v2.u32 [%0], {%1, %2};" ::"l"(peers[r] + 2 * row), "r"(uv), "r"(e) : "memory");
}
__device__ __forceinline__ float2 tk_epilogue_preload(const tk_phase &ph, int seg, int u, int n_past) {
    const fl_mv_args &A = ph.a;
    if (ph.swiglu) return make_float2(0.f, 0.f);
    const int r2 = 2 * u;
    if (A.epi == FL_EPI_QKV) {
        if (seg < 2) return __ldg((const float2 *)A.rope_cs + (size_t)n_past * (A.head_dim >> 1) + ((r2 % A.head_dim) >> 1));
        return make_float2(0.f, 0.f);
    }
    if (A.epi == FL_EPI_RESADD) {
        if (A.res_ll) {                                   // {value, epoch} words; the vector was polled completely by an earlier step of this CTA
            const float4 t = __ldcg((const float4 *)(A.res + 2 * r2));
            return make_float2(t.x, t.z);
        }
        return __ldcg((const float2 *)(A.res + r2));
    }
    return make_float2(0.f, 0.f);
}
__device__ __forceinline__ void tk_epilogue(const tk_phase &ph, int seg, int u, float a, float b, int n_past, float2 pre, unsigned ll_epoch) {
    const fl_mv_args &A = ph.a;
    if (ph.swiglu) {
        const uint16_t h = __half_as_ushort(__float2half_rn(a));
        const float o = __fmul_rn(__half2float(__ushort_as_half(__ldg(A.silu_tab + h))), b);
        if (A.out_ll) tk_store_ll(A.seg_dst[0], u, o, ll_epoch, A.dst_peer, A.n_dst_peer);
        else A.seg_dst[0][u] = o;
        return;
    }
    const int r2 = 2 * u;
    if (A.epi == FL_EPI_QKV) {
        if (seg < 2) {
            const float2 cs = pre;
            const float y0 = __fmaf_rn(a, cs.x, -__fmul_rn(b, cs.y));
            const float y1 = __fmaf_rn(a, cs.y, __fmul_rn(b, cs.x));
            float *o = (seg == 0) ? (A.seg_dst[0] + r2) : (A.kcache + (size_t)n_past * A.n_embd + r2);
            *(float2 *)o = make_float2(y0, y1);
        } else {
            A.vcache[(size_t)r2 * A.n_ctx + n_past] = a;
            A.vcache[(size_t)(r2 + 1) * A.n_ctx + n_past] = b;
        }
        return;
    }
    if (A.epi == FL_EPI_RESADD) {
        a = __fadd_rn(a, pre.x);
        b = __fadd_rn(b, pre.y);
    }
    if (A.out_ll) {
        // every value travels with the epoch in one 8-byte word; seg_dst[0] and dst_peer[] are LL vectors (8 bytes per row)
        tk_store_ll(A.seg_dst[seg], r2, a, ll_epoch, A.dst_peer, A.n_dst_peer);
        tk_store_ll(A.seg_dst[seg], r2 + 1, b, ll_epoch, A.dst_peer, A.n_dst_peer);
        return;
    }
    *(float2 *)(A.seg_dst[seg] + r2) = make_float2(a, b);
}

// ---- the tile stream of a tile group --------------------------------------------------------------
// Tasks (4 units = 8 rows; tk_tile_of) of a phase are dealt to the tile groups round robin, continuing where the previous phase
// stopped (T0), and inside a group to its four consumer warps: the group's k-th task goes to warp k % 4.  The group's tiles are
// streamed round by round (a round = up to four tasks, one per warp), chunk by chunk, warp by warp, so the four warps advance
// through K together.  Producer and consumers enumerate the same sequence from the same closed forms; position idx of the group's
// stream (counted over the whole launch) lives in slot 4 * (idx % Sg) + g with parity (idx / Sg) & 1.
struct tk_stream {
    int first, n_g;              // first task of this group in the phase, number of its tasks
};
__device__ __forceinline__ tk_stream tk_stream_of(int g, int T0, int ntasks) {
    tk_stream st;
    st.first = ((g - (T0 & 3)) + 4) & 3;
    st.n_g = st.first < ntasks ? (ntasks - st.first + 3) >> 2 : 0;
    return st;
}
__device__ __forceinline__ void tk_slot_of(const tk_params &prm, int g, uint32_t idx, int &s, uint32_t &par) {
    const uint32_t q = tk_div(idx, prm.s_magic, prm.s_shift);          // idx / Sg
    s = (int)(idx - q * (uint32_t)prm.Sg) * TK_TG + g;
    par = q & 1u;
}

// ---- main loop of a matvec phase for one consumer warp ------------------------------------------------
__device__ __forceinline__ unsigned tk_clock() {
    unsigned c;
    asm volatile("mov.u32 %0, %%clock;" : "=r"(c));
    return c;
}
template <int TYPE, bool PROF>
__device__ __forceinline__ void tk_consume(const tk_phase &ph, const tk_params &prm, const tk_slice &sl, int T0, uint32_t &cg, const tk_yblock *ysm,
                                           uint8_t *stage0, volatile uint32_t *tags, uint32_t bar0, int warp, int lane, unsigned *pw, unsigned lle) {
    unsigned c_begin = 0, c_wait = 0, c_dot = 0, c_tail = 0, c_rounds = 0, c_t = 0;
    if (PROF) { c_begin = tk_clock(); c_t = c_begin; }
    constexpr int BB = (TYPE == FL_TYPE_Q4_0) ? 20 : 24, QOFF = (TYPE == FL_TYPE_Q4_0) ? 4 : 8;
    const fl_mv_args &A = ph.a;
    const int S = prm.S;
    // group g = warp % 4: its four warps (g, g + 4, g + 8, g + 12) share one SM sub-partition, and a phase with few tasks (wo, w2: four per
    // CTA, one per group, all on warp-of-group 0) runs on warps 0 .. 3, i.e. on four DIFFERENT sub-partitions.  (warp / 4 put those four
    // chains on one scheduler: w2's tile loop measured 17.7 us instead of ~5.)
    const int g = warp % TK_TG, wl = warp / TK_TG;
    const int r = lane >> 2, jj = lane & 3;
    const bool swiglu = ph.swiglu != 0;
    const int C = ph.nchunks, nb = ph.nb;
    const tk_stream st = tk_stream_of(g, T0, sl.ntiles);
    const int n_past = (A.epi == FL_EPI_QKV) ? *A.n_past : 0;
    // the lane that runs the epilogue of pair p: default rows (2p, 2p+1) -> lane 8p; swiglu rows (p, p + 4) -> lane 4p
    const bool leader = swiglu ? ((lane & 3) == 0 && lane < 16) : ((lane & 7) == 0);
    const int pr = swiglu ? (lane >> 2) : (lane >> 3);
    const uint32_t row_off = (uint32_t)r * ph.srow + (uint32_t)(QOFF + 4 * jj);
    for (int k = wl; k < st.n_g; k += TK_WPG) {
        const int k0 = k - wl, n_r = min(TK_WPG, st.n_g - k0);
        int seg, unit0, nunits;
        tk_tile_of(sl, TK_GMAX, st.first + 4 * k, seg, unit0, nunits);
        float2 pre = make_float2(0.f, 0.f);
        if (leader && pr < nunits) pre = tk_epilogue_preload(ph, seg, unit0 + pr, n_past);
        float a0 = 0.0f, a1 = 0.0f, sm = 0.0f;
        for (int c = 0; c < C; c++) {
            int s;
            uint32_t par;
            const uint32_t idx = cg + (uint32_t)(k0 * C + c * n_r + wl);
            tk_slot_of(prm, g, idx, s, par);
            // A parity wait is only meaningful once the slot's PREVIOUS tile has completed its phase: the slots of a group are shared by
            // its four warps, so the previous tenant may be another warp's tile that has not even been issued yet -- and a parity wait
            // answers "done" for a phase two ahead (seen with shallow rings: garbage tiles, launch failures).  The producer
            // tags the slot with the stream position once it owns it again (the previous tenant was consumed), then the wait is exact.
            tk_tag_wait(tags + s, idx + 1u, prm.err, 0x600u + (unsigned)warp, (unsigned)s);
            tk_mbar_wait(bar0 + 8u * s, par, prm.err, 0x400u + (unsigned)warp, (unsigned)s);
            if (PROF) { const unsigned t = tk_clock(); c_wait += t - c_t; c_t = t; c_rounds++; }
            if (!(prm.diag & 2)) {
                const uint8_t *wp = stage0 + (size_t)s * prm.slot_bytes + row_off;
                const tk_yblock *yp = ysm + c * TK_CHB;
                const int nbc = min(TK_CHB, nb - c * TK_CHB);
#pragma unroll 8
                for (int i = 0; i < nbc; i++) {
                    const uint32_t w = *(const uint32_t *)(wp + i * BB);
                    const float dx = *(const float *)(wp + i * BB - (QOFF + 4 * jj));
                    const uint4 y = *(const uint4 *)yp[i].q[jj];
                    const float2 ds = *(const float2 *)&yp[i].d;
                    if (TYPE == FL_TYPE_Q4_1) sm = __fmaf_rn(*(const float *)(wp + i * BB - (QOFF + 4 * jj) + 4), ds.y, sm);
                    fx_block(w, __fmul_rn(dx, ds.x), y, a0, a1);
                }
            }
            // the tile has been read (the chains above consumed every shared load of the warp): hand the slot back
            __syncwarp();
            if (lane == 0) fl_mbar_arrive(bar0 + 8u * (S + s));
            if (PROF) { const unsigned t = tk_clock(); c_dot += t - c_t; c_t = t; }
        }
        float tot = fx_reduce(a0, a1);                                  // valid in lane 4r
        if (TYPE == FL_TYPE_Q4_1) tot = __fadd_rn(tot, sm);
        const float other = __shfl_down_sync(0xffffffffu, tot, swiglu ? 16 : 4);
        if (leader && pr < nunits) tk_epilogue(ph, seg, unit0 + pr, tot, other, n_past, pre, lle);
        if (PROF) { const unsigned t = tk_clock(); c_tail += t - c_t; c_t = t; }
    }
    cg += (uint32_t)(st.n_g * C);
    if (PROF && lane == 0 && pw) {
        pw[0] = 0; pw[1] = c_wait; pw[2] = c_dot; pw[3] = c_tail; pw[4] = c_rounds; pw[5] = tk_clock() - c_begin; pw[6] = (unsigned)sl.ntiles; pw[7] = 0;
    }
}

// ---- attention phase: one head, all consumer threads of the CTA ------------------------------------
__device__ __forceinline__ void tk_attention(const tk_phase &ph, const tk_params &prm, float *sc, double *red, int head, int part_id, int warp, int lane, int tid, unsigned lle_out) {
    float *redf = (float *)(red + 20);                // [16] floats; red[0..16] are the double partials
    const int hd = ph.head_dim;
    const int n_pos = *ph.a.n_past + 1;
    const float *q = ph.q + (size_t)head * hd;
    const float *kbase = ph.kcache + (size_t)head * hd;
    if (hd == 128) {                                  // 8 positions per warp pass, all 36 loads of a lane in flight at once
        float qe[4];
#pragma unroll
        for (int c = 0; c < 4; c++) qe[c] = __ldcg(q + lane + 32 * c);
        for (int j0 = warp * 8; j0 < n_pos; j0 += TK_CW * 8) {
            float kv[8][4], acc[8];
#pragma unroll
            for (int u = 0; u < 8; u++)
#pragma unroll
                for (int c = 0; c < 4; c++) kv[u][c] = __ldcg(kbase + (size_t)min(j0 + u, n_pos - 1) * ph.k_row_stride + lane + 32 * c);
#pragma unroll
            for (int u = 0; u < 8; u++) {
                acc[u] = 0.f;
#pragma unroll
                for (int c = 0; c < 4; c++) acc[u] = __fmaf_rn(kv[u][c], qe[c], acc[u]);
            }
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const float a = fx_reduce_f32(acc[u]);             // ggml_vec_dot_f32's order: lane l = element l of its 32-float step
                if (lane == 0 && j0 + u < n_pos) sc[j0 + u] = __fmul_rn(a, ph.scale);
            }
        }
    } else {
        for (int j0 = warp * 4; j0 < n_pos; j0 += TK_CW * 4) {
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
            for (int e = lane; e < hd; e += 32) {
                const float qe = __ldcg(q + e);
#pragma unroll
                for (int u = 0; u < 4; u++) acc[u] = __fmaf_rn(__ldcg(kbase + (size_t)min(j0 + u, n_pos - 1) * ph.k_row_stride + e), qe, acc[u]);
            }
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const float a = fx_reduce_f32(acc[u]);
                if (lane == 0 && j0 + u < n_pos) sc[j0 + u] = __fmul_rn(a, ph.scale);
            }
        }
    }
    tk_bar_consumers(12);
    float mx = -INFINITY;
    for (int j = tid; j < n_pos; j += TK_NT) mx = fmaxf(mx, sc[j]);
    mx = fl_warp_max(mx);
    if (lane == 0) redf[warp] = mx;
    tk_bar_consumers(12);
    mx = redf[0];
    for (int w = 1; w < TK_CW; w++) mx = fmaxf(mx, redf[w]);
    double sum = 0.0;
    for (int j = tid; j < n_pos; j += TK_NT) {
        const uint16_t hh = __half_as_ushort(__float2half_rn(__fsub_rn(sc[j], mx)));
        const float e = __half2float(__ushort_as_half(__ldg(prm.exp_tab + hh)));
        sc[j] = e;
        sum += (double)e;
    }
    sum = fl_warp_sum_d(sum);
    if (lane == 0) red[warp] = sum;
    tk_bar_consumers(12);
    double tot = 0.0;
    for (int w = 0; w < TK_CW; w++) tot += red[w];
    const float inv = (float)(1.0 / tot);
    // each thread normalises exactly the entries it wrote above, so no barrier is needed in between
    for (int j = tid; j < n_pos; j += TK_NT) sc[j] = __fmul_rn(sc[j], inv);
    tk_bar_consumers(12);
    // P*V, one warp per output dimension, in ggml_vec_dot_f32's order (src0 row = the dimension's cached values over the positions,
    // src1 row = the probabilities): 32-float steps into lane-wise accumulators, the reference's reduction tree, then the
    // n_pos % 32 leftovers one by one (fx_left_nma).  This CTA owns dpc = head_dim / head_split dimensions.
    const int dpc = hd / ph.head_split;
    const int np = n_pos & ~31, rem = n_pos - np, nma = fx_left_nma(rem);
    for (int dl = warp; dl < dpc; dl += TK_CW) {
        const int d = part_id * dpc + dl;
        const float *vrow = ph.vcache + ((size_t)head * hd + d) * ph.n_ctx;
        float acc = 0.0f;
        const float lx = (lane < rem) ? __ldcg(vrow + np + lane) : 0.0f, ly = (lane < rem) ? sc[np + lane] : 0.0f;
        const float lv = __fmul_rn(lx, ly);
        for (int k = lane; k < np; k += 32) acc = __fmaf_rn(__ldcg(vrow + k), sc[k], acc);
        float o = fx_reduce_f32(acc);
        for (int k = 0; k < nma; k++) o = __fadd_rn(o, __shfl_sync(0xffffffffu, lv, k));
        for (int k = nma; k < rem; k++) o = __fmaf_rn(__shfl_sync(0xffffffffu, lx, k), __shfl_sync(0xffffffffu, ly, k), o);
        if (lane == 0) {
            if (ph.out_ll) tk_store_ll(ph.out, head * hd + d, o, lle_out, ph.out_peer, ph.n_out_peer);
            else ph.out[(size_t)head * hd + d] = o;
        }
    }
}
// pull the cached positions of this head (all < n_past: the token's own row is stored in wq|wk|wv) towards L2.  The producer warps
// (threads tid of nt) issue it when their walk reaches the attention, which is while the consumers still run wq|wk|wv: the transfer
// then overlaps that phase's tile loop instead of the grid barrier in front of the attention (issued right before that barrier, it
// made the barrier grow with n_past: 6.0 us at n_past 128, 9.7 us at 400 per layer on 7B).  Not inlined: inside the producer loop
// (64 registers after setmaxnreg) it made ptxas spill.
__device__ __noinline__ void tk_attention_prefetch(const tk_phase &ph, int head, int part_id, int tid, int nt) {
    const int hd = ph.head_dim, n_past = *ph.a.n_past;
    for (int j = tid; j < n_past; j += nt)                                // cached K rows of the head: hd floats each
        for (int l = 0; l < hd; l += 32) asm volatile("prefetch.global.L2 [%0];" ::"l"(ph.kcache + (size_t)j * ph.k_row_stride + (size_t)head * hd + l));
    const int dpc = hd / ph.head_split;
    const float *v0 = ph.vcache + ((size_t)head * hd + (size_t)part_id * dpc) * ph.n_ctx;
    for (int dl = 0; dl < dpc; dl++)                                      // cached V rows of this CTA's dimensions: n_past floats each
        for (int l = 32 * tid; l < n_past; l += 32 * nt) asm volatile("prefetch.global.L2 [%0];" ::"l"(v0 + (size_t)dl * ph.n_ctx + l));
}

template <bool PROF>
__global__ void __launch_bounds__(TK_THREADS, 1) k_decode_token(const tk_params prm) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t *bars = (uint64_t *)smem;
    volatile uint32_t *tags = (volatile uint32_t *)(smem + (size_t)16 * prm.S);     // behind the 2 * S mbarriers: which tile of its group's stream a slot holds
    tk_yblock *ysm = (tk_yblock *)(smem + prm.off_y);
    double *red = (double *)(smem + prm.off_red);            // 32 doubles
    float *sc = (float *)(smem + prm.off_sc);                // attention: [n_ctx] + [256]
    uint8_t *stage0 = smem + prm.off_stage0;
    // Phase descriptors are read from shared memory: every gpu-scope acquire invalidates L1, so reading them from
    // global would put a chain of L2 round trips right behind each grid barrier.  Descriptor pi+1 is copied in
    // by warp 15 while phase pi runs and becomes visible through the next barrier's bar.sync.
    __shared__ __align__(16) tk_phase phs[2];
    __shared__ tk_slice sl_sh;                                // this CTA's slice of the current phase (computed once, read by all)
    const int S = prm.S;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t bar0 = fl_smem_u32(bars);

    if (warp >= TK_CW) {
        // ------------------------------ producers: warp TK_CW + g streams the tiles of tile group g, all phases, as far ahead as its slots allow ------
        // One producer per tile group: the groups drift apart by a tile or two (epilogues differ), and a single in-order producer
        // made every group wait for the slowest one's slot.
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(TK_REGS_PRODUCER));
        const int pg = warp - TK_CW;
        if (pg == 0 && lane == 0) {
            for (int s = 0; s < S; s++) {
                fl_mbar_init(bar0 + 8u * s, 1);                  // full: the producer's expect_tx arrival + the copies' bytes
                fl_mbar_init(bar0 + 8u * (S + s), 1);            // empty: the one consumer warp that owns the tile
                tags[s] = 0u;
            }
            fl_mbar_fence_init();
        }
        __syncwarp();
        asm volatile("bar.sync 14, %0;" ::"r"(TK_THREADS) : "memory");          // barriers initialised (consumers and the other producers wait here too)
        {
            // All 32 lanes walk the stream; lane 0 waits for the slot and posts the byte count, lanes 0-7 issue one row piece each.
            const uint64_t pol = fl_policy_evict_first();
            int T0 = 0;                                                          // tasks of all earlier phases (this CTA): rotates the groups
            uint32_t cg = 0;                                                     // tiles of all earlier phases in this group's stream
            for (int pi = 0; pi < prm.n_phases; pi++) {
                // The descriptor lives in global memory; everything the tile loop needs is pulled into registers once per phase
                // (one L2 round trip, hidden because the producer runs ahead).
                const tk_phase *gp = prm.phases + pi;
                if (__ldg(&gp->kind) != TK_PH_MATVEC) {                      // attention: its KV rows towards L2 (tk_attention_prefetch)
                    const int hs = __ldg(&gp->head_split);
                    if ((int)blockIdx.x < __ldg(&gp->n_head) * hs)
                        tk_attention_prefetch(*gp, (int)blockIdx.x / hs, (int)blockIdx.x % hs, pg * 32 + lane, 32 * TK_PW);
                    continue;
                }
                const int swiglu = __ldg(&gp->swiglu), C = __ldg(&gp->nchunks), nb = __ldg(&gp->nb), type = __ldg(&gp->a.type);
                const int m0 = __ldg(&gp->units[0]), m1 = __ldg(&gp->units[1]), m2 = __ldg(&gp->units[2]);
                const uint32_t row_bytes = __ldg(&gp->row_bytes), srow = __ldg(&gp->srow);
                const uint32_t bb = (type == FL_TYPE_Q4_0) ? 20u : 24u;
                const uint8_t *w0 = (const uint8_t *)__ldg((const unsigned long long *)&gp->a.seg_w[0]);
                const uint8_t *w1 = (const uint8_t *)__ldg((const unsigned long long *)&gp->a.seg_w[1]);
                const uint8_t *w2 = (const uint8_t *)__ldg((const unsigned long long *)&gp->a.seg_w[2]);
                const tk_slice sl = tk_make_slice_u(m0, m1, m2, 2, prm.grid_magic, prm.grid_shift);
                const tk_stream st = tk_stream_of(pg, T0, sl.ntiles);
                for (int k0 = 0; k0 < st.n_g; k0 += TK_WPG) {
                    const int n_r = min(TK_WPG, st.n_g - k0);
                    for (int c = 0; c < C; c++) {
                        const uint32_t cbytes = (uint32_t)min(TK_CHB, nb - c * TK_CHB) * bb;
                        for (int wl = 0; wl < n_r; wl++) {
                            int seg, unit0, nunits;
                            tk_tile_of(sl, TK_GMAX, st.first + 4 * (k0 + wl), seg, unit0, nunits);
                            int s;
                            uint32_t par;
                            const uint32_t idx = cg + (uint32_t)(k0 * C + c * n_r + wl);
                            tk_slot_of(prm, pg, idx, s, par);
                            // row piece of this lane: default rows 2*unit0 .. 2*unit0 + 2*nunits - 1 of the segment's matrix;
                            // swiglu: lanes 0-3 rows unit0.. of w1, lanes 4-7 the same rows of w3
                            const uint8_t *src = nullptr;
                            if (lane < 8) {
                                if (swiglu) { if ((lane & 3) < nunits) src = ((lane < 4) ? w0 : w1) + (size_t)(unit0 + (lane & 3)) * row_bytes; }
                                else if (lane < 2 * nunits) src = (seg == 0 ? w0 : seg == 1 ? w1 : w2) + (size_t)(2 * unit0 + lane) * row_bytes;
                            }
                            if (lane == 0) {
                                tk_mbar_wait(bar0 + 8u * (S + s), par ^ 1u, prm.err, 0x500u + (unsigned)pg, (unsigned)s);
                                tags[s] = idx + 1u;                  // the slot is ours again: consumers may now wait for this tile's phase
                                if (prm.diag & 1) fl_mbar_arrive(bar0 + 8u * s);
                                else fl_mbar_expect_tx(bar0 + 8u * s, 2u * (uint32_t)nunits * cbytes);
                            }
                            __syncwarp();
                            if (src && !(prm.diag & 1))
                                fl_bulk_g2s_hint(fl_smem_u32(stage0 + (size_t)s * prm.slot_bytes + (size_t)lane * srow), src + (size_t)c * (TK_CHB * bb), cbytes, bar0 + 8u * s, pol);
                        }
                    }
                }
                cg += (uint32_t)(st.n_g * C);
                T0 += sl.ntiles;
            }
        }
        return;
    }

    // ------------------------------ consumers ------------------------------
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(TK_REGS_CONSUMER));
    const int tid = threadIdx.x;
    static_assert(sizeof(tk_phase) % 4 == 0 && sizeof(tk_phase) / 4 <= TK_NT, "descriptor copy is one word per thread");
    if (warp == TK_CW - 1)
        for (int i = lane; i < (int)(sizeof(tk_phase) / 4); i += 32) ((uint32_t *)&phs[0])[i] = ((const uint32_t *)&prm.phases[0])[i];
    tk_bar_consumers(15);
    asm volatile("bar.sync 14, %0;" ::"r"(TK_THREADS) : "memory");     // mbarriers initialised
    int T0 = 0;
    uint32_t cg = 0;                                         // tiles of all earlier phases in this warp's group's stream
    unsigned epoch = 0;
    // LL vectors: every element carries (number of LL exchanges before this launch) + (index inside the launch) + 1.  The running count
    // lives next to the vectors (fl_token_plan_create_ll), so words left behind by earlier launches or plans never satisfy a later poll.
    unsigned ll_base = 0;
    if (prm.n_ll > 0) asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(ll_base) : "l"(prm.ll_count) : "memory");
    unsigned *err = prm.err;
    for (int pi = 0; pi < prm.n_phases; pi++) {
        const tk_phase &ph = phs[pi & 1];
        unsigned long long *pr = (prm.prof && tid == 0) ? prm.prof + ((size_t)pi * gridDim.x + blockIdx.x) * 4 : nullptr;
        if (pr) pr[0] = tk_now();
        // attention: CTA b works on head b / head_split, output dimensions part b % head_split
        const bool attn_here = ph.kind == TK_PH_ATTN && (int)blockIdx.x < ph.n_head * ph.head_split;
        const int a_head = attn_here ? (int)blockIdx.x / ph.head_split : 0, a_part = attn_here ? (int)blockIdx.x % ph.head_split : 0;
        const bool ll_in = ph.kind == TK_PH_MATVEC && ph.a.x_ll;      // input arrives element by element with epochs: no grid barrier at all
        const unsigned lle_in = ll_in ? ll_base + (unsigned)ph.a.x_seq + 1u : 0u;
        const unsigned lle_out = ph.kind == TK_PH_MATVEC ? (ph.a.out_ll ? ll_base + (unsigned)ph.a.out_seq + 1u : 0u) : (ph.out_ll ? ll_base + (unsigned)ph.out_seq + 1u : 0u);
        if (pi > 0 && ll_in) {
            tk_bar_consumers(13);                                // only this CTA's warps: the previous phase's tiles have been consumed
        } else if (pi > 0) {
            epoch++;
            if (!(prm.diag & 4)) tk_grid_sync(prm, epoch * gridDim.x, 0u);   // results of phase pi-1 are visible everywhere
            else tk_bar_consumers(13);           // still a CTA barrier: sl_sh and phs[] are rewritten below while slower warps may read them
        }
        if (pr) pr[1] = tk_now();
        // Descriptor pi+1: the load is issued now, the store into phs[(pi+1)&1] (which nobody reads any more: everybody is
        // past the barrier) happens after this phase's prologue, so its L2 latency hides behind the prologue's own loads.
        uint32_t next_word = 0;
        const bool copies = tid < (int)(sizeof(tk_phase) / 4) && pi + 1 < prm.n_phases;
        if (copies) next_word = __ldcg((const uint32_t *)&prm.phases[pi + 1] + tid);
        if (ph.kind == TK_PH_ATTN) {
            if (attn_here && !(prm.diag & 16)) tk_attention(ph, prm, sc, red, a_head, a_part, warp, lane, tid, lle_out);
            if (copies) ((uint32_t *)&phs[(pi + 1) & 1])[tid] = next_word;
            tk_bar_consumers(15);                                // the next iteration reads the new descriptor before its grid barrier
            if (pr) pr[2] = pr[3] = tk_now();
            continue;
        }
        const int K = ph.nb * 32;
        if (tid == TK_NT - 1) sl_sh = tk_make_slice_u(ph.units[0], ph.units[1], ph.units[2], 2, prm.grid_magic, prm.grid_shift);
        if (!(prm.diag & 8)) tk_prologue(ph.a, K, ysm, red, warp, lane, tid, lle_in, err);
        if (copies) ((uint32_t *)&phs[(pi + 1) & 1])[tid] = next_word;
        tk_bar_consumers(15);                                    // activations, slice and next descriptor are in shared memory
        if (pr) pr[2] = tk_now();
        const tk_slice &sl = sl_sh;
        unsigned *pw = (PROF && prm.prof2) ? prm.prof2 + (((size_t)pi * gridDim.x + blockIdx.x) * TK_CW + warp) * 8 : nullptr;
        if (ph.a.type == FL_TYPE_Q4_0) tk_consume<FL_TYPE_Q4_0, PROF>(ph, prm, sl, T0, cg, ysm, stage0, tags, bar0, warp, lane, pw, lle_out);
        else                           tk_consume<FL_TYPE_Q4_1, PROF>(ph, prm, sl, T0, cg, ysm, stage0, tags, bar0, warp, lane, pw, lle_out);
        T0 += sl.ntiles;
        if (pr) pr[3] = tk_now();
    }
    if (prm.n_ll > 0 && blockIdx.x == 0 && tid == 0) *prm.ll_count = ll_base + (unsigned)prm.n_ll;     // the next launch continues from here
}

// =================================================================================================
// host side
// =================================================================================================
struct fl_token_plan_impl {
    tk_phase *d_phases = nullptr;
    unsigned *d_bar = nullptr;
    unsigned *h_err = nullptr;
    unsigned long long *d_prof = nullptr;
    unsigned *d_prof2 = nullptr;
    tk_params prm;
    size_t smem = 0;
    int n_kernels = 0;
};

// n / d for n < 2^31 as umulhi(n, magic) >> shift: with 2^k < d < 2^(k+1), magic = ceil(2^(32+k) / d) < 2^32
static void tk_magic(uint32_t d, uint32_t &magic, uint32_t &shift) {
    uint32_t k = 0;
    while ((2u << k) <= d) k++;                 // k = floor(log2 d)
    shift = k;
    magic = ((d & (d - 1)) == 0) ? 0u : (uint32_t)((((uint64_t)1 << (32 + k)) + d - 1) / d);
}

static int tk_geometry(tk_phase &ph, size_t &tile_bytes) {
    const fl_mv_args &a = ph.a;
    const int bb = fl_block_bytes(a.type);
    const int nb = a.K / 32;
    const size_t row_bytes = a.row_stride_bytes ? a.row_stride_bytes : (size_t)nb * bb;
    FL_REQUIRE(bb > 0 && a.K > 0 && a.K % 32 == 0 && row_bytes % 16 == 0, "token kernel: unsupported matrix K=%d", a.K);
    // the 32 lanes of a warp (8 rows x 4 lanes) hit 32 different banks when the row pitch is an odd multiple of 16 bytes
    const uint32_t chunk_bytes = (uint32_t)std::min(nb, TK_CHB) * bb;
    FL_REQUIRE(chunk_bytes % 16 == 0 && ((size_t)nb * bb) % 16 == 0, "token kernel: K=%d gives row pieces that are not multiples of 16 bytes", a.K);
    const uint32_t srow = (chunk_bytes / 16) % 2 ? chunk_bytes : chunk_bytes + 16;
    ph.units[0] = ph.units[1] = ph.units[2] = 0;
    if (ph.swiglu) {
        ph.units[0] = a.seg_rows[0];
    } else {
        for (int i = 0; i < a.nseg; i++) {
            FL_REQUIRE(a.seg_rows[i] > 0 && a.seg_rows[i] % 2 == 0, "token kernel: segment %d has an odd row count", i);
            ph.units[i] = a.seg_rows[i] / 2;
        }
    }
    for (int i = 0; i < a.nseg; i++) {
        FL_REQUIRE(((uintptr_t)a.seg_w[i] & 15) == 0, "token kernel: segment %d is not 16-byte aligned", i);
        FL_REQUIRE(a.epi == FL_EPI_QKV || ph.swiglu || ((uintptr_t)a.seg_dst[i] & 7) == 0, "token kernel: output %d is not 8-byte aligned", i);
    }
    FL_REQUIRE(a.epi != FL_EPI_RESADD || ((uintptr_t)a.res & 7) == 0, "token kernel: residual is not 8-byte aligned");
    FL_REQUIRE((long)ph.units[0] + ph.units[1] + ph.units[2] < (1 << 23), "token kernel: too many rows");
    ph.kind = TK_PH_MATVEC;
    ph.nb = nb; ph.nchunks = (nb + TK_CHB - 1) / TK_CHB; ph.srow = srow; ph.row_bytes = (uint32_t)row_bytes;
    tile_bytes = (size_t)2 * TK_GMAX * srow;
    return 0;
}

int flk_token_plan_create(const fl_token_step *steps, int n_steps, const uint16_t *silu_tab, const uint16_t *exp_tab, const void *rope_cs, unsigned *epoch_counter, void **out) {
    std::vector<tk_phase> phases((size_t)n_steps);
    for (int i = 0; i < n_steps; i++) {
        tk_phase &ph = phases[i];
        memset(&ph, 0, sizeof(ph));
        if (steps[i].kind == 1) {
            ph.kind = TK_PH_ATTN;
            ph.q = steps[i].q; ph.kcache = steps[i].kcache; ph.vcache = steps[i].vcache; ph.out = steps[i].out;
            ph.k_row_stride = steps[i].k_row_stride; ph.n_head = steps[i].n_head; ph.head_dim = steps[i].head_dim; ph.n_ctx = steps[i].n_ctx;
            ph.scale = steps[i].scale;
            ph.a.n_past = steps[i].n_past;
            ph.out_ll = steps[i].out_ll; ph.out_seq = steps[i].out_seq; ph.n_out_peer = steps[i].n_out_peer;
            for (int r = 0; r < 7; r++) ph.out_peer[r] = steps[i].out_peer[r];
        } else {
            ph.kind = TK_PH_MATVEC;
            ph.a = steps[i].mv;
            ph.a.silu_tab = silu_tab;
            ph.a.rope_cs = rope_cs;
        }
    }
    // w1|w3 followed by a silu(.)*(.) prologue over exactly their outputs: fuse the activation into the first phase (dataflow plans ask for it)
    for (int i = 0; i < n_steps; i++)
        if (phases[i].kind == TK_PH_MATVEC && phases[i].a.swiglu) {
            const fl_mv_args &a = phases[i].a;
            FL_REQUIRE(a.nseg == 2 && a.epi == FL_EPI_STORE && a.seg_rows[0] == a.seg_rows[1], "token kernel: a swiglu step needs two equal segments and a plain store");
            phases[i].swiglu = 1;
        }
    for (int i = 0; i + 1 < n_steps; i++) {
        tk_phase &p0 = phases[i], &p1 = phases[i + 1];
        if (p0.kind != TK_PH_MATVEC || p1.kind != TK_PH_MATVEC || p0.swiglu) continue;
        const fl_mv_args &a = p0.a;
        if (a.nseg == 2 && a.epi == FL_EPI_STORE && a.seg_rows[0] == a.seg_rows[1] && p1.a.pro == FL_PRO_SILUMUL && p1.a.x == a.seg_dst[0] &&
            p1.a.b == a.seg_dst[1] && p1.a.K == a.seg_rows[0] && p1.a.xadd == nullptr) {
            p0.swiglu = 1;
            p1.a.pro = FL_PRO_PLAIN;            // reads silu(w1 x) * (w3 x) from seg_dst[0]
            p1.a.b = nullptr;
        }
    }
    size_t max_tile = 0, max_y = 0;
    int max_ctx = 0;
    int sm_count = 0;
    {
        int dev0 = 0;
        FL_CUDA_OK(cudaGetDevice(&dev0));
        FL_CUDA_OK(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev0));
    }
    for (int i = 0; i < n_steps; i++) {
        tk_phase &ph = phases[i];
        if (ph.kind == TK_PH_ATTN) {
            FL_REQUIRE(ph.n_ctx % 4 == 0 && ph.head_dim >= 32 && ph.head_dim <= 256 && (ph.head_dim & (ph.head_dim - 1)) == 0 && ph.n_head <= sm_count,
                       "token kernel: unsupported attention shape");
            ph.head_split = 1;
            for (int c = 4; c > 1; c /= 2)
                if (c * ph.n_head <= sm_count && ph.head_dim / c >= 32) { ph.head_split = c; break; }
            max_ctx = std::max(max_ctx, ph.n_ctx);
        } else {
            size_t tb = 0;
            if (tk_geometry(ph, tb)) return -1;
            max_tile = std::max(max_tile, tb);
            max_y = std::max(max_y, (size_t)ph.nb * sizeof(tk_yblock));
        }
    }
    int dev = 0, sm = 0, optin = 0;
    FL_CUDA_OK(cudaGetDevice(&dev));
    FL_CUDA_OK(cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, dev));
    FL_CUDA_OK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    fl_token_plan_impl *pl = new fl_token_plan_impl();
    struct plan_guard {                               // every error return below frees what has been allocated so far
        fl_token_plan_impl *p;
        ~plan_guard() { if (p) flk_token_plan_destroy(p); }
    } guard{pl};
    tk_params &p = pl->prm;
    const size_t slot = (max_tile + 127) & ~(size_t)127;
    int S = 64;
    if (getenv("FASTLLAMA_B200_TK_SLOTS")) S = std::max(8, std::min(64, atoi(getenv("FASTLLAMA_B200_TK_SLOTS")) / 4 * 4));      // testing aid: a shallower ring
    size_t off = 0;
    for (;; S -= 4) {
        if (S < 8) { fl_set_error("token kernel: tiles of %zu bytes do not fit shared memory", slot); return -1; }
        p.off_y = ((size_t)(2 * S) * 8 + (size_t)S * 4 + 127) & ~(size_t)127;          // 2 * S mbarriers, S slot tags
        p.off_red = (p.off_y + max_y + 127) & ~(size_t)127;
        p.off_sc = (p.off_red + 32 * sizeof(double) + 127) & ~(size_t)127;
        off = (p.off_sc + ((size_t)max_ctx + 32) * sizeof(float) + 127) & ~(size_t)127;
        if (off + (size_t)S * slot <= (size_t)optin - 1024) break;
    }
    p.off_rowbuf = p.off_cnt = 0;
    p.off_stage0 = (uint32_t)off;
    p.S = S;
    p.Sg = S / TK_TG;
    tk_magic((uint32_t)sm, p.grid_magic, p.grid_shift);
    tk_magic((uint32_t)p.Sg, p.s_magic, p.s_shift);
    p.slot_bytes = (uint32_t)slot;
    p.n_phases = n_steps;
    p.exp_tab = exp_tab;
    p.diag = getenv("FASTLLAMA_B200_TK_DIAG") ? atoi(getenv("FASTLLAMA_B200_TK_DIAG")) : 0;
    pl->smem = off + (size_t)S * slot;
    FL_CUDA_OK(cudaMalloc((void **)&pl->d_phases, sizeof(tk_phase) * (size_t)n_steps));
    FL_CUDA_OK(cudaMemcpy(pl->d_phases, phases.data(), sizeof(tk_phase) * (size_t)n_steps, cudaMemcpyHostToDevice));
    FL_CUDA_OK(cudaMalloc((void **)&pl->d_bar, 256));
    p.phases = pl->d_phases;
    p.grid_bar = pl->d_bar;
    FL_CUDA_OK(cudaMemset(pl->d_bar, 0, 256));
    FL_CUDA_OK(cudaHostAlloc((void **)&pl->h_err, 64, cudaHostAllocMapped));
    memset(pl->h_err, 0, 64);
    FL_CUDA_OK(cudaHostGetDevicePointer((void **)&p.err, pl->h_err, 0));
    p.rank = 0; p.world = 1; p.ll_count = epoch_counter; p.n_ll = 0;
    for (int i = 0; i < n_steps; i++) {
        const tk_phase &ph = phases[i];
        if (ph.kind == TK_PH_MATVEC) {
            if (ph.a.out_ll) p.n_ll = std::max(p.n_ll, ph.a.out_seq + 1);
            if (ph.a.x_ll) p.n_ll = std::max(p.n_ll, ph.a.x_seq + 1);
            if (ph.a.out_ll && ph.a.nseg != 1 && !ph.swiglu) { fl_set_error("token kernel: an LL output needs a single segment (or a w1|w3 pair)"); return -1; }
        } else if (ph.out_ll) p.n_ll = std::max(p.n_ll, ph.out_seq + 1);
    }
    if (p.n_ll > 0 && !epoch_counter) { fl_set_error("token kernel: steps use LL vectors but no epoch counter was given (fl_token_plan_create_ll)"); return -1; }
    p.prof = nullptr;
    p.prof2 = nullptr;
    if (getenv("FASTLLAMA_B200_TOKEN_PROF")) {
        FL_CUDA_OK(cudaMalloc((void **)&pl->d_prof, sizeof(unsigned long long) * 4 * (size_t)n_steps * sm));
        FL_CUDA_OK(cudaMemset(pl->d_prof, 0, sizeof(unsigned long long) * 4 * (size_t)n_steps * sm));
        p.prof = pl->d_prof;
        const size_t n2 = (size_t)n_steps * sm * TK_CW * 8;
        FL_CUDA_OK(cudaMalloc((void **)&pl->d_prof2, n2 * sizeof(unsigned)));
        FL_CUDA_OK(cudaMemset(pl->d_prof2, 0, n2 * sizeof(unsigned)));
        p.prof2 = pl->d_prof2;
    }
    cudaFuncAttributes fa;
    FL_CUDA_OK(cudaFuncGetAttributes(&fa, k_decode_token<false>));
    FL_CUDA_OK(cudaFuncSetAttribute(k_decode_token<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int)fa.sharedSizeBytes));
    FL_CUDA_OK(cudaFuncGetAttributes(&fa, k_decode_token<true>));
    FL_CUDA_OK(cudaFuncSetAttribute(k_decode_token<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int)fa.sharedSizeBytes));
    // setmaxnreg re-distributes the registers the CTA was LAUNCHED with; an over-subscribed request would spin forever inside the kernel
    FL_REQUIRE((size_t)TK_REGS_CONSUMER * TK_NT + (size_t)TK_REGS_PRODUCER * 32 * TK_PW <= (size_t)fa.numRegs * TK_THREADS,
               "token kernel: register re-allocation (%d x %d + %d x %d) exceeds the launch allocation (%d x %d)", TK_REGS_CONSUMER, TK_NT, TK_REGS_PRODUCER,
               32 * TK_PW, fa.numRegs, TK_THREADS);
    int per_sm = 0;
    FL_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_decode_token<false>, TK_THREADS, pl->smem));
    if (per_sm < 1) { const size_t need = pl->smem; fl_set_error("token kernel: one CTA per SM does not fit (smem %zu)", need); return -1; }
    pl->n_kernels = sm;
    guard.p = nullptr;
    *out = pl;
    return 0;
}

int flk_token_plan_launch(cudaStream_t st, void *plan) {
    fl_token_plan_impl *pl = (fl_token_plan_impl *)plan;
    FL_CUDA_OK(cudaMemsetAsync(pl->d_bar, 0, 4, st));
    void *args[] = {(void *)&pl->prm};
    // cooperative launch: all CTAs (one per SM) are guaranteed co-resident, which the grid barrier needs
    const void *fn = pl->prm.prof2 ? (const void *)k_decode_token<true> : (const void *)k_decode_token<false>;
    FL_CUDA_OK(cudaLaunchCooperativeKernel(fn, dim3(pl->n_kernels), dim3(TK_THREADS), args, pl->smem, st));
    fl_count_launch();
    return 0;
}

// tooling: stamps of the last launch, [n_steps][n_ctas][4] nanoseconds (needs FASTLLAMA_B200_TOKEN_PROF at create time)
int flk_token_plan_profile(void *plan, unsigned long long *out, size_t max_words, int *n_ctas) {
    fl_token_plan_impl *pl = (fl_token_plan_impl *)plan;
    FL_REQUIRE(pl && pl->d_prof, "token plan was created without FASTLLAMA_B200_TOKEN_PROF");
    const size_t words = (size_t)4 * pl->prm.n_phases * pl->n_kernels;
    FL_REQUIRE(max_words >= words, "profile buffer too small (%zu words needed)", words);
    FL_CUDA_OK(cudaMemcpy(out, pl->d_prof, words * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    *n_ctas = pl->n_kernels;
    return 0;
}

int flk_token_plan_profile2(void *plan, unsigned *out, size_t max_words) {
    fl_token_plan_impl *pl = (fl_token_plan_impl *)plan;
    FL_REQUIRE(pl && pl->d_prof2, "token plan was created without FASTLLAMA_B200_TOKEN_PROF");
    const size_t words = (size_t)pl->prm.n_phases * pl->n_kernels * TK_CW * 8;
    FL_REQUIRE(max_words >= words, "profile buffer too small (%zu words needed)", words);
    FL_CUDA_OK(cudaMemcpy(out, pl->d_prof2, words * sizeof(unsigned), cudaMemcpyDeviceToHost));
    return 0;
}

int flk_token_plan_error(void *plan) {
    fl_token_plan_impl *pl = (fl_token_plan_impl *)plan;
    if (!pl || !pl->h_err) return 0;
    const volatile unsigned *e = pl->h_err;      // written by the kernel straight into host memory; the caller has synchronised the stream
    if (e[0])
        fl_set_error("token kernel timeout: %s (code 0x%x), waited for / slot %u, last saw / parity %u, CTA %u, rank %d of %d",
                     (e[1] & 0x700u) == 0x600u ? "consumer warp waiting for a slot tag" : (e[1] & 0x700u) == 0x400u ? "consumer warp waiting for a weight tile" : (e[1] & 0x700u) == 0x500u ? "producer waiting for a free ring slot" :
                     (e[1] & 0x300u) == 0x300u ? "LL vector element" : "grid barrier counter", e[1], e[2], e[3], e[4], pl->prm.rank, pl->prm.world);
    return (int)e[0];
}

int flk_token_plan_destroy(void *plan) {
    fl_token_plan_impl *pl = (fl_token_plan_impl *)plan;
    if (!pl) return 0;
    if (pl->d_phases) cudaFree(pl->d_phases);
    if (pl->d_bar) cudaFree(pl->d_bar);
    if (pl->h_err) cudaFreeHost(pl->h_err);
    if (pl->d_prof) cudaFree(pl->d_prof);
    if (pl->d_prof2) cudaFree(pl->d_prof2);
    delete pl;
    return 0;
}
