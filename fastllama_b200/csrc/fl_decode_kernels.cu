// fl_decode_kernels.cu -- the fused decode step (N = 1): 5 kernels per transformer layer.
//
//   k_mv_fused     the TMA-ring matvec of fl_quant_kernels.cu with
//                    * up to 3 weight matrices sharing one input in ONE launch (wq|wk|wv, w1|w3):
//                      the CTA's contiguous slice of the concatenated row space is cut into tiles that
//                      never straddle a matrix, each tile still one 1-D bulk copy;
//                    * a fused PROLOGUE that builds the q8_0 activations in shared memory from f32:
//                        PRO_PLAIN    y = q8(x)
//                        PRO_RMSNORM  y = q8(gamma * rms_norm(x))        (reference lib/ggml.c:7378-7434 + mul)
//                        PRO_SILUMUL  y = q8(silu_f16tab(a) * b)          (reference lib/ggml.c:3207-3215 + mul)
//                      replacing the rms_norm / mul / silu / quantize_row_q8_0 launches (and the q8 work
//                      buffer round trip); every CTA rebuilds the vector itself (K*4 bytes from L2);
//                    * a fused EPILOGUE:
//                        EPI_STORE    dst = W y
//                        EPI_RESADD   dst = W y + residual                (the ggml_add after wo / w2)
//                        EPI_QKV      q -> rope -> q buffer; k -> rope -> K cache slot n_past;
//                                     v -> V cache column n_past          (rope + the two ggml_cpy,
//                                     reference lib/llama.cpp:328-343)
//   k_attn_decode  one CTA per head: scores over the cached positions, fp16-table soft_max, weighted
//                  sum of V (reference lib/llama.cpp:346-398 for N = 1)
//
// n_past is read from device memory so that a captured CUDA graph of the whole token step can be
// replayed for every token.  Arithmetic per element is identical to the unfused kernels (same
// roundings, same table lookups); see DESIGN.md "Parity".
#include <cuda_fp16.h>
#include <stdlib.h>

#include <algorithm>

#include "fl_common.cuh"
#include "fl_decode.h"
#include "fl_decode_dev.cuh"
#include "fl_kernels.h"

#define FD_MAX_THREADS 576

// device-side copy of the launch description (fl_mv_args) plus the ring geometry
struct fd_params {
    fl_mv_args a;
    int nb;
    uint32_t row_bytes;
    int R, S, kparts, G, TG, P;
    uint32_t stage_bytes;
    uint32_t off_y, off_red, off_rowbuf, off_cnt, off_stage0;
    int mtot;
};

template <int TYPE, int NFULL>
__global__ void __launch_bounds__(FD_MAX_THREADS, 1) k_mv_fused(const fd_params prm) {
    constexpr int BB = (TYPE == FL_TYPE_Q4_0) ? 20 : 24;
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t *bars = (uint64_t *)smem;
    fl_block_q8_0 *ysm = (fl_block_q8_0 *)(smem + prm.off_y);
    double *red = (double *)(smem + prm.off_red);            // [16] block-reduce scratch + [1] scale slot
    float *rowbuf = (float *)(smem + prm.off_rowbuf);        // [S][R][kparts] per-part row sums
    int *cnt = (int *)(smem + prm.off_cnt);                  // [S][R] arrival counters of the combine groups
    uint8_t *stage0 = smem + prm.off_stage0;

    const fl_mv_args &A = prm.a;
    const int S = prm.S, R = prm.R, kparts = prm.kparts, G = prm.G, TG = prm.TG;
    const int WPG = kparts * G, CW = WPG * TG;
    const int NT = CW * 32;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int K = prm.nb * 32;
    const fd_slice sl = fd_make_slice(A, prm.mtot, R);
    const int ntiles = sl.ntiles;
    const uint32_t bar0 = fl_smem_u32(bars);
    // Programmatic dependent launch: let the next kernel of the stream start as soon as SMs free up
    // (its producer streams its own weights while we finish); nothing below reads or writes an
    // activation before griddepcontrol.wait, which returns only when the previous kernel has completed.
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

    if (warp == CW) {
        // ------------------------------ producer ------------------------------
        // Initialises the mbarriers itself and starts streaming weights immediately: the weight stream
        // does not depend on anything the consumers compute in their prologue.
        if (lane == 0) {
            for (int s = 0; s < S; s++) {
                fl_mbar_init(bar0 + 8u * s, 1);
                fl_mbar_init(bar0 + 8u * (S + s), WPG);
            }
            fl_mbar_fence_init();
        }
        __syncwarp();
        asm volatile("bar.arrive 14, %0;" ::"r"(NT + 32) : "memory");      // consumers wait on 14 before touching the mbarriers
        if (lane == 0) {
            const uint64_t pol = fl_policy_evict_first();
            int s = 0;
            uint32_t ph = 1;
            for (int t = 0; t < ntiles; t++) {
                int seg, row0, rows;
                fd_tile_of(sl, R, t, seg, row0, rows);
                fl_mbar_wait(bar0 + 8u * (S + s), ph);
                const uint32_t bytes = (uint32_t)rows * prm.row_bytes;
                const uint8_t *src = (const uint8_t *)A.seg_w[seg] + (size_t)row0 * prm.row_bytes;
                fl_mbar_expect_tx(bar0 + 8u * s, bytes);
                fl_bulk_g2s_hint(fl_smem_u32(stage0 + (size_t)s * prm.stage_bytes), src, bytes, bar0 + 8u * s, pol);
                if (++s == S) { s = 0; ph ^= 1u; }
            }
        }
        return;
    }

    const int tid = threadIdx.x;                     // consumers are threads [0, NT)
    for (int i = tid; i < S * R; i += NT) cnt[i] = 0;
    asm volatile("griddepcontrol.wait;" ::: "memory");   // the producer warp never waits: weights depend on nothing

    // ------------------------------ consumers: prologue ------------------------------
    // Build the q8_0 activation vector in shared memory.  Each thread owns float4 groups i, i + NT, ...
    // (K/4 groups); 8 consecutive lanes hold one 32-element block, so amax / sum are 3-step shuffles.
    // Loads go through the read-only path (__ldg) and are issued two iterations ahead of their use.
    {
        const int nvec = K >> 2;
        const float4 *x4 = (const float4 *)A.x;
        const float4 *xa4 = (const float4 *)A.xadd;          // optional residual add in front of everything
        float scale = 1.0f;
        if (A.pro == FL_PRO_RMSNORM) {
            double acc = 0.0;
            // thread t adds the values of the 8-element units t, t + NT, ... in order (the token kernel's order)
            for (int u = tid; u < (nvec >> 1); u += NT) {
#pragma unroll
                for (int k = 0; k < 2; k++) {
                    const int i = 2 * u + k;
                    float4 v = __ldcg(x4 + i);
                    if (xa4) { const float4 w = __ldcg(xa4 + i); v.x = __fadd_rn(v.x, w.x); v.y = __fadd_rn(v.y, w.y); v.z = __fadd_rn(v.z, w.z); v.w = __fadd_rn(v.w, w.w); }
                    acc += (double)__fmul_rn(v.x, v.x);
                    acc += (double)__fmul_rn(v.y, v.y);
                    acc += (double)__fmul_rn(v.z, v.z);
                    acc += (double)__fmul_rn(v.w, v.w);
                }
            }
            acc = fl_warp_sum_d(acc);
            if (lane == 0) red[warp] = acc;
            asm volatile("bar.sync 15, %0;" ::"r"(NT) : "memory");
            if (tid == 0) {
                double t = 0.0;
                for (int w = 0; w < CW; w++) t += red[w];
                const float mean = (float)(t / (double)K);
                ((float *)(red + 16))[0] = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(mean, 1e-6f)));
            }
            asm volatile("bar.sync 15, %0;" ::"r"(NT) : "memory");
            scale = ((float *)(red + 16))[0];
        }
        const float4 *g4 = (const float4 *)A.gamma, *b4 = (const float4 *)A.b;
        const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
        // software pipeline: the loads of group i + NT are in flight while group i is quantised
        int i = warp * 32 + lane;                    // == tid; whole warps advance together (uniform trip count)
        auto load_x = [&](int idx) -> float4 {
            float4 v = __ldcg(x4 + idx);
            if (xa4) { const float4 w = __ldcg(xa4 + idx); v.x = __fadd_rn(v.x, w.x); v.y = __fadd_rn(v.y, w.y); v.z = __fadd_rn(v.z, w.z); v.w = __fadd_rn(v.w, w.w); }
            return v;
        };
        float4 xv = (i < nvec) ? load_x(i) : zero4;
        float4 ov = zero4;
        if (A.pro == FL_PRO_RMSNORM) ov = (i < nvec) ? __ldg(g4 + i) : zero4;
        else if (A.pro == FL_PRO_SILUMUL) ov = (i < nvec) ? __ldg(b4 + i) : zero4;
        for (int base = warp * 32; base < nvec; base += NT) {
            const int inext = i + NT;
            float4 xn = zero4, on = zero4;
            if (base + NT < nvec) {
                xn = (inext < nvec) ? load_x(inext) : zero4;
                if (A.pro == FL_PRO_RMSNORM) on = (inext < nvec) ? __ldg(g4 + inext) : zero4;
                else if (A.pro == FL_PRO_SILUMUL) on = (inext < nvec) ? __ldg(b4 + inext) : zero4;
            }
            float v[4] = {xv.x, xv.y, xv.z, xv.w};
            const float o[4] = {ov.x, ov.y, ov.z, ov.w};
            if (A.sum_out && blockIdx.x == 0 && i < nvec) ((float4 *)A.sum_out)[i] = xv;
            if (A.pro == FL_PRO_RMSNORM) {
#pragma unroll
                for (int c = 0; c < 4; c++) v[c] = __fmul_rn(o[c], __fmul_rn(v[c], scale));
                if (A.normed_out && blockIdx.x == 0 && i < nvec) ((float4 *)A.normed_out)[i] = make_float4(v[0], v[1], v[2], v[3]);
            } else if (A.pro == FL_PRO_SILUMUL) {
#pragma unroll
                for (int c = 0; c < 4; c++) {
                    const uint16_t h = __half_as_ushort(__float2half_rn(v[c]));
                    v[c] = __fmul_rn(__half2float(__ushort_as_half(__ldg(A.silu_tab + h))), o[c]);
                }
            }
            float amax = fmaxf(fmaxf(fabsf(v[0]), fabsf(v[1])), fmaxf(fabsf(v[2]), fabsf(v[3])));
            amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
            amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
            amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 4));
            const float d = __fdiv_rn(amax, 127.f);
            const float id = (amax != 0.0f) ? __fdiv_rn(127.f, amax) : 0.0f;
            int q[4], sum = 0;
#pragma unroll
            for (int c = 0; c < 4; c++) {
                q[c] = max(-128, min(127, __float2int_rn(__fmul_rn(v[c], id))));
                sum += q[c];
            }
            sum += __shfl_xor_sync(0xffffffffu, sum, 1);
            sum += __shfl_xor_sync(0xffffffffu, sum, 2);
            sum += __shfl_xor_sync(0xffffffffu, sum, 4);
            if (i < nvec) {
                fl_block_q8_0 *yb = ysm + (i >> 3);
                const uint32_t packed = (uint32_t)(q[0] & 0xFF) | ((uint32_t)(q[1] & 0xFF) << 8) | ((uint32_t)(q[2] & 0xFF) << 16) | ((uint32_t)(q[3] & 0xFF) << 24);
                ((uint32_t *)yb->qs)[i & 7] = packed;
                if ((i & 7) == 0) {
                    yb->d = d;
                    yb->s = __fmul_rn(d, (float)sum);
                }
            }
            xv = xn; ov = on; i = inext;
        }
        asm volatile("bar.sync 15, %0;" ::"r"(NT) : "memory");
    }

    const int tg = warp / WPG;
    const int wl = warp - tg * WPG;
    const int p = wl % kparts, g = wl / kparts;
    const int b0 = p * prm.P;
    const int b1 = min(prm.nb, b0 + prm.P);

    fd_yprep yp[FD_NBL];
    bool valid[FD_NBL];
#pragma unroll
    for (int j = 0; j < FD_NBL; j++) {
        const int ib = b0 + lane + 32 * j;
        valid[j] = (j < NFULL) || ib < b1;
        if (valid[j]) {
            fd_prep_y<TYPE>(ysm + ib, yp[j]);
        } else {
            yp[j].d = 0.f; yp[j].s = 0.f; yp[j].c = 0;
#pragma unroll
            for (int q = 0; q < 4; q++) { yp[j].ye[q] = 0; yp[j].yo[q] = 0; }
        }
    }

    // ------------------------------ consumers: main loop ------------------------------
    // Results that need more than one warp (K split over `kparts` warps, or a rope pair computed by two
    // warps) are combined by whichever warp arrives last at a per-group counter, always summing the
    // parts in index order -- deterministic, and no barrier in the loop.
    asm volatile("bar.sync 14, %0;" ::"r"(NT + 32) : "memory");          // mbarriers are initialised
    const bool pair = (A.epi == FL_EPI_QKV);
    const bool staged = (kparts > 1) || pair;
    const int target = pair ? 2 * kparts : kparts;
    const int n_past = pair ? *A.n_past : 0;
    int s = tg % S;
    uint32_t ph = (uint32_t)(tg / S) & 1u;
    const int s_step = TG % S, u_step = TG / S;
    for (int t = tg; t < ntiles; t += TG) {
        int seg, row0, rows;
        fd_tile_of(sl, R, t, seg, row0, rows);
        fl_mbar_wait(bar0 + 8u * s, ph);
        const uint8_t *tile = stage0 + (size_t)s * prm.stage_bytes;
        float *dseg = A.seg_dst[seg];
        for (int rr = g; rr < rows; rr += G) {
            const uint8_t *wrow = tile + (size_t)rr * prm.row_bytes + (size_t)(b0 + lane) * BB;
            float acc = 0.0f, accm = 0.0f;
#pragma unroll
            for (int j = 0; j < FD_NBL; j++) {
                if (j < NFULL) fd_block<TYPE>(wrow + (size_t)(32 * j) * BB, yp[j], acc, accm);
                else if (valid[j]) fd_block<TYPE>(wrow + (size_t)(32 * j) * BB, yp[j], acc, accm);
            }
            float tot = fl_warp_sum(acc);
            if (TYPE == FL_TYPE_Q4_1) tot = __fadd_rn(tot, fl_warp_sum(accm));
            if (lane == 0) {
                const int row = row0 + rr;
                if (!staged) {
                    dseg[row] = (A.epi == FL_EPI_RESADD) ? __fadd_rn(tot, A.res[row]) : tot;
                } else {
                    volatile float *rb = rowbuf + (size_t)s * R * kparts;
                    rb[rr * kparts + p] = tot;
                    __threadfence_block();
                    const int gid = pair ? (rr >> 1) : rr;
                    const int old = atomicAdd(&cnt[s * R + gid], 1);
                    if (old == target - 1) {                                  // last arriver combines
                        cnt[s * R + gid] = 0;
                        __threadfence_block();
                        if (pair) {
                            const int ra = gid << 1;
                            float x0 = rb[ra * kparts], x1 = rb[(ra + 1) * kparts];
                            for (int q = 1; q < kparts; q++) { x0 = __fadd_rn(x0, rb[ra * kparts + q]); x1 = __fadd_rn(x1, rb[(ra + 1) * kparts + q]); }
                            const int r2 = row0 + ra;                            // even row of the pair
                            if (seg < 2) {
                                const int ip = (r2 % A.head_dim) >> 1;
                                const float2 cs = ((const float2 *)A.rope_cs)[(size_t)n_past * (A.head_dim >> 1) + ip];
                                const float y0 = __fmaf_rn(x0, cs.x, -__fmul_rn(x1, cs.y));
                                const float y1 = __fmaf_rn(x0, cs.y, __fmul_rn(x1, cs.x));
                                float *o = (seg == 0) ? (dseg + r2) : (A.kcache + (size_t)n_past * A.n_embd + r2);
                                o[0] = y0; o[1] = y1;
                            } else {
                                A.vcache[(size_t)r2 * A.n_ctx + n_past] = x0;
                                A.vcache[(size_t)(r2 + 1) * A.n_ctx + n_past] = x1;
                            }
                        } else {
                            float tsum = rb[rr * kparts];
                            for (int q = 1; q < kparts; q++) tsum = __fadd_rn(tsum, rb[rr * kparts + q]);
                            dseg[row] = (A.epi == FL_EPI_RESADD) ? __fadd_rn(tsum, A.res[row]) : tsum;
                        }
                    }
                }
            }
        }
        __syncwarp();
        if (lane == 0) fl_mbar_arrive(bar0 + 8u * (S + s));
        s += s_step; ph ^= (uint32_t)(u_step & 1);
        if (s >= S) { s -= S; ph ^= 1u; }
    }
}

// =================================================================================================
// attention for one new token: one CTA per head
// =================================================================================================
struct fd_attn_params {
    const float *q;        // [n_embd] rope'd query
    const float *kcache;   // layer base: [pos][n_embd]
    const float *vcache;   // layer base: [n_embd][n_ctx]
    float *out;            // [n_embd]
    const int *n_past;
    int n_embd, n_ctx, head_dim;
    float scale;
    const uint16_t *exp_tab;
};

// The KV cache of a layer was last touched one token ago and has long left L2 (4 GB of weights went
// through since), so this kernel is bound by DRAM round trips, not bytes: every phase is written to
// have many independent loads in flight (4 positions per warp iteration for the scores, one output
// dimension per thread with 4 independent float4 streams for P*V).
__global__ void __launch_bounds__(256) k_attn_decode(const fd_attn_params P) {
    extern __shared__ float sc[];                   // [n_ctx] scores / probabilities, then [FD_PV_SUBS][head_dim] partials
    __shared__ double redd[8];
    __shared__ float redf[8];
    float *part = sc + P.n_ctx;
    const int h = blockIdx.x, hd = P.head_dim;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");              // q / K / V of this step come from the previous kernel
    const int n_pos = *P.n_past + 1;
    const float *q = P.q + (size_t)h * hd;

    // scores_j = scale * <K_j, q>   (ggml_mul_mat K,Q then ggml_scale; the mask is a no-op for N = 1)
    for (int j0 = warp * 4; j0 < n_pos; j0 += nw * 4) {
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        for (int e = lane; e < hd; e += 32) {
            const float qe = q[e];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const int j = min(j0 + u, n_pos - 1);                 // clamp: loads stay in range, result discarded below
                acc[u] = __fmaf_rn(P.kcache[(size_t)j * P.n_embd + (size_t)h * hd + e], qe, acc[u]);
            }
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const float a = fl_warp_sum(acc[u]);
            if (lane == 0 && j0 + u < n_pos) sc[j0 + u] = __fmul_rn(a, P.scale);
        }
    }
    __syncthreads();
    // soft_max with the fp16 exp table (reference lib/ggml.c:8521-8589)
    float mx = -INFINITY;
    for (int j = threadIdx.x; j < n_pos; j += blockDim.x) mx = fmaxf(mx, sc[j]);
    mx = fl_warp_max(mx);
    if (lane == 0) redf[warp] = mx;
    __syncthreads();
    mx = redf[0];
    for (int w = 1; w < nw; w++) mx = fmaxf(mx, redf[w]);
    double sum = 0.0;
    for (int j = threadIdx.x; j < n_pos; j += blockDim.x) {
        const uint16_t hh = __half_as_ushort(__float2half_rn(__fsub_rn(sc[j], mx)));
        const float e = __half2float(__ushort_as_half(P.exp_tab[hh]));
        sc[j] = e;
        sum += (double)e;
    }
    sum = fl_warp_sum_d(sum);
    if (lane == 0) redd[warp] = sum;
    __syncthreads();
    double tot = 0.0;
    for (int w = 0; w < nw; w++) tot += redd[w];
    const float inv = (float)(1.0 / tot);
    for (int j = threadIdx.x; j < n_pos; j += blockDim.x) sc[j] = __fmul_rn(sc[j], inv);
    __syncthreads();
    // out_d = sum_j p_j * V[d][j]   (ggml_mul_mat V, soft_max) in the canonical order of fd_pv_partials
    const int npt = blockDim.x / hd;                               // threads per output dimension (2 for head_dim 128)
    const int ns = FD_PV_SUBS / npt;                               // subsequences per thread
    if ((int)threadIdx.x < npt * hd) {
        const int d = threadIdx.x % hd, sub0 = (threadIdx.x / hd) * ns;
        fd_pv_store_partials<16>(P.vcache + ((size_t)h * hd + d) * P.n_ctx, sc, n_pos, sub0, ns, part, hd, d);
    }
    __syncthreads();
    if ((int)threadIdx.x < hd) P.out[(size_t)h * hd + threadIdx.x] = fd_pv_combine(part, hd, threadIdx.x);
}

// =================================================================================================
// host side
// =================================================================================================
static int g_sm = 0, g_smem_optin = 0;
static int fd_query() {
    if (g_sm) return 0;
    int dev = 0;
    FL_CUDA_OK(cudaGetDevice(&dev));
    FL_CUDA_OK(cudaDeviceGetAttribute(&g_sm, cudaDevAttrMultiProcessorCount, dev));
    FL_CUDA_OK(cudaDeviceGetAttribute(&g_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    return 0;
}

static bool fd_use_pdl() {
    static int v = -1;
    // with PDL the 7B decode step was slower, so it is opt-in
    if (v < 0) v = getenv("FASTLLAMA_B200_PDL") ? 1 : 0;
    return v != 0;
}

typedef void (*fd_kernel_t)(const fd_params);
static fd_kernel_t fd_kernel(int type, int nfull) {
    if (type == FL_TYPE_Q4_0) {
        switch (nfull) {
            case 4: return k_mv_fused<FL_TYPE_Q4_0, 4>;
            case 3: return k_mv_fused<FL_TYPE_Q4_0, 3>;
            case 2: return k_mv_fused<FL_TYPE_Q4_0, 2>;
            case 1: return k_mv_fused<FL_TYPE_Q4_0, 1>;
            default: return k_mv_fused<FL_TYPE_Q4_0, 0>;
        }
    }
    switch (nfull) {
        case 4: return k_mv_fused<FL_TYPE_Q4_1, 4>;
        case 3: return k_mv_fused<FL_TYPE_Q4_1, 3>;
        case 2: return k_mv_fused<FL_TYPE_Q4_1, 2>;
        case 1: return k_mv_fused<FL_TYPE_Q4_1, 1>;
        default: return k_mv_fused<FL_TYPE_Q4_1, 0>;
    }
}

int flk_mv_fused_supported(int type, int K, int mtot) {
    if (type != FL_TYPE_Q4_0 && type != FL_TYPE_Q4_1) return 0;
    if (K <= 0 || K % 32 != 0) return 0;
    const size_t row_bytes = (size_t)(K / 32) * fl_block_bytes(type);
    if (row_bytes % 16 != 0) return 0;
    if (K / 32 > 8 * 128) return 0;
    if (fd_query() != 0) return 0;
    return mtot >= 2 && mtot % 2 == 0;
}

int flk_mv_fused(cudaStream_t st, const fl_mv_args *args) {
    if (fd_query() != 0) return -1;
    const fl_mv_args &a = *args;
    FL_REQUIRE(a.nseg >= 1 && a.nseg <= 3, "mv_fused: nseg=%d", a.nseg);
    int mtot = 0;
    for (int i = 0; i < a.nseg; i++) {
        FL_REQUIRE(a.seg_rows[i] > 0 && a.seg_rows[i] % 2 == 0 && ((uintptr_t)a.seg_w[i] & 15) == 0, "mv_fused: bad segment %d", i);
        mtot += a.seg_rows[i];
    }
    FL_REQUIRE((a.type == FL_TYPE_Q4_0 || a.type == FL_TYPE_Q4_1) && a.K > 0 && a.K % 32 == 0 && mtot >= 2, "mv_fused: unsupported shape type=%d K=%d M=%d", a.type, a.K, mtot);
    FL_REQUIRE(a.row_stride_bytes ? (a.row_stride_bytes % 16 == 0 && a.row_stride_bytes >= (size_t)(a.K / 32) * fl_block_bytes(a.type))
                                  : flk_mv_fused_supported(a.type, a.K, mtot),
               "mv_fused: rows of K=%d (stride %zu) are not 16-byte multiples", a.K, a.row_stride_bytes);
    FL_REQUIRE(((uintptr_t)a.x & 15) == 0 && ((uintptr_t)a.xadd & 15) == 0 && ((uintptr_t)a.gamma & 15) == 0 && ((uintptr_t)a.b & 15) == 0 &&
               ((uintptr_t)a.sum_out & 15) == 0 && ((uintptr_t)a.normed_out & 15) == 0, "mv_fused: activation vectors must be 16-byte aligned");
    fd_params p;
    p.a = a;
    p.mtot = mtot;
    const int bb = fl_block_bytes(a.type);
    const int nb = a.K / 32;
    const size_t row_bytes = a.row_stride_bytes ? a.row_stride_bytes : (size_t)nb * bb;
    int kparts = 1;
    while (kparts * 128 < nb) kparts *= 2;                      // power of two so that 16 consumer warps divide evenly
    const int P = (nb + kparts - 1) / kparts;
    const int last = nb - (kparts - 1) * P;
    FL_REQUIRE(last > 0, "mv_fused: K=%d splits badly", a.K);
    int nfull = std::min(P, last) / 32;
    if (nfull > FD_NBL) nfull = FD_NBL;
    static int tile_target = -1;
    if (tile_target < 0) {
        const char *e = getenv("FASTLLAMA_B200_RING_TILE_KB");
        tile_target = (e ? atoi(e) : 16) * 1024;
    }
    const int Gmax = std::max(1, 16 / kparts);
    int G = Gmax, TG = 1;
    for (int tgc = 1; tgc <= 4; tgc *= 2) {
        const int gc = std::max(1, Gmax / tgc);
        G = gc; TG = tgc;
        if ((size_t)gc * row_bytes <= (size_t)tile_target || gc == 1) break;
    }
    int R = G;
    if (R % 2) { R = (R > 1) ? R - 1 : 2; G = std::min(G, R); }      // even tiles keep rope pairs together
    const size_t stage_bytes = (size_t)R * row_bytes;
    const size_t y_bytes = (size_t)nb * 40;
    int S = 16;
    size_t off_y = 0, off_red = 0, off_rowbuf = 0, off_cnt = 0, off = 0;
    for (;; S--) {
        FL_REQUIRE(S >= 2, "mv_fused: shape does not fit shared memory (K=%d)", a.K);
        off_y = ((size_t)(2 * S) * 8 + 127) & ~(size_t)127;
        off_red = (off_y + y_bytes + 127) & ~(size_t)127;
        off_rowbuf = (off_red + 17 * sizeof(double) + 8 + 127) & ~(size_t)127;
        off_cnt = (off_rowbuf + (size_t)S * R * kparts * sizeof(float) + 127) & ~(size_t)127;
        off = (off_cnt + (size_t)S * R * sizeof(int) + 127) & ~(size_t)127;
        if (off + (size_t)S * stage_bytes <= (size_t)g_smem_optin - 1024) break;       // 1 KB left for static shared memory
    }
    if (TG > S) TG = S;
    const int CW = kparts * G * TG;
    FL_REQUIRE((CW + 1) * 32 <= FD_MAX_THREADS, "mv_fused: too many warps");
    p.nb = nb; p.row_bytes = (uint32_t)row_bytes; p.R = R; p.S = S; p.kparts = kparts; p.G = G; p.TG = TG; p.P = P;
    p.stage_bytes = (uint32_t)stage_bytes;
    p.off_y = (uint32_t)off_y; p.off_red = (uint32_t)off_red;
    p.off_rowbuf = (uint32_t)off_rowbuf; p.off_cnt = (uint32_t)off_cnt; p.off_stage0 = (uint32_t)off;
    const size_t smem_bytes = off + (size_t)S * stage_bytes;
    fd_kernel_t kern = fd_kernel(a.type, nfull);
    static bool attr_set[2][FD_NBL + 1] = {{false}};
    const int ti = a.type == FL_TYPE_Q4_0 ? 0 : 1;
    if (!attr_set[ti][nfull]) {
        cudaFuncAttributes fa;
        FL_CUDA_OK(cudaFuncGetAttributes(&fa, kern));
        FL_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, g_smem_optin - (int)fa.sharedSizeBytes));
        attr_set[ti][nfull] = true;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(g_sm);
    cfg.blockDim = dim3((CW + 1) * 32);
    cfg.dynamicSmemBytes = smem_bytes;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = fd_use_pdl() ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    FL_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, p));
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

int flk_attn_decode(cudaStream_t st, const float *q, const float *kcache, const float *vcache, float *out, const int *n_past,
                    int n_embd, int n_head, int head_dim, int n_ctx, float scale, const uint16_t *exp_tab) {
    fd_attn_params P;
    P.q = q; P.kcache = kcache; P.vcache = vcache; P.out = out; P.n_past = n_past;
    P.n_embd = n_embd; P.n_ctx = n_ctx; P.head_dim = head_dim; P.scale = scale; P.exp_tab = exp_tab;
    const size_t smem = ((size_t)n_ctx + (size_t)FD_PV_SUBS * head_dim) * sizeof(float);
    FL_REQUIRE(smem <= 200 * 1024, "attn_decode: n_ctx=%d too large for the score buffer", n_ctx);
    static size_t attr = 0;
    if (smem > 48 * 1024 && attr < smem) {
        FL_CUDA_OK(cudaFuncSetAttribute(k_attn_decode, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr = smem;
    }
    FL_REQUIRE(n_ctx % 4 == 0 && head_dim >= 16 && head_dim <= 256 && (head_dim & (head_dim - 1)) == 0,
               "attn_decode: n_ctx must be a multiple of 4 and head_dim a power of two in [16, 256]");
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(n_head);
    cfg.blockDim = dim3(256);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute lattr[1];
    lattr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    lattr[0].val.programmaticStreamSerializationAllowed = fd_use_pdl() ? 1 : 0;
    cfg.attrs = lattr;
    cfg.numAttrs = 1;
    FL_CUDA_OK(cudaLaunchKernelEx(&cfg, k_attn_decode, P));
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}
