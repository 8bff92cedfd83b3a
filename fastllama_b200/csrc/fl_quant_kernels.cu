// fl_quant_kernels.cu -- sm_90a kernels for the q4_0/q4_1 x q8_0 hot path.
//
//   k_quantize_q8_0      activations -> q8_0 blocks      (reference lib/ggml.c:1299-1441, AVX2 semantics)
//   k_quantize_q4_{0,1}  weights -> q4 blocks            (reference lib/ggml.c:630-664, :917-956)
//   k_dequantize_rows    q4 rows -> f32 (get_rows)       (reference lib/ggml.c:1443-1665, :8333-8360)
//   k_mul_mat_q_plain    warp-per-row LDG matvec/matmul  (reference lib/ggml.c:8125-8163 + :2368-2714)
//   k_matvec_q4_ring     decode matvec: weights streamed HBM -> smem by the TMA unit (1-D bulk
//                        copies, mbarrier ring), activations resident in registers, dp4a block dots
//
// Arithmetic contract (see DESIGN.md "Parity"): q8_0 / q4 quantisation and dequantisation are
// bit-exact with the reference; in the dot products the per-block integer sums are exact and each
// block contributes fma(dx*dy, float(sum_i), acc) exactly as in the reference, only the order in
// which the per-block terms are added in fp32 differs (lane-strided + shuffle tree here, 8 AVX
// lanes there).
#include <cuda_fp16.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "fl_common.cuh"
#include "fl_kernels.h"

// =================================================================================================
// q8_0 quantisation of activations: one warp per 32-element block
// =================================================================================================
__global__ void k_quantize_q8_0(const float *__restrict__ x, size_t x_row_stride_bytes,
                                fl_block_q8_0 *__restrict__ y, int k, int nrows) {
    const int nb = k / FL_QK;
    const long total = (long)nb * nrows;
    const int lane = threadIdx.x & 31;
    const long wid = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long nw = ((long)gridDim.x * blockDim.x) >> 5;
    for (long b = wid; b < total; b += nw) {
        const int row = (int)(b / nb), ib = (int)(b % nb);
        const float *xr = (const float *)((const char *)x + (size_t)row * x_row_stride_bytes);
        const float v = xr[ib * FL_QK + lane];
        const float amax = fl_warp_max(fabsf(v));
        const float d = __fdiv_rn(amax, 127.f);
        const float id = (amax != 0.0f) ? __fdiv_rn(127.f, amax) : 0.0f;
        int q = __float2int_rn(__fmul_rn(v, id));   // round-half-even == _mm256_round_ps(NEAREST)
        q = max(-128, min(127, q));
        const int sum = fl_warp_sum_i(q);
        fl_block_q8_0 *yb = y + b;
        yb->qs[lane] = (int8_t)q;
        if (lane == 0) {
            yb->d = d;
            yb->s = __fmul_rn(d, (float)sum);
        }
    }
}

// =================================================================================================
// q4_0 / q4_1 weight quantisation ("_reference" semantics: roundf = half away from zero)
// =================================================================================================
// One block per warp, element `lane` in v.  Writes the block and returns the lane's stored nibble
// (the value ggml_quantize_q4_* counts in its histogram).
__device__ __forceinline__ int fl_quantize_block_q4_0(float v, int lane, fl_block_q4_0 *yb) {
    const float amax = fl_warp_max(fabsf(v));
    const float d = __fdiv_rn(amax, 7.0f);
    const float id = (d != 0.0f) ? __fdiv_rn(1.0f, d) : 0.0f;
    const int q = (int)(int8_t)roundf(__fmul_rn(v, id)) + 8;
    const int qn = __shfl_down_sync(0xffffffffu, q, 1);
    if ((lane & 1) == 0) yb->qs[lane >> 1] = (uint8_t)((q & 0xFF) | (qn << 4));
    if (lane == 0) yb->d = d;
    return q & 0xF;
}

// FIRST_MIN: m is the block's first element equal to the minimum, as the reference's `if (v < min)`
// scan keeps it.  That differs from the fminf tree only in the sign of a zero minimum, when the block
// holds both +0 and -0 (as f32 values below 2^-25 do once rounded to f16).
template <bool FIRST_MIN = false>
__device__ __forceinline__ int fl_quantize_block_q4_1(float v, int lane, fl_block_q4_1 *yb) {
    float mn = v, mx = v;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    if (FIRST_MIN) {
        const unsigned at = __ballot_sync(0xffffffffu, v == mn);
        if (at) mn = __shfl_sync(0xffffffffu, v, __ffs(at) - 1);
    }
    const float d = __fdiv_rn(__fsub_rn(mx, mn), 15.0f);
    const float id = (d != 0.0f) ? __fdiv_rn(1.0f, d) : 0.0f;
    const int q = (int)(uint8_t)roundf(__fmul_rn(__fsub_rn(v, mn), id));
    const int qn = __shfl_down_sync(0xffffffffu, q, 1);
    if ((lane & 1) == 0) yb->qs[lane >> 1] = (uint8_t)((q & 0xFF) | (qn << 4));
    if (lane == 0) {
        yb->d = d;
        yb->m = mn;
    }
    return q & 0xF;
}

__global__ void k_quantize_q4_0(const float *__restrict__ x, fl_block_q4_0 *__restrict__ y, long nblocks) {
    const int lane = threadIdx.x & 31;
    const long wid = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long nw = ((long)gridDim.x * blockDim.x) >> 5;
    for (long b = wid; b < nblocks; b += nw) fl_quantize_block_q4_0(x[b * FL_QK + lane], lane, y + b);
}

__global__ void k_quantize_q4_1(const float *__restrict__ x, fl_block_q4_1 *__restrict__ y, long nblocks) {
    const int lane = threadIdx.x & 31;
    const long wid = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long nw = ((long)gridDim.x * blockDim.x) >> 5;
    for (long b = wid; b < nblocks; b += nw) fl_quantize_block_q4_1(x[b * FL_QK + lane], lane, y + b);
}

// Model-file quantisation (the reference's fastllama::quantize, lib/llama.cpp:585-646): a tensor's
// rows as the input file stores them, f32 or f16, to q4 blocks, plus the 16-bin histogram of the
// stored nibbles that ggml_quantize_chunk reports.  f16 -> f32 is exact, so __half2float gives the
// reference's ggml_fp16_to_fp32 inputs and the blocks carry the bits of k_quantize_q4_*, except that a
// q4_1 block's m keeps the sign of its first zero when its minimum is a zero of both signs.  SRC 2 is
// f32 rounded to f16 (round to nearest even, as numpy's astype(float16) in the reference's converter)
// and widened back: the values the reference's tool reads from the f16 file converted from an f32
// checkpoint.  SRC 3 is f16 data of an f32 file (an f16 checkpoint converted to f32): the values of
// SRC 1, merged by the f32 rule below.
// DELTA (FL_DELTA_F32 / FL_DELTA_F16): a LoRA delta of the same [rows][k] layout is merged first, as
// the reference's attach_lora merges it into an unquantised model (ggml_add_inplace, lib/ggml.c):
// into an f32 file (SRC 0, 3) w + d (add_f32); into an f16 file (SRC 1, 2; for SRC 2 w is already the
// f16-rounded value) fp16_rn(w + fp32(d)) (add_f16_f32 / add_f16_f16: widening f16 is exact, so both
// are this one formula), then widened back for the quantiser.
// Histogram: four ballots (one per bit of the nibble) give every lane the warp's count for bin
// `lane` (lanes 0..15); the counts stay in a register across the warp's blocks, then go through
// shared memory to one set of 16 64-bit global atomics per CTA.
#define FL_DELTA_NONE (-1)
#define FL_DELTA_F32 0
#define FL_DELTA_F16 1
template <int TYPE, int SRC, int DELTA>
__global__ void __launch_bounds__(256) k_quantize_q4_file(const void *__restrict__ x, const void *__restrict__ delta, void *__restrict__ y,
                                                          long nblocks, unsigned long long *__restrict__ hist) {
    __shared__ unsigned sh_hist[16];
    const int lane = threadIdx.x & 31;
    if (threadIdx.x < 16) sh_hist[threadIdx.x] = 0;
    __syncthreads();
    const long wid = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long nw = ((long)gridDim.x * blockDim.x) >> 5;
    unsigned cnt = 0;                                        // lanes 0..15: this warp's count of nibble value `lane`
    for (long b = wid; b < nblocks; b += nw) {
        const long e = b * FL_QK + lane;
        float v = (SRC == 1 || SRC == 3) ? __half2float(((const __half *)x)[e])
                  : SRC == 2             ? __half2float(__float2half_rn(((const float *)x)[e]))
                                         : ((const float *)x)[e];
        if (DELTA != FL_DELTA_NONE) {
            const float d = DELTA == FL_DELTA_F16 ? __half2float(((const __half *)delta)[e]) : ((const float *)delta)[e];
            v = __fadd_rn(v, d);
            if (SRC == 1 || SRC == 2) v = __half2float(__float2half_rn(v));
        }
        const int q = (TYPE == FL_TYPE_Q4_0) ? fl_quantize_block_q4_0(v, lane, (fl_block_q4_0 *)y + b)
                                             : fl_quantize_block_q4_1<true>(v, lane, (fl_block_q4_1 *)y + b);
        unsigned m = 0xffffffffu;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const unsigned plane = __ballot_sync(0xffffffffu, (q >> j) & 1);
            m &= ((lane >> j) & 1) ? plane : ~plane;
        }
        cnt += __popc(m);
    }
    if (hist) {
        if (lane < 16 && cnt) atomicAdd(&sh_hist[lane], cnt);
        __syncthreads();
        if (threadIdx.x < 16 && sh_hist[threadIdx.x]) atomicAdd(hist + threadIdx.x, (unsigned long long)sh_hist[threadIdx.x]);
    }
}

// =================================================================================================
// dequantise rows (get_rows on a quantised matrix): one thread per nibble pair
// =================================================================================================
template <int TYPE>
__global__ void k_dequantize_rows(const uint8_t *__restrict__ W, size_t w_row_stride, int K,
                                  const int32_t *__restrict__ ids, int n_ids, float *__restrict__ dst,
                                  size_t dst_row_stride) {
    constexpr int BB = (TYPE == FL_TYPE_Q4_0) ? 20 : 24;
    const int nb = K / FL_QK;
    const long total = (long)n_ids * nb * 16;
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long)gridDim.x * blockDim.x) {
        const int j = (int)(t & 15);
        const long bi = t >> 4;
        const int ib = (int)(bi % nb);
        const int i = (int)(bi / nb);
        const long r = ids ? (long)ids[i] : (long)i;
        const uint8_t *blk = W + (size_t)r * w_row_stride + (size_t)ib * BB;
        const float d = *(const float *)blk;
        float2 o;
        if (TYPE == FL_TYPE_Q4_0) {
            const uint8_t b = blk[4 + j];
            o.x = __fmul_rn((float)((int)(b & 0x0F) - 8), d);
            o.y = __fmul_rn((float)((int)(b >> 4) - 8), d);
        } else {
            const float m = *(const float *)(blk + 4);
            const uint8_t b = blk[8 + j];
            o.x = __fmaf_rn((float)(b & 0x0F), d, m);
            o.y = __fmaf_rn((float)(b >> 4), d, m);
        }
        float *out = dst + (size_t)i * dst_row_stride + ib * FL_QK + 2 * j;
        *(float2 *)out = o;
    }
}

// =================================================================================================
// Shared block arithmetic
// =================================================================================================
// Activation block in "prepared" form: the 32 int8 are split into even / odd elements so that the
// low-nibble word and the high-nibble word of a q4 qs word each meet one contiguous dp4a operand:
//   qs word j holds elements 8j..8j+7; (w & 0x0F0F0F0F) = elements 8j+{0,2,4,6},
//   (w & 0xF0F0F0F0) = 16 * elements 8j+{1,3,5,7}.
struct fl_yprep {
    uint32_t ye[4], yo[4];
    float d;     // q8 block scale
    float s;     // q8 block d*sum (q4_1 only)
    int c;       // -8 * sum(y) for q4_0 (folds the "-8" offset of the nibbles), 0 for q4_1
};

template <int TYPE>
__device__ __forceinline__ void fl_prep_y(const fl_block_q8_0 *yb, fl_yprep &p) {
    const uint32_t *q = (const uint32_t *)yb->qs;   // 40-B blocks on an 8-B aligned base: 4-B loads are safe
    int sum = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const uint32_t a = q[2 * j], b = q[2 * j + 1];
        p.ye[j] = __byte_perm(a, b, 0x6420);
        p.yo[j] = __byte_perm(a, b, 0x7531);
        sum = fl_dp4a_ss(0x01010101u, a, sum);
        sum = fl_dp4a_ss(0x01010101u, b, sum);
    }
    p.d = yb->d;
    p.s = yb->s;
    p.c = (TYPE == FL_TYPE_Q4_0) ? -8 * sum : 0;
}

// exact integer sum_{e<32} (q4_e - off) * q8_e for one block (off = 8 for q4_0, 0 for q4_1)
__device__ __forceinline__ int fl_block_isum(const uint32_t w[4], const fl_yprep &p) {
    int lo = p.c, hi = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        lo = fl_dp4a_us(w[j] & 0x0F0F0F0Fu, p.ye[j], lo);
        hi = fl_dp4a_us(w[j] & 0xF0F0F0F0u, p.yo[j], hi);   // = 16 * (odd-element dot), exact
    }
    return lo + (hi >> 4);
}

// =================================================================================================
// Plain matmul: one warp per weight row, lanes stride over the row's blocks, loop over the N
// activation rows.  Correct for any M, K (multiple of 32), N and any 4-B aligned row stride; used
// for small/odd shapes, for N > 1 until the tensor-core path takes over, and as the in-library
// cross-check of the ring kernel.
// =================================================================================================
template <int TYPE>
__global__ void __launch_bounds__(256)
k_mul_mat_q_plain(const uint8_t *__restrict__ W, size_t w_row_stride, int M, int K,
                  const fl_block_q8_0 *__restrict__ Y, int N, float *__restrict__ dst, size_t dst_row_stride) {
    constexpr int BB = (TYPE == FL_TYPE_Q4_0) ? 20 : 24;
    constexpr int QOFF = (TYPE == FL_TYPE_Q4_0) ? 1 : 2;     // word offset of qs inside the block
    const int nb = K / FL_QK;
    const int lane = threadIdx.x & 31;
    const long wid = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long nw = ((long)gridDim.x * blockDim.x) >> 5;
    for (long m = wid; m < M; m += nw) {
        const uint8_t *wrow = W + (size_t)m * w_row_stride;
        for (int n = 0; n < N; n++) {
            const fl_block_q8_0 *yrow = Y + (size_t)n * nb;
            float acc = 0.0f, accm = 0.0f;
            for (int ib = lane; ib < nb; ib += 32) {
                const uint32_t *bw = (const uint32_t *)(wrow + (size_t)ib * BB);
                const float dx = __uint_as_float(__ldg(bw));
                uint32_t w[4];
#pragma unroll
                for (int j = 0; j < 4; j++) w[j] = __ldg(bw + QOFF + j);
                fl_yprep p;
                fl_prep_y<TYPE>(yrow + ib, p);
                const int isum = fl_block_isum(w, p);
                acc = __fmaf_rn(__fmul_rn(dx, p.d), (float)isum, acc);
                if (TYPE == FL_TYPE_Q4_1) accm = __fmaf_rn(__uint_as_float(__ldg(bw + 1)), p.s, accm);
            }
            float tot = fl_warp_sum(acc);
            if (TYPE == FL_TYPE_Q4_1) tot = __fadd_rn(tot, fl_warp_sum(accm));
            if (lane == 0) dst[(size_t)n * dst_row_stride + m] = tot;
        }
    }
}

// =================================================================================================
// Decode matvec (N = 1): persistent, TMA-fed.
//
//   grid  = one CTA per SM; CTA b owns the contiguous row range [M*b/G, M*(b+1)/G) -- a single
//           contiguous byte range of HBM, so every tile is ONE 1-D bulk copy (UBLKCP), no tensor
//           map needed, and the per-CTA byte imbalance is at most one row.
//   smem  = the q8_0 activation vector (staged once by a bulk copy) + a ring of S stages x
//           (R rows x row_bytes).  A producer lane keeps all S stages in flight (mbarrier
//           full/empty pairs), so ~200 KB per SM of HBM reads are outstanding.
//   warps = TG tile-groups x G row-groups x kparts K-slices of consumer warps + 1 producer warp.
//           Tile t is consumed by tile-group t % TG, so several tiles are worked on at once and a
//           tile can be small (fine-grained ring: data is usable as soon as ~20 KB have landed).
//           A consumer warp is bound to one K-slice ("part", <= 128 blocks) of the row for the
//           whole kernel, so the activations of its slice live in registers in prepared form; it
//           walks the rows of its tiles that belong to its row-group.  Lanes stride over the
//           slice's blocks: lane t reads block t, t+32, ... with 5 x LDS.32 (q4_0, stride 5 words:
//           conflict-free) or 3 x LDS.64 (q4_1, stride 6 words: conflict-free per half-warp).
//   reduce: per-lane sequential fma over its blocks -> 5-step xor-shuffle tree -> (kparts > 1)
//           fixed-order sum of the parts through smem.  Deterministic.
// =================================================================================================
#define FL_RING_NBL 4          // blocks per lane per part (part <= 128 blocks = 4096 weights)
#define FL_RING_MAX_STAGES 16
#define FL_RING_MAX_PARTS 8
#define FL_RING_MAX_THREADS 576   // (16 consumer warps + producer) rounded up; 65536/576 = 113 regs/thread

struct fl_ring_params {
    const uint8_t *W;
    const fl_block_q8_0 *Y;
    float *dst;
    int M, nb;
    uint32_t row_bytes;
    int R;            // rows per tile
    int S;            // stages
    int kparts, G, TG;   // consumer warps = TG * G * kparts
    int P;            // blocks per part
    uint32_t stage_bytes;
    uint32_t y_bytes;                              // nb * 40, multiple of 16
    uint32_t off_y, off_partial, off_stage0;       // dynamic smem layout
};

// one block of one row: weights from smem, activations from registers
template <int TYPE>
__device__ __forceinline__ void fl_ring_block(const uint8_t *blk, const fl_yprep &yp, float &acc, float &accm) {
    uint32_t w[4];
    float dx;
    if (TYPE == FL_TYPE_Q4_0) {
        const uint32_t *bw = (const uint32_t *)blk;
        dx = __uint_as_float(bw[0]);
        w[0] = bw[1]; w[1] = bw[2]; w[2] = bw[3]; w[3] = bw[4];
    } else {
        const uint2 *bw = (const uint2 *)blk;     // 24-B blocks, 8-B aligned
        const uint2 dm = bw[0], q01 = bw[1], q23 = bw[2];
        dx = __uint_as_float(dm.x);
        accm = __fmaf_rn(__uint_as_float(dm.y), yp.s, accm);
        w[0] = q01.x; w[1] = q01.y; w[2] = q23.x; w[3] = q23.y;
    }
    const int isum = fl_block_isum(w, yp);
    acc = __fmaf_rn(__fmul_rn(dx, yp.d), (float)isum, acc);
}

// NFULL = number of leading block slots (of FL_RING_NBL) that are valid for EVERY lane of every
// part; the remaining slots are lane-predicated.  K = 4096 -> NFULL = 4: no predication at all.
template <int TYPE, int NFULL>
__global__ void __launch_bounds__(FL_RING_MAX_THREADS, 1) k_matvec_q4_ring(const fl_ring_params prm) {
    constexpr int BB = (TYPE == FL_TYPE_Q4_0) ? 20 : 24;
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t *bars = (uint64_t *)smem;                       // [0..S) full, [S..2S) empty, [2S] activations
    const fl_block_q8_0 *ysm = (const fl_block_q8_0 *)(smem + prm.off_y);
    float *partial = (float *)(smem + prm.off_partial);      // [S][R][kparts]
    uint8_t *stage0 = smem + prm.off_stage0;

    const int S = prm.S, R = prm.R, kparts = prm.kparts, G = prm.G, TG = prm.TG;
    const int WPG = kparts * G;                              // warps per tile-group
    const int CW = WPG * TG;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    const int r0 = (int)(((long)prm.M * blockIdx.x) / gridDim.x);
    const int r1 = (int)(((long)prm.M * (blockIdx.x + 1)) / gridDim.x);
    const int nrows = r1 - r0;
    const int ntiles = (nrows + R - 1) / R;

    const uint32_t bar0 = fl_smem_u32(bars);
    const uint32_t bar_y = bar0 + 8u * (2 * S);
    if (threadIdx.x == 0) {
        for (int s = 0; s < S; s++) {
            fl_mbar_init(bar0 + 8u * s, 1);                 // full: producer's expect_tx arrive
            fl_mbar_init(bar0 + 8u * (S + s), WPG);         // empty: one arrive per consuming warp
        }
        fl_mbar_init(bar_y, 1);
        fl_mbar_fence_init();
    }
    __syncthreads();

    if (warp == CW) {
        // ------------------------------ producer ------------------------------
        if (lane == 0) {
            // activations first (tiny, L2-resident), then the weight stream
            fl_mbar_expect_tx(bar_y, prm.y_bytes);
            fl_bulk_g2s(fl_smem_u32(ysm), prm.Y, prm.y_bytes, bar_y);
            const uint64_t pol = fl_policy_evict_first();
            const uint8_t *src = prm.W + (size_t)r0 * prm.row_bytes;
            int s = 0;
            uint32_t ph = 1;                                // parity to wait for on the empty barrier
            for (int t = 0; t < ntiles; t++) {
                fl_mbar_wait(bar0 + 8u * (S + s), ph);
                const int rows = min(R, nrows - t * R);
                const uint32_t bytes = (uint32_t)rows * prm.row_bytes;
                fl_mbar_expect_tx(bar0 + 8u * s, bytes);
                fl_bulk_g2s_hint(fl_smem_u32(stage0 + (size_t)s * prm.stage_bytes), src + (size_t)t * R * prm.row_bytes, bytes,
                                 bar0 + 8u * s, pol);
                if (++s == S) { s = 0; ph ^= 1u; }
            }
        }
        return;
    }

    // ------------------------------ consumers ------------------------------
    const int tg = warp / WPG;
    const int wl = warp - tg * WPG;                          // warp index inside the tile-group
    const int p = wl % kparts, g = wl / kparts;
    const int b0 = p * prm.P;
    const int b1 = min(prm.nb, b0 + prm.P);

    fl_mbar_wait(bar_y, 0);
    fl_yprep yp[FL_RING_NBL];
    bool valid[FL_RING_NBL];
#pragma unroll
    for (int j = 0; j < FL_RING_NBL; j++) {
        const int ib = b0 + lane + 32 * j;
        valid[j] = (j < NFULL) || ib < b1;
        if (valid[j]) {
            fl_prep_y<TYPE>(ysm + ib, yp[j]);
        } else {
            yp[j].d = 0.f; yp[j].s = 0.f; yp[j].c = 0;
#pragma unroll
            for (int q = 0; q < 4; q++) { yp[j].ye[q] = 0; yp[j].yo[q] = 0; }
        }
    }

    // this warp consumes tiles tg, tg + TG, ...; stage of tile t is t % S, its use count t / S
    int s = tg % S;
    uint32_t ph = (uint32_t)(tg / S) & 1u;
    const int s_step = TG % S, u_step = TG / S;
    for (int t = tg; t < ntiles; t += TG) {
        fl_mbar_wait(bar0 + 8u * s, ph);
        const uint8_t *tile = stage0 + (size_t)s * prm.stage_bytes;
        const int rows = min(R, nrows - t * R);
        for (int rr = g; rr < rows; rr += G) {
            const uint8_t *wrow = tile + (size_t)rr * prm.row_bytes + (size_t)(b0 + lane) * BB;
            float acc = 0.0f, accm = 0.0f;
#pragma unroll
            for (int j = 0; j < FL_RING_NBL; j++) {
                if (j < NFULL) {
                    fl_ring_block<TYPE>(wrow + (size_t)(32 * j) * BB, yp[j], acc, accm);
                } else if (valid[j]) {
                    fl_ring_block<TYPE>(wrow + (size_t)(32 * j) * BB, yp[j], acc, accm);
                }
            }
            float tot = fl_warp_sum(acc);
            if (TYPE == FL_TYPE_Q4_1) tot = __fadd_rn(tot, fl_warp_sum(accm));
            if (lane == 0) {
                if (kparts == 1) prm.dst[r0 + t * R + rr] = tot;
                else partial[((size_t)s * R + rr) * kparts + p] = tot;
            }
        }
        __syncwarp();
        if (lane == 0) fl_mbar_arrive(bar0 + 8u * (S + s));      // this warp is done reading stage s
        if (kparts > 1) {
            // barrier of this tile-group's consumer warps only (ids 1..TG; the producer never joins)
            asm volatile("bar.sync %0, %1;" ::"r"(tg + 1), "r"(WPG * 32) : "memory");
            const int tl = (int)threadIdx.x - tg * WPG * 32;
            if (tl < rows) {
                const float *pp = partial + ((size_t)s * R + tl) * kparts;
                float tot = pp[0];
                for (int q = 1; q < kparts; q++) tot = __fadd_rn(tot, pp[q]);
                prm.dst[r0 + t * R + tl] = tot;
            }
        }
        s += s_step; ph ^= (uint32_t)(u_step & 1);
        if (s >= S) { s -= S; ph ^= 1u; }
    }
}

// =================================================================================================
// Launchers
// =================================================================================================
static int g_sm_count = 0;
static int g_smem_optin = 0;

int flk_query_device() {
    int dev = 0;
    FL_CUDA_OK(cudaGetDevice(&dev));
    FL_CUDA_OK(cudaDeviceGetAttribute(&g_sm_count, cudaDevAttrMultiProcessorCount, dev));
    FL_CUDA_OK(cudaDeviceGetAttribute(&g_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    return 0;
}
int flk_sm_count() { return g_sm_count; }

static inline int grid_for_warps(long nwarps, int threads) {
    const long wpb = threads / 32;
    long g = (nwarps + wpb - 1) / wpb;
    const long cap = (long)g_sm_count * 16;
    if (g > cap) g = cap;
    if (g < 1) g = 1;
    return (int)g;
}

int flk_quantize_q8_0(cudaStream_t st, const float *x, size_t x_row_stride_bytes, void *y, int k, int nrows) {
    FL_REQUIRE(k > 0 && k % FL_QK == 0, "quantize_q8_0: k=%d is not a multiple of 32", k);
    if (nrows <= 0) return 0;
    const long nblocks = (long)(k / FL_QK) * nrows;
    k_quantize_q8_0<<<grid_for_warps(nblocks, 256), 256, 0, st>>>(x, x_row_stride_bytes, (fl_block_q8_0 *)y, k, nrows);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

int flk_quantize_q4(cudaStream_t st, int type, const float *x, void *y, int k, int nrows) {
    FL_REQUIRE(k > 0 && k % FL_QK == 0, "quantize_q4: k=%d is not a multiple of 32", k);
    FL_REQUIRE(type == FL_TYPE_Q4_0 || type == FL_TYPE_Q4_1, "quantize_q4: unsupported type %d", type);
    if (nrows <= 0) return 0;
    const long nblocks = (long)(k / FL_QK) * nrows;
    if (type == FL_TYPE_Q4_0)
        k_quantize_q4_0<<<grid_for_warps(nblocks, 256), 256, 0, st>>>(x, (fl_block_q4_0 *)y, nblocks);
    else
        k_quantize_q4_1<<<grid_for_warps(nblocks, 256), 256, 0, st>>>(x, (fl_block_q4_1 *)y, nblocks);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

typedef void (*q4_file_kernel_t)(const void *, const void *, void *, long, unsigned long long *);
template <int TYPE>
static q4_file_kernel_t q4_file_kernel(int src_type, int delta_type) {
    if (delta_type == FL_DELTA_NONE) {
        switch (src_type) {
            case 0: return k_quantize_q4_file<TYPE, 0, FL_DELTA_NONE>;
            case 1: case 3: return k_quantize_q4_file<TYPE, 1, FL_DELTA_NONE>;      // the same values with nothing to merge
            case 2: return k_quantize_q4_file<TYPE, 2, FL_DELTA_NONE>;
        }
    } else if (delta_type == FL_DELTA_F32) {
        switch (src_type) {
            case 0: return k_quantize_q4_file<TYPE, 0, FL_DELTA_F32>;
            case 1: return k_quantize_q4_file<TYPE, 1, FL_DELTA_F32>;
            case 2: return k_quantize_q4_file<TYPE, 2, FL_DELTA_F32>;
            case 3: return k_quantize_q4_file<TYPE, 3, FL_DELTA_F32>;
        }
    } else if (delta_type == FL_DELTA_F16) {
        switch (src_type) {
            case 1: return k_quantize_q4_file<TYPE, 1, FL_DELTA_F16>;
            case 2: return k_quantize_q4_file<TYPE, 2, FL_DELTA_F16>;
        }
    }
    return nullptr;
}

int flk_quantize_q4_file_lora(cudaStream_t st, int type, int src_type, const void *x, int delta_type, const void *delta, void *y, int k,
                              int nrows, unsigned long long *hist) {
    FL_REQUIRE(k > 0 && k % FL_QK == 0, "quantize_q4_file: k=%d is not a multiple of 32", k);
    FL_REQUIRE(type == FL_TYPE_Q4_0 || type == FL_TYPE_Q4_1, "quantize_q4_file: unsupported type %d (q4_0 = 2, q4_1 = 3)", type);
    FL_REQUIRE(src_type >= 0 && src_type <= 3,
               "quantize_q4_file: unsupported source type %d (0 f32, 1 f16, 2 f32 via f16, 3 f16 of an f32 file)", src_type);
    FL_REQUIRE(delta_type >= FL_DELTA_NONE && delta_type <= FL_DELTA_F16, "quantize_q4_file: unsupported delta type %d (-1 none, 0 f32, 1 f16)",
               delta_type);
    FL_REQUIRE((delta_type == FL_DELTA_NONE) == (delta == nullptr), "quantize_q4_file: delta type %d with a %s delta buffer", delta_type,
               delta ? "non-null" : "null");
    FL_REQUIRE(!(delta_type == FL_DELTA_F16 && (src_type == 0 || src_type == 3)),
               "quantize_q4_file: an f16 delta cannot be merged into an f32 file (the reference's add_f32 has no f16 operand)");
    if (nrows <= 0) return 0;
    const long nblocks = (long)(k / FL_QK) * nrows;
    const q4_file_kernel_t kern = type == FL_TYPE_Q4_0 ? q4_file_kernel<FL_TYPE_Q4_0>(src_type, delta_type)
                                                       : q4_file_kernel<FL_TYPE_Q4_1>(src_type, delta_type);
    kern<<<grid_for_warps(nblocks, 256), 256, 0, st>>>(x, delta, y, nblocks, hist);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

int flk_quantize_q4_file(cudaStream_t st, int type, int src_type, const void *x, void *y, int k, int nrows,
                         unsigned long long *hist) {
    FL_REQUIRE(src_type >= 0 && src_type <= 2, "quantize_q4_file: unsupported source type %d (0 f32, 1 f16, 2 f32 via f16)",
               src_type);
    return flk_quantize_q4_file_lora(st, type, src_type, x, FL_DELTA_NONE, nullptr, y, k, nrows, hist);
}

int flk_dequantize_rows(cudaStream_t st, int type, const void *W, size_t w_row_stride, int K, const int32_t *ids,
                        int n_ids, float *dst, size_t dst_row_stride) {
    FL_REQUIRE(K > 0 && K % FL_QK == 0, "dequantize_rows: K=%d is not a multiple of 32", K);
    FL_REQUIRE(type == FL_TYPE_Q4_0 || type == FL_TYPE_Q4_1, "dequantize_rows: unsupported type %d", type);
    if (n_ids <= 0) return 0;
    const long total = (long)n_ids * (K / FL_QK) * 16;
    long g = (total + 255) / 256;
    if (g > (long)g_sm_count * 32) g = (long)g_sm_count * 32;
    if (type == FL_TYPE_Q4_0)
        k_dequantize_rows<FL_TYPE_Q4_0><<<(int)g, 256, 0, st>>>((const uint8_t *)W, w_row_stride, K, ids, n_ids, dst, dst_row_stride);
    else
        k_dequantize_rows<FL_TYPE_Q4_1><<<(int)g, 256, 0, st>>>((const uint8_t *)W, w_row_stride, K, ids, n_ids, dst, dst_row_stride);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

static int launch_plain(cudaStream_t st, int type, const void *W, size_t wrs, int M, int K, const void *Y, int N,
                        float *dst, size_t drs) {
    const int grid = grid_for_warps(M, 256);
    if (type == FL_TYPE_Q4_0)
        k_mul_mat_q_plain<FL_TYPE_Q4_0><<<grid, 256, 0, st>>>((const uint8_t *)W, wrs, M, K, (const fl_block_q8_0 *)Y, N, dst, drs);
    else
        k_mul_mat_q_plain<FL_TYPE_Q4_1><<<grid, 256, 0, st>>>((const uint8_t *)W, wrs, M, K, (const fl_block_q8_0 *)Y, N, dst, drs);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

// ring configuration for a given shape; returns false when the shape does not qualify
static bool ring_config(int type, const void *W, size_t wrs, int M, int K, fl_ring_params &p, int &threads,
                        size_t &smem_bytes, int &nfull) {
    const int bb = fl_block_bytes(type);
    const int nb = K / FL_QK;
    const size_t row_bytes = (size_t)nb * bb;
    if (wrs != row_bytes) return false;                       // rows must be contiguous (one bulk copy per tile)
    if (row_bytes % 16 != 0 || ((uintptr_t)W & 15) != 0) return false;
    if (((size_t)nb * 40) % 16 != 0) return false;            // activation vector is bulk-copied too
    const int kparts = (nb + 127) / 128;
    if (kparts > FL_RING_MAX_PARTS) return false;
    if (M < 2 * g_sm_count) return false;                     // too few rows to be worth a persistent grid
    const int P = (nb + kparts - 1) / kparts;
    const int last = nb - (kparts - 1) * P;                   // size of the last (smallest) part
    if (last <= 0) return false;
    nfull = std::min(P, last) / 32;
    if (nfull > FL_RING_NBL) nfull = FL_RING_NBL;
    // 16 consumer warps = TG tile-groups x G row-groups x kparts K-slices; a tile holds G rows (one
    // per row-group).  Smallest TG in {1,2,4} whose tile fits the target size (fine-grained ring:
    // data is usable as soon as one tile has landed, and several tiles are consumed concurrently).
    static int tile_target = -1;
    if (tile_target < 0) {
        const char *e = getenv("FASTLLAMA_B200_RING_TILE_KB");
        tile_target = (e ? atoi(e) : 24) * 1024;
    }
    const int Gmax = std::max(1, 16 / kparts);
    int G = Gmax, TG = 1;
    for (int tgc = 1; tgc <= 4; tgc *= 2) {
        const int gc = std::max(1, Gmax / tgc);
        G = gc; TG = tgc;
        if ((size_t)gc * row_bytes <= (size_t)tile_target || gc == 1) break;
    }
    const int R = G;
    const size_t stage_bytes = (size_t)R * row_bytes;          // multiple of 16
    const size_t y_bytes = (size_t)nb * 40;
    int S = FL_RING_MAX_STAGES;
    size_t off_y = 0, off_partial = 0, off = 0;
    for (;; S--) {
        if (S < 2) return false;
        off_y = ((size_t)(2 * S + 1) * 8 + 127) & ~(size_t)127;
        off_partial = (off_y + y_bytes + 127) & ~(size_t)127;
        off = off_partial + (size_t)S * R * kparts * sizeof(float);
        off = (off + 127) & ~(size_t)127;
        if (off + (size_t)S * stage_bytes <= (size_t)g_smem_optin) break;
    }
    if (TG > S) TG = S;
    const int CW = kparts * G * TG;
    p.M = M; p.nb = nb; p.row_bytes = (uint32_t)row_bytes; p.R = R; p.S = S; p.kparts = kparts; p.G = G; p.TG = TG; p.P = P;
    p.stage_bytes = (uint32_t)stage_bytes;
    p.y_bytes = (uint32_t)y_bytes;
    p.off_y = (uint32_t)off_y;
    p.off_partial = (uint32_t)off_partial;
    p.off_stage0 = (uint32_t)off;
    smem_bytes = off + (size_t)S * stage_bytes;
    threads = (CW + 1) * 32;
    return threads <= FL_RING_MAX_THREADS;
}

typedef void (*ring_kernel_t)(const fl_ring_params);
static ring_kernel_t ring_kernel(int type, int nfull) {
    if (type == FL_TYPE_Q4_0) {
        switch (nfull) {
            case 4: return k_matvec_q4_ring<FL_TYPE_Q4_0, 4>;
            case 3: return k_matvec_q4_ring<FL_TYPE_Q4_0, 3>;
            case 2: return k_matvec_q4_ring<FL_TYPE_Q4_0, 2>;
            case 1: return k_matvec_q4_ring<FL_TYPE_Q4_0, 1>;
            default: return k_matvec_q4_ring<FL_TYPE_Q4_0, 0>;
        }
    }
    switch (nfull) {
        case 4: return k_matvec_q4_ring<FL_TYPE_Q4_1, 4>;
        case 3: return k_matvec_q4_ring<FL_TYPE_Q4_1, 3>;
        case 2: return k_matvec_q4_ring<FL_TYPE_Q4_1, 2>;
        case 1: return k_matvec_q4_ring<FL_TYPE_Q4_1, 1>;
        default: return k_matvec_q4_ring<FL_TYPE_Q4_1, 0>;
    }
}

static int launch_ring(cudaStream_t st, int type, int nfull, fl_ring_params &p, int threads, size_t smem_bytes) {
    static bool attr_set[2][FL_RING_NBL + 1] = {{false}};
    const int ti = (type == FL_TYPE_Q4_0) ? 0 : 1;
    ring_kernel_t kern = ring_kernel(type, nfull);
    if (!attr_set[ti][nfull]) {
        FL_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, g_smem_optin));
        attr_set[ti][nfull] = true;
    }
    kern<<<g_sm_count, threads, smem_bytes, st>>>(p);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

// Fewest activation columns for which the tiled reference-order kernel beats k_mul_mat_q_ref (tools/time_exact_ingest.py).
#define FL_REF_TILED_MIN_N 8

int flk_mul_mat_q(cudaStream_t st, int type, const void *W, size_t wrs, int M, int K, const void *Yq8, int N,
                  float *dst, size_t drs, int impl) {
    FL_REQUIRE(type == FL_TYPE_Q4_0 || type == FL_TYPE_Q4_1, "mul_mat_q: unsupported weight type %d", type);
    FL_REQUIRE(K > 0 && K % FL_QK == 0, "mul_mat_q: K=%d is not a multiple of 32", K);
    FL_REQUIRE(((uintptr_t)W & 3) == 0 && (wrs & 3) == 0, "mul_mat_q: weight rows must be 4-byte aligned");
    if (M <= 0 || N <= 0) return 0;
    // impl 0 (what the graph executor passes): results carry the reference's bits -- the reference-order kernel of fl_exact_kernels.cu --
    // except for multi-token evals of N >= 16 columns, which go to the wgmma GEMM (same per-block arithmetic, block terms added in
    // another fp32 order: within the stated budget, not bit-identical) unless FASTLLAMA_B200_INGEST=exact.
    // The reference-order results come from the tiled kernel from FL_REF_TILED_MIN_N columns on, when its TMA copies take the operands
    // (16-byte aligned rows), and from the warp-per-8-rows kernel otherwise: the same arithmetic, the same bits.
    // The other kernels stay selectable for measurements and their own tests: 1 plain, 2 TMA ring matvec, 3 mma.sync,
    // 4-7 wgmma (column tile chosen / 32 / 64 / 64), 8 reference order (k_mul_mat_q_ref), 9 reference order tiled (k_mul_mat_q_ref_tiled).
    if (impl == 0) {
        static const int umma_auto = getenv("FASTLLAMA_B200_UMMA") ? atoi(getenv("FASTLLAMA_B200_UMMA")) : 1;     // FASTLLAMA_B200_UMMA=0: no tensor-core path
        const char *ing = getenv("FASTLLAMA_B200_INGEST");               // read per call: tests and callers may switch it between evals
        const bool exact_ingest = ing && !strcmp(ing, "exact");
        if (umma_auto && !exact_ingest && N >= 16 && flk_mul_mat_q_umma_supported(type, W, wrs, M, K, N)) return flk_mul_mat_q_umma(st, type, W, wrs, M, K, Yq8, N, dst, drs, 0);
        if (N >= FL_REF_TILED_MIN_N && flk_mul_mat_q_ref_tiled_supported(type, W, wrs, M, K, N)) return flk_mul_mat_q_ref_tiled(st, type, W, wrs, M, K, Yq8, N, dst, drs);
        return flk_mul_mat_q_ref(st, type, W, wrs, M, K, Yq8, N, dst, drs);
    }
    if (impl == 8) return flk_mul_mat_q_ref(st, type, W, wrs, M, K, Yq8, N, dst, drs);
    if (impl == 9) return flk_mul_mat_q_ref_tiled(st, type, W, wrs, M, K, Yq8, N, dst, drs);
    if (impl >= 4 && impl <= 7) return flk_mul_mat_q_umma(st, type, W, wrs, M, K, Yq8, N, dst, drs, impl == 4 ? 0 : 16 << (impl - 4));
    if (impl == 3) return flk_mul_mat_q_mma(st, type, W, wrs, M, K, Yq8, N, dst, drs);
    if (impl == 2) {
        fl_ring_params p;
        int threads = 0;
        size_t smem = 0;
        int nfull = 0;
        const bool ring_ok = (N == 1) && ring_config(type, W, wrs, M, K, p, threads, smem, nfull);
        FL_REQUIRE(ring_ok, "mul_mat_q: shape M=%d K=%d N=%d does not qualify for the ring kernel", M, K, N);
        p.W = (const uint8_t *)W;
        p.Y = (const fl_block_q8_0 *)Yq8;
        p.dst = dst;
        return launch_ring(st, type, nfull, p, threads, smem);
    }
    return launch_plain(st, type, W, wrs, M, K, Yq8, N, dst, drs);
}
