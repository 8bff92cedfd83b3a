// fl_mma_kernel.cu -- ggml_compute_forward_mul_mat_q_f32 for N > 1 (prompt ingest) on the tensor cores.
//
// Reference semantics (lib/ggml.c:8125-8163 + :2368-2714): dst[n][m] = sum over 32-element blocks kb of
//     d_w[m][kb] * d_y[n][kb] * ( sum_i (q4[m][kb][i] - 8) * q8[n][kb][i] )            (q4_0)
//     d_w * d_y * sum_i q4 * q8  +  m_w[m][kb] * s_y[n][kb]                            (q4_1)
// with an exact integer sum per block and fp32 accumulation over blocks.  The integer block sums are what
// the tensor cores compute here: one mma.sync.m16n8k32 (u8 x s8 -> s32) is exactly 16 weight rows x 8
// activation columns x one 32-element block.  The per-block scales stay in fp32 on the CUDA cores
// (I2F, d_w * d_y, FFMA per output and block), as in every other kernel of this backend, so the result
// differs from the reference only in the order of the fp32 additions over blocks (sequential here).
//
// The nibbles never get expanded to a byte plane in memory: with the MMA's k index ordered as
// "low nibbles of qs[0..15], then high nibbles of qs[0..15]", thread (g, t) of the warp builds its A
// fragment from ONE 32-bit word of the block ((w & 0x0F0F0F0F) and ((w >> 4) & 0x0F0F0F0F) for rows g
// and g + 8), and the matching B fragment is the even / odd byte planes (ye[t], yo[t]) of the q8_0
// block -- the same prepared layout the decode kernels use.  The -8 of q4_0 is folded in as
// c[n][kb] = -8 * sum(q8), added to the integer result.
//
#include "fl_common.cuh"
#include "fl_kernels.h"

#define MM_ROWS 32            // weight rows per CTA: 2 row groups of 16
#define MM_COLS 128           // activation columns per pass: 2 column groups of 64
#define MM_THREADS 128

struct __align__(16) mm_yblock {
    uint32_t ye[4], yo[4];
    float d, s;
    int c, pad;
};

__device__ __forceinline__ void mm_mma(int c[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%10, %10, %10, %10};"
                 : "=r"(c[0]), "=r"(c[1]), "=r"(c[2]), "=r"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1), "r"(0));
}

#define MM_KC 4               // k-blocks staged per barrier (2 x 4 x 128 prepared blocks = 48 KB of static shared memory)

template <int TYPE>
__global__ void __launch_bounds__(MM_THREADS)
k_mul_mat_q_mma(const uint8_t *__restrict__ W, size_t w_row_stride, int M, int K, const fl_block_q8_0 *__restrict__ Y, int N,
                float *__restrict__ dst, size_t dst_row_stride) {
    constexpr int BB = (TYPE == FL_TYPE_Q4_0) ? 20 : 24;
    constexpr int QOFF = (TYPE == FL_TYPE_Q4_0) ? 1 : 2;      // word offset of qs inside a block
    __shared__ mm_yblock ysm[2][MM_KC][MM_COLS];
    const int nb = K / FL_QK;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;
    const int rg = warp & 1, cg = warp >> 1;                  // row group (16 rows), column group (64 columns)
    const int row_a = blockIdx.x * MM_ROWS + rg * 16 + g, row_b = row_a + 8;
    const uint8_t *wa = W + (size_t)min(row_a, M - 1) * w_row_stride;       // clamped: tail rows compute garbage that is never stored
    const uint8_t *wb = W + (size_t)min(row_b, M - 1) * w_row_stride;

    for (int n0 = 0; n0 < N; n0 += MM_COLS) {
        const int ncols = min(MM_COLS, N - n0);
        const int ntiles = max(0, min(8, (ncols - cg * 64 + 7) / 8));       // 8-column tiles of this warp
        float acc[8][4], accm[8][4];
#pragma unroll
        for (int j = 0; j < 8; j++)
#pragma unroll
            for (int e = 0; e < 4; e++) { acc[j][e] = 0.f; accm[j][e] = 0.f; }

        // stage the activation blocks of k-blocks [kb0, kb0 + MM_KC) for all columns of this pass: thread n prepares column n
        auto stage = [&](int kb0, int buf) {
            const int n = threadIdx.x;
            if (n < ncols) {
#pragma unroll
                for (int i = 0; i < MM_KC; i++) {
                    if (kb0 + i < nb) {
                        const fl_block_q8_0 *yb = Y + (size_t)(n0 + n) * nb + kb0 + i;
                        const uint32_t *q = (const uint32_t *)yb->qs;
                        mm_yblock o;
                        int sum = 0;
#pragma unroll
                        for (int j = 0; j < 4; j++) {
                            const uint32_t a = __ldg(q + 2 * j), b = __ldg(q + 2 * j + 1);
                            o.ye[j] = __byte_perm(a, b, 0x6420);
                            o.yo[j] = __byte_perm(a, b, 0x7531);
                            sum = fl_dp4a_ss(0x01010101u, a, sum);
                            sum = fl_dp4a_ss(0x01010101u, b, sum);
                        }
                        o.d = __ldg(&yb->d);
                        o.s = __ldg(&yb->s);
                        o.c = -8 * sum;
                        o.pad = 0;
                        ysm[buf][i][n] = o;
                    }
                }
            }
        };
        stage(0, 0);
        __syncthreads();
        for (int kb0 = 0; kb0 < nb; kb0 += MM_KC) {
            const int buf = (kb0 / MM_KC) & 1;
            // A fragments of the whole chunk first (independent loads in flight), then the next chunk's activations
            uint32_t qa[MM_KC], qb[MM_KC];
            float da[MM_KC], db[MM_KC], ma[MM_KC], mb[MM_KC];
#pragma unroll
            for (int i = 0; i < MM_KC; i++) {
                const int kb = min(kb0 + i, nb - 1);
                const uint32_t *ba = (const uint32_t *)(wa + (size_t)kb * BB), *bbp = (const uint32_t *)(wb + (size_t)kb * BB);
                qa[i] = __ldg(ba + QOFF + t); qb[i] = __ldg(bbp + QOFF + t);
                da[i] = __uint_as_float(__ldg(ba)); db[i] = __uint_as_float(__ldg(bbp));
                ma[i] = mb[i] = 0.f;
                if (TYPE == FL_TYPE_Q4_1) { ma[i] = __uint_as_float(__ldg(ba + 1)); mb[i] = __uint_as_float(__ldg(bbp + 1)); }
            }
            if (kb0 + MM_KC < nb) stage(kb0 + MM_KC, buf ^ 1);   // read by nobody until the barrier at the end of this iteration
#pragma unroll
            for (int i = 0; i < MM_KC; i++) {
                if (kb0 + i < nb) {
                    const uint32_t a0 = qa[i] & 0x0F0F0F0Fu, a1 = qb[i] & 0x0F0F0F0Fu, a2 = (qa[i] >> 4) & 0x0F0F0F0Fu, a3 = (qb[i] >> 4) & 0x0F0F0F0Fu;
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        if (j < ntiles) {
                            const int cb = cg * 64 + 8 * j;           // first column of the tile (relative to n0)
                            const mm_yblock &yb = ysm[buf][i][min(cb + g, ncols - 1)];
                            int c[4];
                            mm_mma(c, a0, a1, a2, a3, yb.ye[t], yb.yo[t]);
                            // outputs of this thread: (row_a, cb + 2t), (row_a, cb + 2t + 1), (row_b, cb + 2t), (row_b, cb + 2t + 1)
                            const mm_yblock &y0 = ysm[buf][i][min(cb + 2 * t, ncols - 1)], &y1 = ysm[buf][i][min(cb + 2 * t + 1, ncols - 1)];
                            const float d0 = y0.d, d1 = y1.d;
                            if (TYPE == FL_TYPE_Q4_0) { c[0] += y0.c; c[1] += y1.c; c[2] += y0.c; c[3] += y1.c; }
                            acc[j][0] = __fmaf_rn(__fmul_rn(da[i], d0), (float)c[0], acc[j][0]);
                            acc[j][1] = __fmaf_rn(__fmul_rn(da[i], d1), (float)c[1], acc[j][1]);
                            acc[j][2] = __fmaf_rn(__fmul_rn(db[i], d0), (float)c[2], acc[j][2]);
                            acc[j][3] = __fmaf_rn(__fmul_rn(db[i], d1), (float)c[3], acc[j][3]);
                            if (TYPE == FL_TYPE_Q4_1) {
                                const float s0 = y0.s, s1 = y1.s;
                                accm[j][0] = __fmaf_rn(ma[i], s0, accm[j][0]);
                                accm[j][1] = __fmaf_rn(ma[i], s1, accm[j][1]);
                                accm[j][2] = __fmaf_rn(mb[i], s0, accm[j][2]);
                                accm[j][3] = __fmaf_rn(mb[i], s1, accm[j][3]);
                            }
                        }
                    }
                }
            }
            __syncthreads();
        }
#pragma unroll
        for (int j = 0; j < 8; j++) {
            if (j < ntiles) {
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    const int row = (e < 2) ? row_a : row_b;
                    const int col = n0 + cg * 64 + 8 * j + 2 * t + (e & 1);
                    if (row < M && col < N) {
                        const float v = (TYPE == FL_TYPE_Q4_1) ? __fadd_rn(acc[j][e], accm[j][e]) : acc[j][e];
                        dst[(size_t)col * dst_row_stride + row] = v;
                    }
                }
            }
        }
        __syncthreads();                                      // the next pass re-stages buffer 0
    }
}

int flk_mul_mat_q_mma(cudaStream_t st, int type, const void *W, size_t wrs, int M, int K, const void *Yq8, int N, float *dst, size_t drs) {
    const int grid = (M + MM_ROWS - 1) / MM_ROWS;
    if (type == FL_TYPE_Q4_0)
        k_mul_mat_q_mma<FL_TYPE_Q4_0><<<grid, MM_THREADS, 0, st>>>((const uint8_t *)W, wrs, M, K, (const fl_block_q8_0 *)Yq8, N, dst, drs);
    else
        k_mul_mat_q_mma<FL_TYPE_Q4_1><<<grid, MM_THREADS, 0, st>>>((const uint8_t *)W, wrs, M, K, (const fl_block_q8_0 *)Yq8, N, dst, drs);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}
