// fl_exact_kernels.cu -- matmuls whose fp32 results carry the reference's bits (fl_exact.cuh explains why that matters).
//
//   k_yx_prepare        q8_0 blocks -> prepared 80-byte blocks (per-quad words and biases)
//   k_mul_mat_q_ref     q4_0 / q4_1 weights x prepared activations, any M, K, N: 8 rows per warp, 4 lanes per row, blocks in
//                       order, NC activation columns per pass.  This is the general path (small prompts, shapes the token
//                       kernel or the wgmma GEMM do not take, FASTLLAMA_B200_INGEST=exact); the decode step runs the same
//                       arithmetic inside k_decode_token.
//   k_mul_mat_q_ref_tiled the same arithmetic as a tiled GEMM for multi-token evals: a CTA owns a 64-row x 32-column output
//                       tile, K streams through a 4-stage shared-memory ring (2-D TMA copies of raw q4 blocks and of prepared
//                       activation blocks, one producer lane, mbarriers), each consumer lane register-blocks 4 rows x 8 columns.
//   k_mul_mat_f32_ref4  f32 x f32 mul_mat on strided 4-D views (attention scores K.Q and the value mix V.P of a multi-token
//                       eval) in ggml_vec_dot_f32's order: lane l of a warp is element l of the reference's 32-float step.
#include <stdlib.h>

#include "fl_common.cuh"
#include "fl_exact.cuh"
#include "fl_kernels.h"
#include "fl_tma.cuh"

// one thread per (activation block, jj)
__global__ void __launch_bounds__(256) k_yx_prepare(const fl_block_q8_0 *__restrict__ y, fl_yx *__restrict__ out, long nblocks, int off) {
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nblocks * 4) return;
    const long b = t >> 2;
    const int jj = (int)(t & 3);
    const uint32_t *q = (const uint32_t *)y[b].qs + 2 * jj;
    const uint32_t ya = q[0], yb = q[1];
    *(uint4 *)out[b].q[jj] = make_uint4(ya, yb, fx_bias(ya, off), fx_bias(yb, off));
    if (jj == 0) { out[b].d = y[b].d; out[b].s = y[b].s; }
}

template <int TYPE, int NC>
__global__ void __launch_bounds__(128) k_mul_mat_q_ref(const uint8_t *__restrict__ W, size_t wrs, int M, int nb, const fl_yx *__restrict__ Y, int N,
                                                       float *__restrict__ dst, size_t drs) {
    constexpr int BB = (TYPE == FL_TYPE_Q4_0) ? 20 : 24, QOFF = (TYPE == FL_TYPE_Q4_0) ? 4 : 8;
    const int lane = threadIdx.x & 31, r = lane >> 2, jj = lane & 3;
    const long nwarps = (long)gridDim.x * (blockDim.x >> 5);
    const int ngroups = (M + 7) >> 3, ctiles = (N + NC - 1) / NC;
    for (long task = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); task < (long)ngroups * ctiles; task += nwarps) {
        const int grp = (int)(task % ngroups), ct = (int)(task / ngroups);
        const int row = min(grp * 8 + r, M - 1);
        const uint8_t *wr = W + (size_t)row * wrs;
        const fl_yx *yc[NC];
#pragma unroll
        for (int c = 0; c < NC; c++) yc[c] = Y + (size_t)min(ct * NC + c, N - 1) * nb;
        float a0[NC], a1[NC], sm[NC];
#pragma unroll
        for (int c = 0; c < NC; c++) a0[c] = a1[c] = sm[c] = 0.0f;
        for (int i = 0; i < nb; i++) {
            const uint8_t *blk = wr + (size_t)i * BB;
            const uint32_t w = __ldg((const uint32_t *)(blk + QOFF) + jj);
            const float dx = __ldg((const float *)blk);
            const float mx = (TYPE == FL_TYPE_Q4_1) ? __ldg((const float *)blk + 1) : 0.0f;
#pragma unroll
            for (int c = 0; c < NC; c++) {
                const uint4 y = __ldg((const uint4 *)yc[c][i].q[jj]);
                const float2 ds = __ldg((const float2 *)&yc[c][i].d);
                if (TYPE == FL_TYPE_Q4_1) sm[c] = __fmaf_rn(mx, ds.y, sm[c]);
                fx_block(w, __fmul_rn(dx, ds.x), y, a0[c], a1[c]);
            }
        }
#pragma unroll
        for (int c = 0; c < NC; c++) {
            float s = fx_reduce(a0[c], a1[c]);
            if (TYPE == FL_TYPE_Q4_1) s = __fadd_rn(s, sm[c]);
            const int n = ct * NC + c;
            if (jj == 0 && n < N && grp * 8 + r < M) dst[(size_t)n * drs + row] = s;
        }
    }
}

static fl_yx *g_yx = nullptr;
static size_t g_yx_cap = 0;

template <int TYPE>
static void launch_ref(cudaStream_t st, int nc, int grid, const uint8_t *W, size_t wrs, int M, int nb, const fl_yx *Y, int N, float *dst, size_t drs) {
    switch (nc) {
        case 1: k_mul_mat_q_ref<TYPE, 1><<<grid, 128, 0, st>>>(W, wrs, M, nb, Y, N, dst, drs); break;
        case 2: k_mul_mat_q_ref<TYPE, 2><<<grid, 128, 0, st>>>(W, wrs, M, nb, Y, N, dst, drs); break;
        case 4: k_mul_mat_q_ref<TYPE, 4><<<grid, 128, 0, st>>>(W, wrs, M, nb, Y, N, dst, drs); break;
        default: k_mul_mat_q_ref<TYPE, 8><<<grid, 128, 0, st>>>(W, wrs, M, nb, Y, N, dst, drs); break;
    }
}

// q8_0 rows -> the prepared blocks in g_yx ([N][nb] x 80 B), shared by both reference-order matmul kernels
static int yx_prepare(cudaStream_t st, int type, const void *Yq8, int N, int nb) {
    const size_t need = (size_t)N * nb * sizeof(fl_yx);
    if (need > g_yx_cap) {
        FL_CUDA_OK(cudaStreamSynchronize(st));                       // earlier launches may still read the old buffer
        if (g_yx) FL_CUDA_OK(cudaFree(g_yx));
        g_yx = nullptr; g_yx_cap = 0;
        const size_t cap = need + need / 2;
        FL_CUDA_OK(cudaMalloc((void **)&g_yx, cap));
        g_yx_cap = cap;
    }
    const long nblocks = (long)N * nb;
    k_yx_prepare<<<(int)((nblocks * 4 + 255) / 256), 256, 0, st>>>((const fl_block_q8_0 *)Yq8, g_yx, nblocks, type == FL_TYPE_Q4_0 ? 8 : 0);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

int flk_mul_mat_q_ref(cudaStream_t st, int type, const void *W, size_t wrs, int M, int K, const void *Yq8, int N, float *dst, size_t drs) {
    FL_REQUIRE(type == FL_TYPE_Q4_0 || type == FL_TYPE_Q4_1, "mul_mat_q_ref: unsupported weight type %d", type);
    FL_REQUIRE(K > 0 && K % FL_QK == 0, "mul_mat_q_ref: K=%d is not a multiple of 32", K);
    FL_REQUIRE(((uintptr_t)W & 3) == 0 && (wrs & 3) == 0, "mul_mat_q_ref: weight rows must be 4-byte aligned");
    if (M <= 0 || N <= 0) return 0;
    const int nb = K / FL_QK;
    if (yx_prepare(st, type, Yq8, N, nb)) return -1;
    const int nc = N >= 8 ? 8 : N >= 4 ? 4 : N >= 2 ? 2 : 1;
    const long tasks = (long)((M + 7) / 8) * ((N + nc - 1) / nc);
    long blocks = (tasks + 3) / 4;
    const long cap = (long)flk_sm_count() * 8;
    if (blocks > cap) blocks = cap;
    if (type == FL_TYPE_Q4_0) launch_ref<FL_TYPE_Q4_0>(st, nc, (int)blocks, (const uint8_t *)W, wrs, M, nb, g_yx, N, dst, drs);
    else launch_ref<FL_TYPE_Q4_1>(st, nc, (int)blocks, (const uint8_t *)W, wrs, M, nb, g_yx, N, dst, drs);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}
// ------------------------------------------------------------------------------------------------
// k_mul_mat_q_ref_tiled: k_mul_mat_q_ref's arithmetic, tiled.  Every output is still computed by the 4 lanes of one row group
// (fx_split / fx_block_split / fx_reduce), blocks 0 .. nb-1 in order: K is never split across lanes, warps or CTAs, because the
// reference's eight accumulators are sequential chains and any split would change the fp32 order.  What changes is where the
// operands come from: a CTA owns a QT_BM x QT_BN output tile and stages KC-block chunks of its weight rows (raw q4 blocks) and of
// its activation columns (80-byte prepared blocks) in shared memory, so each weight byte leaves HBM once per column tile instead
// of once per 8 columns, and each staged value is read from shared memory once per block for R rows or C columns.
//
//   warps 0 .. 7  consumers, QT_WR x QT_WC: warp (wr, wc) owns tile rows wr*32 + g + 8k (k < R, g = lane / 4) and tile
//                 columns wc*8 + c (c < C); lane jj = lane % 4 owns accumulators 2jj, 2jj + 1 of each of its R x C outputs.
//                 Per block a lane splits its R weight words once (reused for C columns) and loads its C activation entries
//                 once (reused for R rows).
//   warp 8        producer (one lane): per chunk one 2-D TMA box of raw weights (BM rows x KC blocks) and one of prepared
//                 activations (BN columns x KC blocks) into a QT_STAGES-deep mbarrier ring.  Rows, columns and blocks past the
//                 operands' ends are zero-filled by the TMA unit; the consumers never read those blocks, and never store those
//                 rows or columns.
//
// Shared-memory banks (tests/test_exact_gemm_math.py restates this): a weight row of a stage is RW = KC * BB / 4 words with
// RW % 8 == 4 (60 words for both types), so the 8 rows g of one load land on 8 disjoint 4-bank groups and the 4 lanes jj of a
// row read 4 consecutive words: 32 distinct banks.  The scale loads read one word per row (a broadcast over jj), again 8
// distinct banks.  All 32 lanes of a warp read the same activation column, so an activation load touches the 4 consecutive
// 16-byte entries of one block (broadcast over g) and its (d, s) pair is a single broadcast.
// ------------------------------------------------------------------------------------------------
#define QT_WR 2                                // consumer warps along rows
#define QT_WC 4                                // consumer warps along columns
#define QT_R 4                                 // rows per lane (g + 8k)
#define QT_C 8                                 // columns per warp
#define QT_BM (QT_WR * 8 * QT_R)               // 64 rows per CTA
#define QT_BN (QT_WC * QT_C)                   // 32 columns per CTA
#define QT_STAGES 4
#define QT_CONSUMERS (QT_WR * QT_WC)
#define QT_THREADS ((QT_CONSUMERS + 1) * 32)

template <int TYPE>
struct qt_layout {
    static constexpr int BB = (TYPE == FL_TYPE_Q4_0) ? 20 : 24;        // bytes per weight block
    static constexpr int WPB = BB / 4, QW = WPB - 4;                   // words per block, first nibble word
    static constexpr int KC = (TYPE == FL_TYPE_Q4_0) ? 12 : 10;        // blocks per chunk: RW % 8 == 4, KC * BB % 16 == 0
    static constexpr int RW = KC * WPB;                                // words per weight row of a stage
    static constexpr int YW = KC * (int)(sizeof(fl_yx) / 4);           // words per activation column of a stage (TMA box <= 256)
    static constexpr int A_BYTES = QT_BM * RW * 4;
    static constexpr int Y_BYTES = QT_BN * YW * 4;
    static constexpr int STAGE = A_BYTES + Y_BYTES;                    // a multiple of 128 (TMA destinations)
    static constexpr int OFF_BAR = QT_STAGES * STAGE;
    static constexpr int SMEM = OFF_BAR + 2 * QT_STAGES * 8;
    static_assert(RW % 8 == 4, "weight rows of a lane group must fall on disjoint bank groups");
    static_assert(A_BYTES % 128 == 0 && Y_BYTES % 128 == 0, "TMA destinations");
    static_assert(RW <= 256 && YW <= 256, "TMA box");
};

template <int TYPE>
__global__ void __launch_bounds__(QT_THREADS, 1) k_mul_mat_q_ref_tiled(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_y,
                                                                      int M, int N, int nb, int ntiles_n, float *__restrict__ dst, size_t drs) {
    using L = qt_layout<TYPE>;
    constexpr int R = QT_R, C = QT_C, SR = (TYPE == FL_TYPE_Q4_1) ? R : 1, SC = (TYPE == FL_TYPE_Q4_1) ? C : 1;
    extern __shared__ __align__(128) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile_n = blockIdx.x % ntiles_n, tile_m = blockIdx.x / ntiles_n;     // neighbouring CTAs share the weight rows (L2)
    const int m0 = tile_m * QT_BM, n0 = tile_n * QT_BN;
    const int nchunks = (nb + L::KC - 1) / L::KC;

    const uint32_t sm0 = fl_smem_u32(smem), bar0 = sm0 + L::OFF_BAR;
    auto full = [&](int s) { return bar0 + 8u * s; };
    auto empty = [&](int s) { return bar0 + 8u * (QT_STAGES + s); };
    if (threadIdx.x == 0) {
        for (int s = 0; s < QT_STAGES; s++) {
            fl_mbar_init(full(s), 1);
            fl_mbar_init(empty(s), QT_CONSUMERS);
        }
        fl_mbar_fence_init();
    }
    __syncthreads();

    if (warp < QT_CONSUMERS) {
        const int wr = warp % QT_WR, wc = warp / QT_WR;
        const int g = lane >> 2, jj = lane & 3;
        const int rt = wr * 8 * R + g, ct = wc * C;                    // tile row of k = 0, first tile column
        // a warp whose rows or columns all lie past the operands only keeps the ring turning
        const bool active = m0 + wr * 8 * R < M && n0 + ct < N;
        float a0[R][C], a1[R][C], sm[SR][SC];
#pragma unroll
        for (int k = 0; k < R; k++)
#pragma unroll
            for (int c = 0; c < C; c++) a0[k][c] = a1[k][c] = 0.0f;
#pragma unroll
        for (int k = 0; k < SR; k++)
#pragma unroll
            for (int c = 0; c < SC; c++) sm[k][c] = 0.0f;

        for (int ch = 0; ch < nchunks; ch++) {
            const int s = ch % QT_STAGES;
            fl_mbar_wait_bounded(full(s), (uint32_t)(ch / QT_STAGES) & 1u);
            if (active) {
                const uint32_t *ws = (const uint32_t *)(smem + (size_t)s * L::STAGE) + rt * L::RW;
                const fl_yx *ys = (const fl_yx *)(smem + (size_t)s * L::STAGE + L::A_BYTES) + ct * L::KC;
                const int kn = min(L::KC, nb - ch * L::KC);            // the last chunk may be short: blocks past nb are never read
#pragma unroll 1
                for (int i = 0; i < kn; i++) {
                    uint32_t wa[R], wb[R];
                    float dx[R], mx[SR];
#pragma unroll
                    for (int k = 0; k < R; k++) {
                        const uint32_t *blk = ws + k * 8 * L::RW + i * L::WPB;
                        dx[k] = __uint_as_float(blk[0]);
                        if (TYPE == FL_TYPE_Q4_1) mx[k % SR] = __uint_as_float(blk[1]);
                        fx_split(blk[L::QW + jj], wa[k], wb[k]);
                    }
#pragma unroll
                    for (int c = 0; c < C; c++) {
                        const fl_yx *yb = ys + c * L::KC + i;
                        const uint4 y = *(const uint4 *)yb->q[jj];
                        const float2 ds = *(const float2 *)&yb->d;
#pragma unroll
                        for (int k = 0; k < R; k++) {
                            if (TYPE == FL_TYPE_Q4_1) sm[k % SR][c % SC] = __fmaf_rn(mx[k % SR], ds.y, sm[k % SR][c % SC]);
                            fx_block_split(wa[k], wb[k], __fmul_rn(dx[k], ds.x), y, a0[k][c], a1[k][c]);
                        }
                    }
                }
            }
            __syncwarp();
            if (lane == 0) fl_mbar_arrive(empty(s));
        }
        if (active) {
#pragma unroll
            for (int k = 0; k < R; k++) {
                const int row = m0 + rt + 8 * k;
#pragma unroll
                for (int c = 0; c < C; c++) {
                    float v = fx_reduce(a0[k][c], a1[k][c]);
                    if (TYPE == FL_TYPE_Q4_1) v = __fadd_rn(v, sm[k % SR][c % SC]);
                    const int col = n0 + ct + c;
                    if (jj == 0 && row < M && col < N) dst[(size_t)col * drs + row] = v;
                }
            }
        }
    } else if (lane == 0) {
        for (int ch = 0; ch < nchunks; ch++) {
            const int s = ch % QT_STAGES;
            fl_mbar_wait_bounded(empty(s), ((uint32_t)(ch / QT_STAGES) & 1u) ^ 1u);
            const uint32_t st = sm0 + (uint32_t)(s * L::STAGE);
            fl_mbar_expect_tx(full(s), (uint32_t)L::STAGE);
            fl_tma_2d(st, &tmap_w, ch * L::RW, m0, full(s));
            fl_tma_2d(st + L::A_BYTES, &tmap_y, ch * L::YW, n0, full(s));
        }
    }
}

int flk_mul_mat_q_ref_tiled_supported(int type, const void *W, size_t wrs, int M, int K, int N) {
    if (type != FL_TYPE_Q4_0 && type != FL_TYPE_Q4_1) return 0;
    if (((uintptr_t)W & 15) != 0 || (wrs & 15) != 0 || K <= 0 || K % FL_QK != 0 || M < 1 || N < 1) return 0;   // TMA: 16-byte base and row stride
    return fl_tma_get_encode() != nullptr;
}

template <int TYPE>
static int launch_ref_tiled(cudaStream_t st, const void *W, size_t wrs, int M, int nb, int N, float *dst, size_t drs) {
    using L = qt_layout<TYPE>;
    CUtensorMap tw, ty;
    const cuuint32_t estr[2] = {1, 1};
    const cuuint64_t wdim[2] = {(cuuint64_t)nb * L::WPB, (cuuint64_t)M}, wstr[1] = {(cuuint64_t)wrs};
    const cuuint32_t wbox[2] = {(cuuint32_t)L::RW, (cuuint32_t)QT_BM};
    CUresult cr = fl_tma_get_encode()(&tw, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, (void *)W, wdim, wstr, wbox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                      CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    FL_REQUIRE(cr == CUDA_SUCCESS, "mul_mat_q_ref_tiled: cuTensorMapEncodeTiled failed (%d) for weights M=%d nb=%d stride=%zu", (int)cr, M, nb, wrs);
    const cuuint64_t ydim[2] = {(cuuint64_t)nb * (sizeof(fl_yx) / 4), (cuuint64_t)N}, ystr[1] = {(cuuint64_t)nb * sizeof(fl_yx)};
    const cuuint32_t ybox[2] = {(cuuint32_t)L::YW, (cuuint32_t)QT_BN};
    cr = fl_tma_get_encode()(&ty, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, (void *)g_yx, ydim, ystr, ybox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    FL_REQUIRE(cr == CUDA_SUCCESS, "mul_mat_q_ref_tiled: cuTensorMapEncodeTiled failed (%d) for activations N=%d nb=%d", (int)cr, N, nb);
    static bool attr_done = false;
    if (!attr_done) {
        FL_CUDA_OK(cudaFuncSetAttribute(k_mul_mat_q_ref_tiled<TYPE>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::SMEM));
        attr_done = true;
    }
    const int ntiles_n = (N + QT_BN - 1) / QT_BN, ntiles_m = (M + QT_BM - 1) / QT_BM;
    k_mul_mat_q_ref_tiled<TYPE><<<ntiles_m * ntiles_n, QT_THREADS, L::SMEM, st>>>(tw, ty, M, N, nb, ntiles_n, dst, drs);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

int flk_mul_mat_q_ref_tiled(cudaStream_t st, int type, const void *W, size_t wrs, int M, int K, const void *Yq8, int N, float *dst, size_t drs) {
    FL_REQUIRE(flk_mul_mat_q_ref_tiled_supported(type, W, wrs, M, K, N),
               "mul_mat_q_ref_tiled: unsupported operands (type %d, W %p, stride %zu, M %d, K %d, N %d; needs q4_0 / q4_1 with 16-byte aligned rows)",
               type, W, wrs, M, K, N);
    const int nb = K / FL_QK;
    if (yx_prepare(st, type, Yq8, N, nb)) return -1;
    if (type == FL_TYPE_Q4_0) return launch_ref_tiled<FL_TYPE_Q4_0>(st, W, wrs, M, nb, N, dst, drs);
    return launch_ref_tiled<FL_TYPE_Q4_1>(st, W, wrs, M, nb, N, dst, drs);
}

void flk_exact_release() {
    if (g_yx) cudaFree(g_yx);
    g_yx = nullptr;
    g_yx_cap = 0;
}

// ------------------------------------------------------------------------------------------------
// f32 x f32 -> f32 mul_mat on strided views, reference summation order (reference lib/ggml.c:7482-7680 calls ggml_vec_dot_f32 per output).
// One warp per (src0 row, CT consecutive src1 rows) of an (i2, i3) slice.
// ------------------------------------------------------------------------------------------------
#define MF_CT 8
// 3 CTAs per SM (<= 80 registers): the kernel is a stream of L1/L2 hits, occupancy is what hides them.  (The first version let ptxas
// unroll the k loop into 202 registers = 8 warps per SM: 535 us per attention product of a 128-token eval, half of the eval.)
__global__ void __launch_bounds__(256, 3) k_mul_mat_f32_ref4(const fl_view a, const fl_view b, const fl_view d) {
    const int lane = threadIdx.x & 31;
    const int K = (int)a.ne[0], np = K & ~31;
    const int64_t M0 = d.ne[0], M1 = d.ne[1];
    const int64_t ct = (M1 + MF_CT - 1) / MF_CT;
    const int64_t total = M0 * ct * d.ne[2] * d.ne[3];
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    const int64_t xs = a.nb[0], ys = b.nb[0], yr = b.nb[1];
    for (int64_t t = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); t < total; t += nwarps) {
        int64_t r = t;
        // consecutive warps: consecutive src0 rows against the SAME src1 rows (which then come from L1)
        const int64_t i0 = r % M0; r /= M0;
        const int64_t c1 = r % ct; r /= ct;
        const int64_t i2 = r % d.ne[2];
        const int64_t i3 = r / d.ne[2];
        const char *x = (const char *)a.data + i0 * a.nb[1] + i2 * a.nb[2] + i3 * a.nb[3];
        const char *y0 = (const char *)b.data + (c1 * MF_CT) * yr + i2 * b.nb[2] + i3 * b.nb[3];
        const int ncol = (int)min((int64_t)MF_CT, M1 - c1 * MF_CT);
        float acc[MF_CT];
        int yoff[MF_CT];                               // column offsets fit 32 bits (8 rows of one operand)
#pragma unroll
        for (int c = 0; c < MF_CT; c++) { acc[c] = 0.0f; yoff[c] = (int)((int64_t)min(c, ncol - 1) * yr); }
#pragma unroll 1
        for (int k = lane; k < np; k += 32) {
            const float xv = *(const float *)(x + (int64_t)k * xs);
            const char *yk = y0 + (int64_t)k * ys;
#pragma unroll
            for (int c = 0; c < MF_CT; c++) acc[c] = __fmaf_rn(xv, *(const float *)(yk + yoff[c]), acc[c]);
        }
        const int rem = K - np, nma = fx_left_nma(rem);
        // lane l fetches leftover element np + l; the sum is continued in order through shuffles (fx_left_nma: products-then-adds, then fmas)
        const float lx = (lane < rem) ? *(const float *)(x + (int64_t)(np + lane) * xs) : 0.0f;
#pragma unroll
        for (int c = 0; c < MF_CT; c++) {
            const float ly = (lane < rem) ? *(const float *)(y0 + yoff[c] + (int64_t)(np + lane) * ys) : 0.0f;
            float s = fx_reduce_f32(acc[c]);
            const float lp = __fmul_rn(lx, ly);
            for (int k = 0; k < nma; k++) s = __fadd_rn(s, __shfl_sync(0xffffffffu, lp, k));
            for (int k = nma; k < rem; k++) s = __fmaf_rn(__shfl_sync(0xffffffffu, lx, k), __shfl_sync(0xffffffffu, ly, k), s);
            if (lane == 0 && c < ncol) *(float *)((char *)d.data + i0 * d.nb[0] + (c1 * MF_CT + c) * d.nb[1] + i2 * d.nb[2] + i3 * d.nb[3]) = s;
        }
    }
}
int flk_mul_mat_f32_ref4(cudaStream_t st, const fl_view &a, const fl_view &b, const fl_view &d) {
    FL_REQUIRE(a.ne[0] == b.ne[0] && d.ne[0] == a.ne[1] && d.ne[1] == b.ne[1], "mul_mat_f32: shapes do not match");
    FL_REQUIRE(a.ne[2] == b.ne[2] && a.ne[3] == b.ne[3] && d.ne[2] == a.ne[2] && d.ne[3] == a.ne[3], "mul_mat_f32: batch dims do not match");
    const int64_t total = d.ne[0] * ((d.ne[1] + MF_CT - 1) / MF_CT) * d.ne[2] * d.ne[3];
    if (total <= 0 || a.ne[0] <= 0) return 0;
    int64_t blocks = (total + 7) / 8;
    const int64_t cap = (int64_t)flk_sm_count() * 3 * 8;          // 3 resident CTAs per SM, a few waves
    if (blocks > cap) blocks = cap;
    k_mul_mat_f32_ref4<<<(int)blocks, 256, 0, st>>>(a, b, d);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}
