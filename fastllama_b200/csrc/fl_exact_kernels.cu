// fl_exact_kernels.cu -- matmuls whose fp32 results carry the reference's bits (fl_exact.cuh explains why that matters).
//
//   k_yx_prepare        q8_0 blocks -> prepared 80-byte blocks (per-quad words and biases)
//   k_mul_mat_q_ref     q4_0 / q4_1 weights x prepared activations, any M, K, N: 8 rows per warp, 4 lanes per row, blocks in
//                       order, NC activation columns per pass.  This is the general path (small prompts, shapes the token
//                       kernel or the wgmma GEMM do not take, FASTLLAMA_B200_INGEST=exact); the decode step runs the same
//                       arithmetic inside k_decode_token.
//   k_mul_mat_f32_ref4  f32 x f32 mul_mat on strided 4-D views (attention scores K.Q and the value mix V.P of a multi-token
//                       eval) in ggml_vec_dot_f32's order: lane l of a warp is element l of the reference's 32-float step.
#include <stdlib.h>

#include "fl_common.cuh"
#include "fl_exact.cuh"
#include "fl_kernels.h"

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

int flk_mul_mat_q_ref(cudaStream_t st, int type, const void *W, size_t wrs, int M, int K, const void *Yq8, int N, float *dst, size_t drs) {
    FL_REQUIRE(type == FL_TYPE_Q4_0 || type == FL_TYPE_Q4_1, "mul_mat_q_ref: unsupported weight type %d", type);
    FL_REQUIRE(K > 0 && K % FL_QK == 0, "mul_mat_q_ref: K=%d is not a multiple of 32", K);
    FL_REQUIRE(((uintptr_t)W & 3) == 0 && (wrs & 3) == 0, "mul_mat_q_ref: weight rows must be 4-byte aligned");
    if (M <= 0 || N <= 0) return 0;
    const int nb = K / FL_QK;
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
