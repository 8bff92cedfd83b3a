// fl_umma_kernel.cu -- ggml_compute_forward_mul_mat_q_f32 for N > 1 (prompt ingest, n_batch = 128) on the
// Hopper tensor cores: wgmma.mma_async with 8-bit integer operands, weights fetched by TMA.
//
// Reference semantics (lib/ggml.c:8105-8163 with ne11 = N, over :2445-2487 / :2639-2687):
//     dst[n][m] = sum over 32-element blocks kb of
//         d_w[m][kb] * d_y[n][kb] * ( sum_i (q4[m][kb][i] - 8) * q8[n][kb][i] )            (q4_0)
//         d_w * d_y * sum_i q4 * q8  +  m_w[m][kb] * s_y[n][kb]                            (q4_1)
// The per-block integer sum is exact in the reference and the scales are fp32.  ONE wgmma with M = 64,
// N = NT, K = 32 (8-bit operands) is exactly one quant block for 64 weight rows x NT activation columns, so
// the kernel issues one MMA per k-block into a fresh register accumulator (scale-d = 0: no accumulation
// across blocks on the tensor core) and the same warpgroup does the reference's fp32 step
// acc = fma(d_w * d_y, float(isum), acc) on the CUDA cores.  Two accumulator sets alternate, so the MMA of
// block kb + 1 runs while the epilogue of block kb does.  Result: exactly the arithmetic of every other kernel
// of this backend (exact block sums, fp32 scales, blocks added sequentially), so the same 2e-6 * sum|d q| budget.
//
// Roles (160 threads, one CTA per 64-row x NT-column output tile):
//   warps 0-3   one consumer warpgroup.  Thread (warp w, lane 4g + t) builds its A fragment (rows 16w + g and
//               16w + g + 8, k = 4t .. 4t + 3 and 16 + 4t .. 16 + 4t + 3) straight from ONE 32-bit word of each
//               raw q4 block in shared memory: the k index inside a block is permuted to "16 low nibbles, then
//               16 high nibbles" (= even elements, then odd elements), the activations are stored in the same
//               order, and integer sums do not care.  q4_0: bytes are (q - 8) as s8; q4_1: q as u8.  B (the
//               activations) is read by the tensor core from shared memory through a matrix descriptor.
//   warp 4      TMA producer: weights by cp.async.bulk.tensor.2d (SASS UTMALDG), prepared activations and their
//               scales by 1-D bulk copies, into a 4-stage mbarrier ring.
#include <cuda.h>
#include <stdlib.h>

#include "fl_common.cuh"
#include "fl_kernels.h"
#include "fl_tma.cuh"

#define UM_M 64               // weight rows per CTA = the M of one wgmma
#define UM_KC 4               // k-blocks per TMA stage
#define UM_STAGES 4
#define UM_THREADS (4 * 32 + 32)

// ---- PTX wrappers --------------------------------------------------------------------------------
// K-major operand, no swizzle: core matrix = 8 rows x 16 bytes, contiguous (128 B); LBO = byte distance between the two
// 16-byte K halves, SBO = byte distance between 8-row groups (wgmma matrix descriptor, swizzle mode 0)
__device__ __forceinline__ uint64_t um_smem_desc(uint32_t addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((addr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(sbo_bytes >> 4) << 32);
}
__device__ __forceinline__ void um_wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void um_wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void um_wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from touching accumulator registers while an MMA that writes them may be in flight
template <int R>
__device__ __forceinline__ void um_fence_regs(int32_t (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; i++) asm volatile("" : "+r"(d[i])::"memory");
}

// D[regs] = A[regs] * B[smem], s32 accumulator, D not read (scale-d = 0).  A: s8 (q4_0, q - 8) or u8 (q4_1); B: s8.
#define UM_R8(i) "+r"(d[i + 0]), "+r"(d[i + 1]), "+r"(d[i + 2]), "+r"(d[i + 3]), "+r"(d[i + 4]), "+r"(d[i + 5]), "+r"(d[i + 6]), "+r"(d[i + 7])
template <int NT, bool A_S8>
__device__ __forceinline__ void um_mma(int32_t (&d)[NT / 2], const uint32_t (&a)[4], uint64_t bdesc);
template <>
__device__ __forceinline__ void um_mma<32, true>(int32_t (&d)[16], const uint32_t (&a)[4], uint64_t bdesc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
                 "{%16, %17, %18, %19}, %20, p;\n\t}"
                 : UM_R8(0), UM_R8(8)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(0));
}
template <>
__device__ __forceinline__ void um_mma<32, false>(int32_t (&d)[16], const uint32_t (&a)[4], uint64_t bdesc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k32.s32.u8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
                 "{%16, %17, %18, %19}, %20, p;\n\t}"
                 : UM_R8(0), UM_R8(8)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(0));
}
#define UM_D64 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}"
template <>
__device__ __forceinline__ void um_mma<64, true>(int32_t (&d)[32], const uint32_t (&a)[4], uint64_t bdesc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 " UM_D64 ", {%32, %33, %34, %35}, %36, p;\n\t}"
                 : UM_R8(0), UM_R8(8), UM_R8(16), UM_R8(24)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(0));
}
template <>
__device__ __forceinline__ void um_mma<64, false>(int32_t (&d)[32], const uint32_t (&a)[4], uint64_t bdesc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k32.s32.u8.s8 " UM_D64 ", {%32, %33, %34, %35}, %36, p;\n\t}"
                 : UM_R8(0), UM_R8(8), UM_R8(16), UM_R8(24)
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(0));
}

struct um_params {
    const uint8_t *yq;          // prepared activations: [ntiles][nbp][2][NT][16] bytes (even elements, odd elements)
    const float *dy, *sy;       // [ntiles][nbp][NT]
    float *dst;
    size_t dst_row_stride;
    int M, N, nbp;              // nbp = k-blocks padded to a multiple of UM_KC
    int ntiles;                 // column tiles
};

template <int TYPE, int NT>
struct um_layout {
    static constexpr int BB = (TYPE == FL_TYPE_Q4_0) ? 20 : 24;
    static constexpr int RAW_A = UM_M * UM_KC * BB;                      // TMA box: 64 rows x KC blocks
    static constexpr int RAW_B = UM_KC * NT * 32;
    static constexpr int RAW_S = UM_KC * NT * 4;
    static constexpr int NSC = (TYPE == FL_TYPE_Q4_1) ? 2 : 1;           // scale arrays per stage (dy [, sy])
    static constexpr int STAGE = RAW_A + RAW_B + NSC * RAW_S;            // a multiple of 128 (TMA destinations)
    static constexpr int OFF_BAR = UM_STAGES * STAGE;
    static constexpr int SMEM = OFF_BAR + 2 * UM_STAGES * 8;
};

// ---- activations: q8_0 rows -> the operand layout of the MMA ------------------------------------------
// One thread per (column n, k-block kb) of the PADDED domain [ntiles * NT][nbp]; padding is written as zeros
// (d = 0, q = 0: contributes exactly +0 to every sum).
template <int NT>
__global__ void k_umma_prep(const fl_block_q8_0 *__restrict__ Y, int N, int nb, int nbp, uint8_t *__restrict__ yq, float *__restrict__ dy,
                            float *__restrict__ sy) {
    const int kb = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = blockIdx.y;
    if (kb >= nbp) return;
    const int tile = n / NT, nl = n % NT;
    uint4 ev = make_uint4(0, 0, 0, 0), od = make_uint4(0, 0, 0, 0);
    float d = 0.f, s = 0.f;
    if (n < N && kb < nb) {
        const fl_block_q8_0 *yb = Y + (size_t)n * nb + kb;
        const uint32_t *q = (const uint32_t *)yb->qs;
        uint32_t e[4], o[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const uint32_t a = __ldg(q + 2 * j), b = __ldg(q + 2 * j + 1);
            e[j] = __byte_perm(a, b, 0x6420);
            o[j] = __byte_perm(a, b, 0x7531);
        }
        ev = make_uint4(e[0], e[1], e[2], e[3]);
        od = make_uint4(o[0], o[1], o[2], o[3]);
        d = __ldg(&yb->d);
        s = __ldg(&yb->s);
    }
    uint8_t *base = yq + ((size_t)tile * nbp + kb) * (size_t)(NT * 32);
    *(uint4 *)(base + (size_t)nl * 16) = ev;
    *(uint4 *)(base + (size_t)NT * 16 + (size_t)nl * 16) = od;
    dy[((size_t)tile * nbp + kb) * NT + nl] = d;
    sy[((size_t)tile * nbp + kb) * NT + nl] = s;
}

template <int TYPE, int NT>
__global__ void __launch_bounds__(UM_THREADS) k_mul_mat_q_umma(const __grid_constant__ CUtensorMap tmap_w, const um_params prm) {
    using L = um_layout<TYPE, NT>;
    constexpr int BB = L::BB, WPB = BB / 4, QOFF = WPB - 4;           // words per block, first qs word
    constexpr int R = NT / 2;                                          // accumulator registers per thread
    extern __shared__ __align__(1024) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile_n = blockIdx.x % prm.ntiles, tile_m = blockIdx.x / prm.ntiles;
    const int m0 = tile_m * UM_M, n0 = tile_n * NT;
    const int nstages = prm.nbp / UM_KC;

    const uint32_t sm0 = fl_smem_u32(smem);
    const uint32_t bar0 = sm0 + L::OFF_BAR;
    auto raw_full = [&](int s) { return bar0 + 8u * s; };
    auto raw_empty = [&](int s) { return bar0 + 8u * (UM_STAGES + s); };

    if (threadIdx.x == 0) {
        for (int s = 0; s < UM_STAGES; s++) {
            fl_mbar_init(raw_full(s), 1);
            fl_mbar_init(raw_empty(s), 4);                             // the four consumer warps, after their MMAs of the stage completed
        }
        fl_mbar_fence_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ------------------------------------------------ consumer warpgroup: MMA + fp32 block scaling ------------
        const int g = lane >> 2, t = lane & 3;
        const int ra = 16 * warp + g, rb = ra + 8;                     // tile rows of this thread's A fragment and outputs
        float acc[R], accm[(TYPE == FL_TYPE_Q4_1) ? R : 1];
#pragma unroll
        for (int j = 0; j < R; j++) acc[j] = 0.f;
#pragma unroll
        for (int j = 0; j < ((TYPE == FL_TYPE_Q4_1) ? R : 1); j++) accm[j] = 0.f;
        int32_t d[2][R];
#pragma unroll
        for (int j = 0; j < R; j++) d[0][j] = d[1][j] = 0;

        for (int st = 0; st < nstages; st++) {
            const int s = st % UM_STAGES;
            fl_mbar_wait_bounded(raw_full(s), (uint32_t)(st / UM_STAGES) & 1u);
            const uint8_t *raw = smem + (size_t)s * L::STAGE;
            const uint32_t *wa = (const uint32_t *)(raw + (size_t)ra * (UM_KC * BB));
            const uint32_t *wb = (const uint32_t *)(raw + (size_t)rb * (UM_KC * BB));
            const float *dys = (const float *)(raw + L::RAW_A + L::RAW_B);
            const uint32_t bstage = sm0 + (uint32_t)(s * L::STAGE + L::RAW_A);
            auto issue = [&](int i, int32_t(&dd)[R]) {
                const uint32_t qa = wa[i * WPB + QOFF + t], qb = wb[i * WPB + QOFF + t];
                uint32_t a[4] = {qa & 0x0F0F0F0Fu, qb & 0x0F0F0F0Fu, (qa >> 4) & 0x0F0F0F0Fu, (qb >> 4) & 0x0F0F0F0Fu};   // k 4t.. low, k 16 + 4t.. high nibbles
                if (TYPE == FL_TYPE_Q4_0) {
#pragma unroll
                    for (int j = 0; j < 4; j++) a[j] = (a[j] + 0x78787878u) ^ 0x80808080u;     // (x - 8) as s8, per byte, no carries
                }
                um_wg_fence();
                um_mma<NT, TYPE == FL_TYPE_Q4_0>(dd, a, um_smem_desc(bstage + (uint32_t)(i * NT * 32), NT * 16, 128));
                um_wg_commit();
            };
            issue(0, d[0]);
#pragma unroll
            for (int i = 0; i < UM_KC; i++) {
                if (i + 1 < UM_KC) {
                    issue(i + 1, d[(i + 1) & 1]);
                    um_wg_wait<1>();
                } else {
                    um_wg_wait<0>();
                }
                int32_t(&v)[R] = d[i & 1];
                um_fence_regs(v);
                // outputs of register 4j + e: row (e < 2 ? ra : rb), column 8j + 2t + (e & 1)
                const float dwa = __uint_as_float(wa[i * WPB]), dwb = __uint_as_float(wb[i * WPB]);
                const float *dyi = dys + i * NT;
#pragma unroll
                for (int j = 0; j < NT / 8; j++) {
                    const float2 y = *(const float2 *)(dyi + 8 * j + 2 * t);
                    acc[4 * j + 0] = __fmaf_rn(__fmul_rn(dwa, y.x), __int2float_rn(v[4 * j + 0]), acc[4 * j + 0]);
                    acc[4 * j + 1] = __fmaf_rn(__fmul_rn(dwa, y.y), __int2float_rn(v[4 * j + 1]), acc[4 * j + 1]);
                    acc[4 * j + 2] = __fmaf_rn(__fmul_rn(dwb, y.x), __int2float_rn(v[4 * j + 2]), acc[4 * j + 2]);
                    acc[4 * j + 3] = __fmaf_rn(__fmul_rn(dwb, y.y), __int2float_rn(v[4 * j + 3]), acc[4 * j + 3]);
                }
                if (TYPE == FL_TYPE_Q4_1) {
                    const float mwa = __uint_as_float(wa[i * WPB + 1]), mwb = __uint_as_float(wb[i * WPB + 1]);
                    const float *syi = dyi + UM_KC * NT;
#pragma unroll
                    for (int j = 0; j < NT / 8; j++) {
                        const float2 y = *(const float2 *)(syi + 8 * j + 2 * t);
                        accm[4 * j + 0] = __fmaf_rn(mwa, y.x, accm[4 * j + 0]);
                        accm[4 * j + 1] = __fmaf_rn(mwa, y.y, accm[4 * j + 1]);
                        accm[4 * j + 2] = __fmaf_rn(mwb, y.x, accm[4 * j + 2]);
                        accm[4 * j + 3] = __fmaf_rn(mwb, y.y, accm[4 * j + 3]);
                    }
                }
            }
            __syncwarp();
            if (lane == 0) fl_mbar_arrive(raw_empty(s));               // every MMA reading this stage has completed (wait_group 0)
        }
        // store: column n of the output is M contiguous floats
#pragma unroll
        for (int j = 0; j < R; j++) {
            const int row = m0 + (((j >> 1) & 1) ? rb : ra);
            const int col = n0 + 8 * (j >> 2) + 2 * t + (j & 1);
            if (row < prm.M && col < prm.N) {
                float o = acc[j];
                if (TYPE == FL_TYPE_Q4_1) o = __fadd_rn(acc[j], accm[j]);
                prm.dst[(size_t)col * prm.dst_row_stride + (size_t)row] = o;
            }
        }
    } else if (lane == 0) {
        // ------------------------------------------------ TMA producer ------------------------------------------------
        const int nbp = prm.nbp;
        const uint8_t *yq = prm.yq + (size_t)tile_n * nbp * (size_t)(NT * 32);
        const float *dy = prm.dy + (size_t)tile_n * nbp * NT;
        const float *sy = prm.sy + (size_t)tile_n * nbp * NT;
        for (int st = 0; st < nstages; st++) {
            const int s = st % UM_STAGES;
            fl_mbar_wait_bounded(raw_empty(s), ((uint32_t)(st / UM_STAGES) & 1u) ^ 1u);
            const uint32_t dst = sm0 + (uint32_t)(s * L::STAGE);
            const int kb0 = st * UM_KC;
            fl_mbar_expect_tx(raw_full(s), (uint32_t)L::STAGE);
            fl_tma_2d(dst, &tmap_w, kb0 * (BB / 4), m0, raw_full(s));                                   // 64 rows x KC blocks of raw q4
            fl_bulk_g2s(dst + L::RAW_A, yq + (size_t)kb0 * (NT * 32), (uint32_t)L::RAW_B, raw_full(s));
            fl_bulk_g2s(dst + L::RAW_A + L::RAW_B, dy + (size_t)kb0 * NT, (uint32_t)L::RAW_S, raw_full(s));
            if (TYPE == FL_TYPE_Q4_1) fl_bulk_g2s(dst + L::RAW_A + L::RAW_B + L::RAW_S, sy + (size_t)kb0 * NT, (uint32_t)L::RAW_S, raw_full(s));
        }
    }
}

// ---- host ------------------------------------------------------------------------------------------
static struct {
    uint8_t *yq = nullptr;
    float *dy = nullptr, *sy = nullptr;
    size_t cap_cols = 0;                 // capacity in (padded column) x (padded k-block) units
} g_um;

int flk_mul_mat_q_umma_supported(int type, const void *W, size_t wrs, int M, int K, int N) {
    if (type != FL_TYPE_Q4_0 && type != FL_TYPE_Q4_1) return 0;
    if (((uintptr_t)W & 15) != 0 || (wrs & 15) != 0 || K % 32 != 0 || M < 1 || N < 1) return 0;
    return fl_tma_get_encode() != nullptr;
}

template <int TYPE, int NT>
static int um_launch(cudaStream_t st, const void *W, size_t wrs, int M, int K, const void *Yq8, int N, float *dst, size_t drs) {
    using L = um_layout<TYPE, NT>;
    const int nb = K / 32, nbp = (nb + UM_KC - 1) / UM_KC * UM_KC;
    const int ntiles = (N + NT - 1) / NT, mtiles = (M + UM_M - 1) / UM_M;
    const size_t units = (size_t)ntiles * NT * nbp;
    if (units > g_um.cap_cols) {
        FL_CUDA_OK(cudaStreamSynchronize(st));
        if (g_um.yq) { cudaFree(g_um.yq); cudaFree(g_um.dy); cudaFree(g_um.sy); }
        g_um.cap_cols = units + units / 4;
        FL_CUDA_OK(cudaMalloc((void **)&g_um.yq, g_um.cap_cols * 32));
        FL_CUDA_OK(cudaMalloc((void **)&g_um.dy, g_um.cap_cols * 4));
        FL_CUDA_OK(cudaMalloc((void **)&g_um.sy, g_um.cap_cols * 4));
    }
    k_umma_prep<NT><<<dim3((nbp + 127) / 128, ntiles * NT), 128, 0, st>>>((const fl_block_q8_0 *)Yq8, N, nb, nbp, g_um.yq, g_um.dy, g_um.sy);
    fl_count_launch();
    CUtensorMap tm;
    const cuuint64_t gdim[2] = {(cuuint64_t)nb * (L::BB / 4), (cuuint64_t)M};
    const cuuint64_t gstr[1] = {(cuuint64_t)wrs};
    const cuuint32_t box[2] = {(cuuint32_t)(UM_KC * L::BB / 4), (cuuint32_t)UM_M};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult cr = fl_tma_get_encode()(&tm, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, (void *)W, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                        CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    FL_REQUIRE(cr == CUDA_SUCCESS, "mul_mat_q (wgmma): cuTensorMapEncodeTiled failed (%d) for M=%d K=%d stride=%zu", (int)cr, M, K, wrs);
    static bool attr_done = false;
    if (!attr_done) {
        FL_CUDA_OK(cudaFuncSetAttribute(k_mul_mat_q_umma<TYPE, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::SMEM));
        attr_done = true;
    }
    um_params p;
    p.yq = g_um.yq; p.dy = g_um.dy; p.sy = g_um.sy; p.dst = dst; p.dst_row_stride = drs; p.M = M; p.N = N; p.nbp = nbp; p.ntiles = ntiles;
    k_mul_mat_q_umma<TYPE, NT><<<mtiles * ntiles, UM_THREADS, L::SMEM, st>>>(tm, p);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

// nt_hint: 0 = choose, else 32 / 64 (128 is taken as 64: two register accumulator sets of 64 columns are the most a
// warpgroup keeps beside its fp32 sums without spilling)
int flk_mul_mat_q_umma(cudaStream_t st, int type, const void *W, size_t wrs, int M, int K, const void *Yq8, int N, float *dst, size_t drs, int nt_hint) {
    FL_REQUIRE(flk_mul_mat_q_umma_supported(type, W, wrs, M, K, N), "mul_mat_q (wgmma): unsupported operands (type %d, W %p, stride %zu, K %d)", type, W, wrs, K);
    int nt = nt_hint;
    if (nt == 0) {
        // wide column tiles re-read the weights less often; narrow ones when the wide tiling leaves SMs idle
        const int mtiles = (M + UM_M - 1) / UM_M;
        nt = (N > 32 && mtiles * ((N + 63) / 64) >= flk_sm_count()) ? 64 : 32;
    }
    if (nt >= 64) {
        if (type == FL_TYPE_Q4_0) return um_launch<FL_TYPE_Q4_0, 64>(st, W, wrs, M, K, Yq8, N, dst, drs);
        return um_launch<FL_TYPE_Q4_1, 64>(st, W, wrs, M, K, Yq8, N, dst, drs);
    }
    if (type == FL_TYPE_Q4_0) return um_launch<FL_TYPE_Q4_0, 32>(st, W, wrs, M, K, Yq8, N, dst, drs);
    return um_launch<FL_TYPE_Q4_1, 32>(st, W, wrs, M, K, Yq8, N, dst, drs);
}
