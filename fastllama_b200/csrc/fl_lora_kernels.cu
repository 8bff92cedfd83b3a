// fl_lora_kernels.cu -- the ops of attach_lora / detach_lora on the device (SURVEY.md section 8 row f4), and the SIMD
// weight quantisers behind quantize_fns[type].quantize_row_q (row a2).
//
// Reference path (lib/llama.cpp:697-944): for every adapted matrix  BA = ggml_mul_mat(loraA, loraB)  (f32 x f32, K = rank),
// then  ggml_add_inplace(W, BA)  with W quantised -> ggml_compute_forward_add_q_f32 (lib/ggml.c:6414-6520): per row
// dequantize_row_q, ggml_vec_acc_f32, quantize_row_q -- the SIMD quantiser (AVX2 branches :739-803 and :965-1038), whose
// arithmetic differs from the _reference quantisers that define file contents:
//   q4_0: id = 7 / amax (not 1 / (amax / 7)), round-half-EVEN; q4_1: round-half-EVEN.
// A cached adapter stored as f16 (convert-lora-to-ggml.py --dtype fp16) takes ggml_compute_forward_add_q_f16 (lib/ggml.c:12372-12483)
// instead: the same row loop with X widened from f16 -- and detach first negates it in place with ggml_compute_forward_scale_f16
// (:12485-12524).
// Everything here is bit-exact against the reference's x86 build (tests/golden/lora_ops.npz and lora_f16_ops.npz, produced by the
// reference library).
#include <cuda_fp16.h>

#include "fl_common.cuh"
#include "fl_exact.cuh"
#include "fl_kernels.h"

// lane = element of the block; returns the 4-bit code of this lane's value and writes the block header from lane 0
template <int TYPE>
__device__ __forceinline__ int lq_quantize_simd(float v, int lane, uint8_t *blk) {
    if (TYPE == FL_TYPE_Q4_0) {
        const float amax = fl_warp_max(fabsf(v));
        const float d = __fdiv_rn(amax, 7.0f);
        const float id = (amax != 0.0f) ? __fdiv_rn(7.0f, amax) : 0.0f;
        // _mm256_round_ps(NEAREST) + cvtps_epi32 = round-half-even; the saturating packs never trigger (|v * id| <= 7 up to rounding)
        const int q = max(-128, min(127, __float2int_rn(__fmul_rn(v, id)))) + 8;
        if (lane == 0) *(float *)blk = d;
        return q & 0x0F;
    } else {
        float mn = v, mx = v;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        }
        const float d = __fdiv_rn(__fsub_rn(mx, mn), 15.0f);
        const float id = (d != 0.0f) ? __fdiv_rn(1.0f, d) : 0.0f;
        const int q = max(-128, min(127, __float2int_rn(__fmul_rn(__fsub_rn(v, mn), id))));
        if (lane == 0) { ((float *)blk)[0] = d; ((float *)blk)[1] = mn; }
        return q & 0x0F;
    }
}
template <int TYPE>
__device__ __forceinline__ void lq_store_codes(int q, int lane, uint8_t *blk) {
    constexpr int QOFF = (TYPE == FL_TYPE_Q4_0) ? 4 : 8;
    const int qn = __shfl_down_sync(0xffffffffu, q, 1);
    if ((lane & 1) == 0) blk[QOFF + (lane >> 1)] = (uint8_t)(q | (qn << 4));     // packNibbles: element 2j low, 2j+1 high
}

// quantize_row_q4_0 / quantize_row_q4_1 (the SIMD variants): one warp per block
template <int TYPE>
__global__ void k_quantize_q4_simd(const float *__restrict__ x, uint8_t *__restrict__ y, long nblocks) {
    constexpr int BB = (TYPE == FL_TYPE_Q4_0) ? 20 : 24;
    const int lane = threadIdx.x & 31;
    const long wid = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long nw = ((long)gridDim.x * blockDim.x) >> 5;
    for (long b = wid; b < nblocks; b += nw) {
        uint8_t *blk = y + b * BB;
        const int q = lq_quantize_simd<TYPE>(x[b * FL_QK + lane], lane, blk);
        lq_store_codes<TYPE>(q, lane, blk);
    }
}

// X's element as fp32: f32 as is; f16 widened exactly (GGML_FP16_TO_FP32, the F16C build's _cvtsh_ss)
__device__ __forceinline__ float lq_widen(float x) { return x; }
__device__ __forceinline__ float lq_widen(uint16_t x) { return __half2float(__ushort_as_half(x)); }

// ggml_compute_forward_add_q_f32 (XT = float) and ggml_compute_forward_add_q_f16 (XT = uint16_t, f16 bits): dst row =
// quantize_row_q(dequantize_row_q(src0 row) + fp32(src1 row)); dst may alias src0 (add_inplace)
template <int TYPE, typename XT>
__global__ void k_add_q(const uint8_t *W, size_t w_row_stride, int M, int K, const XT *__restrict__ X, size_t x_row_stride, uint8_t *D,
                        size_t d_row_stride) {
    constexpr int BB = (TYPE == FL_TYPE_Q4_0) ? 20 : 24;
    constexpr int QOFF = (TYPE == FL_TYPE_Q4_0) ? 4 : 8;
    const int nb = K / FL_QK;
    const int lane = threadIdx.x & 31;
    const long wid = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long nw = ((long)gridDim.x * blockDim.x) >> 5;
    for (long t = wid; t < (long)M * nb; t += nw) {
        const long r = t / nb;
        const int ib = (int)(t % nb);
        const uint8_t *src = W + (size_t)r * w_row_stride + (size_t)ib * BB;
        const float d = *(const float *)src;
        const uint8_t byte = src[QOFF + (lane >> 1)];
        const int code = (lane & 1) ? (byte >> 4) : (byte & 0x0F);
        float v;
        if (TYPE == FL_TYPE_Q4_0) v = __fmul_rn((float)(code - 8), d);                       // dequantize_row_q4_0, lib/ggml.c:1449-1481
        else v = __fmaf_rn((float)code, d, *(const float *)(src + 4));                       // dequantize_row_q4_1 (fused in the GNU-mode build), :1567-1596
        v = __fadd_rn(v, lq_widen(X[(size_t)r * x_row_stride + (size_t)ib * FL_QK + lane])); // ggml_vec_acc_f32 :2286 / the f16 loop :12476-12478
        __syncwarp();                                                                        // every lane has read the block before it is overwritten in place
        uint8_t *dst = D + (size_t)r * d_row_stride + (size_t)ib * BB;
        const int q = lq_quantize_simd<TYPE>(v, lane, dst);
        lq_store_codes<TYPE>(q, lane, dst);
    }
}

// ggml_compute_forward_scale_f16 (ggml_scale is a view, so this is in place): x = fp16_rn(fp32(x) * v), the F16C build's
// _cvtsh_ss / _cvtss_sh(., 0)
__global__ void k_scale_f16(uint16_t *x, long n, float v) {
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
        x[i] = __half_as_ushort(__float2half_rn(__fmul_rn(lq_widen(x[i]), v)));
}

// ggml_mul_mat on two f32 matrices in the reference's summation order (ggml_vec_dot_f32, lib/ggml.c:2295-2325, AVX2 + FMA build):
// out[j * ldo + i] = dot(a row i, b row j).  One warp per output: lane L is lane L % 8 of accumulator L / 8 of the 4 x 8-lane
// SIMD part (fma per 32-element step), the GGML_F32x8_REDUCE tree, then the leftovers added as rounded products by lane 0.
__global__ void k_mul_mat_f32_ref(const float *__restrict__ A, size_t lda, int Ma, const float *__restrict__ B, size_t ldb, int Mb, int K, float *__restrict__ out,
                                  size_t ldo) {
    const int lane = threadIdx.x & 31;
    const long wid = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long nw = ((long)gridDim.x * blockDim.x) >> 5;
    const int np = K & ~31;
    for (long t = wid; t < (long)Ma * Mb; t += nw) {
        const int i = (int)(t % Ma);
        const long j = t / Ma;
        const float *a = A + (size_t)i * lda, *b = B + (size_t)j * ldb;
        float acc = 0.0f;
        for (int k = 0; k < np; k += 32) acc = __fmaf_rn(a[k + lane], b[k + lane], acc);
        // sum[0] += sum[1]; sum[2] += sum[3]; sum[0] += sum[2]  (lanes 0-7 | 8-15 | 16-23 | 24-31 are the four accumulators)
        float t1 = __fadd_rn(acc, __shfl_down_sync(0xffffffffu, acc, 8));          // valid in lanes 0-7 and 16-23
        float t2 = __fadd_rn(t1, __shfl_down_sync(0xffffffffu, t1, 16));           // valid in lanes 0-7
        // t0[l] = x[l] + x[l + 4]; t1 = hadd(t0, t0): (t0[0] + t0[1], t0[2] + t0[3]); res = t1[0] + t1[1]
        float u = __fadd_rn(t2, __shfl_down_sync(0xffffffffu, t2, 4));             // lanes 0-3
        float p = __fadd_rn(u, __shfl_down_sync(0xffffffffu, u, 1));               // lane 0: u0 + u1, lane 2: u2 + u3
        float s = __fadd_rn(p, __shfl_down_sync(0xffffffffu, p, 2));               // lane 0
        if (lane == 0) {
            const int nma = np + fx_left_nma(K - np);
            for (int k = np; k < nma; k++) s = __fadd_rn(s, __fmul_rn(a[k], b[k]));
            for (int k = nma; k < K; k++) s = __fmaf_rn(a[k], b[k], s);
            out[(size_t)j * ldo + i] = s;
        }
    }
}
// K < 32: no SIMD part, one thread per output
__global__ void k_mul_mat_f32_ref_small(const float *__restrict__ A, size_t lda, int Ma, const float *__restrict__ B, size_t ldb, int Mb, int K,
                                        float *__restrict__ out, size_t ldo) {
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < (long)Ma * Mb; t += (long)gridDim.x * blockDim.x) {
        const int i = (int)(t % Ma);
        const long j = t / Ma;
        const float *a = A + (size_t)i * lda, *b = B + (size_t)j * ldb;
        float s = 0.0f;
        const int nma = fx_left_nma(K);
        for (int k = 0; k < nma; k++) s = __fadd_rn(s, __fmul_rn(a[k], b[k]));
        for (int k = nma; k < K; k++) s = __fmaf_rn(a[k], b[k], s);
        out[(size_t)j * ldo + i] = s;
    }
}

static inline int lq_grid(long nwarps, int threads) {
    const long blocks = (nwarps * 32 + threads - 1) / threads;
    const long cap = (long)flk_sm_count() * 16;
    return (int)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

int flk_quantize_q4_simd(cudaStream_t st, int type, const float *x, void *y, int k, int nrows) {
    FL_REQUIRE(k > 0 && k % FL_QK == 0, "quantize_q4_simd: k=%d is not a multiple of 32", k);
    FL_REQUIRE(type == FL_TYPE_Q4_0 || type == FL_TYPE_Q4_1, "quantize_q4_simd: unsupported type %d", type);
    if (nrows <= 0) return 0;
    const long nblocks = (long)(k / FL_QK) * nrows;
    if (type == FL_TYPE_Q4_0) k_quantize_q4_simd<FL_TYPE_Q4_0><<<lq_grid(nblocks, 256), 256, 0, st>>>(x, (uint8_t *)y, nblocks);
    else k_quantize_q4_simd<FL_TYPE_Q4_1><<<lq_grid(nblocks, 256), 256, 0, st>>>(x, (uint8_t *)y, nblocks);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

template <typename XT>
static int add_q(cudaStream_t st, int type, const void *W, size_t w_row_stride, int M, int K, const XT *X, size_t x_row_stride_elems, void *dst,
                 size_t dst_row_stride) {
    FL_REQUIRE(K > 0 && K % FL_QK == 0, "add_q: K=%d is not a multiple of 32", K);
    FL_REQUIRE(type == FL_TYPE_Q4_0 || type == FL_TYPE_Q4_1, "add_q: unsupported type %d", type);
    if (M <= 0) return 0;
    const long nblocks = (long)(K / FL_QK) * M;
    if (type == FL_TYPE_Q4_0)
        k_add_q<FL_TYPE_Q4_0, XT><<<lq_grid(nblocks, 256), 256, 0, st>>>((const uint8_t *)W, w_row_stride, M, K, X, x_row_stride_elems, (uint8_t *)dst, dst_row_stride);
    else
        k_add_q<FL_TYPE_Q4_1, XT><<<lq_grid(nblocks, 256), 256, 0, st>>>((const uint8_t *)W, w_row_stride, M, K, X, x_row_stride_elems, (uint8_t *)dst, dst_row_stride);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}
int flk_add_q_f32(cudaStream_t st, int type, const void *W, size_t w_row_stride, int M, int K, const float *X, size_t x_row_stride_elems, void *dst,
                  size_t dst_row_stride) {
    return add_q(st, type, W, w_row_stride, M, K, X, x_row_stride_elems, dst, dst_row_stride);
}
int flk_add_q_f16(cudaStream_t st, int type, const void *W, size_t w_row_stride, int M, int K, const uint16_t *X, size_t x_row_stride_elems, void *dst,
                  size_t dst_row_stride) {
    return add_q(st, type, W, w_row_stride, M, K, X, x_row_stride_elems, dst, dst_row_stride);
}

int flk_scale_f16(cudaStream_t st, uint16_t *x, long n, float v) {
    if (n <= 0) return 0;
    k_scale_f16<<<lq_grid((n + 31) / 32, 256), 256, 0, st>>>(x, n, v);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}

int flk_mul_mat_f32_ref(cudaStream_t st, const float *A, size_t lda, int Ma, const float *B, size_t ldb, int Mb, int K, float *out, size_t ldo) {
    if (Ma <= 0 || Mb <= 0) return 0;
    FL_REQUIRE(K > 0, "mul_mat_f32: K=%d", K);
    const long n = (long)Ma * Mb;
    if (K < 32) k_mul_mat_f32_ref_small<<<lq_grid((n + 31) / 32, 256), 256, 0, st>>>(A, lda, Ma, B, ldb, Mb, K, out, ldo);
    else k_mul_mat_f32_ref<<<lq_grid(n, 256), 256, 0, st>>>(A, lda, Ma, B, ldb, Mb, K, out, ldo);
    fl_count_launch();
    FL_CUDA_OK(cudaGetLastError());
    return 0;
}
