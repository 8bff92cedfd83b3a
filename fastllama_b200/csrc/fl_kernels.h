// fl_kernels.h -- internal (C++) launcher interface between the kernel translation units and the
// runtime / graph executor.  Not part of the public C ABI (that is include/fl_cuda.h, fl_ggml.h).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "fl_cuda.h"

// bookkeeping implemented in fl_runtime.cu
void fl_count_launch();
void fl_set_error(const char *fmt, ...);

// ---- fl_quant_kernels.cu ------------------------------------------------------------------------
int flk_query_device();
int flk_sm_count();
int flk_quantize_q8_0(cudaStream_t st, const float *x, size_t x_row_stride_bytes, void *y, int k, int nrows);
int flk_quantize_q4(cudaStream_t st, int type, const float *x, void *y, int k, int nrows);
int flk_quantize_q4_file(cudaStream_t st, int type, int src_type, const void *x, void *y, int k, int nrows,
                         unsigned long long *hist);
int flk_dequantize_rows(cudaStream_t st, int type, const void *W, size_t w_row_stride, int K, const int32_t *ids,
                        int n_ids, float *dst, size_t dst_row_stride);
int flk_mul_mat_q(cudaStream_t st, int type, const void *W, size_t w_row_stride, int M, int K, const void *Yq8, int N,
                  float *dst, size_t dst_row_stride, int impl);

// fl_mma_kernel.cu: N > 1, integer block sums on the tensor cores (mma.sync m16n8k32 u8 x s8), scales in fp32
int flk_mul_mat_q_mma(cudaStream_t st, int type, const void *W, size_t w_row_stride, int M, int K, const void *Yq8, int N, float *dst,
                      size_t dst_row_stride);

// ---- fl_ops_kernels.cu: the non-matmul ops Model::eval emits (reference lib/llama.cpp:301-465) ----
// A strided 4-D view of device memory: ne = element counts, nb = byte strides (ggml conventions,
// reference include/ggml.h:279-309).
// (struct fl_view is declared in include/fl_cuda.h)

enum { FLK_ADD = 0, FLK_MUL = 1 };

int flk_rms_norm(cudaStream_t st, const fl_view &src, const fl_view &dst, float eps);
int flk_binary(cudaStream_t st, int op, const fl_view &a, const fl_view &b, const fl_view &dst);
int flk_repeat(cudaStream_t st, const fl_view &src, const fl_view &dst);
int flk_scale(cudaStream_t st, const fl_view &t, float v);
int flk_silu(cudaStream_t st, const fl_view &src, const fl_view &dst, const uint16_t *silu_table_f16);
int flk_diag_mask_inf(cudaStream_t st, const fl_view &t, int n_past);
int flk_soft_max(cudaStream_t st, const fl_view &t, const uint16_t *exp_table_f16);
// cs: [n_pos][n_dims/2] (cos, sin) pairs for absolute positions 0..n_pos-1, built on the host
int flk_rope(cudaStream_t st, const fl_view &t, int n_past, int n_dims, int mode, const float2 *cs, int n_pos);
int flk_cpy_f32(cudaStream_t st, const fl_view &src, const fl_view &dst);
int flk_mul_mat_f32(cudaStream_t st, const fl_view &src0, const fl_view &src1, const fl_view &dst);
// [world][N][n_local] (an all-gather's output) -> [N][world * n_local], + residual [N][world * n_local] when it is not null
int flk_tp_unshard(cudaStream_t st, const float *gathered, int world, int N, int n_local, const float *residual, float *dst);
int flk_tp_unshard_v(cudaStream_t st, const float *gathered, int world, int N, int stride, const int *first, const int *count, const float *residual,
                     float *dst);

// fl_umma_kernel.cu: N > 1 on the Hopper tensor cores: one wgmma (M = 64, K = 32, 8-bit operands) per quant block into registers,
// weights by TMA, exact fp32 block scaling by the same warpgroup.  nt_hint: column-tile width (0 = choose; 32 / 64; 128 is taken as 64)
int flk_mul_mat_q_umma_supported(int type, const void *W, size_t w_row_stride, int M, int K, int N);
int flk_mul_mat_q_umma(cudaStream_t st, int type, const void *W, size_t w_row_stride, int M, int K, const void *Yq8, int N, float *dst,
                       size_t dst_row_stride, int nt_hint);

// fl_lora_kernels.cu: the SIMD weight quantisers (quantize_fns[].quantize_row_q) and the ops of attach_lora / detach_lora
int flk_quantize_q4_simd(cudaStream_t st, int type, const float *x, void *y, int k, int nrows);
int flk_add_q_f32(cudaStream_t st, int type, const void *W, size_t w_row_stride, int M, int K, const float *X, size_t x_row_stride_elems, void *dst,
                  size_t dst_row_stride);
int flk_add_q_f16(cudaStream_t st, int type, const void *W, size_t w_row_stride, int M, int K, const uint16_t *X, size_t x_row_stride_elems, void *dst,
                  size_t dst_row_stride);
int flk_scale_f16(cudaStream_t st, uint16_t *x, long n, float v);
int flk_mul_mat_f32_ref(cudaStream_t st, const float *A, size_t lda, int Ma, const float *B, size_t ldb, int Mb, int K, float *out, size_t ldo);

// fl_exact_kernels.cu: results with the reference's fp32 bits (fl_exact.cuh): q4 x q8_0 matmul for any M, K, N, and the f32 mul_mat
int flk_mul_mat_q_ref(cudaStream_t st, int type, const void *W, size_t w_row_stride, int M, int K, const void *Yq8, int N, float *dst,
                      size_t dst_row_stride);
// the same bits as a tiled GEMM (shared-memory ring, TMA) for multi-token evals; operands: q4_0 / q4_1, 16-byte aligned W and rows
int flk_mul_mat_q_ref_tiled_supported(int type, const void *W, size_t w_row_stride, int M, int K, int N);
int flk_mul_mat_q_ref_tiled(cudaStream_t st, int type, const void *W, size_t w_row_stride, int M, int K, const void *Yq8, int N, float *dst,
                            size_t dst_row_stride);
int flk_mul_mat_f32_ref4(cudaStream_t st, const fl_view &a, const fl_view &b, const fl_view &d);
void flk_exact_release();
