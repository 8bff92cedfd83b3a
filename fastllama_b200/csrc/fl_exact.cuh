// fl_exact.cuh -- the q4 x q8_0 block dot in the REFERENCE'S OWN fp32 ORDER, shared by the general matmul kernel
// (fl_exact_kernels.cu) and the persistent token kernel (fl_token_kernel.cu).
//
// The reference's x86 row kernels (ggml_vec_dot_q4_0_q8_0 / _q4_1_q8_0, AVX2 branches, reference lib/ggml.c:2445-2487 and
// :2639-2687) keep EIGHT fp32 accumulators per output: accumulator l takes, block after block,
//     acc[l] = fma(dx * dy, float(sum of the 4 products of elements 4l .. 4l+3), acc[l])
// and the row result is ((a0+a4)+(a2+a6)) + ((a1+a5)+(a3+a7)) (+ the scalar chain summs = fma(m, s, summs) for q4_1).
// Every activation vector is re-quantised to q8_0 before the next matmul, which turns a one-ulp difference of an input into
// per-cent differences a few matmuls later (DESIGN.md section 5), so "the same sum in another order" is NOT good enough for
// identical greedy tokens.  Here the order is reproduced exactly:
//   * lane mapping: 4 lanes per weight row, lane jj owns accumulators 2jj and 2jj+1 (the 8 values of bytes 4jj .. 4jj+3 of a block);
//   * the four-product integer sums are dp4a results (exact), biased with 0x4B400000 so that float(q) is one FADD;
//   * blocks are visited in order 0 .. nb-1 by every lane, the lane reduction is the reference's tree.
#pragma once
#include "fl_common.cuh"

// One q8_0 activation block prepared for the dot: 80 bytes.
//   q[jj] = { y[8jj .. 8jj+3], y[8jj+4 .. 8jj+7] (int8 x 4 each, natural order), bias_a, bias_b }
//   bias  = 0x4B400000 - off * (sum of the four y values), off = 8 for q4_0 (the nibble offset), 0 for q4_1
struct __align__(16) fl_yx {
    uint32_t q[4][4];
    float d, s;                 // the q8_0 block's scale and d * sum(q)
    uint32_t pad[2];
};
static_assert(sizeof(fl_yx) == 80, "prepared activation block");

#define FX_MAGIC_I 0x4B400000
#define FX_MAGIC_F 12582912.0f

#ifdef __CUDACC__
__device__ __forceinline__ uint32_t fx_bias(uint32_t y4, int off) { return (uint32_t)(FX_MAGIC_I - off * fl_dp4a_ss(0x01010101u, y4, 0)); }

// w: the 4 weight bytes (8 nibbles) of this lane -> its elements 0,1,2,3 (wa) and 4,5,6,7 (wb) as unsigned bytes
__device__ __forceinline__ void fx_split(uint32_t w, uint32_t &wa, uint32_t &wb) {
    const uint32_t lo = w & 0x0F0F0F0Fu, hi = (w >> 4) & 0x0F0F0F0Fu;      // elements 0,2,4,6 | 1,3,5,7
    wa = __byte_perm(lo, hi, 0x5140);                                        // elements 0,1,2,3
    wb = __byte_perm(lo, hi, 0x7362);                                        // elements 4,5,6,7
}
// wa, wb: fx_split of the lane's weight word (split once, used against any number of activation columns);
// d = dx * dy already rounded; y: this lane's entry of the prepared block
__device__ __forceinline__ void fx_block_split(uint32_t wa, uint32_t wb, float d, const uint4 y, float &a0, float &a1) {
    const float qa = __fsub_rn(__int_as_float(fl_dp4a_us(wa, y.x, (int)y.z)), FX_MAGIC_F);    // |sum| <= 4 * 15 * 128 < 2^22: exact
    const float qb = __fsub_rn(__int_as_float(fl_dp4a_us(wb, y.y, (int)y.w)), FX_MAGIC_F);
    a0 = __fmaf_rn(d, qa, a0);
    a1 = __fmaf_rn(d, qb, a1);
}
// w: the 4 weight bytes (8 nibbles) of this lane; d = dx * dy already rounded; y: this lane's entry of the prepared block
__device__ __forceinline__ void fx_block(uint32_t w, float d, const uint4 y, float &a0, float &a1) {
    uint32_t wa, wb;
    fx_split(w, wa, wb);
    fx_block_split(wa, wb, d, y, a0, a1);
}
// the reference's lane reduction; lanes 4r .. 4r+3 hold (a[2jj], a[2jj+1]); the row total is valid in lane 4r
__device__ __forceinline__ float fx_reduce(float a0, float a1) {
    a0 = __fadd_rn(a0, __shfl_xor_sync(0xffffffffu, a0, 2));                 // jj 0: a0+a4, a1+a5   jj 1: a2+a6, a3+a7
    a1 = __fadd_rn(a1, __shfl_xor_sync(0xffffffffu, a1, 2));
    a0 = __fadd_rn(a0, __shfl_xor_sync(0xffffffffu, a0, 1));                 // (a0+a4)+(a2+a6)
    a1 = __fadd_rn(a1, __shfl_xor_sync(0xffffffffu, a1, 1));                 // (a1+a5)+(a3+a7)
    return __fadd_rn(a0, a1);
}

// ggml_vec_dot_f32's reduction of the 32 partial sums of its four 8-lane accumulators (reference lib/ggml.c GGML_F32x8_REDUCE):
// lane l of the warp = element l of the 32-float step; the total is valid in lane 0
__device__ __forceinline__ float fx_reduce_f32(float acc) {
    const float t1 = __fadd_rn(acc, __shfl_down_sync(0xffffffffu, acc, 8));      // sum[0] += sum[1]; sum[2] += sum[3]
    const float t2 = __fadd_rn(t1, __shfl_down_sync(0xffffffffu, t1, 16));       // sum[0] += sum[2]
    const float u = __fadd_rn(t2, __shfl_down_sync(0xffffffffu, t2, 4));         // x[l] + x[l + 4]
    const float p = __fadd_rn(u, __shfl_down_sync(0xffffffffu, u, 1));           // hadd
    return __fadd_rn(p, __shfl_down_sync(0xffffffffu, p, 2));                    // hadd
}
// The leftover elements (n % 32) of ggml_vec_dot_f32 as the reference BUILD adds them (oracle/q4_oracle.c orc_vec_dot_f32): gcc
// vectorises "sumf += x[i]*y[i]" -- groups of 8 and one group of 4 become rounded product + rounded add, the last <= 3 elements an fma.
// Returns how many leftovers take the product + add form.
__device__ __forceinline__ int fx_left_nma(int rem) { return (rem & ~7) + ((rem & 4) ? 4 : 0); }
#endif
