// fl_common.cuh -- block formats, PTX wrappers and error plumbing shared by the sm_90a kernels.
//
// Block formats are the reference's on-disk / in-memory layouts and are kept byte for byte
// (reference lib/ggml.c:590-626): q4_0 {f32 d; u8 qs[16]} 20 B, q4_1 {f32 d; f32 m; u8 qs[16]}
// 24 B, q8_0 {f32 d; f32 s; i8 qs[32]} 40 B; qs[j] = q[2j] | q[2j+1] << 4.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#define FL_QK 32
#define FL_TYPE_F32 0
#define FL_TYPE_F16 1
#define FL_TYPE_Q4_0 2
#define FL_TYPE_Q4_1 3
#define FL_TYPE_Q8_0 6

struct fl_block_q4_0 { float d; uint8_t qs[FL_QK / 2]; };
struct fl_block_q4_1 { float d; float m; uint8_t qs[FL_QK / 2]; };
struct fl_block_q8_0 { float d; float s; int8_t qs[FL_QK]; };
static_assert(sizeof(fl_block_q4_0) == 20, "q4_0 block");
static_assert(sizeof(fl_block_q4_1) == 24, "q4_1 block");
static_assert(sizeof(fl_block_q8_0) == 40, "q8_0 block");

__host__ __device__ inline int fl_block_bytes(int type) {
    return type == FL_TYPE_Q4_0 ? 20 : type == FL_TYPE_Q4_1 ? 24 : type == FL_TYPE_Q8_0 ? 40 : 0;
}

// ---- error plumbing (host) -------------------------------------------------------------------
void fl_set_error(const char *fmt, ...);
#define FL_CUDA_OK(expr)                                                                     \
    do {                                                                                     \
        cudaError_t _e = (expr);                                                             \
        if (_e != cudaSuccess) {                                                             \
            fl_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return -1;                                                                       \
        }                                                                                    \
    } while (0)
#define FL_REQUIRE(cond, ...)                 \
    do {                                      \
        if (!(cond)) {                        \
            fl_set_error(__VA_ARGS__);        \
            return -2;                        \
        }                                     \
    } while (0)

#ifdef __CUDACC__
// ---- device helpers ----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t fl_smem_u32(const void *p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}

// unsigned-byte x signed-byte 4-way dot with int32 accumulate (SASS: IDP.4A.U8.S8)
__device__ __forceinline__ int fl_dp4a_us(uint32_t a_u8x4, uint32_t b_s8x4, int c) {
    int r;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(r) : "r"(a_u8x4), "r"(b_s8x4), "r"(c));
    return r;
}
__device__ __forceinline__ int fl_dp4a_ss(uint32_t a_s8x4, uint32_t b_s8x4, int c) {
    int r;
    asm("dp4a.s32.s32 %0, %1, %2, %3;" : "=r"(r) : "r"(a_s8x4), "r"(b_s8x4), "r"(c));
    return r;
}

// mbarrier (shared::cta) -- the async-copy completion mechanism of sm_90
__device__ __forceinline__ void fl_mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fl_mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fl_mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void fl_mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool fl_mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void fl_mbar_wait(uint32_t bar, uint32_t parity) {
    while (!fl_mbar_try_wait(bar, parity)) {
    }
}
// bounded mbarrier wait: a protocol bug traps (the launch fails with an error) instead of hanging the GPU
__device__ __forceinline__ void fl_mbar_wait_bounded(uint32_t bar, uint32_t parity) {
    for (uint32_t n = 0; !fl_mbar_try_wait(bar, parity); n++)
        if (n > (1u << 24)) asm volatile("trap;");
}

// 1-D bulk async copy global -> shared through the TMA unit (SASS: UBLKCP.S.G); completion is
// signalled on `bar` as `bytes` transaction bytes.  dst/src 16-B aligned, bytes % 16 == 0.
__device__ __forceinline__ void fl_bulk_g2s(uint32_t dst_smem, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
        "l"(src), "r"(bytes), "r"(bar)
        : "memory");
}
// same, with an L2 eviction-priority hint (weights are streamed once per token: evict_first)
__device__ __forceinline__ void fl_bulk_g2s_hint(uint32_t dst_smem, const void *src, uint32_t bytes, uint32_t bar,
                                                 uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::
            "r"(dst_smem),
        "l"(src), "r"(bytes), "r"(bar), "l"(policy)
        : "memory");
}
// ask L2 to fetch [src, src + bytes) (16-byte granular); no completion signal, no shared memory involved
__device__ __forceinline__ void fl_bulk_prefetch_l2(const void *src, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ uint64_t fl_policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}

__device__ __forceinline__ float fl_warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float fl_warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ double fl_warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ int fl_warp_sum_i(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
#endif  // __CUDACC__
