// Microbenchmark: how fast can one CTA per SM stream a contiguous HBM range into shared memory with
// 1-D bulk copies (UBLKCP) through an mbarrier ring, with NO compute?  Sweeps tile size / stage count /
// CTAs per SM.  Decides the ring geometry of the matvec kernels.   nvcc -arch=sm_90a -O3 tma_stream.cu
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include "../../fastllama_b200/csrc/fl_common.cuh"
void fl_set_error(const char *, ...) {}

__global__ void __launch_bounds__(128) k_stream(const uint8_t *src, size_t bytes_per_cta, uint32_t tile, int S, int use_hint, unsigned *sink) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t *bars = (uint64_t *)smem;
    uint8_t *stage0 = smem + 1024;
    const uint32_t bar0 = fl_smem_u32(bars);
    const int ntiles = (int)(bytes_per_cta / tile);
    if (threadIdx.x == 0) {
        for (int s = 0; s < S; s++) { fl_mbar_init(bar0 + 8u * s, 1); fl_mbar_init(bar0 + 8u * (S + s), 1); }
        fl_mbar_fence_init();
    }
    __syncthreads();
    const uint8_t *base = src + (size_t)blockIdx.x * bytes_per_cta;
    if (threadIdx.x == 0) {
        const uint64_t pol = fl_policy_evict_first();
        int s = 0; uint32_t ph = 1;
        for (int t = 0; t < ntiles; t++) {
            fl_mbar_wait(bar0 + 8u * (S + s), ph);
            fl_mbar_expect_tx(bar0 + 8u * s, tile);
            if (use_hint) fl_bulk_g2s_hint(fl_smem_u32(stage0 + (size_t)s * tile), base + (size_t)t * tile, tile, bar0 + 8u * s, pol);
            else fl_bulk_g2s(fl_smem_u32(stage0 + (size_t)s * tile), base + (size_t)t * tile, tile, bar0 + 8u * s);
            if (++s == S) { s = 0; ph ^= 1u; }
        }
    } else if (threadIdx.x == 32) {
        int s = 0; uint32_t ph = 0; unsigned acc = 0;
        for (int t = 0; t < ntiles; t++) {
            fl_mbar_wait(bar0 + 8u * s, ph);
            acc ^= *(volatile unsigned *)(stage0 + (size_t)s * tile);
            fl_mbar_arrive(bar0 + 8u * (S + s));
            if (++s == S) { s = 0; ph ^= 1u; }
        }
        if (acc == 0x12345u) *sink = acc;
    }
}

int main() {
    int sm = 0; cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, 0);
    const size_t total = (size_t)1 << 30;       // 1 GiB buffer, far larger than L2
    uint8_t *buf; cudaMalloc(&buf, total); cudaMemset(buf, 1, total);
    unsigned *sink; cudaMalloc(&sink, 4);
    cudaFuncSetAttribute(k_stream, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    const int tiles_kb[] = {2, 4, 8, 16, 32};
    const int cps[] = {1, 2};
    printf("sm=%d\n", sm);
    for (int cpsm : cps) for (int tk : tiles_kb) for (int inflight_kb : {32, 64, 128, 200}) for (int hint : {0, 1}) for (size_t mb : {28, 224}) {
        const uint32_t tile = tk * 1024;
        const int budget = inflight_kb / cpsm;
        int S = budget * 1024 / tile; if (S < 2) continue; if (S > 64) S = 64;
        const size_t smem = 1024 + (size_t)S * tile;
        if (smem * cpsm > 227 * 1024) continue;
        const int grid = sm * cpsm;
        size_t per_cta = (mb << 20) / grid / tile * tile;
        float best = 1e9;
        for (int rep = 0; rep < 3; rep++) {
            // rotate through the 1 GiB buffer so every launch reads cold data
            const size_t off = ((size_t)rep * (mb << 20)) % (total - (mb << 20));
            cudaEventRecord(e0);
            k_stream<<<grid, 128, smem>>>(buf + (off & ~(size_t)255), per_cta, tile, S, hint, sink);
            cudaEventRecord(e1); cudaEventSynchronize(e1);
            float ms; cudaEventElapsedTime(&ms, e0, e1); if (ms < best) best = ms;
        }
        const double gb = (double)per_cta * grid / 1e9;
        printf("cta/sm=%d tile=%2dKB stages=%2d inflight/SM=%3dKB hint=%d total=%4zuMB  %7.2f us  %7.1f GB/s  err=%s\n", cpsm, tk, S, inflight_kb, hint, mb,
               best * 1e3, gb / (best * 1e-3), cudaGetErrorString(cudaGetLastError()));
    }
    return 0;
}
