// grid_sync.cu -- cost of a software grid barrier, one CTA per SM x 544 threads (the token kernel's shape).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o grid_sync grid_sync.cu && ./grid_sync
#include <cstdio>
#include <cuda_runtime.h>
#define NT 512
__device__ __forceinline__ void bar512() { asm volatile("bar.sync 13, 512;" ::: "memory"); }

template <int V>
__global__ void __launch_bounds__(544, 1) k_sync(unsigned *ctr, unsigned *flag, unsigned *sub, int iters, float *sink) {
    if (threadIdx.x >= NT) return;
    float acc = 0.f;
    for (int e = 1; e <= iters; e++) {
        bar512();
        if (threadIdx.x == 0) {
            if (V == 0) {          // release increment, acquire spin on the counter
                asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory");
                unsigned v;
                do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory"); } while (v < (unsigned)e * gridDim.x);
            } else if (V == 1) {   // __threadfence + atomicAdd + spin + __threadfence (cooperative-groups style)
                __threadfence();
                atomicAdd(ctr, 1u);
                unsigned v;
                do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory"); } while (v < (unsigned)e * gridDim.x);
                __threadfence();
            } else if (V == 2) {   // last arriver publishes a flag on its own line; everybody else spins on the flag
                unsigned old;
                asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(old) : "l"(ctr) : "memory");
                if (old == (unsigned)e * gridDim.x - 1) {
                    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(flag), "r"((unsigned)e) : "memory");
                } else {
                    unsigned v;
                    do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory"); } while (v < (unsigned)e);
                }
            } else if (V == 3) {   // relaxed spin, one acquire fence at the end
                asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory");
                unsigned v;
                do { asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory"); } while (v < (unsigned)e * gridDim.x);
                asm volatile("fence.acq_rel.gpu;" ::: "memory");
            } else if (V == 4) {   // two levels: 8 sub-counters, the last arriver of each bumps the top counter
                const int grp = blockIdx.x & 7;
                const unsigned gsz = (gridDim.x + 7 - grp) / 8;
                unsigned old;
                asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(old) : "l"(sub + 32 * grp) : "memory");
                if (old == (unsigned)e * gsz - 1) asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory");
                unsigned v;
                do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory"); } while (v < (unsigned)e * 8u);
            } else if (V == 5) {   // relaxed increment only (no ordering): lower bound
                asm volatile("red.relaxed.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory");
                unsigned v;
                do { asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory"); } while (v < (unsigned)e * gridDim.x);
            }
        }
        bar512();
        acc += 1.f;
    }
    if (acc < 0) sink[0] = acc;
}

template <int V>
static void run(const char *name) {
    unsigned *ctr, *flag, *sub; float *sink;
    cudaMalloc(&ctr, 256); cudaMalloc(&flag, 256); cudaMalloc(&sub, 8 * 128 + 128); cudaMalloc(&sink, 4);
    int sm = 0; cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, 0);
    const int iters = 2000;
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    float best = 1e9f;
    for (int rep = 0; rep < 3; rep++) {
        cudaMemset(ctr, 0, 256); cudaMemset(flag, 0, 256); cudaMemset(sub, 0, 8 * 128 + 128);
        int it = iters;
        void *args[] = {&ctr, &flag, &sub, &it, &sink};
        cudaEventRecord(a);
        cudaLaunchCooperativeKernel((const void *)k_sync<V>, dim3(sm), dim3(544), args, 0, 0);
        cudaEventRecord(b);
        cudaError_t e = cudaEventSynchronize(b);
        if (e != cudaSuccess) { printf("%s: %s\n", name, cudaGetErrorString(e)); return; }
        float ms; cudaEventElapsedTime(&ms, a, b);
        if (ms < best) best = ms;
    }
    printf("%-60s %6.3f us per barrier (%d CTAs)\n", name, best * 1e3f / iters, sm);
}
int main() {
    run<0>("V0 red.release + ld.acquire spin on counter");
    run<1>("V1 threadfence + atomicAdd + acquire spin + threadfence");
    run<2>("V2 atom.acq_rel, last arriver st.release flag, spin on flag");
    run<3>("V3 red.release + relaxed spin + fence.acq_rel");
    run<4>("V4 two-level (8 sub-counters)");
    run<5>("V5 relaxed only (no ordering; lower bound)");
    return 0;
}
