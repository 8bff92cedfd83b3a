// fl_tma.cuh -- 2-D tensor-map copies (TMA) shared by the GEMM kernels that stage tiles through shared memory
// (fl_umma_kernel.cu, fl_exact_kernels.cu).
#pragma once
#include <cuda.h>

#include "fl_common.cuh"

#ifdef __CUDACC__
// box at element coordinates (c0 inner, c1 outer) -> shared memory at dst; completion is signalled on `bar` as the box's bytes
// (elements outside the tensor are zero-filled and counted too).  SASS: UTMALDG.
__device__ __forceinline__ void fl_tma_2d(uint32_t dst, const CUtensorMap *tm, int c0, int c1, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst), "l"(tm), "r"(c0),
                 "r"(c1), "r"(bar)
                 : "memory");
}
#endif

// the driver's cuTensorMapEncodeTiled, found through the runtime (no link against libcuda); nullptr when the driver lacks it
typedef CUresult (*fl_tma_encode_fn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                     const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static inline fl_tma_encode_fn fl_tma_get_encode() {
    static fl_tma_encode_fn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = (fl_tma_encode_fn)p;
    }
    return fn;
}
